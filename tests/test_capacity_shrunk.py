"""The capacity limits of the statistics and text kernels at CPU-test sizes: the emulated library (tests/simt_emu.py) built
with its capacity #defines shrunk — one SM's grid caps, staging rounds and groups of a few dozen segments, two-entry
long lists, "long" at a few hundred bytes — runs tests/capacity.py's batches, built from the same shrunk constants, against
the oracle.  Every path tests/test_gpu_capacity.py reaches at full size on the GPU runs here: the second and later staging
rounds of k_cycle_stats and both of its early exits, several segment groups (with CS_GROUP a multiple of CS_STAGE and not),
the lone-warp fallbacks behind KF_LIST and RQ_LIST, warps looping over several reads, per-block flushes of several reads,
k_fastq_pack and k_emit_copy with more records than warps.  One path runs here only: the lone warps behind RQ_LIST in
k_read_qual_exc, which at the product's constants want a list of 25 000 reads of 96 KiB.  The k_read_qual batches run on both
quality passes (scan="fast": k_read_qual itself; "jit": k_scan_jit's counts and k_read_qual_exc), and every quality case
asserts which one ran."""
import numpy as np
import pytest

import capacity
import simt_emu

SMALL = dict(FPL_NUM_SMS=1, CS_STAGE=24, KF_LIST=2, RQ_LIST=2, RQ_LONG=300, KF_LONG=200)
BUILDS = {"group_of_2_stages": dict(SMALL, CS_GROUP=48), "group_of_2.5_stages": dict(SMALL, CS_GROUP=60)}


LIBS = {}      # build name -> (library, constants); tools/mutate_kernels.py puts a mutant's shrunk build here


def shrunk(name):
    """(path of the shrunk emulated library, its constants as capacity.constants reads them back)"""
    if name not in LIBS:
        texts = capacity.shrunk_sources(**BUILDS[name])
        k = capacity.constants(texts)
        for key, v in BUILDS[name].items():
            assert k[key] == v, key
        LIBS[name] = (simt_emu.build_library(texts), k)
    return LIBS[name]


# scan kernel (simt_emu.EmuEngine) -> the quality pass capacity.RQ_OPT takes with it
SCANS = {"jit": "scan", "fast": "read_qual"}


def engine(name, opt, scan="jit"):
    return simt_emu.EmuEngine(opt, scan=scan, lib=shrunk(name)[0])


def test_constants_are_read_from_the_sources():
    """every constant and grid cap is found in the product sources, and the shrunk texts change only what was asked"""
    k = capacity.constants()
    assert set(capacity.DEFINES) <= set(k)
    assert k["k_kmer_fix_BLOCKS"] % k["FPL_NUM_SMS"] == 0 and k["k_fastq_pack_WARPS"] == k["k_emit_copy_WARPS"] == 8
    assert set(capacity.GRID_CAPS) == {key[:-7] for key in k if key.endswith("_BLOCKS")} and "k_read_qual_exc" in capacity.GRID_CAPS
    renamed = {"fpl_stats.cu": open(capacity.CSRC + "/fpl_stats.cu").read().replace("void launch_read_qual_exc(", "void launch_rq_exc(")}
    with pytest.raises(AssertionError, match="launch_read_qual_exc"):
        capacity.constants(renamed)
    assert k["CS_GROUP"] <= 4095 and 127 * k["CS_GROUP"] < (1 << 20)       # the packed counter's fields
    s = capacity.constants(capacity.shrunk_sources(**BUILDS["group_of_2.5_stages"]))
    for key in k:
        if key in BUILDS["group_of_2.5_stages"]:
            continue
        if key.endswith("_BLOCKS"):
            assert s[key] * k["FPL_NUM_SMS"] == k[key], key
        else:
            assert s[key] == k[key], key
    with pytest.raises(KeyError):
        capacity.shrunk_sources(NOT_A_CONSTANT=1)


@pytest.mark.parametrize("build", sorted(BUILDS))
@pytest.mark.parametrize("optset", sorted(capacity.CS_SETS))
def test_cycle_stats_staging_rounds_and_groups(build, optset):
    """pre-filter segment counts CS_STAGE - 1 .. 2 * CS_GROUP + 1: ties of equal length, reads that stop reaching the second
    tile exactly at a staging round's end and three past it; the post-filter list of the same reads by the plain (no -N/-b)
    or the 5-mer (--mask) variant"""
    lib, k = shrunk(build)
    opt = capacity.CS_SETS[optset]
    for count in capacity.cycle_counts(k):
        for kind in ("ties", "falloff", "falloff_plus"):
            if kind != "ties" and count <= k["CS_STAGE"] + 3:
                continue
            batch = capacity.cycle_stats_batch(k, count, kind, seed=count)
            capacity.compare_with_oracle(engine(build, opt), opt, batch, f"{build}/{optset}/{count}/{kind}",
                                         qual_pass=capacity.CS_PASS[optset])


@pytest.mark.parametrize("build", sorted(BUILDS))
@pytest.mark.parametrize("optset", sorted(capacity.CS_SETS))
def test_cycle_stats_post_filter_counts(build, optset):
    """post-filter lists of exactly CS_STAGE - 1 .. 2 * CS_GROUP + 1 passing segments, none of them on a 16-byte boundary"""
    lib, k = shrunk(build)
    opt = capacity.CS_SETS[optset]
    for count in capacity.cycle_counts(k):
        batch = capacity.post_count_batch(k, count, seed=count)
        exp = capacity.compare_with_oracle(engine(build, opt), opt, batch, f"{build}/{optset}/post{count}", qual_pass=capacity.CS_PASS[optset])
        assert capacity.passing_segments(exp) == count


@pytest.mark.parametrize("build", ["group_of_2_stages"])
def test_kmer_fix_long_range_list(build):
    """blocks with exactly KF_LIST, KF_LIST + 1 and more long removed ranges (the ones past the list go to a lone warp), and
    a batch past the grid cap whose warps loop onto more reads with long ranges"""
    lib, k = shrunk(build)
    opt = capacity.KF_OPT
    batch = capacity.kmer_fix_batch(k, 5)
    res = capacity.compare_with_oracle(engine(build, opt), opt, batch, f"{build}/kmer_fix", qual_pass="scan")
    per_block = capacity.long_ranges(batch, res, k["KF_LONG"]).reshape(-1, k["KF_WARPS"]).sum(axis=1)
    assert list(per_block[:3]) == capacity.kf_targets(k) and per_block[0] == k["KF_LIST"]
    batch = capacity.kmer_fix_loop_batch(k, 6)
    res = capacity.compare_with_oracle(engine(build, opt), opt, batch, f"{build}/kmer_fix_loop", qual_pass="scan")
    assert batch.n_reads > k["KF_WARPS"] * k["k_kmer_fix_BLOCKS"]
    assert capacity.long_ranges(batch, res, k["KF_LONG"]).sum() == 2 * 3 * k["KF_WARPS"]


@pytest.mark.parametrize("build", ["group_of_2_stages"])
def test_read_qual_long_list_and_stride(build):
    """k_read_qual (the fast scan): RQ_LIST + 1 long reads in one block and exactly RQ_LIST in the next; then more reads than
    the capped grid has warps.  On the jit scan the same batches are parity cases of k_read_qual_exc, whose list has another
    order"""
    lib, k = shrunk(build)
    opt = capacity.RQ_OPT
    batch = capacity.read_qual_batch(k, 7)
    assert (batch.lens > k["RQ_LONG"]).sum() == 2 * k["RQ_LIST"] + 1
    stride = capacity.stride_batch(k, 8)
    assert stride.n_reads > k["RQ_WARPS"] * k["k_read_qual_BLOCKS"]
    for scan, qual_pass in SCANS.items():
        capacity.compare_with_oracle(engine(build, opt, scan), opt, batch, f"{build}/read_qual/{scan}", qual_pass=qual_pass)
        capacity.compare_with_oracle(engine(build, opt, scan), opt, stride, f"{build}/stride/{scan}", qual_pass=qual_pass)


@pytest.mark.parametrize("build", ["group_of_2_stages"])
def test_read_qual_exc_list(build):
    """k_read_qual_exc on both sides of its limits, for every order of its list: a list of long reads of every kind of which
    block 0 meets more than RQ_LIST (the rest go to lone warps); long listed reads among short ones; a list longer than the
    capped grid has warps, with quality bytes over 1..127 (many windows taken out of the post-filter sums per flush); an
    empty list and one of every read"""
    lib, k = shrunk(build)
    opt = capacity.RQ_OPT

    def check(batch, what):
        res = capacity.compare_with_oracle(engine(build, opt), opt, batch, f"{build}/{what}", qual_pass="scan")
        return res, capacity.listed(res)

    batch = capacity.exc_overflow_batch(k, 21)
    res, listed = check(batch, "exc_overflow")
    assert listed.sum() >= capacity.exc_min_overflow(k) and (batch.lens[listed] > k["RQ_LONG"]).all()
    assert batch.n_reads >= k["RQ_WARPS"] * k["k_read_qual_exc_BLOCKS"]         # the grid is at its cap
    capacity.check_exc_kinds(batch, res, k)
    batch = capacity.exc_kinds_batch(k, 22)
    capacity.check_exc_kinds(batch, check(batch, "exc_kinds")[0], k)
    batch = capacity.exc_loop_batch(k, 23)
    res, listed = check(batch, "exc_loop")
    assert listed.sum() > k["RQ_WARPS"] * k["k_read_qual_exc_BLOCKS"]
    capacity.check_exc_kinds(batch, res, k)
    for every in (False, True):
        batch = capacity.exc_list_batch(k, 24 + every, every)
        assert check(batch, f"exc_list/every{int(every)}")[1].sum() == (batch.n_reads if every else 0)


@pytest.mark.parametrize("build", ["group_of_2_stages"])
def test_text_path_more_records_than_warps(build):
    lib, k = shrunk(build)
    for name, opt in (("rq", capacity.RQ_OPT), ("plain", capacity.CS_SETS["plain"])):
        capacity.check_text(engine(build, opt), opt, capacity.text_batch(k, 9), f"{build}/text/{name}")


def test_long_range_count_mirrors_the_kernel():
    """capacity.long_ranges on hand-made records: a failed read, trimmed ends, a split with its gap"""
    from fastplong_b200 import PackedBatch, abi
    lens = np.array([5000, 5000, 5000, 30], np.int32)
    b = PackedBatch(np.zeros(15200, np.uint8), np.zeros(15200, np.uint8), np.array([0, 5008, 10016, 15024], np.int64), lens)
    res = np.zeros(4, dtype=abi.RESULT_DTYPE)
    res[0]["n_segments"], res[0]["seg_result"][0] = 1, abi.FAIL_LENGTH
    res[1]["n_segments"], res[1]["seg_lo"][0], res[1]["seg_len"][0] = 1, 2100, 500
    res[2]["n_segments"] = 2
    res[2]["seg_lo"][:2], res[2]["seg_len"][:2] = (10, 2500), (400, 2400)
    assert list(capacity.long_ranges(b, res, 2048)) == [1, 2, 1, 0]
