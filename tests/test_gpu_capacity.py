"""The statistics and text kernels on both sides of their fixed capacities, at the sizes the product's constants put them
(tests/capacity.py reads every constant and grid cap from the sources): k_cycle_stats around CS_STAGE and CS_GROUP segments,
pre- and post-filter, plain and 5-mer variant; its packed count << 20 | sum(q) counter at its fullest (CS_GROUP equal
reads at quality byte 127); k_kmer_fix with KF_LIST and KF_LIST + 1 long removed ranges in a block and past its grid cap;
k_read_qual with RQ_LIST and RQ_LIST + 1 reads over RQ_LONG in a block and past its grid cap; k_read_qual_exc with long
listed reads of every kind, a list longer than its capped grid has warps, an empty list and a full one; one FASTQ chunk
with more records than k_fastq_pack and k_emit_copy have warps.  Everything is compared with the oracle: records, both Stats
blocks, counters, the -N/-b lists, the output text.  The k_read_qual batches run on both quality passes — k_read_qual itself
(FPL_NO_JIT=1: k_scan_fast) and k_scan_jit's counts with k_read_qual_exc — and every quality case asserts which one ran.

Runs on the GPU and, with FPL_EMULATE=1, on the emulated library, where the batches of more than a few thousand reads are
skipped: tests/test_capacity_shrunk.py runs the same paths with shrunk constants in the CPU suite."""
import os

import pytest

import capacity

pytestmark = pytest.mark.gpu

EMULATE = os.environ.get("FPL_EMULATE", "") not in ("", "0")
K = capacity.constants()
EMU_MAX_READS = 10000


# scan kernel -> (environment of fpl_create, the quality pass capacity.RQ_OPT takes with it)
SCANS = {"jit": ({}, "scan"), "no_jit": ({"FPL_NO_JIT": "1"}, "read_qual")}


def engine(opt, scan="jit"):
    from fastplong_b200.binding import Engine
    with pytest.MonkeyPatch.context() as mp:
        mp.delenv("FPL_NO_JIT", raising=False)
        for key, v in SCANS[scan][0].items():
            mp.setenv(key, v)
        return Engine(opt)


def emulator_limit(n_reads):
    if EMULATE and n_reads > EMU_MAX_READS:
        pytest.skip(f"{n_reads} reads: too slow for the emulator (tests/test_capacity_shrunk.py covers the path)")


@pytest.mark.parametrize("optset", sorted(capacity.CS_SETS))
@pytest.mark.parametrize("count", capacity.cycle_counts(K))
def test_cycle_stats_staging_rounds_and_groups(count, optset):
    """count pre-filter segments (CS_STAGE - 1 .. 2 * CS_GROUP + 1): equal lengths, and reads that stop reaching the second
    tile exactly at a staging round's end or three past it; the post-filter Stats of the same reads"""
    emulator_limit(count)
    opt = capacity.CS_SETS[optset]
    for kind in ("ties", "falloff", "falloff_plus"):
        if kind != "ties" and count <= K["CS_STAGE"] + 3:
            continue
        batch = capacity.cycle_stats_batch(K, count, kind, seed=count)
        capacity.compare_with_oracle(engine(opt), opt, batch, f"{optset}/{count}/{kind}")


@pytest.mark.parametrize("optset", sorted(capacity.CS_SETS))
@pytest.mark.parametrize("count", capacity.cycle_counts(K))
def test_cycle_stats_post_filter_counts(count, optset):
    """exactly `count` passing segments in the post-filter list, none on a 16-byte boundary"""
    emulator_limit(count)
    opt = capacity.CS_SETS[optset]
    batch = capacity.post_count_batch(K, count, seed=count)
    exp = capacity.compare_with_oracle(engine(opt), opt, batch, f"{optset}/post{count}", qual_pass=capacity.CS_PASS[optset])
    assert capacity.passing_segments(exp) == count


@pytest.mark.parametrize("mixed", [False, True])
def test_packed_counter_at_its_fullest(mixed):
    """2 * CS_GROUP + 1 equal reads at quality byte 127: CS_GROUP per column and 127 * CS_GROUP in the quality sum of group 0,
    pre-filter (5-mer variant) and post-filter (plain variant); with a second base bin and one N per read"""
    batch = capacity.headroom_batch(K, mixed)
    emulator_limit(batch.n_reads)
    capacity.compare_with_oracle(engine(capacity.HEADROOM_OPT), capacity.HEADROOM_OPT, batch, f"headroom/mixed{int(mixed)}")


def test_kmer_fix_long_range_list():
    """blocks with exactly KF_LIST, KF_LIST + 1 and more long removed ranges: cut low-quality heads and tails, failed reads,
    splits whose gap runs from a start to an end adapter"""
    batch = capacity.kmer_fix_batch(K, 5)
    res = capacity.compare_with_oracle(engine(capacity.KF_OPT), capacity.KF_OPT, batch, "kmer_fix", qual_pass="scan")
    per_block = capacity.long_ranges(batch, res, K["KF_LONG"]).reshape(-1, K["KF_WARPS"]).sum(axis=1)
    assert list(per_block[:3]) == capacity.kf_targets(K) and per_block[0] == K["KF_LIST"]


def test_kmer_fix_warps_loop():
    batch = capacity.kmer_fix_loop_batch(K, 6)
    emulator_limit(batch.n_reads)
    assert batch.n_reads > K["KF_WARPS"] * K["k_kmer_fix_BLOCKS"]
    res = capacity.compare_with_oracle(engine(capacity.KF_OPT), capacity.KF_OPT, batch, "kmer_fix_loop", qual_pass="scan")
    assert capacity.long_ranges(batch, res, K["KF_LONG"]).sum() == 2 * 3 * K["KF_WARPS"]


def test_read_qual_long_read_list():
    """k_read_qual (the no_jit scan): RQ_LIST + 1 reads over RQ_LONG at the indices block 0 visits and RQ_LIST at block 1's,
    among empty and 1-base reads.  On the jit scan the same batch is a parity case of k_read_qual_exc, whose list has
    another order"""
    batch = capacity.read_qual_batch(K, 7)
    emulator_limit(batch.n_reads)
    assert (batch.lens > K["RQ_LONG"]).sum() == 2 * K["RQ_LIST"] + 1
    for scan, (_, qual_pass) in SCANS.items():
        capacity.compare_with_oracle(engine(capacity.RQ_OPT, scan), capacity.RQ_OPT, batch, f"read_qual/{scan}", qual_pass=qual_pass)


def test_more_reads_than_the_capped_grids_have_warps():
    batch = capacity.stride_batch(K, 8)
    emulator_limit(batch.n_reads)
    assert batch.n_reads > K["RQ_WARPS"] * K["k_read_qual_BLOCKS"]
    for scan, (_, qual_pass) in SCANS.items():
        capacity.compare_with_oracle(engine(capacity.RQ_OPT, scan), capacity.RQ_OPT, batch, f"stride/{scan}", qual_pass=qual_pass)


def test_read_qual_exc_long_reads_of_every_kind():
    """listed reads over RQ_LONG — dropped by the cut, split with two, one and no passing part, the gap as the largest part,
    a lone right part, an unsplit failing read, a split window well inside the read — few enough for the block-wide list
    (the lone warps behind RQ_LIST take tests/test_capacity_shrunk.py's list: here that is 25 000 reads of 96 KiB)"""
    batch = capacity.exc_kinds_batch(K, 22)
    res = capacity.compare_with_oracle(engine(capacity.RQ_OPT), capacity.RQ_OPT, batch, "exc_kinds", qual_pass="scan")
    capacity.check_exc_kinds(batch, res, K)


def test_read_qual_exc_list_longer_than_the_grid_has_warps():
    """warps loop over the list and a block takes hundreds of windows out of the post-filter sums before its flush"""
    batch = capacity.exc_loop_batch(K, 23)
    emulator_limit(batch.n_reads)
    res = capacity.compare_with_oracle(engine(capacity.RQ_OPT), capacity.RQ_OPT, batch, "exc_loop", qual_pass="scan")
    listed = capacity.listed(res)
    assert listed.sum() > K["RQ_WARPS"] * K["k_read_qual_exc_BLOCKS"] and 2 * (batch.lens[listed] <= K["RQ_LONG"]).sum() > listed.sum()
    capacity.check_exc_kinds(batch, res, K)


@pytest.mark.parametrize("every", [False, True])
def test_read_qual_exc_empty_and_full_list(every):
    batch = capacity.exc_list_batch(K, 24 + every, every)
    res = capacity.compare_with_oracle(engine(capacity.RQ_OPT), capacity.RQ_OPT, batch, f"exc_list/every{int(every)}", qual_pass="scan")
    assert capacity.listed(res).sum() == (batch.n_reads if every else 0)


def test_text_path_more_records_than_warps():
    batch = capacity.text_batch(K, 9)
    emulator_limit(batch.n_reads)
    capacity.check_text(engine(capacity.RQ_OPT), capacity.RQ_OPT, batch, "text")
