"""The report and merge kernels past their limits at CPU-test sizes: the emulated library (tests/simt_emu.py) built with one SM's
grid caps and HTML_CHUNK 40 (no multiple of 32: every chunk ends in a partial warp round) runs tests/capacity.py's report
batches, built from the same shrunk constants.  Each case compares the records, both Stats blocks and the counters with the
oracle, and the JSON and HTML reports with the plain-Python twins (tests/report_twin.py, tests/report_html_twin.py); each
asserts that its batch reaches the path it is there for:
  - the grouping by median (k_html_hist / k_html_scatter) over one chunk, several chunks, one block and six blocks, every bin
    0..129 spread over chunks and blocks, warp rounds of one bin, of distinct bins and of bins 0 / 128 and 1 / 129 side by side,
    entries of one bin of distinct lengths; the post-filter list by both capture paths, and lists past k_html_capture's and
    k_html_lenhist's grid caps;
  - Stats::calcLengthHistogram's ties (median and N50 exactly at half) and edges (only empty reads, one entry, one length, a
    post-filter block without cycles);
  - the per-cycle curves at 40, 41, 300 and 301 cycles and past the grid caps of k_report_cycles, k_html_bins and k_html_values;
  - fpl_merge_stats over three capacities (a source whose longest read fills its capacity, rows == C), into an empty
    destination and into a larger one, past k_merge_stats' grid cap, with the sources' list boundaries inside chunks;
  - k_emit_batch_copy with more output reads than its capped grid has warps."""
import numpy as np
import pytest

import capacity
import simt_emu
from fastplong_b200 import abi

SHRUNK = dict(FPL_NUM_SMS=1, HTML_CHUNK=40)
LIBS = {}            # tools/mutate_kernels.py puts a mutant's shrunk build here


def shrunk():
    """(path of the shrunk emulated library, its constants as capacity.constants reads them back)"""
    if "lib" not in LIBS:
        texts = capacity.shrunk_sources(**SHRUNK)
        k = capacity.constants(texts)
        assert all(k[key] == v for key, v in SHRUNK.items()) and k["HTML_CHUNK"] % 32
        LIBS["lib"] = (simt_emu.build_library(texts), k)
    return LIBS["lib"]


def engine(opt):
    return simt_emu.EmuEngine(opt, lib=shrunk()[0])


def test_grid_caps_cover_every_launch_of_the_sources():
    """every `FPL_NUM_SMS *` of fastplong_b200/csrc/*.cu lies in a launch capacity.GRID_CAPS reads, and a new one does not"""
    assert capacity.uncapped() == []
    k = capacity.constants()
    for kern in ("k_html_capture", "k_html_lenhist", "k_html_bins", "k_report_cycles", "k_merge_stats"):
        assert k[kern + "_BLOCKS"] == 8 * k["FPL_NUM_SMS"] and k[kern + "_WARPS"] == 8, kern
    assert k["k_html_values_BLOCKS"] == k["k_emit_batch_copy_BLOCKS"] == 16 * k["FPL_NUM_SMS"]
    src = open(capacity.CSRC + "/fpl_stats.cu").read()
    new = src + "\nvoid launch_new(int64_t n, cudaStream_t s) { k_new<<<grid_for(n, FPL_NUM_SMS * 4), 256, 0, s>>>(n); }\n"
    assert capacity.uncapped({"fpl_stats.cu": new}) == [("fpl_stats.cu", new.count("\n"))]
    with pytest.raises(AssertionError, match="launch_html_capture"):
        capacity.constants({"fpl_stats.cu": src.replace("void launch_html_capture(", "void launch_capture(")})
    with pytest.raises(AssertionError, match="k_html_values"):
        capacity.constants({"fpl_stats.cu": src.replace("grid_for(11 * T, FPL_NUM_SMS * 16)", "grid_for(11 * T, 2112)")})


@pytest.mark.parametrize("which", range(6))
def test_grouping_by_median_across_chunks_and_blocks(which):
    lib, k = shrunk()
    ch, n = k["HTML_CHUNK"], capacity.grouping_lengths(k)[which]
    opt = capacity.REPORT_OPT
    batch = capacity.grouping_batch(k, n, seed=which)
    res, (pre, post) = capacity.report_run(engine(opt), opt, [batch], f"grouping{n}")
    entries = [pre, capacity.post_slots(res)]
    bins = [capacity.html_bins(e) for e in entries]
    assert len(bins[0]) == n and len(bins[1]) == 2 * n
    for e, b in zip(entries, bins):          # entries of one bin have distinct lengths
        lens = {}
        for (L, m), x in zip(e, b):
            if x < 128:
                lens.setdefault(x, []).append(L)
        assert all(len(v) == len(set(v)) for v in lens.values())
    assert set(bins[1]) - set(bins[0]) == {129}
    rounds = [capacity.warp_rounds(b, ch) for b in bins]
    assert any(len(r) < 32 for r in rounds[0]) and any(len(r) < 32 for r in rounds[1])       # chunks end inside a round
    if which == 5:
        nch = (n + ch - 1) // ch
        assert nch // 4 >= 5 and nch % 4
        assert set(bins[0]) == set(range(129)) and set(bins[1]) == set(range(128)) | {129}
        for x in range(129):    # each bin in several chunks and blocks
            where = {i // ch for i, y in enumerate(bins[0]) if y == x}
            assert len({c // 4 for c in where}) >= 2, x
    if n > 2 * ch:
        assert any(len(r) == 32 and len(set(r)) == 1 for r in rounds[0])
        assert any(len(r) == 32 and len(set(r)) == 32 for r in rounds[0])
    if which == 5:
        assert any({0, 128} <= set(r) for r in rounds[0]) and any({1, 129} <= set(r) for r in rounds[1])


@pytest.mark.parametrize("kind", ["slots", "segments_above", "segments_below"])
def test_lists_past_the_capture_cap(kind):
    """the post-filter list by both capture paths: two slots per record, and the --mask/--break list with more and with fewer
    output reads than reads; the lists past k_html_capture's and k_html_lenhist's capped grids"""
    lib, k = shrunk()
    cap = max(k["k_html_capture_BLOCKS"], k["k_html_lenhist_BLOCKS"]) * 256
    opt = {"slots": capacity.REPORT_OPT, "segments_above": capacity.MASK_OPT, "segments_below": capacity.BREAK_OPT}[kind]
    batch = capacity.capture_cap_batch(k, 3) if kind == "slots" else capacity.segment_batch(k, 4, kind == "segments_above")
    eng = engine(opt)
    res, (pre, post) = capacity.report_run(eng, opt, [batch], f"capture/{kind}")
    assert len(pre) == batch.n_reads
    if kind == "slots":
        assert batch.n_reads > cap and 2 * batch.n_reads > cap
    else:
        n_segs = len(eng.segments())
        assert (n_segs > batch.n_reads) == (kind == "segments_above") and n_segs != batch.n_reads
        assert kind == "segments_above" or (n_segs > cap and batch.n_reads > cap)


@pytest.mark.parametrize("name", sorted(capacity.LENGTH_CASES))
def test_length_statistics_ties_and_edges(name):
    lens, opt = capacity.LENGTH_CASES[name]
    batch = capacity.length_batch(lens, seed=len(name))
    eng = engine(opt)
    res, (pre, post) = capacity.report_run(eng, opt, [batch], f"lengths/{name}")
    assert eng.stats(0)[16 * eng.cycles:][abi.STATS_READS] == len(lens) and max(lens) == max(L for L, _ in pre)
    if name in ("median_tie", "n50_tie"):
        assert capacity.length_ties(lens) == (name == "median_tie", name == "n50_tie")
        assert capacity.length_ties([L for L, _ in post]) == capacity.length_ties(lens)
    if name == "post_empty":
        assert post == [] and b'"total_cycles": 0' in eng.report_json() and b'"total_cycles": 45' in eng.report_json()


@pytest.mark.parametrize("which", range(6))
def test_curves_down_sampling_and_past_the_grid_caps(which):
    lib, k = shrunk()
    total = capacity.curve_totals(k)[which]
    opt = capacity.CURVE_OPT
    eng = engine(opt)
    capacity.report_run(eng, opt, [capacity.curve_batch(total, seed=total)], f"curves{total}")
    js = eng.report_json()
    assert b'"total_cycles": %d,' % total in js and b'"total_cycles": %d,' % (total - 8) in js
    assert total % 32 or which == 5
    assert eng.cycles > total or (which == 5 and eng.cycles == total)
    if which == 4:
        assert min(total, eng.cycles) > max(k["k_report_cycles_BLOCKS"], k["k_html_bins_BLOCKS"]) * 256
        assert 11 * (total - 8) > k["k_html_values_BLOCKS"] * 256


def test_down_sampled_ranges_are_never_empty():
    """k_html_sums' empty-range branch (and the "0.0" k_html_text prints for it) is unreachable: past 300 cycles the x list is
    1..40, then int(40 * 1.05^i) while below the cycles, then the cycles — and int(p * 1.05) > int(p) for every p >= 20, so
    every range holds at least one cycle"""
    import report_html_twin
    pos, last = 40.0, 40
    while pos < 2 ** 31:
        pos *= 1.05
        assert int(pos) > last
        last = int(pos)
    for cycles in list(range(1, 700)) + [2 ** 21 + 1, 270373, 10 ** 7]:
        x = report_html_twin.curve_x(cycles)
        assert x[-1] == cycles and all(b > a for a, b in zip([0] + x, x))


def test_merge_three_capacities_past_the_merge_cap():
    """three sources of C 1024 (its longest read 1024 cycles: rows == C), 2048 and 4096 merged into a fresh destination, which
    grows, and two of them into the context of the third; both equal one context over the same reads in the same order and the
    oracle's Stats, counters and lists"""
    import test_gpu_merge as M
    lib, k = shrunk()
    opt = capacity.REPORT_OPT
    batches = capacity.merge_sources(k, seed=9)
    srcs = [engine(opt) for _ in batches]
    for e, b in zip(srcs, batches):
        e.keep_read_lists(True)
        e.process(b)
    assert srcs[0].cycles == max(batches[0].lens) == 1024 and len({e.cycles for e in srcs}) == 3
    assert all(b.n_reads % k["HTML_CHUNK"] for b in batches)
    assert 2 * 16 * int(max(batches[2].lens)) > k["k_merge_stats_BLOCKS"] * 256
    whole = engine(opt)
    _, lists = capacity.report_run(whole, opt, batches, "merge/whole")
    fresh = engine(opt)
    fresh.keep_read_lists(True)
    assert fresh.cycles == 1024
    fresh.merge(*srcs)
    M.assert_equal_contexts(fresh, whole)
    capacity.check_reports(fresh, opt, lists, "merge/fresh")
    # the 2048-cycle context takes the 1024- and the 4096-cycle one: its own reads come first
    into = engine(opt)
    _, lists = capacity.report_run(into, opt, [batches[1]], "merge/into")
    into.merge(srcs[0], srcs[2])
    whole = engine(opt)
    _, lists = capacity.report_run(whole, opt, [batches[1], batches[0], batches[2]], "merge/whole2")
    M.assert_equal_contexts(into, whole)
    capacity.check_reports(into, opt, lists, "merge/into")


def test_emit_batch_copy_more_reads_than_warps():
    """fpl_emit_batch_device with more output reads than k_emit_batch_copy's capped grid has warps"""
    import test_gpu_emit_batch as EB
    from oracle_lib import OracleEngine
    lib, k = shrunk()
    opt = capacity.CS_SETS["plain"]
    batch = capacity.text_batch(k, 9)
    g = engine(opt)
    o = OracleEngine(opt)
    res = g.process(batch)
    exp_out, exp_failed = EB.expected(opt, batch, o, o.process(batch))
    assert len(exp_out["lens"]) > k["k_emit_batch_copy_BLOCKS"] * k["k_emit_batch_copy_WARPS"]
    out, failed = g.emit_batch(True, device="cpu")
    EB.compare_batch(out, exp_out, "grid/out")
    EB.compare_batch(failed, exp_failed, "grid/failed")
    assert np.count_nonzero(res["n_segments"])
