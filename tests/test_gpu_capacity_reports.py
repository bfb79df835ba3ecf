"""The report and merge kernels past their limits at the product's constants (tests/capacity.py reads them from the sources):
the grouping by median over 1 .. 22 chunks of HTML_CHUNK entries, the lists past k_html_capture's and k_html_lenhist's grid caps
(270 336 entries and more), the length statistics' ties and edges, the per-cycle curves at 40 .. 301 cycles and past the grid
caps of k_report_cycles, k_html_bins and k_html_values, fpl_merge_stats over three capacities past its grid cap
(k_emit_batch_copy past its cap: tests/test_gpu_emit_batch.py).  Records, both Stats blocks and the counters against the oracle, both reports against the twins, merges
against one context over the same reads.  tests/test_capacity_shrunk_reports.py runs the same builders at CPU-test sizes.

With FPL_EMULATE=1 on the emulated library, the cases of more than EMU_MAX_ENTRIES list entries or cycles are skipped."""
import os

import pytest

import capacity

pytestmark = pytest.mark.gpu

EMULATE = os.environ.get("FPL_EMULATE", "") not in ("", "0")
K = capacity.constants()
EMU_MAX_ENTRIES = 20000


def engine(opt):
    from fastplong_b200.binding import Engine
    return Engine(opt)


def emulator_limit(n):
    if EMULATE and n > EMU_MAX_ENTRIES:
        pytest.skip(f"{n} entries or cycles: too slow for the emulator (tests/test_capacity_shrunk_reports.py covers the path)")


@pytest.mark.parametrize("which", range(6))
def test_grouping_by_median_across_chunks_and_blocks(which):
    n = capacity.grouping_lengths(K)[which]
    emulator_limit(2 * n)
    opt = capacity.REPORT_OPT
    res, (pre, post) = capacity.report_run(engine(opt), opt, [capacity.grouping_batch(K, n, seed=which)], f"grouping{n}")
    bins = capacity.html_bins(pre)
    assert len(bins) == n and set(bins) == set(range(129))
    assert set(capacity.html_bins(capacity.post_slots(res))) == set(range(128)) | {129}
    if which == 5:
        assert (n + K["HTML_CHUNK"] - 1) // K["HTML_CHUNK"] % 4


@pytest.mark.parametrize("kind", ["slots", "segments_above", "segments_below"])
def test_lists_past_the_capture_cap(kind):
    cap = max(K["k_html_capture_BLOCKS"], K["k_html_lenhist_BLOCKS"]) * 256
    opt = {"slots": capacity.REPORT_OPT, "segments_above": capacity.MASK_OPT, "segments_below": capacity.BREAK_OPT}[kind]
    if kind != "segments_above":
        emulator_limit(cap)
    batch = capacity.capture_cap_batch(K, 3) if kind == "slots" else capacity.segment_batch(K, 4, kind == "segments_above")
    eng = engine(opt)
    capacity.report_run(eng, opt, [batch], f"capture/{kind}")
    if kind == "slots":
        assert batch.n_reads > cap
    else:
        n_segs = len(eng.segments())
        assert (n_segs > batch.n_reads) == (kind == "segments_above")
        assert kind == "segments_above" or (n_segs > cap and batch.n_reads > cap)


@pytest.mark.parametrize("name", sorted(capacity.LENGTH_CASES))
def test_length_statistics_ties_and_edges(name):
    lens, opt = capacity.LENGTH_CASES[name]
    capacity.report_run(engine(opt), opt, [capacity.length_batch(lens, seed=len(name))], f"lengths/{name}")


@pytest.mark.parametrize("which", range(6))
def test_curves_down_sampling_and_past_the_grid_caps(which):
    total = capacity.curve_totals(K)[which]
    emulator_limit(total)
    opt = capacity.CURVE_OPT
    eng = engine(opt)
    capacity.report_run(eng, opt, [capacity.curve_batch(total, seed=total)], f"curves{total}")
    js = eng.report_json()
    assert b'"total_cycles": %d,' % total in js and b'"total_cycles": %d,' % (total - 8) in js
    if which == 4:
        assert total > max(K["k_report_cycles_BLOCKS"], K["k_html_bins_BLOCKS"]) * 256
        assert 11 * (total - 8) > K["k_html_values_BLOCKS"] * 256


def test_merge_three_capacities_past_the_merge_cap():
    """sources of C 1024 (rows == C), 2048 and 16384 (a read of 8.5 kb: more words than k_merge_stats' capped grid has threads)"""
    import test_gpu_merge as M
    batches = capacity.merge_sources(K, seed=9)
    emulator_limit(sum(int(b.lens.sum()) for b in batches) // 100)
    opt = capacity.REPORT_OPT
    srcs = [engine(opt) for _ in batches]
    for e, b in zip(srcs, batches):
        e.keep_read_lists(True)
        e.process(b)
    assert srcs[0].cycles == max(batches[0].lens) == 1024 and len({e.cycles for e in srcs}) == 3
    assert 2 * 16 * int(max(batches[2].lens)) > K["k_merge_stats_BLOCKS"] * 256
    whole = engine(opt)
    _, lists = capacity.report_run(whole, opt, batches, "merge/whole")
    fresh = engine(opt)
    fresh.keep_read_lists(True)
    fresh.merge(*srcs)
    M.assert_equal_contexts(fresh, whole)
    capacity.check_reports(fresh, opt, lists, "merge/fresh")
    into = engine(opt)
    capacity.report_run(into, opt, [batches[1]], "merge/into")
    into.merge(srcs[0], srcs[2])
    whole = engine(opt)
    _, lists = capacity.report_run(whole, opt, [batches[1], batches[0], batches[2]], "merge/whole2")
    M.assert_equal_contexts(into, whole)
    capacity.check_reports(into, opt, lists, "merge/into")

