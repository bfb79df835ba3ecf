"""The quality histograms counted in the adapter scan (k_scan_jit built with FPL_DO_QHIST: the quality or the length
filter is on, so the scan loads the quality bytes anyway, and neither --mask nor --break).

The scan counts every alive read's window and trimmed ends, writes the pre-filter median and keeps the window's median
for k_final.  A read whose one passing segment is its window takes that median; every other read — dropped by the
cut, split (with zero, one or two passing parts), or with a failing segment — goes to k_final's exception list, and
k_read_qual_exc takes its window out of the post-filter sums and counts it the way k_read_qual does.  k_count adds the
per-read sums.  These batches put reads of every exception kind through that path (next to ordinary ones, including
reads past RQ_LONG, which k_read_qual_exc streams block-wide) and compare records, both Stats blocks and the counters
with the oracle; the kernel times say which path ran (capacity.quality_pass).  FPL_NO_JIT=1 runs the same cases on
k_scan_fast, which keeps k_read_qual.  One submission also runs in several tiles (read tiling of a device batch, upload
pieces of a host batch): the exception list restarts per tile and the striped sums are folded once per call.

Runs on the GPU and, with FPL_EMULATE=1, on the emulated library."""
import numpy as np
import pytest

import capacity
import cases
from fastplong_b200 import Options, pack_reads
from oracle_lib import OracleEngine, compare_results, compare_stats

pytestmark = pytest.mark.gpu

S, E = capacity.S, capacity.E
OPT = Options(start_adapter=S, end_adapter=E, cut_front=True, cut_tail=True, length_required=50)
# -Q -L: the scan has no filter counts to take, loads no quality bytes and leaves the histograms to k_read_qual
OPT_QL = Options(start_adapter=S, end_adapter=E, disable_quality_filtering=True, disable_length_filtering=True)
SCANS = {"jit": {}, "no_jit": {"FPL_NO_JIT": "1"}}


def _read(rng, kind, L):
    """one read of an exception kind (or an ordinary one: "plain")"""
    if kind == "short_fails":                    # passes everything but the length filter
        s, q = capacity.decided_read(rng, "plain", L)
        return s[:30], q[:30]
    return capacity.decided_read(rng, kind, L)


KINDS = ("plain", "split", "left_fails", "none_pass", "fails", "dead", "cut_head", "short_fails")


def exception_batch(seed, n=160, long_reads=True):
    rng = np.random.default_rng(seed)
    reads = []
    for i in range(n):
        kind = KINDS[i % len(KINDS)]
        reads.append(_read(rng, kind, int(rng.integers(400, 3000))))
    reads += [(b"", b""), (b"A", b"5"), (b"C", b"#"), (b"", b"")]
    if long_reads:
        rq_long = capacity.constants()["RQ_LONG"]
        for j, kind in enumerate(("plain", "split", "left_fails", "dead", "cut_head")):
            reads.insert(7 * j + 3, _read(rng, kind, rq_long + 1 + 101 * j))
    return pack_reads(reads)


def make_engine(opt, env, monkeypatch):
    from fastplong_b200.binding import Engine
    for k in ("FPL_NO_JIT", "FPL_TILE_MBASES", "FPL_PIECE_MB"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    g = Engine(opt)
    g.set_timing(True)
    return g


def check_path(g, scan, opt):
    counts = not (opt.disable_quality_filtering and opt.disable_length_filtering)
    expected = "scan" if scan == "jit" and counts and not (opt.mask or opt.break_reads) else "read_qual"
    assert capacity.quality_pass(g) == expected, g.kernel_times()


def run(opt, batches, scan, what, monkeypatch):
    """batches: processed one call after the other on the same context (the accumulators add up)"""
    g, o = make_engine(opt, SCANS[scan], monkeypatch), OracleEngine(opt)
    try:
        cyc = 1
        for i, b in enumerate(batches):
            res = g.process(b)
            exp = o.process(b)
            compare_results(res, exp, f"{what}/call{i}")
            cyc = max(cyc, int(b.lens.max()) if b.n_reads else 1)
        for w in (0, 1):
            compare_stats(g.stats(w, cyc), o.stats(w, cyc), f"{what}/stats{w}")
        compare_stats(g.counters(), o.counters(), what + "/counters")
        check_path(g, scan, opt)
        return exp
    finally:
        g.close()


@pytest.mark.parametrize("scan", sorted(SCANS))
def test_exception_kinds(scan, monkeypatch):
    exp = run(OPT, [exception_batch(1)], scan, f"kinds/{scan}", monkeypatch)
    # every exception kind is there (on the oracle's records)
    from fastplong_b200 import abi
    flags, nseg, sr = exp["flags"], exp["n_segments"], exp["seg_result"]
    split = (flags & abi.FLAG_MIDDLE_ADAPTER) != 0
    npass = ((sr == abi.PASS_FILTER) & (np.arange(2)[None, :] < nseg[:, None])).sum(axis=1)
    assert ((flags & abi.FLAG_DROPPED_BY_CUT) != 0).any()
    for k in (0, 1, 2):
        assert (split & (npass == k)).any(), k
    assert (~split & (nseg == 1) & (npass == 0)).any()


@pytest.mark.parametrize("scan", sorted(SCANS))
def test_quiet_filters(scan, monkeypatch):
    """-Q -L: k_read_qual on either scan"""
    run(OPT_QL, [exception_batch(2)], scan, f"QL/{scan}", monkeypatch)


@pytest.mark.parametrize("scan", sorted(SCANS))
def test_several_calls(scan, monkeypatch):
    """one submission split into three calls: the striped sums are folded once per call, the exception list restarts"""
    b = exception_batch(3, n=120, long_reads=False)
    parts = [pack_reads([b.read(i) for i in range(lo, hi)]) for lo, hi in ((0, 50), (50, 51), (51, b.n_reads))]
    run(OPT, parts, scan, f"calls/{scan}", monkeypatch)


@pytest.mark.parametrize("name", sorted(cases.QUALITY_SETS))
@pytest.mark.parametrize("scan", sorted(SCANS))
def test_quality_domain(name, scan, monkeypatch):
    """quality bytes over 1..127 with the quality options at their ends (the --mask / --break sets keep k_read_qual)"""
    run(cases.QUALITY_SETS[name], [cases.quality_domain_batch(5)], scan, f"{name}/{scan}", monkeypatch)


@pytest.mark.parametrize("how", ["tiles", "pieces"])
def test_one_submission_in_several_tiles(how, monkeypatch):
    """one call whose reads run tile by tile — FPL_TILE_MBASES=1 on a device batch, 1 MiB upload pieces of a host batch: the
    exception list restarts and moves on with each tile, the stripes are indexed by the tile's read numbers, one fold"""
    import layouts
    from test_gpu_layout import device_buffers
    b = exception_batch(4, n=2400)
    assert b.n_bases > 4000000
    g = make_engine(OPT, {"tiles": {"FPL_TILE_MBASES": "1"}, "pieces": {"FPL_PIECE_MB": "1"}}[how], monkeypatch)
    o = OracleEngine(OPT)
    try:
        if how == "tiles":
            relaid = layouts.relayout(b, tail=64)
            n_bytes = layouts.end_of_reads(relaid)
            bufs = device_buffers(relaid, n_bytes)
            g.process_device(*(x.data_ptr() for x in bufs), b.n_reads, n_bytes)
            g.sync()
            res = g.fetch_results(b.n_reads)
        else:
            res = g.process(b)
        compare_results(res, o.process(b), how)
        cyc = int(b.lens.max())
        for w in (0, 1):
            compare_stats(g.stats(w, cyc), o.stats(w, cyc), f"{how}/stats{w}")
        compare_stats(g.counters(), o.counters(), how + "/counters")
        check_path(g, "jit", OPT)
        kt = g.kernel_times()
        assert kt[capacity.QUAL_TIMERS["scan"]][1] >= 3 and kt["k_qhist_fold"][1] == 1, kt
    finally:
        g.close()
