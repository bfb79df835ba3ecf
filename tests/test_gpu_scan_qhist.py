"""The quality histograms counted in the adapter scan (k_scan_jit built with FPL_DO_QHIST: the quality or the length
filter is on, so the scan loads the quality bytes anyway, and neither --mask nor --break).

The scan counts every alive read's window and trimmed ends, writes the pre-filter median and keeps the window's median
for k_final.  A read whose one passing segment is its window takes that median; every other read — dropped by the
cut, split (with zero, one or two passing parts), or with a failing segment — goes to k_final's exception list, and
k_read_qual_exc takes its window out of the post-filter sums and counts it the way k_read_qual does.  k_count adds the
per-read sums.  These batches put reads of every exception kind through that path (next to ordinary ones, including
reads past RQ_LONG, which k_read_qual_exc streams block-wide) and compare records, both Stats blocks and the counters
with the oracle; the kernel times say which path ran.  FPL_NO_JIT=1 runs the same cases on k_scan_fast, which keeps
k_read_qual.

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
EXC, FULL = "k_read_qual(exceptions)", "k_read_qual(pre+post)"


def _read(rng, kind, L):
    """one read of an exception kind (or an ordinary one: "plain")"""
    s = bytearray(capacity._bases(rng, L))
    q = bytearray(capacity._quals(rng, L, 20, 40))
    a = L // 2
    if kind == "split2":                         # a start adapter in the middle: two passing parts
        s[a:a + len(S)] = S.encode()
    elif kind == "split1":                       # ... whose left part fails the filter (N bases)
        s[a:a + len(S)] = S.encode()
        s[a // 4:a // 4 + a // 4] = b"N" * (a // 4)
    elif kind == "split0":                       # ... whose two parts both fail
        s[a:a + len(S)] = S.encode()
        s[:] = bytes(b if i % 3 else ord("N") for i, b in enumerate(s))
        s[a:a + len(S)] = S.encode()
    elif kind == "fails":                        # unsplit, the one segment fails the quality filter
        q[:] = capacity._quals(rng, L, 1, 12)
        q[:40] = capacity._q(40, 30)
        q[-40:] = capacity._q(40, 30)
    elif kind == "dead":                         # the quality cut drops it
        q[:] = capacity._q(L, 0)
    elif kind == "cut_head":                     # a long low-quality head that the front cut removes
        h = L // 3
        q[:h] = capacity._q(h, 2)
    elif kind == "short_fails":                  # passes everything but the length filter
        s, q = s[:30], q[:30]
    return bytes(s), bytes(q)


KINDS = ("plain", "split2", "split1", "split0", "fails", "dead", "cut_head", "short_fails")


def exception_batch(seed, n=160, long_reads=True):
    rng = np.random.default_rng(seed)
    reads = []
    for i in range(n):
        kind = KINDS[i % len(KINDS)]
        reads.append(_read(rng, kind, int(rng.integers(400, 3000))))
    reads += [(b"", b""), (b"A", b"5"), (b"C", b"#"), (b"", b"")]
    if long_reads:
        rq_long = capacity.constants()["RQ_LONG"]
        for j, kind in enumerate(("plain", "split2", "split1", "dead", "cut_head")):
            reads.insert(7 * j + 3, _read(rng, kind, rq_long + 1 + 101 * j))
    return pack_reads(reads)


def make_engine(opt, env, monkeypatch):
    from fastplong_b200.binding import Engine
    for k in ("FPL_NO_JIT",):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    g = Engine(opt)
    g.set_timing(True)
    return g


def check_path(g, scan, opt):
    kt = g.kernel_times()
    counts = not (opt.disable_quality_filtering and opt.disable_length_filtering)
    if scan == "jit" and counts and not (opt.mask or opt.break_reads):
        assert kt[EXC][1] > 0 and kt[FULL][1] == 0, kt
    else:
        assert kt[EXC][1] == 0 and kt[FULL][1] > 0, kt


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
