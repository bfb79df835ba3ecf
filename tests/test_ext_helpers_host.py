"""The --mask / --break stage's own helpers (fpl_ext.cu), cut out of the source and compiled for the host
(tests/device_helpers.py:load_ext): its copy of passFilter, the region detection, the break walk and the clamp of
maskRegionWithN, against plain transcriptions of the reference (src/filter.cpp:12-128, src/read.cpp:217-262) over input spaces
the GPU tests can only sample: every tie of the filter thresholds, and every quality string of up to 10 bytes over the bytes
just below, on and just above a window's threshold (and one below '!') for every window of 1..12 bases.  Last, which edge of
the stage each set of cases.MASK_BREAK_EDGE_SETS reaches on cases.mask_break_edge_batch, read off the oracle's lists."""
import ctypes as C

import numpy as np
import pytest

import cases
import device_helpers
from fastplong_b200 import abi
from oracle_lib import OracleEngine
from test_device_helpers_host import _reference_pass_filter, pass_filter_tie_space


@pytest.fixture(scope="module")
def ext():
    return device_helpers.load_ext()


def test_pass_filter_ext_on_every_tie(ext):
    """k_ext_filter's pass_filter_ext against the reference's double forms, and against k_final's pass_filter, over the tie
    space of test_pass_filter_integer_forms_on_every_tie: the two integer copies cannot drift apart."""
    scan = device_helpers.load()
    n = 0
    for o, rlen, lowq, nn, totalq, diff in pass_filter_tie_space():
        got = ext.e_pass_filter(C.byref(o), rlen, lowq, nn, totalq, diff)
        assert got == _reference_pass_filter(o, rlen, lowq, nn, totalq, diff), (rlen, lowq, nn, totalq, diff)
        assert got == scan.h_pass_filter(C.byref(o), rlen, lowq, nn, totalq, diff), (rlen, lowq, nn, totalq, diff)
        n += 1
    assert n > 150000


# ---- the reference, transcribed line by line ----
def _char(b):
    return b - 256 if b >= 128 else b           # qualstr is a `const char*` (signed on the reference's targets)


def detect_low_quality_regions(qual, window_size, quality):
    """Filter::detectLowQualityRegions (src/filter.cpp:83-128).  The prep loop starts at `start` but stops at
    window_size - 1 (an absolute bound): after the first region it adds nothing and the running sum restarts from 0."""
    results = []
    if len(qual) == 0 or window_size <= 0:
        return results
    l = len(qual)
    q = [_char(b) for b in qual]
    start = 0
    while start + window_size <= l:
        total = 0
        i = start
        while i < window_size - 1 and i < l:
            total += q[i]
            i += 1
        window_start = -1
        s = start
        while s + window_size < l:
            if total < (33 + quality) * window_size:
                window_start = s
                break
            total += q[s + window_size]
            total -= q[s]
            s += 1
        if window_start == -1:
            break
        e = window_start
        while e + window_size < l:
            total += q[e + window_size]
            total -= q[e]
            if total >= (33 + quality) * window_size:
                break
            e += 1
        results.append((window_start, e + window_size - 1))
        start = e + window_size
    return results


def break_by_regions(length, regions):
    """Read::breakByRegions (src/read.cpp:227-262): the pieces as (lo, len, k) with name prefix "r<k>-"."""
    out, last_end = [], -1
    for i, (start, end) in enumerate(regions):
        if start < 0:
            start = 0
        if end >= length:
            end = length - 1
        if start > end or start >= length:
            continue
        if start > last_end + 1:
            out.append((last_end + 1, start - last_end - 1, i + 1))
        last_end = end
    if last_end < length - 1:
        out.append((last_end + 1, length - last_end - 1, len(regions) + 1))
    return out


def mask_region_with_n(seq, start, length):
    """Read::maskRegionWithN (src/read.cpp:217-225) on a bytearray; the range it painted, or None"""
    if start < 0 or length <= 0 or start >= len(seq):
        return None
    if start + length > len(seq):
        length = len(seq) - start
    seq[start:start + length] = b"N" * length
    return start, length


def expected(qual, w, Q):
    """what the stage does with one read for --break / --mask at window w, quality Q (src/seprocessor.cpp:235-262): the regions,
    walk_break's return (-1 when there is no region: the read stays whole) and pieces, the masked ranges and sequence"""
    regions = detect_low_quality_regions(qual, w, Q)
    pieces = break_by_regions(len(qual), regions) if regions else None
    seq = bytearray(b"A" * len(qual))
    masked = [m for m in (mask_region_with_n(seq, a, b - a + 1) for a, b in regions) if m is not None]
    return regions, pieces, masked, bytes(seq)


# ---- the same transcription run in lock step over many strings at once (numpy), for the exhaustive space ----
def _lockstep(q, w, Q, maxr):
    """q: (N, l) signed quality values.  Every string runs the loops of detect_low_quality_regions / break_by_regions /
    mask_region_with_n; a string takes part in a step only where its own loop would be at that index."""
    N, l = q.shape
    nreg = np.zeros(N, np.int64)
    reg = np.full((N, maxr, 2), -7, np.int64)
    rows = np.arange(N)
    if l > 0 and w > 0:
        need = (33 + Q) * w
        start = np.zeros(N, np.int64)
        live = np.ones(N, bool)
        while True:
            live &= start + w <= l
            if not live.any():
                break
            total = np.zeros(N, np.int64)
            for i in range(min(w - 1, l)):                          # for (i = start; i < w - 1 && i < l; i++)
                total += np.where(live & (i >= start), q[:, i], 0)
            ws = np.full(N, -1, np.int64)
            look = live.copy()
            for s in range(l - w):                                  # for (s = start; s + w < l; s++)
                at = look & (s >= start)
                hit = at & (total < need)
                ws[hit] = s
                look &= ~hit
                total += np.where(at & ~hit, q[:, min(s + w, l - 1)] - q[:, s], 0)
            live &= ws >= 0
            e, grow = ws.copy(), live.copy()
            for x in range(l - w):                                  # for (e = ws; e + w < l; e++)
                at = grow & (e == x)
                total += np.where(at, q[:, min(x + w, l - 1)] - q[:, x], 0)
                stop = at & (total >= need)
                grow &= ~stop
                e = np.where(at & ~stop, x + 1, e)
            k = nreg[live]
            assert (k < maxr).all()
            reg[rows[live], k, 0] = ws[live]
            reg[rows[live], k, 1] = e[live] + w - 1
            nreg += live
            start = np.where(live, e + w, start)
    # break_by_regions, compacted per string
    npc = np.where(nreg > 0, 0, -1)
    pc = np.full((N, maxr, 3), -7, np.int64)
    last_end = np.full(N, -1, np.int64)

    def put(where, lo, ln, k):
        pc[rows[where], npc[where], 0] = lo[where]
        pc[rows[where], npc[where], 1] = ln[where]
        pc[rows[where], npc[where], 2] = k[where]
        npc[where] += 1
    nmax = int(nreg.max(initial=0))
    for k in range(nmax):
        valid = nreg > k
        start = np.maximum(reg[:, k, 0], 0)
        end = np.where(reg[:, k, 1] >= l, l - 1, reg[:, k, 1])
        act = valid & ~((start > end) | (start >= l))
        put(act & (start > last_end + 1), last_end + 1, start - last_end - 1, np.full(N, k + 1))
        last_end = np.where(act, end, last_end)
    put((nreg > 0) & (last_end < l - 1), last_end + 1, l - last_end - 1, nreg + 1)
    # mask_region_with_n(first, last - first + 1)
    nmask = np.zeros(N, np.int64)
    mreg = np.full((N, maxr, 2), -7, np.int64)
    seq = np.full((N, l), ord("A"), np.uint8)
    cols = np.arange(l)
    for k in range(nmax):
        a, ln = reg[:, k, 0], reg[:, k, 1] - reg[:, k, 0] + 1
        act = (nreg > k) & ~((a < 0) | (ln <= 0) | (a >= l))
        ln = np.where(a + ln > l, l - a, ln)
        mreg[rows[act], nmask[act], 0] = a[act]
        mreg[rows[act], nmask[act], 1] = ln[act]
        nmask += act
        seq[act[:, None] & (cols[None, :] >= a[:, None]) & (cols[None, :] < (a + ln)[:, None])] = ord("N")
    return nreg, reg, npc, pc, nmask, mreg, seq


def _device(ext, qs, w, Q, maxr):
    """the fpl_ext.cu helpers over the rows of qs (uint8, (N, l))"""
    N, l = qs.shape
    assert l < 4096
    qs = np.ascontiguousarray(qs)
    nreg, npc, nmask = (np.zeros(N, np.int32) for _ in range(3))
    reg, pc, mreg = (np.full((N, maxr, k), -7, np.int32) for k in (2, 3, 2))
    mseq = np.zeros((N, max(l, 1)), np.uint8)
    ext.e_regions(qs.ctypes.data, N, l, w, Q, maxr, nreg.ctypes.data, reg.ctypes.data, npc.ctypes.data, pc.ctypes.data,
                  nmask.ctypes.data, mreg.ctypes.data, mseq.ctypes.data)
    return nreg, reg, npc, pc, nmask, mreg, mseq[:, :l]


FIELDS = ("regions", "region list", "walk_break return", "pieces", "mask count", "masked ranges", "masked sequence")


def _compare(got, exp, qs, w, Q):
    for name, g, e in zip(FIELDS, got, exp):
        if not np.array_equal(g, e):
            bad = np.nonzero((g != e).reshape(len(g), -1).any(axis=1))[0]
            i = int(bad[0])
            raise AssertionError(f"w={w} Q={Q} {name} differ on {len(bad)} strings, first {list(qs[i])}: {g[i].tolist()} vs {e[i].tolist()}")


def _alphabet(Q):
    """the bytes just below, on and just above 33 + Q, and one below '!'"""
    return np.array([33 + Q - 1, 33 + Q, 33 + Q + 1, 20], np.uint8)


def _strings(al, l):
    """every string of l bytes over the alphabet al, one per row"""
    idx = np.arange(len(al) ** l)
    return al[(idx[:, None] // len(al) ** np.arange(l)[None, :]) % len(al)]


@pytest.mark.parametrize("Q", [1, 15, 93])
def test_regions_pieces_and_masks_on_every_short_string(ext, Q):
    """Every quality string of 0..10 bytes over _alphabet(Q), and of 0..8 bytes over that alphabet with byte 127 added, every
    window of 1..12 bases: detect_regions' regions, walk_break's pieces (lo, len, r<k> index) and its -1 "no region" return,
    k_ext_mask_count's count and k_ext_mask_emit's clamped ranges and painted bases, against the reference's loops run in lock
    step.  The rolling sum of the reference holds w - 1 bytes (the prep loop stops at w - 1, the roll skips base s + w - 1), so
    over bytes near 33 + Q alone the first window is always low and the region runs to the end; byte 127 is what lets a read
    keep a head piece or a region end early."""
    reached = {"head piece": 0, "no head piece": 0, "region not on the last base": 0, "region on the last base": 0,
               "tail piece shorter than w": 0, "later region": 0, "vanished": 0, "no region": 0}
    for al, top in ((_alphabet(Q), 10), (np.unique(np.append(_alphabet(Q), 127)).astype(np.uint8), 8)):
        for l in range(0, top + 1):
            qs = _strings(al, l)
            q = qs.astype(np.int64)
            maxr = l + 2
            rows = np.arange(len(q))
            for w in range(1, 13):
                exp = _lockstep(q, w, Q, maxr)
                _compare(_device(ext, qs, w, Q, maxr), exp, qs, w, Q)
                nreg, reg, npc, pc = exp[:4]
                has = nreg > 0
                last = reg[rows, np.maximum(nreg - 1, 0), 1]
                tail = pc[rows, np.maximum(npc - 1, 0)]
                reached["head piece"] += int((has & (reg[:, 0, 0] > 0)).sum())
                reached["no head piece"] += int((has & (reg[:, 0, 0] == 0)).sum())
                reached["region on the last base"] += int((has & (last == l - 1)).sum())
                reached["region not on the last base"] += int((has & (last < l - 1)).sum())
                reached["tail piece shorter than w"] += int(((npc > 0) & (tail[:, 1] < w) & (tail[:, 2] == nreg + 1)).sum())
                reached["later region"] += int((nreg > 1).sum())
                reached["vanished"] += int((npc == 0).sum())
                reached["no region"] += int((npc == -1).sum())
    if Q == 93:     # 126 * w over w - 1 bytes of at most 127: every first window is low, every region runs to the end
        assert reached["head piece"] == reached["region not on the last base"] == reached["later region"] == 0, reached
        assert reached["vanished"] and reached["no region"], reached
    else:
        assert all(reached.values()), reached


def test_lockstep_transcription_is_the_plain_one():
    """the lock-step form above against the line-by-line transcription, string by string"""
    rng = np.random.default_rng(3)
    for Q in (1, 15, 93):
        al = _alphabet(Q)
        for l in (0, 1, 2, 3, 5, 8, 13, 40):
            qs = al[rng.integers(0, 4, size=(300, l))]
            for w in (1, 2, 3, 5, 12, 40, 41):
                maxr = l + 2
                nreg, reg, npc, pc, nmask, mreg, seq = _lockstep(qs.astype(np.int64), w, Q, maxr)
                for i in range(len(qs)):
                    regions, pieces, masked, mseq = expected(bytes(qs[i]), w, Q)
                    assert [tuple(r) for r in reg[i, :nreg[i]].tolist()] == regions
                    assert (npc[i] == -1) if pieces is None else [tuple(p) for p in pc[i, :npc[i]].tolist()] == pieces
                    assert [tuple(m) for m in mreg[i, :nmask[i]].tolist()] == masked and seq[i].tobytes() == mseq


@pytest.mark.parametrize("Q", [1, 15, 20, 93])
def test_regions_on_random_long_strings(ext, Q):
    """longer strings, one transcription call per string: blocks of good and bad bytes around the threshold, runs below '!',
    windows much shorter and much longer than the read"""
    rng = np.random.default_rng(Q)
    for case in range(150):
        l = int(rng.integers(1, 400))
        w = int(rng.choice([1, 2, 3, 4, 5, 7, 10, 12, 30, 64, l, l - 1, l + 1]))
        if w <= 0:
            continue
        if case % 3 == 0:
            q = rng.integers(max(1, 33 + Q - 3), min(127, 33 + Q + 3) + 1, size=l)
        elif case % 3 == 1:
            q = np.where(rng.random(l) < 0.3, rng.integers(1, 33, size=l), rng.integers(33 + Q, 128, size=l))
        else:
            q = np.concatenate([rng.integers(1, 128, size=int(k)) for k in rng.integers(1, 60, size=20)])[:l]
            q = np.resize(q, l)
        qs = q.astype(np.uint8).reshape(1, l)
        maxr = l + 2
        nreg, reg, npc, pc, nmask, mreg, seq = _device(ext, qs, w, Q, maxr)
        regions, pieces, masked, mseq = expected(qs[0].tobytes(), w, Q)
        assert [tuple(r) for r in reg[0, :nreg[0]].tolist()] == regions, (case, l, w)
        assert (npc[0] == -1) if pieces is None else [tuple(p) for p in pc[0, :npc[0]].tolist()] == pieces, (case, l, w)
        assert [tuple(m) for m in mreg[0, :nmask[0]].tolist()] == masked and seq[0].tobytes() == mseq, (case, l, w)


# ---- what cases.mask_break_edge_batch reaches, read off the oracle's lists (tests/test_gpu_mask_break_edges.py runs it) ----
def _pieces(opt, batch):
    """the oracle's records, output reads and mask regions, and per output read (segment, masked sequence as k_ext_filter sees
    it, quality values, the masked byte behind the read's end or None)"""
    o = OracleEngine(opt)
    res = o.process(batch)
    segs, regs = o.segments(), o.mask_regions()
    mseq = batch.seq.copy()
    for r in regs:
        a = int(batch.offsets[r["read"]]) + int(r["lo"])
        mseq[a:a + int(r["len"])] = ord("N")
    out = []
    for s in segs:
        a = int(batch.offsets[s["read"]]) + int(s["lo"])
        n = int(s["len"])
        end = int(s["lo"]) + n
        nxt = int(mseq[a + n]) if end < int(batch.lens[s["read"]]) else None
        out.append((s, mseq[a:a + n].tobytes(), batch.qual[a:a + n].astype(np.int64), nxt))
    o.close()
    return res, segs, regs, out


def _diff(sq):
    return sum(sq[i] != sq[i + 1] for i in range(len(sq) - 1))


def test_edge_batch_reaches_every_edge():
    """each edge tests/test_gpu_mask_break_edges.py is meant to reach, found in the oracle's lists for that set"""
    batch = cases.mask_break_edge_batch()
    assert batch.n_reads % 8 and batch.n_reads % 256 and 2 * batch.n_reads > 4 * 256      # k_ext_count / _emit: several blocks
    S = cases.MASK_BREAK_EDGE_SETS

    opt = S["break_lengths_mean"]
    res, segs, regs, pcs = _pieces(opt, batch)
    by_len = {}
    for s, sq, q, nxt in pcs:
        by_len.setdefault(int(s["len"]), set()).add(int(s["result"]))
    assert abi.FAIL_LENGTH in by_len[opt.length_required - 1]
    assert by_len[opt.length_required] - {abi.FAIL_LENGTH} and by_len[opt.length_limit] - {abi.FAIL_TOO_LONG}
    assert abi.FAIL_TOO_LONG in by_len[opt.length_limit + 1] and by_len[opt.length_limit + 1] - {abi.FAIL_TOO_LONG} <= {abi.FAIL_QUALITY}
    means = [(int((q - 33).sum()), len(q), int(s["result"])) for s, sq, q, nxt in pcs if len(q)]
    assert any(t < 0 for t, n, r in means)                                                  # a negative totalQual
    assert any(int(t / n) == opt.mean_qual for t, n, r in means)                            # the mean exactly on --mean_qual
    assert any(int(t / n) == opt.mean_qual - 1 and r == abi.FAIL_QUALITY for t, n, r in means)

    opt = S["mask_n_limits"]
    res, segs, regs, pcs = _pieces(opt, batch)
    nn = [(sq.count(b"N"), len(sq), int(s["result"]), sq, q) for s, sq, q, nxt in pcs]
    assert len(regs) and any(c == opt.n_base_limit and r == abi.PASS_FILTER for c, n, r, sq, q in nn)   # N count on -n, masked
    assert any(c == opt.n_base_limit + 1 and r == abi.FAIL_N_BASE for c, n, r, sq, q in nn)
    assert any(c * 100 == n * opt.n_percent_limit and c for c, n, r, sq, q in nn)                      # the N share on the limit
    qq = 33 + opt.qualified_quality_phred
    ties = [(int((q < qq).sum()), n, r) for c, n, r, sq, q in nn if (q == qq).any()]
    assert any(lo * 100 == n * opt.unqualified_percent_limit for lo, n, r in ties)                     # -u on the limit ...
    assert any((lo + int((q == qq).sum())) * 100 > n * opt.unqualified_percent_limit >= lo * 100 and r == abi.PASS_FILTER
               for (lo, n, r), (c, _, _, sq, q) in zip(ties, [x for x in nn if (x[4] == qq).any()]))  # ... decided by bytes on -q

    opt = S["mask_break_cplx"]
    res, segs, regs, pcs = _pieces(opt, batch)
    pct = opt.complexity_threshold
    assert {1, 2} <= {int(s["len"]) for s, sq, q, nxt in pcs}
    tie = [(sq, nxt, int(s["break_index"])) for s, sq, q, nxt in pcs if len(sq) > 1 and _diff(sq) * 100 == pct * (len(sq) - 1)]
    assert any(b"NN" in sq for sq, nxt, bi in tie)                                          # a tie on the masked copy
    assert any(nxt is not None and nxt != sq[-1] and bi for sq, nxt, bi in tie)            # the byte behind the piece differs
    assert int(res["n_segments"].min()) == 0                                                # vanishing reads

    opt = S["cplx_only_w1"]
    res, segs, regs, pcs = _pieces(opt, batch)
    results = {int(s["result"]) for s, sq, q, nxt in pcs}
    assert results == {abi.PASS_FILTER, abi.FAIL_COMPLEXITY} and len(pcs) % 8
    assert any(int(r["lo"]) == int(s["lo"]) for r in regs for s in segs[segs["read"] == r["read"]][:1])   # a mask region at base 0

    opt = S["break_w1_qual_only"]
    res, segs, regs, pcs = _pieces(opt, batch)
    assert {abi.PASS_FILTER, abi.FAIL_QUALITY, abi.FAIL_N_BASE} <= {int(s["result"]) for s, sq, q, nxt in pcs}
    one_base = [r for r in range(batch.n_reads)
                if any(a == b for a, b in detect_low_quality_regions(batch.read(r)[1], 1, opt.break_mean_quality))]
    assert any(int(res["n_segments"][r]) for r in one_base)                                # a one-base region before a piece

    opt = S["split_break_mask"]
    res, segs, regs, pcs = _pieces(opt, batch)
    assert int(res["n_segments"].max()) >= 3                                                # more than the two inline slots
    assert ((segs["split_side"] == 1) & (segs["break_index"] > 0)).any()
    assert ((segs["split_side"] == 2) & (segs["break_index"] > 0)).any()
    assert (segs["len"] > 32).any() and (segs["result"] == abi.PASS_FILTER).any()
    # median ties: a passing even-length piece whose running quality count lands exactly on half
    def half_tie(q):
        h = np.bincount(q & 127, minlength=128).cumsum()
        return len(q) % 2 == 0 and (h == len(q) // 2).any()
    assert any(half_tie(q) for s, sq, q, nxt in pcs if int(s["result"]) == abi.PASS_FILTER)
