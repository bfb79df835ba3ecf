"""Output assembly into packed device batches (fpl_emit_batch_device): after any fpl_process_* call the library hands back the
output reads as two valid fpl_batch layouts — `out` and `failed` — with 16-byte slots, zero padding and one fpl_segment per read.
Expected output: the text the Python mirror of the writers (hostside.emit_fastq / emit_fastq_ext, held to the reference binary's
output files by tests/test_oracle_golden.py) makes from the ORACLE's records, with a unique name per read, parsed back into reads;
the side and break index come from the name tags, the window, median and is_r1 from the oracle's list of output reads.  The
buffers are compared whole, padding included.  Runs on the GPU and, with FPL_EMULATE=1, on the emulated library."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import cases
import layouts
from fastplong_b200 import Options, abi, hostside, pack_reads, synth
from oracle_lib import OracleEngine, compare_lists, compare_results, compare_stats

pytestmark = pytest.mark.gpu

EMULATE = os.environ.get("FPL_EMULATE", "") not in ("", "0")
DEVICE = "cpu" if EMULATE else None       # the emulated library's device memory is host memory
CODES = {v: k for k, v in abi.FAILED_TYPES.items()}
OUT_NAME = re.compile(rb"@(?:r(\d+)-)?(?:split-by-adapter-(left|right)-)?q(\d+)$")
FAILED_NAME = re.compile(rb"@q(\d+) (\w+)$")


def engine(opt, monkeypatch=None, env=None):
    from fastplong_b200.binding import Engine
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    try:
        return Engine(opt)
    finally:
        for k in (env or {}):
            monkeypatch.delenv(k)


def oracle_output_reads(opt, o, ores):
    """read -> the oracle's output reads of that read, in order: (lo, len, result, median, side, break_index, is_r1)"""
    per = {}
    if opt.mask or opt.break_reads:
        for s in o.segments():
            per.setdefault(int(s["read"]), []).append(tuple(int(s[f]) for f in ("lo", "len", "result", "median_qual", "split_side",
                                                                                  "break_index", "is_r1")))
        return per
    for i, r in enumerate(ores):
        for k in range(int(r["n_segments"])):
            side = 0
            if r["flags"] & abi.FLAG_MIDDLE_ADAPTER:
                side = 2 if (k == 1 or r["flags"] & abi.FLAG_SEG0_IS_RIGHT) else 1
            per.setdefault(i, []).append((int(r["seg_lo"][k]), int(r["seg_len"][k]), int(r["seg_result"][k]),
                                          int(r["seg_median_qual"][k]), side, 0, int(side == 0)))
    return per


def packed(reads, segs):
    """the expected fpl_batch: reads at 16-byte slots, zero padding, FPL_BATCH_BYTES long (empty: no buffers)"""
    lens = np.array([len(s) for s, _ in reads], np.int32)
    slots = (lens.astype(np.int64) + 15) // 16 * 16
    offsets = np.concatenate([[0], np.cumsum(slots)[:-1]]).astype(np.int64) if len(reads) else np.zeros(0, np.int64)
    n_bytes = int(slots.sum())
    size = abi.batch_bytes(n_bytes) if len(reads) else 0
    seq, qual = np.zeros(size, np.uint8), np.zeros(size, np.uint8)
    for (s, q), o in zip(reads, offsets):
        seq[o:o + len(s)] = np.frombuffer(s, np.uint8)
        qual[o:o + len(q)] = np.frombuffer(q, np.uint8)
    return dict(seq=seq, qual=qual, offsets=offsets, lens=lens, n_bytes=n_bytes,
                segs=np.array(segs, dtype=abi.SEGMENT_DTYPE) if segs else np.zeros(0, abi.SEGMENT_DTYPE), reads=reads)


def expected(opt, batch, o, ores):
    """(out, failed) expected from the writers' text"""
    names = [b"@q%d" % i for i in range(batch.n_reads)]
    if opt.mask or opt.break_reads:
        out_t, failed_t = hostside.emit_fastq_ext(batch, names, ores, o.segments(), o.mask_regions())
    else:
        out_t, failed_t = hostside.emit_fastq(batch, names, ores)
    per = oracle_output_reads(opt, o, ores)
    taken = {}
    res = []
    for text, is_failed in ((out_t, False), (failed_t, True)):
        reads, segs = [], []
        p = 0
        while p < len(text):        # quality bytes may be '\n': the record is cut by the window length
            e = text.index(b"\n", p)
            name, p = text[p:e], e + 1
            if is_failed:
                m = FAILED_NAME.match(name)
                i, code, side, bidx = int(m.group(1)), CODES[m.group(2).decode()], 0, 0
                (lo_, len_, code_, med, _, _, r1), = per[i]          # the read's only output read
                assert code_ == code
                lo, ln = int(ores[i]["trim_lo"]), int(ores[i]["trim_len"])
            else:
                m = OUT_NAME.match(name)
                i, code = int(m.group(3)), abi.PASS_FILTER
                bidx = int(m.group(1)) if m.group(1) else 0
                side = {None: 0, b"left": 1, b"right": 2}[m.group(2)]
                passing = [x for x in per[i] if x[2] == abi.PASS_FILTER]
                lo, ln, _, med, side_, bidx_, r1 = passing[taken.get(i, 0)]
                taken[i] = taken.get(i, 0) + 1
                assert (side_, bidx_) == (side, bidx)
            s, q = text[p:p + ln], text[p + ln + 3:p + 2 * ln + 3]
            assert text[p + ln:p + ln + 3] == b"\n+\n" and text[p + 2 * ln + 3:p + 2 * ln + 4] == b"\n"
            p += 2 * ln + 4
            reads.append((s, q))
            segs.append((i, lo, ln, code, med, side, r1, bidx))
        res.append(packed(reads, segs))
    return res


def compare_batch(got, exp, what):
    hb, segs = got.to_host()
    assert got.n_reads == len(exp["lens"]) and got.n_bytes == exp["n_bytes"], (what, got.n_reads, got.n_bytes, exp["n_bytes"])
    assert np.array_equal(hb.lens, exp["lens"]), what + "/lens"
    assert np.array_equal(hb.offsets, exp["offsets"]), what + "/offsets"
    for f in ("seq", "qual"):
        a, b = getattr(hb, f), exp[f]
        assert a.shape == b.shape, (what, f, a.shape, b.shape)
        if not np.array_equal(a, b):
            k = int(np.flatnonzero(a != b)[0])
            raise AssertionError(f"{what}/{f}: {int((a != b).sum())} bytes differ, first at {k}")
    compare_lists(segs, exp["segs"], what + "/segs")


def fastq_text(batch):
    return b"".join(b"@q%d\n%s\n+\n%s\n" % ((i,) + batch.read(i)) for i in range(batch.n_reads))


def device_buffers(batch, n_bytes):
    """seq, qual, offsets, lens as tensors, the byte buffers exactly FPL_BATCH_BYTES(n_bytes) long"""
    import torch
    dev = torch.device("cpu" if EMULATE else "cuda:0")
    size = abi.batch_bytes(n_bytes)
    out = [torch.from_numpy(batch.seq[:size].copy()).to(dev), torch.from_numpy(batch.qual[:size].copy()).to(dev),
           torch.from_numpy(batch.offsets.astype(np.int64)).to(dev), torch.from_numpy(batch.lens.astype(np.int32)).to(dev)]
    if dev.type == "cuda":
        torch.cuda.synchronize()
    return out


def process(g, batch, entry, keep):
    """run one fpl_process_* entry point on `batch` (whose reads are the canonical ones)"""
    if entry == "host":
        g.process(batch)
    elif entry == "device":
        relaid = layouts.relayout(batch, align=16, order="shuffled", gaps=1, poison="acgt", tail=32, seed=batch.n_reads)
        n_bytes = layouts.end_of_reads(relaid)
        bufs = device_buffers(relaid, n_bytes)
        keep.append(bufs)
        g.process_device(*(t.data_ptr() for t in bufs), relaid.n_reads, n_bytes)
    else:
        got = g.process_fastq(fastq_text(batch))
        assert got is not None and len(got[0]) == batch.n_reads


def check(opt, batch, what, entry="host", monkeypatch=None, env=None):
    """-> (expected out, expected failed) after comparing both with what the library emits"""
    g, o = engine(opt, monkeypatch, env), OracleEngine(opt)
    keep = []
    try:
        process(g, batch, entry, keep)
        ores = o.process(batch)
        exp_out, exp_failed = expected(opt, batch, o, ores)
        out, failed = g.emit_batch(True, device=DEVICE)
        compare_batch(out, exp_out, what + "/out")
        compare_batch(failed, exp_failed, what + "/failed")
        return exp_out, exp_failed
    finally:
        g.close()


def test_every_option_set_on_the_adversarial_batch():
    b = cases.adversarial_batch(3)
    for name in sorted(cases.OPTION_SETS):
        check(cases.OPTION_SETS[name], b, f"{name}/adv")


def test_mask_break_sets():
    """every -N/-b set; between them, failed reads whose output read is r1 (masked bases) and failed reads whose is not"""
    r1, pieces = set(), 0
    for name in sorted(cases.MASK_BREAK_SETS):
        for k, b in enumerate((cases.blocky_quality_batch(77), cases.adversarial_batch(6))):
            exp_out, exp_failed = check(cases.MASK_BREAK_SETS[name], b, f"{name}/{k}")
            r1 |= set(int(x) for x in exp_failed["segs"]["is_r1"])
            pieces += int((exp_out["segs"]["break_index"] > 0).sum())
    assert r1 == {0, 1} and pieces > 0


def test_split_reads_and_seg0_is_right():
    import capacity
    from test_gpu_long_read_decisions import OPT, long_decision_batch
    batch, _ = long_decision_batch(capacity.constants(), 11)
    res = OracleEngine(OPT).process(batch)
    assert (res["flags"] & abi.FLAG_SEG0_IS_RIGHT).any() and (res["flags"] & abi.FLAG_DROPPED_BY_CUT).any()
    exp_out, _ = check(OPT, batch, "split")
    assert set(exp_out["segs"]["split_side"]) == {0, 1, 2}


def test_ont_batch_with_chimeras_and_reads_over_96_kb():
    check(cases.OPTION_SETS["cut_polyx_cplx"], cases.ont_batch(91, n=300, mean=2500, p_chimera=0.3), "ont")
    long_ = synth.ont_like(4, 110000, 31, p_chimera=0.7, p_n=0.001)
    long_ = pack_reads([long_.read(i) for i in range(long_.n_reads)] + [(b"ACGTN" * 7, b"I" * 35)])
    assert long_.lens.max() > 96 * 1024
    for name in ("cut_polyx_cplx", "mask_and_break"):
        opt = cases.OPTION_SETS.get(name) or cases.MASK_BREAK_SETS[name]
        check(opt, long_, f"{name}/long")


def test_quality_sets_on_the_quality_domain_batch():
    b = cases.quality_domain_batch(5)
    for name in sorted(cases.QUALITY_SETS):
        check(cases.QUALITY_SETS[name], b, f"{name}/quality")


def test_empty_all_dropped_and_all_failed():
    opt = cases.OPTION_SETS["default_se"]
    out, failed = check(opt, pack_reads([]), "empty")
    assert len(out["lens"]) == len(failed["lens"]) == 0
    short = pack_reads([(b"ACGTACGTAC"[:k], b"IIIIIIIIII"[:k]) for k in range(1, 10)])
    drop = Options(start_adapter=synth.ADAPTER_START, trim_front=20)
    res = OracleEngine(drop).process(short)
    assert (res["flags"] & abi.FLAG_DROPPED_BY_CUT).all()
    out, failed = check(drop, short, "all dropped")
    assert len(out["lens"]) == len(failed["lens"]) == 0
    out, failed = check(Options(start_adapter=synth.ADAPTER_START, length_required=50), short, "all failed")
    assert len(out["lens"]) == 0 and len(failed["lens"]) == short.n_reads


@pytest.mark.parametrize("tiling", [None, "1"])
@pytest.mark.parametrize("name", ["cut_polyx_cplx", "mask_and_break", "fasta5"])
def test_device_batch_entry_point(name, tiling, monkeypatch):
    """fpl_process_device on 16-byte slots, shuffled, poisoned, exactly FPL_BATCH_BYTES long, with and without read tiling"""
    opt = cases.OPTION_SETS.get(name) or cases.MASK_BREAK_SETS[name]
    check(opt, cases.adversarial_batch(4), f"{name}/device/{tiling}", entry="device", monkeypatch=monkeypatch,
          env={"FPL_TILE_MBASES": tiling} if tiling else {})


@pytest.mark.parametrize("name", ["cut_polyx_cplx", "mask_and_break", "trims_limits"])
def test_fastq_entry_point_formats_to_the_writers_text(name):
    """after fpl_process_fastq_host, the emitted batches formatted with the record table's names and '+' lines are exactly
    fpl_emit_fastq_host's text"""
    from test_gpu_emit import fastq_of
    opt = cases.OPTION_SETS.get(name) or cases.MASK_BREAK_SETS[name]
    batch = cases.adversarial_batch(5)
    check(opt, batch, f"{name}/fastq", entry="fastq")
    text, names, plus = fastq_of(batch)
    g = engine(opt)
    try:
        recs, res, _ = g.process_fastq(text)
        want_out, want_failed = g.emit_fastq(True)
        out, failed = g.emit_batch(True, device=DEVICE)
    finally:
        g.close()
    for em, want, is_failed in ((out, want_out, False), (failed, want_failed, True)):
        hb, segs = em.to_host()
        parts = []
        for j in range(hb.n_reads):
            i = int(segs[j]["read"])
            nm = names[i]
            if is_failed:
                nm += b" " + abi.FAILED_TYPES[int(segs[j]["result"])].encode()
            else:
                tag = b""
                if segs[j]["break_index"]:
                    tag += b"r%d-" % int(segs[j]["break_index"])
                if segs[j]["split_side"]:
                    tag += b"split-by-adapter-right-" if segs[j]["split_side"] == 2 else b"split-by-adapter-left-"
                nm = nm[:1] + tag + nm[1:]
            s, q = hb.read(j)
            parts.append(nm + b"\n" + s + b"\n" + plus[i] + b"\n" + q + b"\n")
        assert b"".join(parts) == want, name


def test_round_trip_through_fpl_process_device():
    """`out` is a valid fpl_batch: a second context on it gives the oracle's records, Stats and counters on the same reads"""
    import torch
    from fastplong_b200.binding import Engine
    opt = cases.OPTION_SETS["cut_polyx_cplx"]
    batch = cases.ont_batch(93, n=300, mean=2000, p_chimera=0.2)
    g = Engine(opt)
    g.process(batch)
    out, _ = g.emit_batch(False, device=DEVICE)
    o = OracleEngine(opt)
    exp_out, _ = expected(opt, batch, o, o.process(batch))
    assert out.n_reads == len(exp_out["lens"]) > 0
    g2, o2 = Engine(opt), OracleEngine(opt)
    res = torch.zeros(out.n_reads * abi.RESULT_DTYPE.itemsize, dtype=torch.uint8, device=out.seq.device)
    g2.process_device(out.seq.data_ptr(), out.qual.data_ptr(), out.offsets.data_ptr(), out.lens.data_ptr(), out.n_reads,
                      out.n_bytes, results_ptr=res.data_ptr())
    g2.sync()
    canon = pack_reads(exp_out["reads"])
    compare_results(res.cpu().numpy().view(abi.RESULT_DTYPE), o2.process(canon), "round trip")
    cyc = int(canon.lens.max())
    for w in (0, 1):
        compare_stats(g2.stats(w, cyc), o2.stats(w, cyc), f"round trip/stats{w}")
    compare_stats(g2.counters(), o2.counters(), "round trip/counters")
    g.close()
    g2.close()


def raw_emit(g, out, failed):
    return g.lib.fpl_emit_batch_device(g.h, C.byref(out), C.byref(failed) if failed is not None else None)


def test_two_phase_contract():
    """the sizing call returns 1 and writes nothing; repeat calls give the same bytes; failed=NULL leaves `out` as it is;
    the next process call invalidates the emit"""
    import torch
    from fastplong_b200.binding import Engine, FplError
    opt = cases.MASK_BREAK_SETS["mask_and_break"]
    g = Engine(opt)
    g.process(cases.blocky_quality_batch(78))
    o, f = abi.FplOutBatch(), abi.FplOutBatch()
    assert raw_emit(g, o, f) == 1 and o.n_reads > 0 and f.n_reads > 0
    dev = torch.device("cpu" if EMULATE else "cuda:0")
    size = abi.batch_bytes(o.n_bytes)
    bufs = [torch.full((size,), 0xA5, dtype=torch.uint8, device=dev) for _ in range(2)]
    idx = [torch.full((o.n_reads,), -7, dtype=t, device=dev) for t in (torch.int64, torch.int32)]
    o.seq, o.qual, o.offsets, o.lens = bufs[0].data_ptr(), bufs[1].data_ptr(), idx[0].data_ptr(), idx[1].data_ptr()
    o.cap_reads, o.cap_bytes = o.n_reads - 1, size                # one read short
    if dev.type == "cuda":
        torch.cuda.synchronize()
    assert raw_emit(g, o, None) == 1
    o.cap_reads, o.cap_bytes = o.n_reads, size - 1                # one byte short
    assert raw_emit(g, o, None) == 1
    g.sync()
    assert all(bool((t == 0xA5).all()) for t in bufs) and all(bool((t == -7).all()) for t in idx)
    a1, fa = g.emit_batch(True, device=DEVICE)
    a2, _ = g.emit_batch(False, device=DEVICE)                    # failed = NULL
    a3, fb = g.emit_batch(True, device=DEVICE)
    for x, y in ((a1, a2), (a1, a3), (fa, fb)):
        for f_ in ("seq", "qual", "offsets", "lens", "segs"):
            assert torch.equal(getattr(x, f_), getattr(y, f_)), f_
    o.cap_reads, o.cap_bytes = o.n_reads, size
    assert raw_emit(g, o, None) == 0
    g.sync()
    assert torch.equal(bufs[0], a1.seq) and torch.equal(bufs[1], a1.qual) and torch.equal(idx[0], a1.offsets)
    g.process(pack_reads([(b"ACGTACGTACGTACGTACGTACGTACGTAC", b"I" * 30)]))     # the emit follows the last call
    one, none = g.emit_batch(True, device=DEVICE)
    assert one.n_reads == 1 and none.n_reads == 0
    bad = pack_reads([(b"ACGT", b"IIII"), (b"ACGT", b"IIII")])
    bad.offsets[1] = 8
    with pytest.raises(FplError, match="multiples of 16"):         # a call that fails leaves nothing to emit
        g.process(bad)
    with pytest.raises(FplError):
        g.emit_batch(device=DEVICE)
    g.close()
    g = Engine(opt)
    with pytest.raises(FplError):                                  # nothing processed yet
        g.emit_batch(device=DEVICE)
    g.close()


def test_more_reads_than_the_copy_grid_has_warps():
    """a batch past k_emit_batch_copy's grid cap, whose warps loop over several reads (a one-SM cap under the emulator)"""
    import capacity
    src = open(os.path.join(capacity.CSRC, "fpl_emit.cu")).read()
    cap = re.search(r"k_emit_batch_copy<<<\(unsigned\)\(want < FPL_NUM_SMS \* (\d+) \? want : FPL_NUM_SMS \* (\d+)\), (\d+)", src)
    assert cap and cap.group(1) == cap.group(2)
    opt = capacity.CS_SETS["plain"]
    if EMULATE:
        import simt_emu
        texts = capacity.shrunk_sources(FPL_NUM_SMS=1)
        k = capacity.constants(texts)
        g = simt_emu.EmuEngine(opt, lib=simt_emu.build_library(texts))
    else:
        from fastplong_b200.binding import Engine
        k = capacity.constants()
        g = Engine(opt)
    batch = capacity.text_batch(k, 9)
    assert batch.n_reads > k["FPL_NUM_SMS"] * int(cap.group(1)) * int(cap.group(3)) // 32
    o = OracleEngine(opt)
    g.process(batch)
    exp_out, exp_failed = expected(opt, batch, o, o.process(batch))
    out, failed = g.emit_batch(True, device=DEVICE)
    compare_batch(out, exp_out, "grid/out")
    compare_batch(failed, exp_failed, "grid/failed")
    g.close()


def test_a_refused_fastq_chunk_leaves_nothing_to_emit():
    """fpl_process_fastq_host overwrites the record table and offsets before it refuses a chunk (here: CR line ends), so the
    emit of the call before it is gone: emit_batch raises instead of copying from the new chunk's offsets"""
    from fastplong_b200.binding import FplError
    opt = cases.OPTION_SETS["cut_polyx_cplx"]
    batch = cases.adversarial_batch(7)
    g = engine(opt)
    try:
        assert g.process_fastq(fastq_text(batch)) is not None
        out, _ = g.emit_batch(True, device=DEVICE)
        assert out.n_reads > 0
        crlf = fastq_text(cases.ont_batch(94, n=50, mean=800)).replace(b"\n", b"\r\n")
        assert g.process_fastq(crlf) is None
        with pytest.raises(FplError):
            g.emit_batch(True, device=DEVICE)
        assert g.process_fastq(fastq_text(batch)) is not None           # a later strict chunk emits as usual
        again, _ = g.emit_batch(True, device=DEVICE)
        for f in ("seq", "qual", "offsets", "lens", "segs"):
            assert bool((getattr(again, f) == getattr(out, f)).all()), f
    finally:
        g.close()


def test_emit_batch_refuses_another_cuda_device():
    from fastplong_b200.binding import FplError
    g = engine(cases.OPTION_SETS["default_se"])
    try:
        g.process(cases.adversarial_batch(3))
        with pytest.raises(FplError, match="cuda:0"):
            g.emit_batch(True, device="cuda:1")
    finally:
        g.close()
