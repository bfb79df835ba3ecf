#!/usr/bin/env python
"""bench_emit_batch.py — device time of fpl_emit_batch_device on config 2 (bench.py's workload), one H100.

  python tools/bench_emit_batch.py [--reads N] [--reps K] [--warmup W] [--mask-reads M]

1. Generates bench.py's c2 input on the device (synth_fast.ont_like_device, same seeds), with the planted adapters (the ones
   Evaluator::evalAdapterAndReadNum detects on this generator's reads).
2. Runs fpl_process_device on it, builds the sizes (the first fpl_emit_batch_device call), then times the copying call over
   K warm repetitions with CUDA events on the library's stream.
3. Prints one JSON line: ms per emit, output reads and bytes, algorithmic bytes (read + write of the sequence and quality of
   every output base, plus 32 B per output read: offset, length, 20-byte segment) per second and their share of the data-sheet
   3.35 TB/s, and the card's name, power limit and maximum SM clock read in the same run.
If `out` and `failed` do not fit in HBM beside the input, the largest prefix of the reads whose output does is used (said in
"reads_used").  Behind the timing the output is checked at full size: for eight read ranges spread over the batch, the last
one ending with the last read, the slots are rebuilt from the records with plain torch indexing (no code shared with the
kernels) and compared byte for byte with the emitted buffers, padding included, and so are offsets, lengths and segments.
A second, masked run (-N, on the first M reads: the masked copy of the sequence buffer needs room too) rebuilds the 'N'
regions from fpl_last_mask_regions the same way."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

PEAK_GBS = 3350.0           # H100 SXM data sheet (HBM3)
RANGES = 8
RANGE_READS = 200


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, pl, mhz = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": pl, "max_sm_clock": mhz}
    except Exception as e:      # reported, never fatal
        return {"error": str(e)[:200]}


def output_reads(res, failed):
    """the output reads of the records, in writer order: (read, lo, len, result, median, side, is_r1) as numpy columns"""
    nseg = res["n_segments"]
    flags = res["flags"].astype(np.int64)
    if failed:
        keep = (nseg == 1) & (res["seg_result"][:, 0] != 0)
        rd = np.flatnonzero(keep)
        r1 = (flags[rd] & 4) == 0       # not split: the output read is r1 itself
        return dict(read=rd, lo=res["trim_lo"][rd].astype(np.int64), len=res["trim_len"][rd].astype(np.int64),
                    result=res["seg_result"][rd, 0].astype(np.int64), median=res["seg_median_qual"][rd, 0].astype(np.int64),
                    side=np.zeros(len(rd), np.int64), is_r1=r1.astype(np.int64))
    ks = np.arange(2)[None, :]
    keep = (ks < nseg[:, None]) & (res["seg_result"] == 0)
    rd, k = np.nonzero(keep)            # row-major: input order, then segment order
    split = (flags[rd] & 4) != 0
    side = np.where(split, np.where((k == 1) | ((flags[rd] & 8) != 0), 2, 1), 0)
    return dict(read=rd, lo=res["seg_lo"][rd, k].astype(np.int64), len=res["seg_len"][rd, k].astype(np.int64),
                result=np.zeros(len(rd), np.int64), median=res["seg_median_qual"][rd, k].astype(np.int64), side=side,
                is_r1=(side == 0).astype(np.int64))


def check(torch, got, exp, in_seq, in_qual, in_off, regions, what):
    """RANGES ranges of output reads (the last one ends with the last) rebuilt with torch indexing vs the emitted batch"""
    dev = in_seq.device
    n = len(exp["read"])
    slots = (exp["len"] + 15) // 16 * 16
    offs = np.concatenate([[0], np.cumsum(slots)[:-1]]) if n else np.zeros(0, np.int64)
    n_bytes = int(slots.sum())
    assert got["n_reads"] == n and got["n_bytes"] == n_bytes, (what, got["n_reads"], n, got["n_bytes"], n_bytes)
    if n == 0:
        return {"reads": 0}
    g_off = got["offsets"].cpu().numpy()
    g_len = got["lens"].cpu().numpy()
    assert np.array_equal(g_off, offs) and np.array_equal(g_len, exp["len"]), what + ": offsets / lens"
    segs = got["segs"].cpu().numpy().view(np.dtype([("read", "<i4"), ("lo", "<i4"), ("len", "<i4"), ("result", "u1"),
                                                     ("median_qual", "u1"), ("split_side", "u1"), ("is_r1", "u1"),
                                                     ("break_index", "<i4")]))
    for a, b in (("read", "read"), ("lo", "lo"), ("len", "len"), ("result", "result"), ("median_qual", "median"),
                 ("split_side", "side"), ("is_r1", "is_r1")):
        assert np.array_equal(segs[a].astype(np.int64), exp[b]), f"{what}: segs.{a}"
    assert not segs["break_index"].any(), what
    spans, nb = [], 0
    for j in range(1, RANGES + 1):
        j1 = max(1, n * j // RANGES)
        j0 = max(0, j1 - RANGE_READS)
        b0, b1 = int(offs[j0]), int(offs[j1 - 1] + slots[j1 - 1])
        # expected bytes of output reads [j0, j1): zero slots, then each window gathered from the input by an index vector
        ln = torch.from_numpy(exp["len"][j0:j1]).to(dev)
        dst0 = torch.from_numpy(offs[j0:j1] - b0).to(dev)
        src0 = torch.from_numpy(in_off[exp["read"][j0:j1]] + exp["lo"][j0:j1]).to(dev)
        within = torch.arange(int(ln.sum()), device=dev) - torch.repeat_interleave(torch.cumsum(ln, 0) - ln, ln)
        src = torch.repeat_interleave(src0, ln) + within
        dst = torch.repeat_interleave(dst0, ln) + within
        for buf, name in ((in_seq, "seq"), (in_qual, "qual")):
            want = torch.zeros(b1 - b0, dtype=torch.uint8, device=dev)
            want[dst] = buf[src]
            if name == "seq" and regions is not None:
                # the -N regions of these reads, painted into the window copies that are masked
                rd_sel = exp["read"][j0:j1]
                masked = exp["is_r1"][j0:j1] if what.endswith("failed") else np.ones(j1 - j0, bool)
                for q in range(j1 - j0):
                    if not masked[q]:
                        continue
                    for lo, l_ in regions.get(int(rd_sel[q]), ()):
                        a = max(lo, int(exp["lo"][j0 + q]))
                        e = min(lo + l_, int(exp["lo"][j0 + q] + exp["len"][j0 + q]))
                        if e > a:
                            d = int(offs[j0 + q] - b0) + a - int(exp["lo"][j0 + q])
                            want[d:d + e - a] = ord("N")
            have = got[name][b0:b1]
            if not torch.equal(have, want):
                k = int(torch.nonzero(have != want)[0])
                raise AssertionError(f"{what}: {name} differs at byte {b0 + k} (output reads [{j0}, {j1}))")
        nb += b1 - b0
        spans.append([j0, j1])
    tail = torch.cat([got["seq"][n_bytes:], got["qual"][n_bytes:]])
    assert not tail.any(), what + ": tail pad"
    return {"reads": n, "output_read_ranges": spans, "bytes_compared": nb, "highest_offset": int(offs[-1])}


def emit(torch, eng, lib, dev, alloc=True):
    """sizing call, then buffers, then the copying call; returns (out, failed) dicts of tensors + sizes"""
    from fastplong_b200 import abi
    d = [abi.FplOutBatch(), abi.FplOutBatch()]
    rc = lib.fpl_emit_batch_device(eng.h, C.byref(d[0]), C.byref(d[1]))
    assert rc in (0, 1), lib.fpl_last_error()
    got = []
    for x in d:
        n, nb = int(x.n_reads), int(x.n_bytes)
        size = abi.batch_bytes(nb) if n else 0
        t = {"n_reads": n, "n_bytes": nb, "seq": torch.empty(size, dtype=torch.uint8, device=dev),
             "qual": torch.empty(size, dtype=torch.uint8, device=dev), "offsets": torch.empty(n, dtype=torch.int64, device=dev),
             "lens": torch.empty(n, dtype=torch.int32, device=dev), "segs": torch.empty(20 * n, dtype=torch.uint8, device=dev)}
        if n:
            x.seq, x.qual, x.offsets, x.lens, x.segs = (t[k].data_ptr() for k in ("seq", "qual", "offsets", "lens", "segs"))
        x.cap_reads, x.cap_bytes = n, size
        got.append(t)
    torch.cuda.synchronize()
    return d, got


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=1 << 20)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--mask-reads", type=int, default=1 << 18, help="reads of the masked (-N) check run")
    args = ap.parse_args()
    import torch
    import bench
    from fastplong_b200 import synth_fast
    from fastplong_b200.binding import Engine
    if not torch.cuda.is_available():
        raise SystemExit("bench_emit_batch.py: no CUDA device")
    dev = torch.device("cuda", 0)
    info = card()
    plan = synth_fast.read_plan(args.reads, bench.MEAN_LEN, bench.SEED)
    tile = synth_fast.ont_like_device(args.reads, bench.MEAN_LEN, bench.SEED + 1000, dev, plan=plan)
    in_off = tile.offsets.astype(np.int64)
    offs = torch.from_numpy(in_off).to(dev)
    lens = torch.from_numpy(tile.lens).to(dev)
    torch.cuda.synchronize()
    # the output is about as large as the input: use the longest prefix whose output fits beside it (5% headroom)
    free = torch.cuda.mem_get_info(dev)[0]
    ends = in_off + tile.lens
    n_use = int(np.searchsorted(2 * ends * 1.05 + (2 << 30), free, side="right"))
    n_use = min(n_use, tile.n_reads)
    opt = bench.workload_options("c2")
    eng = Engine(opt)
    lib = eng.lib
    ext = torch.cuda.ExternalStream(eng.stream_ptr, device=dev)
    eng.process_device(tile.seq.data_ptr(), tile.qual.data_ptr(), offs.data_ptr(), lens.data_ptr(), n_use, tile.n_bytes)
    eng.sync()
    eng.set_timing(True)
    d, got = emit(torch, eng, lib, dev)
    for _ in range(args.warmup):
        assert lib.fpl_emit_batch_device(eng.h, C.byref(d[0]), C.byref(d[1])) == 0, lib.fpl_last_error()
    eng.sync()
    evs = []
    for _ in range(args.reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(ext)
        assert lib.fpl_emit_batch_device(eng.h, C.byref(d[0]), C.byref(d[1])) == 0, lib.fpl_last_error()
        b.record(ext)
        evs.append((a, b))
    eng.sync()
    ms = sorted(a.elapsed_time(b) for a, b in evs)
    d_sizes = [(x.n_reads, x.n_bytes) for x in d]
    kt = eng.kernel_times()
    eng.set_timing(False)
    out_bases = int(sum(int(g["lens"].sum()) for g in got))
    out_reads = sum(g["n_reads"] for g in got)
    alg = 4 * out_bases + 32 * out_reads
    med = ms[len(ms) // 2]
    res = eng.fetch_results(n_use)
    t0 = time.time()
    checked = {}
    for g, failed in ((got[0], False), (got[1], True)):
        checked["failed" if failed else "out"] = check(torch, g, output_reads(res, failed), tile.seq, tile.qual, in_off, None,
                                                       "plain/" + ("failed" if failed else "out"))
    del got, d
    eng.close()
    torch.cuda.empty_cache()
    # masked run: the inline segments of the records are still the output reads (-N without -b)
    mopt = bench.workload_options("c2")
    mopt.mask, mopt.mask_window_size, mopt.mask_mean_quality = True, 20, 8    # some reads of this input get regions, a few then fail
    m = min(args.mask_reads, n_use)
    meng = Engine(mopt)
    meng.process_device(tile.seq.data_ptr(), tile.qual.data_ptr(), offs.data_ptr(), lens.data_ptr(), m, tile.n_bytes)
    meng.sync()
    mres = meng.fetch_results(m)
    regs = {}
    for rg in meng.mask_regions():
        regs.setdefault(int(rg["read"]), []).append((int(rg["lo"]), int(rg["len"])))
    d, mgot = emit(torch, meng, meng.lib, dev)
    assert meng.lib.fpl_emit_batch_device(meng.h, C.byref(d[0]), C.byref(d[1])) == 0
    meng.sync()
    for g, failed in ((mgot[0], False), (mgot[1], True)):
        checked["masked_" + ("failed" if failed else "out")] = check(torch, g, output_reads(mres, failed), tile.seq, tile.qual,
                                                                     in_off, regs, "masked/" + ("failed" if failed else "out"))
    checked["masked_reads"] = m
    checked["masked_regions"] = sum(len(v) for v in regs.values())
    assert checked["masked_regions"] > 0, "the masked run painted nothing"
    meng.close()
    line = {"metric": "fpl_emit_batch_device, config 2", "card": info, "reads_used": n_use, "reads_generated": tile.n_reads,
            "input_bases": int(tile.lens[:n_use].sum(dtype=np.int64)),
            "out": {"reads": int(d_sizes[0][0]), "bytes": int(d_sizes[0][1])},
            "failed": {"reads": int(d_sizes[1][0]), "bytes": int(d_sizes[1][1])},
            "ms_per_emit": round(med, 3), "ms_min": round(ms[0], 3), "ms_max": round(ms[-1], 3), "reps": args.reps,
            "output_reads": out_reads, "output_bases": out_bases,
            "alg_bytes": alg, "alg_gbs": round(alg / (med * 1e-3) / 1e9, 1),
            "share_of_3350_gbs": round(alg / (med * 1e-3) / 1e9 / PEAK_GBS, 4),
            "kernels": {k: {"ms": round(v[0], 3), "launches": v[1]} for k, v in kt.items() if v[1]},
            "check": checked, "check_s": round(time.time() - t0, 1), "ok": True}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
