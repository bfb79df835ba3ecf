#!/usr/bin/env python
"""bench_state.py — fpl_state_export and fpl_state_merge on bench.py's c2 and c5-500k contexts, one H100.

  python tools/bench_state.py [--workloads c2,c5-500k] [--reps K]

For each workload: generates bench.py's input on the device (c2: 1 M reads of 15 kb; c5-500k: 20 k reads of 500 kb, so the Stats
blocks have millions of rows), runs fpl_process_device on it with the read lists kept, then K times exports the
context's image into host memory (the wall time of the fpl_state_export call, which ends synchronised, into a buffer
already paged in) and merges it into a second context
(the wall time of fpl_state_merge up to fpl_sync, after one untimed merge that grows the lists; the device time of its one
k_merge_stats launch from fpl_last_kernel_times).  One JSON line, with the image size and the card's name and power limit read
in the same run."""
import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402

from bench_report_html import card, stats  # noqa: E402


def run(name, reps):
    import torch
    import bench
    from fastplong_b200 import synth_fast
    from fastplong_b200.binding import Engine
    dev = torch.device("cuda", 0)
    n_reads, _, mean_len, gen_kw, _ = bench.WORKLOADS[name]
    plan = synth_fast.read_plan(n_reads, mean_len, bench.SEED, **{k: v for k, v in gen_kw.items() if k in ("min_len",)})
    tile = synth_fast.ont_like_device(n_reads, mean_len, bench.SEED + 1000, dev, plan=plan)
    offs = torch.from_numpy(tile.offsets.astype(np.int64)).to(dev)
    lens = torch.from_numpy(tile.lens).to(dev)
    torch.cuda.synchronize()
    src, dst = Engine(bench.workload_options(name)), Engine(bench.workload_options(name))
    for e in (src, dst):
        e.keep_read_lists(True)
    src.process_device(tile.seq.data_ptr(), tile.qual.data_ptr(), offs.data_ptr(), lens.data_ptr(), tile.n_reads, tile.n_bytes)
    src.sync()
    rows = int(tile.lens.max())
    del tile, offs, lens
    torch.cuda.empty_cache()
    img = src.export_state()                      # warm-up: the first export, and the merge that grows dst's capacities
    dst.merge_state(img)
    dst.sync()
    export_ms, merge_ms = [], []
    buf, n = np.zeros(len(img), np.uint8), C.c_int64()      # the export's own time: into a buffer already paged in
    dst.set_timing(True)
    for _ in range(reps):
        t0 = time.perf_counter()
        rc = src.lib.fpl_state_export(src.h, buf.ctypes.data, buf.size, C.byref(n))
        export_ms.append(1e3 * (time.perf_counter() - t0))
        assert rc == 0 and n.value == buf.size
        img = buf
        t0 = time.perf_counter()
        dst.merge_state(img)
        dst.sync()
        merge_ms.append(1e3 * (time.perf_counter() - t0))
    ms, n = dst.kernel_times()["k_merge_stats"]
    out = {"reads": n_reads, "rows": rows, "image_bytes": len(img), "export_wall_ms": stats(export_ms),
           "merge_wall_ms": stats(merge_ms), "k_merge_stats_ms": round(ms / max(n, 1), 4), "k_merge_stats_launches": n,
           "export_gb_per_s": round(len(img) / (stats(export_ms)["median"] * 1e6), 2),
           "merge_gb_per_s": round(len(img) / (stats(merge_ms)["median"] * 1e6), 2)}
    src.close()
    dst.close()
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c2,c5-500k")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    line = {"metric": "fpl_state_export / fpl_state_merge, one context's image", "card": card()}
    for name in args.workloads.split(","):
        line[name] = run(name, args.reps)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
