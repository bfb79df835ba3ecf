#!/usr/bin/env python
"""bench_merge.py — fpl_merge_stats on a pair of config-2-sized contexts, one H100.

  python tools/bench_merge.py [--reps K]

Generates bench.py's c2 input on the device (1 M reads of 15 kb), runs fpl_process_device on it in two contexts with the read
lists kept, then merges the second into the first K times (after one untimed merge that grows the lists): the device time of
k_merge_stats per call (fpl_last_kernel_times) and the wall time of the call up to a fpl_sync, list copies included.  Also
prints the bytes the kernel reads and writes, counted from the capacities.  One JSON line, with the card's name and power limit
read in the same run."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402

from bench_report_html import card, stats  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    import torch
    import bench
    from fastplong_b200 import abi, synth_fast
    from fastplong_b200.binding import Engine
    dev = torch.device("cuda", 0)
    n_reads, _, mean_len, gen_kw, _ = bench.WORKLOADS["c2"]
    plan = synth_fast.read_plan(n_reads, mean_len, bench.SEED, **{k: v for k, v in gen_kw.items() if k in ("min_len",)})
    tile = synth_fast.ont_like_device(n_reads, mean_len, bench.SEED + 1000, dev, plan=plan)
    offs = torch.from_numpy(tile.offsets.astype(np.int64)).to(dev)
    lens = torch.from_numpy(tile.lens).to(dev)
    torch.cuda.synchronize()
    ptrs = (tile.seq.data_ptr(), tile.qual.data_ptr(), offs.data_ptr(), lens.data_ptr(), tile.n_reads, tile.n_bytes)
    dst, src = Engine(bench.workload_options("c2")), Engine(bench.workload_options("c2"))
    for e in (dst, src):
        e.keep_read_lists(True)
        e.process_device(*ptrs)
        e.sync()
    dst.merge(src)                         # warm-up: the lists grow once
    dst.sync()
    dst.set_timing(True)
    wall = []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        dst.merge(src)
        dst.sync()
        wall.append(1e3 * (time.perf_counter() - t0))
    ms, n = dst.kernel_times()["k_merge_stats"]
    rows = int(tile.lens.max())
    words = 2 * (16 * rows + abi.STATS_TAIL) + dst.lib.fpl_counter_words(dst.h)
    moved = 8 * words * 3                  # per word: the destination read and written, one source read
    line = {"metric": "fpl_merge_stats, two c2 contexts", "card": card(), "reads_per_context": tile.n_reads, "rows": rows,
            "k_merge_stats_ms": round(ms / max(n, 1), 4), "launches": n, "kernel_bytes": moved,
            "kernel_gb_per_s": round(moved / (ms / max(n, 1)) / 1e6, 1) if ms else None,
            "call_wall_ms": stats(wall), "list_entries_copied_per_call": tile.n_reads * 3}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
