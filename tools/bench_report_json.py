#!/usr/bin/env python
"""bench_report_json.py — fpl_report_json on config 5 at 500 kb (bench.py --workload c5-500k's input), one H100.

  python tools/bench_report_json.py [--reads N] [--reps K] [--warmup W] [--no-twin]

1. Generates c5-500k's input on the device (synth_fast.ont_like_device, bench.py's seeds: 20k reads, mean 500 kb, so the
   longest read and total_cycles are in the millions) and runs fpl_process_device on it with bench.py's c5 options.
2. Times Engine.report_json over K warm repetitions.  Every repetition rebuilds the text (the "command" value changes, so
   the cached text does not apply): the device time of the report kernels (fpl_last_kernel_times: k_report(cycles),
   k_report(sizes), k_report(text)) and the wall time of the call, D2H copy of the whole text included.
3. Builds the same report with the plain-Python twin (tests/report_twin.py) from the downloaded blocks — its time is a
   Python number, not the reference's C++ reporter — and compares the two texts byte for byte at full size.
Prints one JSON line, with the card's name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, pl, mhz = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": pl, "max_sm_clock": mhz}
    except Exception as e:      # reported, never fatal
        return {"error": str(e)[:200]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=0, help="reads (default: c5-500k's 20k)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--no-twin", action="store_true", help="skip the Python twin (no equality check)")
    args = ap.parse_args()
    import torch
    import bench
    from fastplong_b200 import synth_fast
    from fastplong_b200.binding import Engine
    if not torch.cuda.is_available():
        raise SystemExit("bench_report_json.py: no CUDA device")
    dev = torch.device("cuda", 0)
    info = card()
    n_reads, _, mean_len, gen_kw, _ = bench.WORKLOADS["c5-500k"]
    n_reads = args.reads or n_reads
    plan = synth_fast.read_plan(n_reads, mean_len, bench.SEED, **{k: v for k, v in gen_kw.items() if k in ("min_len",)})
    tile = synth_fast.ont_like_device(n_reads, mean_len, bench.SEED + 1000, dev, plan=plan)
    offs = torch.from_numpy(tile.offsets.astype(np.int64)).to(dev)
    lens = torch.from_numpy(tile.lens).to(dev)
    torch.cuda.synchronize()
    eng = Engine(bench.workload_options("c5-500k"))
    eng.process_device(tile.seq.data_ptr(), tile.qual.data_ptr(), offs.data_ptr(), lens.data_ptr(), tile.n_reads, tile.n_bytes)
    eng.sync()
    longest = int(tile.lens.max())
    del tile
    torch.cuda.empty_cache()
    for i in range(args.warmup):
        eng.report_json(command=f"warmup {i}")
    eng.set_timing(True)
    walls = []
    for i in range(args.reps):
        t0 = time.perf_counter()
        text = eng.report_json(command=f"rep {i}")
        walls.append((time.perf_counter() - t0) * 1e3)
    kt = eng.kernel_times()
    eng.set_timing(False)
    report_ms = {k: round(v[0] / max(v[1], 1), 3) for k, v in kt.items() if k.startswith("k_report") and v[1]}
    rep = json.loads(text)
    line = {"metric": "fpl_report_json, config 5 at 500 kb (c5-500k input)", "card": info, "reads": n_reads,
            "longest_read": longest, "total_cycles": {"pre": rep["read_before_filtering"]["total_cycles"],
                                                      "post": rep["read_after_filtering"]["total_cycles"]},
            "report_bytes": len(text), "reps": args.reps,
            "device_ms_per_report": {"kernels": report_ms, "sum": round(sum(report_ms.values()), 3)},
            "wall_ms_per_call_incl_d2h": {"median": round(sorted(walls)[len(walls) // 2], 2), "min": round(min(walls), 2),
                                          "max": round(max(walls), 2)}}
    if not args.no_twin:
        import report_twin
        t0 = time.perf_counter()
        pre, post, cnt = eng.stats(0), eng.stats(1), eng.counters()
        dl = time.perf_counter() - t0
        t0 = time.perf_counter()
        want = report_twin.report(pre, post, cnt, eng.options, command=f"rep {args.reps - 1}")
        line["python_twin_s"] = round(time.perf_counter() - t0, 2)
        line["python_twin_download_s"] = round(dl, 2)
        line["equal_to_twin"] = want == text
        if want != text:
            i = next((i for i in range(min(len(want), len(text))) if want[i] != text[i]), min(len(want), len(text)))
            line["first_difference"] = i
    eng.close()
    line["ok"] = line.get("equal_to_twin", True)
    print(json.dumps(line), flush=True)
    if not line["ok"]:
        sys.exit(1)


if __name__ == "__main__":
    main()
