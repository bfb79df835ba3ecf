#!/usr/bin/env python
"""bench_report_html.py — fpl_report_html and its read-list capture, one H100.

  python tools/bench_report_html.py [--workloads c2,c5-500k] [--reps K] [--capture-steps S] [--no-twin]

For each workload (bench.py's input and options: c2 = 1 M reads of 15 kb, so the density lists are at full size; c5-500k =
20 k reads of 500 kb, so the down-sampled sums run over millions of cycles):
1. generates the input on the device and runs fpl_process_device on it with the read lists kept;
2. times Engine.report_html over K repetitions, each rebuilding the text (the command changes): device time per report
   kernel (fpl_last_kernel_times) and wall time of the call, D2H copy of the whole text included;
3. builds the same report with the plain-Python twin (tests/report_html_twin.py) from the downloaded accumulators and the
   library's own records (the records themselves are held to the oracle by the GPU test suite) and compares the texts.
On c2 it also measures what capture costs on the processing path: fpl_process_device step time (CUDA events) with the lists
off and on, two engines alternated step by step in one process, the lists emptied between steps (fpl_reset, untimed).
Prints one JSON line per workload, with the card's name and power limit read in the same run."""
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


def stats(v):
    v = sorted(v)
    return {"median": round(v[len(v) // 2], 3), "min": round(v[0], 3), "max": round(v[-1], 3), "n": len(v)}


def run(name, args, info):
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
    ptrs = (tile.seq.data_ptr(), tile.qual.data_ptr(), offs.data_ptr(), lens.data_ptr(), tile.n_reads, tile.n_bytes)
    line = {"metric": f"fpl_report_html, {name} input", "card": info, "reads": tile.n_reads, "bases": int(tile.lens.sum())}
    if name == "c2" and args.capture_steps:
        engines = {"off": Engine(bench.workload_options(name)), "on": Engine(bench.workload_options(name))}
        engines["on"].keep_read_lists(True)
        ms = {"off": [], "on": []}
        stream = {k: torch.cuda.ExternalStream(e.stream_ptr) for k, e in engines.items()}
        for step in range(args.capture_steps + 2):
            for k in (("off", "on") if step % 2 == 0 else ("on", "off")):
                e = engines[k]
                e.reset()
                e.sync()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(stream[k])
                e.process_device(*ptrs)
                b.record(stream[k])
                e.sync()
                if step >= 2:          # two warm-up rounds
                    ms[k].append(a.elapsed_time(b))
        line["capture_cost_c2"] = {"step_ms_lists_off": stats(ms["off"]), "step_ms_lists_on": stats(ms["on"]),
                                   "median_delta_ms": round(stats(ms["on"])["median"] - stats(ms["off"])["median"], 3)}
        engines["on"].set_timing(True)
        engines["on"].reset()
        engines["on"].process_device(*ptrs)
        engines["on"].sync()
        line["capture_cost_c2"]["k_html_capture_ms"] = round(engines["on"].kernel_times()["k_html(capture)"][0], 3)
        for e in engines.values():
            e.close()
    eng = Engine(bench.workload_options(name))
    eng.keep_read_lists(True)
    eng.process_device(*ptrs)
    eng.sync()
    res = eng.fetch_results(tile.n_reads) if not args.no_twin else None
    host_lens = tile.lens.copy()
    del tile, offs, lens
    torch.cuda.empty_cache()
    eng.report_html(command="warmup", time_text="t")
    eng.set_timing(True)
    walls = []
    for i in range(args.reps):
        t0 = time.perf_counter()
        text = eng.report_html(command=f"rep {i}", time_text="t")
        walls.append((time.perf_counter() - t0) * 1e3)
    kt = eng.kernel_times()
    eng.set_timing(False)
    per = {k: round(v[0] / args.reps, 3) for k, v in kt.items() if k.startswith("k_html") and v[1]}
    line.update({"report_bytes": len(text), "reps": args.reps, "device_ms_per_report": {"kernels": per, "sum": round(sum(per.values()), 3)},
                 "wall_ms_per_call_incl_d2h": stats(walls)})
    if not args.no_twin:
        import report_html_twin
        t0 = time.perf_counter()
        pre, post = report_html_twin.read_lists(host_lens, res)
        want = report_html_twin.report(eng.stats(0), eng.stats(1), eng.counters(), eng.options, pre, post,
                                       command=f"rep {args.reps - 1}", time_text="t")
        line["python_twin_s"] = round(time.perf_counter() - t0, 1)
        line["equal_to_twin"] = want == text
        if want != text:
            line["first_difference"] = next((i for i in range(min(len(want), len(text))) if want[i] != text[i]), min(len(want), len(text)))
    eng.close()
    line["ok"] = line.get("equal_to_twin", True)
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c2,c5-500k")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--capture-steps", type=int, default=10, help="alternated off/on steps on c2 (0: skip)")
    ap.add_argument("--no-twin", action="store_true", help="skip the Python twin (no equality check)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_report_html.py: no CUDA device")
    info = card()
    ok = True
    for name in args.workloads.split(","):
        line = run(name, args, info)
        ok &= line["ok"]
        print(json.dumps(line), flush=True)
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
