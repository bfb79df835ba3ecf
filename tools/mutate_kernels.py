"""Development aid (CPU): mutation testing of the GPU tests' grip on the KERNELS.  A sample of single-token mutants of the kernel
sources (comparison operators, && / ||, +-1) is built into the emulated library (tests/simt_emu.py) and run against the oracle on
a battery — crafted boundaries, option matrix on adversarial reads, RNA, -N/-b, FASTQ text, and the capacity limits of the
statistics and text kernels (tests/test_capacity_shrunk.py's cases on the mutant built with shrunk constants, the packed
counter of k_cycle_stats at its fullest).  A surviving mutant is kernel
behaviour the parity tests do not pin — or an equivalent mutant: the one-sided filters (a filter that says "maybe" more often
changes no result by design), min / max ties, guards that cannot fire.
--range FROM[:TO] samples the lines from the first one containing FROM to the first one after it containing TO (or the end);
--only reports runs only the report and merge cases (tests/test_capacity_shrunk_reports.py), which are the only ones that reach
the report / merge code: the rest of the battery calls none of fpl_report_json, fpl_report_html, fpl_merge_stats.
--only ext runs only the --mask / --break cases, the only ones that reach fpl_ext.cu (fpl_ext_run runs only with one of the two
flags on): the same verdict as the whole battery for a mutant of that file, in a fraction of the time.
--only state runs the in-process cases of tests/test_gpu_state.py, the only ones that call fpl_state_export / fpl_state_merge
(its processes of their own, the gloo ranks and the cases past k_merge_stats' grid cap are left out).
usage: python tools/mutate_kernels.py <file.cu> <n_mutants> [seed] [workers] [--range FROM[:TO]] [--only reports|ext|state]
       (internal: --battery <lib.so|-> [<shrunk lib.so>] [reports|ext|state])"""
import os
import random
import re
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
OPS = [(r"<=", "<"), (r">=", ">"), (r"(?<![<>=!-])<(?![<=])", "<="), (r"(?<![<>=!-])>(?![>=])", ">="), (r"==", "!="), (r"!=", "=="),
       (r"&&", "||"), (r"\|\|", "&&"), (r"\+ 1\b", "+ 0"), (r"- 1\b", "- 0")]


SHRUNK = "group_of_2_stages"       # tests/test_capacity_shrunk.py: the build whose capacities the battery's small cases reach


def shrunk_values():
    """the shrunk constants of the battery's small build: tests/test_capacity_shrunk.py's SHRUNK build with the grouping chunk of
    tests/test_capacity_shrunk_reports.py"""
    import test_capacity_shrunk as CS
    import test_capacity_shrunk_reports as R
    v = dict(CS.BUILDS[SHRUNK], **R.SHRUNK)
    assert v["FPL_NUM_SMS"] == R.SHRUNK["FPL_NUM_SMS"]
    return v


def report_cases(small):
    """tests/test_capacity_shrunk_reports.py's cases on the mutant's shrunk build"""
    import capacity
    import test_capacity_shrunk_reports as R
    R.LIBS["lib"] = (small, capacity.constants(capacity.shrunk_sources(**shrunk_values())))
    R.test_down_sampled_ranges_are_never_empty()
    for which in range(len(capacity.grouping_lengths(R.LIBS["lib"][1]))):
        R.test_grouping_by_median_across_chunks_and_blocks(which)
    for kind in ("slots", "segments_above", "segments_below"):
        R.test_lists_past_the_capture_cap(kind)
    for name in sorted(capacity.LENGTH_CASES):
        R.test_length_statistics_ties_and_edges(name)
    for which in range(len(capacity.curve_totals(R.LIBS["lib"][1]))):
        R.test_curves_down_sampling_and_past_the_grid_caps(which)
    R.test_merge_three_capacities_past_the_merge_cap()
    R.test_emit_batch_copy_more_reads_than_warps()


def ext_cases(T):
    """every case of the battery that turns --mask or --break on"""
    import cases
    for name, opt in cases.MASK_BREAK_SETS.items():
        T.check(opt, cases.blocky_quality_batch(5, n=40), name)
    edges = cases.mask_break_edge_batch()
    for name, opt in cases.MASK_BREAK_EDGE_SETS.items():
        T.check(opt, edges, name + "/edges")
    T.check_text(cases.MASK_BREAK_SETS["mask_and_break"], cases.blocky_quality_batch(5, n=30), "text/ext")
    T.check_text(cases.MASK_BREAK_EDGE_SETS["split_break_mask"], edges, "text/ext/edges")
    for name, (opt, b) in cases.edge_cases().items():
        if opt.mask or opt.break_reads:
            T.check(opt, b, name)


def state_cases():
    """tests/test_gpu_state.py's cases that run in this process, on the mutant"""
    import simt_emu
    import test_gpu_state as S
    from fastplong_b200 import binding
    binding.LIB_PATH, binding._lib = simt_emu.build_library(), None
    for name in sorted(S.M.SHARD_SETS):
        S.test_round_trip(name)
        S.test_shards_into_a_destination_holding_data(name)
    for case in (S.test_source_longer_than_the_destination, S.test_destination_reserved_far_above,
                 S.test_empty_sources_and_the_same_image_twice, S.test_capture_off, S.test_merged_flag_travels,
                 S.test_processing_after_the_merge_continues_the_sequence,
                 S.test_refusals_leave_the_destination_unchanged, S.test_two_phase_export, S.test_one_launch_per_merge):
        case()


def battery(lib, small=None, only=None):
    import signal
    import simt_emu
    if lib != "-":
        simt_emu._emu_lib_path = lib
    import capacity
    import cases
    import test_capacity_shrunk as CS
    import test_simt_kernels as T
    signal.alarm(300 if only in ("reports", "ext", "state") else 900)       # the report cases take well under a minute
    try:
        if only == "state":
            state_cases()
            print("SURVIVED")
            return
        if only == "reports":
            report_cases(small)
            print("SURVIVED")
            return
        if only == "ext":
            ext_cases(T)
            print("SURVIVED")
            return
        # the capacity limits: the mutant built with shrunk constants, and the packed counter at its fullest at full size
        if small:
            report_cases(small)
            CS.LIBS[SHRUNK] = (small, capacity.constants(capacity.shrunk_sources(**shrunk_values())))
            for optset in sorted(capacity.CS_SETS):
                CS.test_cycle_stats_staging_rounds_and_groups(SHRUNK, optset)
                CS.test_cycle_stats_post_filter_counts(SHRUNK, optset)
            CS.test_kmer_fix_long_range_list(SHRUNK)
            CS.test_read_qual_long_list_and_stride(SHRUNK)
            CS.test_read_qual_exc_list(SHRUNK)
            CS.test_text_path_more_records_than_warps(SHRUNK)
        T.check(capacity.HEADROOM_OPT, capacity.headroom_batch(capacity.constants(), False), "packed counter at its fullest")
        for name, (opt, b) in cases.edge_cases().items():
            T.check(opt, b, name)
        adv = cases.adversarial_batch(1)
        for name in T.PLAIN_SETS:
            T.check(cases.OPTION_SETS[name], adv, name)
        for name, opt in cases.RNA_SETS.items():
            T.check(opt, cases.rna_batch(41, n=40, mean=1000, mixed=True), name)
        ext_cases(T)
        for n in (33, 65, 129):
            T.check(cases.OPTION_SETS[f"long_adapter_{n}"], cases.long_adapter_batch(n, 900 + n, n=16), f"long{n}")
        T.check(cases.OPTION_SETS["fasta64_polyx"], cases.hifi_fasta64_batch(3, n=40), "fasta64")
        from fastplong_b200 import synth
        T.check(cases.OPTION_SETS["cut_polyx_cplx"], synth.ont_like(2, 110000, 5, p_chimera=1.0), "reads beyond 96 kb")      # block-wide paths
        T.check_text(cases.OPTION_SETS["cut_polyx_cplx"], cases.adversarial_batch(3), "text")
        print("SURVIVED")
    except AssertionError:
        print("KILLED")
    except BaseException as e:
        print("KILLED (%s)" % type(e).__name__)


def line_range(text, spec):
    """[first, last) line indices of --range FROM[:TO]"""
    lines = text.split("\n")
    frm, _, to = spec.partition(":")
    a = next(i for i, ln in enumerate(lines) if frm in ln)
    b = next((i for i in range(a + 1, len(lines)) if to in lines[i]), len(lines)) if to else len(lines)
    return a, b


def candidates(text, rng_lines=None):
    out = []
    in_comment = False
    for li, line in enumerate(text.split("\n")):
        code = line
        if in_comment:
            if "*/" not in code:
                continue
            code = " " * (code.index("*/") + 2) + code[code.index("*/") + 2:]
            in_comment = False
        if "/*" in code and "*/" not in code[code.index("/*"):]:
            in_comment = True
            code = code[:code.index("/*")]
        code = re.sub(r"/\*.*?\*/", lambda m: " " * len(m.group(0)), code).split("//")[0]
        st = code.strip()
        if not st or st.startswith("#") or st.startswith("template") or "static_assert" in st or "<<<" in st or "asm" in st:
            continue
        if rng_lines and not rng_lines[0] <= li < rng_lines[1]:
            continue
        for pat, rep in OPS:
            for m in re.finditer(pat, code):
                out.append((li, m.start(), m.end(), rep))
    return out


def run_one(args):
    import capacity
    import simt_emu
    k, fn, text, (li, a, b, rep), only = args
    lines = text.split("\n")
    new = lines[li][:a] + rep + lines[li][b:]
    mutated = "\n".join(lines[:li] + [new] + lines[li + 1:])
    try:
        lib = simt_emu.build_library({fn: mutated}) if only != "reports" else "-"
        small = (simt_emu.build_library(capacity.shrunk_sources({fn: mutated}, **shrunk_values()))
                 if only not in ("ext", "state") else None)
    except Exception:
        return k, "nocompile", lines[li], new
    try:
        p = subprocess.run([sys.executable, os.path.abspath(__file__), "--battery", lib, small or "-"] + ([only] if only else []),
                           capture_output=True, text=True, timeout=1200)
        out = p.stdout.strip().split("\n")[-1] if p.stdout.strip() else "KILLED (crash)"
    except subprocess.TimeoutExpired:
        out = "KILLED (timeout)"
    subprocess.run(["rm", "-rf"] + [os.path.dirname(p) for p in (small, lib) if p and p != "-"])
    return k, out, lines[li], new


if __name__ == "__main__":
    if sys.argv[1] == "--battery":
        battery(*sys.argv[2:5])
        sys.exit(0)
    argv, flags = [], {}
    it = iter(sys.argv[1:])
    for a in it:
        if a in ("--range", "--only"):
            flags[a] = next(it)
        else:
            argv.append(a)
    fn, count = argv[0], int(argv[1])
    rng = random.Random(int(argv[2]) if len(argv) > 2 else 1)
    text = open(os.path.join(ROOT, "fastplong_b200", "csrc", fn)).read()
    span = line_range(text, flags["--range"]) if "--range" in flags else None
    cand = candidates(text, span)
    picks = rng.sample(cand, min(count, len(cand)))
    print(f"{fn}: {len(cand)} candidate mutants" + (f" in lines {span[0] + 1}..{span[1]}" if span else "") + f", running {len(picks)}",
          flush=True)
    tally = {}
    with ThreadPoolExecutor(int(argv[3]) if len(argv) > 3 else 6) as ex:
        for k, out, old, new in ex.map(run_one, [(k, fn, text, c, flags.get("--only")) for k, c in enumerate(picks)]):
            tally[out.split(" ")[0]] = tally.get(out.split(" ")[0], 0) + 1
            if out.startswith("SURVIVED"):
                print(f"SURVIVED  line {picks[k][0] + 1}: {old.strip()[:110]}   ==>   {new.strip()[:110]}", flush=True)
    print(tally)
