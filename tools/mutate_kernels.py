"""Development aid (CPU): mutation testing of the GPU tests' grip on the KERNELS.  A sample of single-token mutants of the kernel
sources (comparison operators, && / ||, +-1) is built into the emulated library (tests/simt_emu.py) and run against the oracle on
a battery — crafted boundaries, option matrix on adversarial reads, RNA, -N/-b, FASTQ text, and the capacity limits of the
statistics and text kernels (tests/test_capacity_shrunk.py's cases on the mutant built with shrunk constants, the packed
counter of k_cycle_stats at its fullest).  A surviving mutant is kernel
behaviour the parity tests do not pin — or an equivalent mutant: the one-sided filters (a filter that says "maybe" more often
changes no result by design), min / max ties, guards that cannot fire.
usage: python tools/mutate_kernels.py <file.cu> <n_mutants> [seed] [workers]      (internal: --battery <lib.so> [<shrunk lib.so>])"""
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


def battery(lib, small=None):
    import signal
    import simt_emu
    simt_emu._emu_lib_path = lib
    import capacity
    import cases
    import test_capacity_shrunk as CS
    import test_simt_kernels as T
    signal.alarm(900)
    try:
        # the capacity limits: the mutant built with shrunk constants, and the packed counter at its fullest at full size
        if small:
            CS.LIBS[SHRUNK] = (small, capacity.constants(capacity.shrunk_sources(**CS.BUILDS[SHRUNK])))
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
        for name, opt in cases.MASK_BREAK_SETS.items():
            T.check(opt, cases.blocky_quality_batch(5, n=40), name)
        for n in (33, 65, 129):
            T.check(cases.OPTION_SETS[f"long_adapter_{n}"], cases.long_adapter_batch(n, 900 + n, n=16), f"long{n}")
        T.check(cases.OPTION_SETS["fasta64_polyx"], cases.hifi_fasta64_batch(3, n=40), "fasta64")
        from fastplong_b200 import synth
        T.check(cases.OPTION_SETS["cut_polyx_cplx"], synth.ont_like(2, 110000, 5, p_chimera=1.0), "reads beyond 96 kb")      # block-wide paths
        T.check_text(cases.OPTION_SETS["cut_polyx_cplx"], cases.adversarial_batch(3), "text")
        T.check_text(cases.MASK_BREAK_SETS["mask_and_break"], cases.blocky_quality_batch(5, n=30), "text/ext")
        print("SURVIVED")
    except AssertionError:
        print("KILLED")
    except BaseException as e:
        print("KILLED (%s)" % type(e).__name__)


def candidates(text):
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
        for pat, rep in OPS:
            for m in re.finditer(pat, code):
                out.append((li, m.start(), m.end(), rep))
    return out


def run_one(args):
    import capacity
    import simt_emu
    import test_capacity_shrunk
    k, fn, text, (li, a, b, rep) = args
    lines = text.split("\n")
    new = lines[li][:a] + rep + lines[li][b:]
    mutated = "\n".join(lines[:li] + [new] + lines[li + 1:])
    try:
        lib = simt_emu.build_library({fn: mutated})
        small = simt_emu.build_library(capacity.shrunk_sources({fn: mutated}, **test_capacity_shrunk.BUILDS[SHRUNK]))
    except Exception:
        return k, "nocompile", lines[li], new
    try:
        p = subprocess.run([sys.executable, os.path.abspath(__file__), "--battery", lib, small], capture_output=True, text=True,
                           timeout=1200)
        out = p.stdout.strip().split("\n")[-1] if p.stdout.strip() else "KILLED (crash)"
    except subprocess.TimeoutExpired:
        out = "KILLED (timeout)"
    subprocess.run(["rm", "-rf", os.path.dirname(lib), os.path.dirname(small)])
    return k, out, lines[li], new


if __name__ == "__main__":
    if sys.argv[1] == "--battery":
        battery(*sys.argv[2:4])
        sys.exit(0)
    fn, count = sys.argv[1], int(sys.argv[2])
    rng = random.Random(int(sys.argv[3]) if len(sys.argv) > 3 else 1)
    text = open(os.path.join(ROOT, "fastplong_b200", "csrc", fn)).read()
    cand = candidates(text)
    picks = rng.sample(cand, min(count, len(cand)))
    print(f"{fn}: {len(cand)} candidate mutants, running {len(picks)}", flush=True)
    tally = {}
    with ThreadPoolExecutor(int(sys.argv[4]) if len(sys.argv) > 4 else 6) as ex:
        for k, out, old, new in ex.map(run_one, [(k, fn, text, c) for k, c in enumerate(picks)]):
            tally[out.split(" ")[0]] = tally.get(out.split(" ")[0], 0) + 1
            if out.startswith("SURVIVED"):
                print(f"SURVIVED  {old.strip()[:110]}   ==>   {new.strip()[:110]}", flush=True)
    print(tally)
