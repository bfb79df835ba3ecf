"""TEST INFRASTRUCTURE: the golden runs of fastplong's HTML report (tests/golden/html_golden.json, made by
tests/golden/make_golden_html.py from the reference binary at -w 1 with -h): how each input is built, and how a report is masked
before its md5 is taken.  Three things are masked, in every text that is compared with a fixture:
  - the time text (the <title> and the footer), replaced by TIME;
  - the footer's <p>command</p>, emptied;
  - quirk 1: the reference prints mReads entries of density arrays that only its reads with bases fill, so the last
    `empty` entries of each block's x and y lists are uninitialised memory there (0 in the library); they are dropped."""
import hashlib
import os
import re
import subprocess

import numpy as np

import cases
from fastplong_b200 import Options, pack_reads, synth

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, "golden", "html_golden.json")
TIME = "2026-10-16      12:00:00"


def quirk_batch():
    """empty reads, medians below 33 (quality char 30) and a few ordinary reads"""
    reads = [(b"", b""), (b"ACGTACGTAC" * 30, b"\x1e" * 300), (b"", b""), (b"ACGT" * 100, b"(" * 400), (b"GATTACA" * 50, b"I" * 350)]
    return pack_reads(reads * 6)


def short_batch(seed):
    """reads of 20..250 bases: total_cycles <= 300, every per-cycle value printed"""
    rng = np.random.default_rng(seed)
    reads = []
    for _ in range(120):
        L = int(rng.integers(20, 251))
        reads.append((synth.BASES[rng.integers(0, 4, L)].tobytes(), (rng.integers(3, 45, L).astype(np.uint8) + 33).tobytes()))
    return pack_reads(reads)


# name: (options, batch maker, is_rna, extra CLI flags, fasta adapters)
RUNS = {
    "default": (lambda: cases.OPTION_SETS["default_se"], lambda: synth.ont_like(150, 1500, 31, p_chimera=0.05, q_mean=17.0)),
    "cut_polyx": (lambda: cases.OPTION_SETS["cut_polyx_cplx"],
                  lambda: synth.ont_like(150, 1500, 32, p_polya=0.05, p_chimera=0.05, q_mean=17.0)),
    "mask": (lambda: cases.MASK_BREAK_SETS["mask_default"], lambda: cases.blocky_quality_batch(33, n=100)),
    "break": (lambda: cases.MASK_BREAK_SETS["break_default"], lambda: cases.blocky_quality_batch(34, n=100)),
    "mask_break": (lambda: cases.MASK_BREAK_SETS["mask_and_break"], lambda: cases.blocky_quality_batch(35, n=100)),
    "rna": (lambda: cases.RNA_SETS["rna_reads_dna_adapters"], lambda: cases.rna_batch(36, n=150)),
    "fasta64": (lambda: cases.OPTION_SETS["fasta64_polyx"], lambda: cases.hifi_fasta64_batch(37, n=120, mean=2500)),
    "cplx_limit": (lambda: Options(start_adapter=synth.ADAPTER_START, low_complexity_filter=True, length_required=500,
                                   length_limit=3000), lambda: synth.ont_like(150, 1500, 38, p_chimera=0.05)),
    "short": (lambda: cases.OPTION_SETS["default_se"], lambda: short_batch(39)),
    "quirks": (lambda: Options(length_required=10), quirk_batch),
}
IS_RNA = {"rna"}
TITLE = {"quirks": "my run"}


def run_input(name):
    opt, mk = RUNS[name]
    return opt(), mk()


def fastq(batch):
    return b"".join(b"@read%d\n%s\n+\n%s\n" % (i, s, q) for i, (s, q) in enumerate(batch.read(i) for i in range(batch.n_reads)))


def input_md5(batch):
    return hashlib.md5(fastq(batch)).hexdigest()


def mask(text, empty):
    """the report with the time text, the footer command and the quirk-1 tail of each density plot masked"""
    text = re.sub(rb"\d+-\d\d-\d\d      \d\d:\d\d:\d\d", b"TIME", text)
    text = re.sub(rb"<div id='footer'> <p>.*?</p>fastplong ", b"<div id='footer'> <p></p>fastplong ", text, flags=re.S)
    parts = text.split(b"var density={x:[")
    for k in range(1, len(parts)):
        xs, rest = parts[k].split(b"],y:[", 1)
        ys, tail = rest.split(b"]", 1)
        drop = empty[k - 1]
        if drop:
            xs = b",".join(xs.split(b",")[:-drop])
            ys = b",".join(ys.split(b",")[:-drop])
        parts[k] = xs + b"],y:[" + ys + b"]" + tail
    return b"var density={x:[".join(parts)


def empties(pre_list, post_list):
    return [sum(1 for L, _ in pre_list if L == 0), sum(1 for L, _ in post_list if L == 0)]


def masked_md5(text, empty):
    return hashlib.md5(mask(text, empty)).hexdigest()


def run_reference(ref_bin, name, workdir):
    """the reference binary at -w 1 on the run's input: the -h report's bytes"""
    opt, batch = run_input(name)
    fq = os.path.join(workdir, "in.fq")
    open(fq, "wb").write(fastq(batch))
    extra = []
    if opt.adapter_fasta:
        fa = os.path.join(workdir, "adapters.fa")
        with open(fa, "w") as f:        # headers chosen so that std::map order == list order (src/options.cpp:50-59)
            for i, s in enumerate(opt.adapter_fasta):
                f.write(f">a{i:03d}\n{s}\n")
        extra += ["-a", fa]
    if name in TITLE:
        extra += ["-R", TITLE[name]]
    html = os.path.join(workdir, "r.html")
    cmd = [ref_bin, "-i", fq, "-o", os.path.join(workdir, "out.fq"), "-j", os.path.join(workdir, "r.json"), "-h", html, "-w", "1"]
    r = subprocess.run(cmd + opt.cli_flags() + extra, capture_output=True, text=True, timeout=600)
    if r.returncode != 0:
        raise RuntimeError(r.stderr[-2000:])
    return open(html, "rb").read()
