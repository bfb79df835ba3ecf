"""Every kernel of libfplgpu executed on the CPU: binding.Engine on the EMULATED library (tests/simt_emu.py: every .cu of
fastplong_b200/csrc, fpl_api.cu and fpl_jit.cu included, built for the host behind the SIMT emulator of tests/simt/) against the
oracle — k_make_preseg, k_trim / k_trim_fasta in their size classes, k_cs_keys / k_cs_gather, k_cycle_stats (5-mer and plain,
cp.async ring and bulk-copy variant), k_scan_jit v2 as fpl_jit.cu generates and "compiles" it per context, k_scan_fast, the
generic k_scan, k_final, k_count, k_kmer_fix, k_read_qual, the --mask/--break kernels, FASTQ text in / text out (k_count_lines,
k_fastq_records, k_fastq_pack, k_emit_sizes, k_emit_copy), k_eval_kmers: every field of every record, every word of both Stats
blocks, every counter, the -N/-b lists, the output text — on the option matrix, adapters up to 1024 bp, the 64-entry FASTA, the
crafted boundaries, RNA reads and seeded random option sets."""
import random

import numpy as np
import pytest

import cases
import simt_emu
from fastplong_b200 import Options, pack_reads, synth
from oracle_lib import OracleEngine, compare_lists, compare_results, compare_stats


def check(opt, batch, what, scan="jit"):
    """scan: which whole-read scan fpl_create sets up on the emulated library — "jit": k_scan_jit v2 specialised through the NVRTC
    stand-in wherever the library specialises, "fast": the precompiled k_scan_fast (FPL_NO_JIT), "generic": k_scan."""
    e, o = simt_emu.EmuEngine(opt, scan=scan), OracleEngine(opt)
    compare_results(e.process(batch), o.process(batch), what)
    if opt.mask or opt.break_reads:
        compare_lists(e.segments(), o.segments(), what + "/segments")
        compare_lists(e.mask_regions(), o.mask_regions(), what + "/regions")
    cyc = max(1, int(batch.lens.max()) if batch.n_reads else 1)
    for w in (0, 1):
        compare_stats(e.stats(w, cyc), o.stats(w, cyc), f"{what}/stats{w}")
    compare_stats(e.counters(), o.counters(), what + "/counters")
    e.close()
    o.close()


PLAIN_SETS = sorted(n for n in cases.OPTION_SETS if not n.startswith("long_adapter_"))


OTHER_SCANS = [(n, sc) for n in ("default_se", "cut_polyx_cplx", "fasta5", "literal_auto", "empty_adapters", "loose_ed") for sc in ("fast", "generic")]


@pytest.mark.parametrize("name,scan", [(n, "jit") for n in PLAIN_SETS] + OTHER_SCANS)
def test_option_matrix_on_adversarial_reads(name, scan):
    check(cases.OPTION_SETS[name], cases.adversarial_batch(1), name + "/adv", scan)


@pytest.mark.parametrize("name", PLAIN_SETS)
def test_option_matrix_on_ont_like_reads(name):
    check(cases.OPTION_SETS[name], cases.ont_batch(77, n=60, mean=2500, p_chimera=0.1, p_polya=0.05), name + "/ont")


@pytest.mark.parametrize("n", sorted(cases.LONG_ADAPTERS))
def test_long_adapters_every_size_class(n):
    """-s / -e of 31..1024 bp: k_trim<0/1/2>, k_final<0/2>, the 64- / 128-bit and multi-word Myers forms; k_scan_jit with 5..8
    count planes and 1..4 halo words up to 128 bp, the generic k_scan beyond"""
    check(cases.OPTION_SETS[f"long_adapter_{n}"], cases.long_adapter_batch(n, 900 + n, n=24), f"long{n}")
    if n <= 128:
        check(cases.OPTION_SETS[f"long_adapter_{n}"], cases.long_adapter_batch(n, 900 + n, n=24), f"long{n}/fast", "fast")


def test_config3_shape_64_entry_fasta():
    check(cases.OPTION_SETS["fasta64_polyx"], cases.hifi_fasta64_batch(3, n=60), "fasta64")


@pytest.mark.parametrize("name", sorted(cases.edge_cases()))
def test_crafted_boundary_cases(name):
    opt, batch = cases.edge_cases()[name]
    check(opt, batch, name)


FILTER_CASES = sorted(n for n in cases.edge_cases() if n.startswith(("filter_ties", "complexity_on_tiny", "qual_filter_without", "length_filter_without",
                                                                     "neither_filter")))


@pytest.mark.parametrize("scan", ["fast", "generic"])
@pytest.mark.parametrize("name", FILTER_CASES)
def test_filter_counts_of_the_other_scan_kernels(name, scan):
    """passFilter's counts (low-quality bases, N, quality sum, unequal neighbours) are taken by whichever scan kernel runs: the
    threshold ties and the tiny reads also through k_scan_fast and the generic k_scan (a mutant of the generic kernel's
    neighbour-byte pick survived the battery: tools/mutate_kernels.py)"""
    opt, batch = cases.edge_cases()[name]
    check(opt, batch, f"{name}/{scan}", scan)


@pytest.mark.parametrize("name", sorted(cases.EXTREME_SETS))
def test_extreme_option_values(name):
    batch = cases.ont_batch(8, n=40, mean=2500, p_chimera=0.2, p_polya=0.2) if name == "fasta_200_entries" else cases.adversarial_batch(12)
    check(cases.EXTREME_SETS[name], batch, name)


@pytest.mark.parametrize("scan", ["jit", "fast", "generic"])
@pytest.mark.parametrize("name", sorted(cases.QUALITY_DOMAIN_SETS))
def test_quality_bytes_1_to_127(name, scan):
    """cases.quality_domain_batch (bytes 1..127, pinned oracle-vs-reference) through each of the three whole-read scans, whose
    quality counts are byte-packed: x = q + (128 - Q) with unsigned and signed dp4a (k_scan_jit), (q | 0x80) - Q (k_scan_fast)"""
    check(cases.QUALITY_DOMAIN_SETS[name], cases.quality_domain_batch(21), f"{name}/{scan}", scan)


@pytest.mark.parametrize("name", sorted(cases.RNA_SETS))
@pytest.mark.parametrize("mixed", [False, True])
def test_rna_reads(name, mixed):
    check(cases.RNA_SETS[name], cases.rna_batch(41, n=60, mean=1200, mixed=mixed), f"{name}/{int(mixed)}")


@pytest.mark.parametrize("name", sorted(cases.MASK_BREAK_SETS))
@pytest.mark.parametrize("kind", ["blocky", "adversarial"])
def test_mask_and_break(name, kind):
    """--mask / --break (fpl_ext.cu: k_ext_count / emit / mask_count / mask_emit / filter / seg_qual / fill_records around two
    exclusive scans): records, the output-read list, the masked regions, the post-filter Stats over the masked bases"""
    batch = cases.blocky_quality_batch(5, n=60) if kind == "blocky" else cases.adversarial_batch(3)
    check(cases.MASK_BREAK_SETS[name], batch, f"{name}/{kind}")


def test_empty_tiny_and_very_long_reads():
    check(cases.OPTION_SETS["cut_polyx_cplx"], pack_reads([]), "empty")
    reads = [((b"ACGTTGCAAC" * 8)[:n], bytes([33 + 30]) * n) for n in (0, 1, 2, 3, 4, 5, 6, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65)] * 2
    check(Options(disable_adapter_trimming=True, length_required=0), pack_reads(reads), "tiny")
    check(cases.OPTION_SETS["cut_polyx_cplx"], pack_reads(reads), "tiny/adapters")
    check(cases.OPTION_SETS["cut_polyx_cplx"], synth.ont_like(3, 60000, 5, p_chimera=1.0), "long reads")
    check(cases.OPTION_SETS["cut_polyx_cplx"], synth.ont_like(3, 60000, 5, p_chimera=1.0), "long reads/generic", "generic")


@pytest.mark.parametrize("family,count", [("random_case", 20), ("random_case_many_adapters", 8), ("random_case_long_reads", 3)])
def test_random_option_sets(family, count):
    rng = random.Random(20260924)
    done = 0
    while done < count:
        opt, batch, what = getattr(cases, family)(rng)
        check(opt, batch, f"{family}[{done}] {what}")
        done += 1


def test_cycle_stats_bulk_copy_variant_in_a_subprocess():
    """FPL_CS_TMA=1 (read once per process): k_cycle_stats<..., TMA = true>, whose rows arrive by one lane's bulk copies; the
    emulator completes a bulk copy at issue, so this checks the variant's addressing and bookkeeping, not its mbarrier waits."""
    import os
    import subprocess
    import sys
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "import cases, test_simt_kernels as t\n"
            "t.check(cases.OPTION_SETS['cut_polyx_cplx'], cases.adversarial_batch(1), 'tma/adv')\n"
            "t.check(cases.OPTION_SETS['default_se'], cases.ont_batch(9, n=40, mean=3000, p_chimera=0.2), 'tma/ont')\n"
            "print('TMA_VARIANT_OK')\n") % (os.path.dirname(os.path.dirname(os.path.abspath(__file__))), os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900, env=dict(os.environ, FPL_CS_TMA="1"))
    assert r.returncode == 0 and "TMA_VARIANT_OK" in r.stdout, r.stdout[-800:] + r.stderr[-1500:]


def test_cp_async_completion_order_does_not_matter():
    """cp.async may complete anywhere between its issue and the wait covering its group: the emulator's default is the latest
    legal moment, this repeats two batches with the earliest one (a kernel correct under both extremes does not lean on when
    the copies land; removing the warp barrier behind k_cycle_stats' wait fails under both, as racecheck reported on the GPU)."""
    lib = simt_emu.emulated_library()
    try:
        lib.emu_set_cp_async_lazy(0)
        check(cases.OPTION_SETS["cut_polyx_cplx"], cases.adversarial_batch(2), "eager/adv")
        check(cases.OPTION_SETS["default_se"], cases.ont_batch(9, n=40, mean=3000, p_chimera=0.2), "eager/ont")
    finally:
        lib.emu_set_cp_async_lazy(1)


# ---- FASTQ text in, FASTQ text out (SURVEY §8f rows 1 and 2): k_count_lines, the newline select, k_fastq_records, k_fastq_pack,
# the kernels above, k_emit_sizes, k_emit_copy — the harness mirrors fpl_process_fastq_host + fpl_emit_fastq_host ----
def _fastq_of(batch):
    """names of varying length, '+' lines that sometimes repeat the name (as tests/test_gpu_emit.py)"""
    names, plus, parts = [], [], []
    for i in range(batch.n_reads):
        s, q = batch.read(i)
        nm = b"@read%d %s" % (i, b"x" * (i % 41))
        pl = b"+" if i % 3 else b"+read%d" % i
        names.append(nm)
        plus.append(pl)
        parts.append(nm + b"\n" + s + b"\n" + pl + b"\n" + q + b"\n")
    return b"".join(parts), names, plus


def check_text(opt, batch, what, want_failed=True, last_newline=True):
    from fastplong_b200 import hostside
    text, names, plus = _fastq_of(batch)
    if not last_newline:
        text = text[:-1]
    e, o = simt_emu.EmuEngine(opt), OracleEngine(opt)
    got = e.process_fastq(text)
    assert got is not None, what
    recs, res, used = got
    out, failed = e.emit_fastq(want_failed)
    assert used == len(text) and len(recs) == batch.n_reads
    ores = o.process(batch)
    compare_results(res, ores, what)
    if opt.mask or opt.break_reads:
        exp_out, exp_failed = hostside.emit_fastq_ext(batch, names, ores, o.segments(), o.mask_regions(), strand=plus)
    else:
        exp_out, exp_failed = hostside.emit_fastq(batch, names, ores, strand=plus)
    assert out == exp_out, f"{what}: --out text differs ({len(out)} bytes, expected {len(exp_out)})"
    assert failed == (exp_failed if want_failed else b""), f"{what}: --failed_out text differs"
    cyc = max(1, int(batch.lens.max()))
    for w in (0, 1):
        compare_stats(e.stats(w, cyc), o.stats(w, cyc), f"{what}/stats{w}")
    compare_stats(e.counters(), o.counters(), what + "/counters")
    e.close()
    o.close()


@pytest.mark.parametrize("name", ["default_se", "cut_polyx_cplx", "trims_limits", "fasta5", "no_adapter_no_filters"])
def test_fastq_text_path(name):
    check_text(cases.OPTION_SETS[name], cases.adversarial_batch(3), name + "/text/adv")
    check_text(cases.OPTION_SETS[name], cases.ont_batch(91, n=50, mean=2000, p_chimera=0.2), name + "/text/ont", last_newline=False)


@pytest.mark.parametrize("name", sorted(cases.MASK_BREAK_SETS))
def test_fastq_text_path_mask_break(name):
    check_text(cases.MASK_BREAK_SETS[name], cases.blocky_quality_batch(5, n=50), name + "/text")


def test_fastq_text_path_without_failed_writer_and_empty_reads():
    check_text(cases.OPTION_SETS["default_se"], cases.adversarial_batch(4), "nofailed", want_failed=False)
    reads = [(b"", b""), (b"A", b"I"), ((b"ACGTTGCAAC" * 9)[:90], b"I" * 90), (b"", b"")]
    check_text(Options(disable_adapter_trimming=True, length_required=0), pack_reads(reads), "empty reads in the text")


@pytest.mark.parametrize("kind", ["crlf", "blank_line", "no_at", "no_plus", "len_mismatch", "three_lines"])
def test_fastq_parser_refuses_non_strict_layouts(kind):
    """what FastqReader would treat by its own rules goes back to the caller (return value 1 of fpl_process_fastq_host)"""
    text = b"@r0\nACGTACGTAC\n+\nIIIIIIIIII\n@r1\nGGGTTTAAAC\n+\nIIIIIIIIII\n"
    text = {"crlf": lambda t: t.replace(b"\n", b"\r\n"), "blank_line": lambda t: t.replace(b"IIIIIIIIII\n@r1", b"IIIIIIIIII\n\n@r1"),
            "no_at": lambda t: t.replace(b"@r1", b"r1x"), "no_plus": lambda t: t.replace(b"\n+\n", b"\n-\n"),
            "len_mismatch": lambda t: t.replace(b"GGGTTTAAAC", b"GGGTTTAAA"),
            "three_lines": lambda t: t[: t.rfind(b"\n", 0, len(t) - 1) + 1]}[kind](text)
    e = simt_emu.EmuEngine(cases.OPTION_SETS["default_se"])
    assert e.process_fastq(text) is None


@pytest.mark.parametrize("side", [0, 1])
def test_adapter_detection_tables(side):
    """k_eval_kmers (fpl_eval.cu, the counting half of Evaluator::evalAdapterAndReadNum) against the numpy restatement, and the
    whole detection — emulated tables + the C ABI's fpl_eval_pick_adapter — finding the planted adapters"""
    from fastplong_b200 import evaluator
    from oracle_lib import kmer10_tables
    reads = synth.adversarial_reads(9) + [synth.ont_like(120, 900, 4).read(i) for i in range(120)]
    batch = pack_reads(reads)
    for shift in (1, 3):
        c, a, t = simt_emu.eval_adapter_kmers(batch, side, shift)
        rc, ra, rt = kmer10_tables(batch, side, shift)
        assert t == rt and np.array_equal(c, rc) and np.array_equal(a, ra)
    if side == 0:
        b = synth.ont_like(400, 1500, 21)
        assert evaluator.detect_adapters(b, kmers=simt_emu.eval_adapter_kmers) == (synth.ADAPTER_START, synth.ADAPTER_END)
