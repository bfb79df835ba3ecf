"""Differential test: the oracle restatement vs the UNMODIFIED reference operators (oracle/_ref/libfplref.so) on
seeded batches beyond the committed fixtures.  Skipped where the prebuilt reference library is absent."""
import numpy as np
import pytest

import cases
from fastplong_b200 import Options, pack_reads, synth
from oracle_lib import OracleEngine, RefEngine, compare_lists, compare_results, compare_stats, have_ref

pytestmark = pytest.mark.skipif(not have_ref(), reason="oracle/_ref/libfplref.so not built")


def check(opt, batch, what):
    o, r = OracleEngine(opt), RefEngine(opt)
    compare_results(o.process(batch), r.process(batch), what)
    cyc = max(1, int(batch.lens.max()) if batch.n_reads else 1)
    for w in (0, 1):
        compare_stats(o.stats(w, cyc), r.stats(w, cyc), f"{what}/stats{w}")
    compare_stats(o.counters(), r.counters(), what + "/counters")


@pytest.mark.parametrize("name", sorted(cases.OPTION_SETS))
@pytest.mark.parametrize("seed", [1, 2])
def test_adversarial(name, seed):
    check(cases.OPTION_SETS[name], cases.adversarial_batch(seed), f"{name}/adv{seed}")


@pytest.mark.parametrize("name", sorted(cases.OPTION_SETS))
def test_ont_like(name):
    check(cases.OPTION_SETS[name], cases.ont_batch(77, n=150, mean=2500, p_chimera=0.05, p_polya=0.05), name + "/ont")


@pytest.mark.parametrize("n", sorted(cases.LONG_ADAPTERS))
def test_long_adapters(n):
    check(cases.OPTION_SETS[f"long_adapter_{n}"], cases.long_adapter_batch(n, 900 + n), f"long{n}")


def test_edit_distance_random_pairs():
    rng = np.random.default_rng(5)
    o, r = OracleEngine(Options()), RefEngine(Options())
    for _ in range(3000):
        la, lb = int(rng.integers(0, 150)), int(rng.integers(0, 150))
        a = synth.BASES[rng.integers(0, 4, size=la)].tobytes()
        b = synth.BASES[rng.integers(0, 4, size=lb)].tobytes()
        if rng.random() < 0.5 and la:
            b = a[: int(rng.integers(0, la + 1))] + b[: int(rng.integers(0, 6))]
        assert o.edit_distance(a, b) == r.edit_distance(a, b)
    for la, lb in ((700, 650), (641, 10), (64, 65), (128, 129), (640, 640)):
        a = synth.BASES[rng.integers(0, 4, size=la)].tobytes()
        b = synth.BASES[rng.integers(0, 4, size=lb)].tobytes()
        assert o.edit_distance(a, b) == r.edit_distance(a, b)


@pytest.mark.parametrize("name", sorted(cases.RNA_SETS))
@pytest.mark.parametrize("mixed", [False, True])
def test_rna_reads(name, mixed):
    """U instead of T: 5-mers through base2val's U case, content bin 5, byte-wise adapter comparison, polyX that does not
    count U."""
    batch = cases.rna_batch(41, mixed=mixed)
    assert (batch.seq == ord("U")).sum() > 10000
    check(cases.RNA_SETS[name], batch, f"{name}/rna{int(mixed)}")


@pytest.mark.parametrize("name", sorted(cases.edge_cases()))
def test_crafted_boundary_cases(name):
    """cases.edge_cases(): the boundaries a mutation run over the oracle found unpinned (more events than inline slots, global
    trims that eat the read exactly, a cut from one side with a trim on the other, N inside polyX runs, one filter without
    the other, ties of the filter thresholds)."""
    opt, batch = cases.edge_cases()[name]
    check(opt, batch, name)


@pytest.mark.parametrize("name", sorted(cases.EXTREME_SETS))
def test_extreme_option_values(name):
    opt = cases.EXTREME_SETS[name]
    batch = cases.ont_batch(8, n=40, mean=2500, p_chimera=0.2, p_polya=0.2) if name == "fasta_200_entries" else cases.adversarial_batch(12)
    o, r = OracleEngine(opt), RefEngine(opt)
    compare_results(o.process(batch), r.process(batch), name)
    if opt.mask or opt.break_reads:
        compare_lists(o.segments(), r.segments(), name + "/segments")
        compare_lists(o.mask_regions(), r.mask_regions(), name + "/regions")
    cyc = int(batch.lens.max())
    for w in (0, 1):
        compare_stats(o.stats(w, cyc), r.stats(w, cyc), f"{name}/stats{w}")
    compare_stats(o.counters(), r.counters(), name + "/counters")


@pytest.mark.parametrize("name", sorted(cases.QUALITY_DOMAIN_SETS))
def test_quality_bytes_1_to_127(name):
    """quality bytes over the whole range the reference takes (1..127: runs below '!', runs of 127, all-low reads whose
    totalQual is negative, windows exactly on a cut / mask / break threshold) under -q 0 / 93, --mean_qual 1 / 93 and the cut,
    mask and break qualities at the ends of what the CLI accepts"""
    opt = cases.QUALITY_DOMAIN_SETS[name]
    batch = cases.quality_domain_batch(21)
    o, r = OracleEngine(opt), RefEngine(opt)
    compare_results(o.process(batch), r.process(batch), name)
    if opt.mask or opt.break_reads:
        compare_lists(o.segments(), r.segments(), name + "/segments")
        compare_lists(o.mask_regions(), r.mask_regions(), name + "/regions")
    cyc = int(batch.lens.max())
    for w in (0, 1):
        compare_stats(o.stats(w, cyc), r.stats(w, cyc), f"{name}/stats{w}")
    compare_stats(o.counters(), r.counters(), name + "/counters")


def test_empty_batch():
    check(cases.OPTION_SETS["default_se"], pack_reads([]), "empty")


@pytest.mark.parametrize("name", sorted(cases.MASK_BREAK_SETS))
@pytest.mark.parametrize("kind", ["blocky", "adversarial", "ont"])
def test_mask_break(name, kind):
    """--mask / --break: records, the output-read list, the masked regions, both Stats blocks, counters."""
    opt = cases.MASK_BREAK_SETS[name]
    batch = {"blocky": lambda: cases.blocky_quality_batch(5, n=100), "adversarial": lambda: cases.adversarial_batch(4),
             "ont": lambda: cases.ont_batch(6, n=80, mean=2000, p_chimera=0.05)}[kind]()
    o, r = OracleEngine(opt), RefEngine(opt)
    what = f"{name}/{kind}"
    compare_results(o.process(batch), r.process(batch), what)
    compare_lists(o.segments(), r.segments(), what + "/segments")
    compare_lists(o.mask_regions(), r.mask_regions(), what + "/regions")
    cyc = max(1, int(batch.lens.max()))
    for w in (0, 1):
        compare_stats(o.stats(w, cyc), r.stats(w, cyc), f"{what}/stats{w}")
    compare_stats(o.counters(), r.counters(), what + "/counters")


@pytest.mark.parametrize("seed", [31, 32, 33])
def test_random_option_sets(seed):
    """Seeded random option sets x batches (cases.random_case; tools/fuzz_oracle_vs_reference.py runs the same for longer)."""
    import random
    rng = random.Random(seed)
    for i in range(40):
        opt, batch, what = cases.random_case(rng)
        o, r = OracleEngine(opt), RefEngine(opt)
        compare_results(o.process(batch), r.process(batch), f"{what}")
        if opt.mask or opt.break_reads:
            compare_lists(o.segments(), r.segments(), what + "/segments")
            compare_lists(o.mask_regions(), r.mask_regions(), what + "/regions")
        cyc = max(1, int(batch.lens.max()))
        for w in (0, 1):
            compare_stats(o.stats(w, cyc), r.stats(w, cyc), f"{what}/stats{w}")
        compare_stats(o.counters(), r.counters(), what + "/counters")


@pytest.mark.parametrize("name", sorted(cases.MASK_BREAK_EDGE_SETS))
def test_mask_break_edges(name):
    """cases.MASK_BREAK_EDGE_SETS on cases.mask_break_edge_batch: pieces on the length limits, filter ties on the masked copy,
    region walks at base 0 and the last base, split reads broken on either side, more than two output reads per read."""
    opt, batch = cases.MASK_BREAK_EDGE_SETS[name], cases.mask_break_edge_batch()
    o, r = OracleEngine(opt), RefEngine(opt)
    what = f"{name}/edges"
    compare_results(o.process(batch), r.process(batch), what)
    compare_lists(o.segments(), r.segments(), what + "/segments")
    compare_lists(o.mask_regions(), r.mask_regions(), what + "/regions")
    cyc = max(1, int(batch.lens.max()))
    for w in (0, 1):
        compare_stats(o.stats(w, cyc), r.stats(w, cyc), f"{what}/stats{w}")
    compare_stats(o.counters(), r.counters(), what + "/counters")
