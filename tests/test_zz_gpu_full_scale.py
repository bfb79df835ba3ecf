"""bench.py's full-size parity check (full_scale_check) on the GPU at a size the whole oracle would need minutes for: a
device-generated batch goes through fpl_process_device exactly as in the bench; the records of read ranges spread over
the batch are held to the oracle, every word of both Stats blocks and every median to the torch restatement
(tests/stats_tables.py, pinned to the oracle by tests/test_stats_tables.py), the filter counters to the records.
(Named to run last: it drives bench.py's own code.)"""
import os

import numpy as np
import pytest


@pytest.mark.gpu
@pytest.mark.parametrize("optset,n,mean", [("cut_polyx_cplx", 20000, 6000), ("default_se", 3000, 40000)])
def test_full_scale_check_on_a_device_resident_batch(optset, n, mean, monkeypatch):
    import torch
    import bench
    import cases
    from fastplong_b200 import synth_fast
    from fastplong_b200.binding import Engine
    monkeypatch.setattr(bench, "FULL_CHECK_BASES", 6_000_000)
    emulated = os.environ.get("FPL_EMULATE", "") not in ("", "0")      # conftest.py: device memory of the emulated library is host memory
    dev = torch.device("cpu" if emulated else "cuda:0")
    if emulated:
        n, mean = max(200, n // 20), min(mean, 6000)
    opt = cases.OPTION_SETS[optset]
    tile = synth_fast.ont_like_device(n, mean, 4242, dev, p_chimera=0.02)
    offs = torch.from_numpy(tile.offsets).to(dev)
    lens = torch.from_numpy(tile.lens).to(dev)
    if not emulated:
        torch.cuda.synchronize()
    eng = Engine(opt)
    eng.process_device(tile.seq.data_ptr(), tile.qual.data_ptr(), offs.data_ptr(), lens.data_ptr(), tile.n_reads, tile.seq.numel())
    eng.sync()
    out = bench.full_scale_check(torch, eng, opt, tile, tile.seq, tile.qual, tile.offsets, tile.lens, tile.n_reads, mean)
    assert out["ok"] is True and out["reads"] == n
    assert out["records_vs_oracle"]["read_ranges"][-1][1] == n and out["stats_vs_torch"]["passing_segments"] > 0
    # the checker does see a difference: one more pass doubles the accumulators but not the restatement
    eng.process_device(tile.seq.data_ptr(), tile.qual.data_ptr(), offs.data_ptr(), lens.data_ptr(), tile.n_reads, tile.seq.numel())
    eng.sync()
    with pytest.raises(AssertionError):
        bench.full_scale_check(torch, eng, opt, tile, tile.seq, tile.qual, tile.offsets, tile.lens, tile.n_reads, mean)
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["rna_adapters", "rna_reads_dna_adapters", "rna_mixed_adapter_fasta"])
@pytest.mark.parametrize("mixed", [False, True])
def test_rna_reads_vs_oracle(name, mixed):
    """Direct-RNA input (U instead of T; cases.RNA_SETS, pinned oracle-vs-reference on the CPU): U inside valid 5-mers
    (k_cycle_stats' exact ACGTU test, k_kmer_fix), content bin 5, U bytes on the bit-plane path of the whole-read scan
    (never an adapter letter, never an N), adapters that contain U (byte-wise paths), polyX that does not count U."""
    import cases
    from test_gpu_parity import check_against_oracle
    check_against_oracle(cases.RNA_SETS[name], cases.rna_batch(41, mixed=mixed), f"{name}/rna{int(mixed)}")


def _edge_names():
    import cases
    return sorted(cases.edge_cases())


@pytest.mark.gpu
@pytest.mark.parametrize("name", _edge_names())
def test_crafted_boundary_cases_vs_oracle(name):
    """cases.edge_cases() (each pinned oracle-vs-reference on the CPU): boundaries no other batch reaches."""
    import cases
    from test_gpu_parity import check_against_oracle
    opt, batch = cases.edge_cases()[name]
    check_against_oracle(opt, batch, name)


def _extreme_names():
    import cases
    return sorted(cases.EXTREME_SETS)


@pytest.mark.gpu
@pytest.mark.parametrize("name", _extreme_names())
def test_extreme_option_values_vs_oracle(name):
    """cases.EXTREME_SETS: option values at the ends of what the CLI accepts (pinned oracle-vs-reference on the CPU)"""
    import cases
    from test_gpu_parity import check_against_oracle
    batch = cases.ont_batch(8, n=40, mean=2500, p_chimera=0.2, p_polya=0.2) if name == "fasta_200_entries" else cases.adversarial_batch(12)
    check_against_oracle(cases.EXTREME_SETS[name], batch, name)


@pytest.mark.gpu
@pytest.mark.parametrize("switch", ["FPL_NO_JIT", "FPL_FORCE_GENERIC_SCAN"])
@pytest.mark.parametrize("name", ["filter_ties", "complexity_on_tiny_reads_30", "qual_filter_without_length_filter"])
def test_filter_counts_of_the_other_scan_kernels(name, switch, monkeypatch):
    """the threshold ties and the tiny reads with passFilter's counts taken by k_scan_fast / the generic k_scan instead of k_scan_jit"""
    import cases
    from test_gpu_parity import check_against_oracle
    monkeypatch.setenv(switch, "1")
    opt, batch = cases.edge_cases()[name]
    check_against_oracle(opt, batch, f"{name}/{switch}")


def _quality_names():
    import cases
    return sorted(cases.QUALITY_DOMAIN_SETS)


@pytest.mark.gpu
@pytest.mark.parametrize("switch", [None, "FPL_NO_JIT", "FPL_FORCE_GENERIC_SCAN"])
@pytest.mark.parametrize("name", _quality_names())
def test_quality_bytes_1_to_127_vs_oracle(name, switch, monkeypatch):
    """cases.quality_domain_batch (quality bytes 1..127, pinned oracle-vs-reference on the CPU) under the extreme quality
    options, through k_scan_jit, k_scan_fast and the generic k_scan: records, both Stats blocks, counters, the -N/-b lists"""
    import capacity
    import cases
    from fastplong_b200.binding import Engine
    if switch:
        monkeypatch.setenv(switch, "1")
    opt = cases.QUALITY_DOMAIN_SETS[name]
    capacity.compare_with_oracle(Engine(opt), opt, cases.quality_domain_batch(21), f"{name}/{switch}")
