"""fpl_report_json / Engine.report_json on the device: the reference's JSON report byte for byte.
  - the six golden runs: the text minus its "command" line has the md5 of the unmodified reference's own report;
  - the plain-Python twin (tests/report_twin.py) on the same accumulators, full text: every option set, RNA, all reads
    failing, a fresh context, accumulation over calls and fpl_reset, reads of 2-3 Mb (total_cycles past 2^21);
  - the two-phase contract (sizing call, short buffer, copy, invalidation by a later call);
  - the reference binary on fresh input (a 64-entry adapter FASTA, direct-RNA reads), where oracle/_ref/fastplong_ref exists."""
import ctypes as C
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

import cases
import report_twin
from fastplong_b200 import Options, abi, pack_reads, synth
from fastplong_b200.binding import Engine, FplError
from oracle_lib import REF_BIN
from test_report_json import GOLDEN, GOLDEN_RUNS, golden_input

pytestmark = pytest.mark.gpu

EMULATED = os.environ.get("FPL_EMULATE", "") not in ("", "0")


def twin(e, opt, **kw):
    return report_twin.report(e.stats(0), e.stats(1), e.counters(), opt, **kw)


def assert_same(got, want):
    if got != want:
        i = next((i for i in range(min(len(got), len(want))) if got[i] != want[i]), min(len(got), len(want)))
        raise AssertionError(f"reports differ at byte {i} of {len(got)} / {len(want)}:\n"
                             f"library: {got[max(0, i - 120):i + 60]!r}\ntwin:    {want[max(0, i - 120):i + 60]!r}")


@pytest.mark.parametrize("name", GOLDEN_RUNS)
def test_report_matches_golden_reference_run(name):
    g = json.load(open(os.path.join(GOLDEN, f"binary_{name}.json")))
    opt, batch = golden_input(name, g)
    e = Engine(opt)
    e.process(batch)
    text = e.report_json(command="fastplong -i in.fq -j out.json")
    assert hashlib.md5(report_twin.without_command(text)).hexdigest() == g["json_text_md5"]
    assert json.loads(text)["command"] == "fastplong -i in.fq -j out.json"


def option_set_batch(name, seed):
    if name.startswith("long_adapter_"):
        return cases.long_adapter_batch(int(name.rsplit("_", 1)[1]), seed, n=60)
    if name == "fasta5":
        return pack_reads(cases.planted_fasta_reads(seed, n=80))
    if name == "fasta64_polyx":
        return cases.hifi_fasta64_batch(seed, n=80, mean=1500)
    return synth.ont_like(80, 1500, seed, p_chimera=0.08, p_polya=0.08, q_mean=17.0)


@pytest.mark.parametrize("name", sorted(cases.OPTION_SETS))
def test_report_equals_twin(name):
    opt = cases.OPTION_SETS[name]
    e = Engine(opt)
    e.process(option_set_batch(name, 300 + len(name)))
    assert_same(e.report_json(command=f"fastplong {name}"), twin(e, opt, command=f"fastplong {name}"))


@pytest.mark.parametrize("name", sorted(cases.MASK_BREAK_SETS))
def test_report_equals_twin_mask_break(name):
    opt = cases.MASK_BREAK_SETS[name]
    e = Engine(opt)
    e.process(cases.blocky_quality_batch(500 + len(name), n=80))
    assert_same(e.report_json(), twin(e, opt))


@pytest.mark.parametrize("name", sorted(cases.RNA_SETS))
def test_report_equals_twin_rna(name):
    opt = cases.RNA_SETS[name]
    e = Engine(opt)
    e.process(cases.rna_batch(70 + len(name), n=80))
    text = e.report_json(is_rna=True)
    assert_same(text, twin(e, opt, is_rna=True))
    rep = json.loads(text)
    assert "U" in rep["read_before_filtering"]["quality_curves"] and "UUUUU" in rep["read_before_filtering"]["kmer_count"]
    assert max(rep["read_before_filtering"]["content_curves"]["U"]) > 0.1


def test_report_all_reads_failing():
    opt = Options(start_adapter=synth.ADAPTER_START, length_required=1_000_000)
    e = Engine(opt)
    e.process(synth.ont_like(50, 1200, 8))
    text = e.report_json()
    assert_same(text, twin(e, opt))
    rep = json.loads(text)
    assert rep["read_after_filtering"]["total_cycles"] == 0 and rep["read_after_filtering"]["quality_curves"]["mean"] == []
    assert rep["filtering_result"]["too_short_reads"] == 50 and rep["summary"]["after_filtering"]["q20_rate"] == 0


def test_report_fresh_context():
    opt = cases.OPTION_SETS["cut_polyx_cplx"]
    e = Engine(opt)
    text = e.report_json()
    assert_same(text, twin(e, opt))
    rep = json.loads(text)
    assert rep["read_before_filtering"]["total_cycles"] == 0 and rep["summary"]["before_filtering"]["read_mean_length"] == 0


def test_report_accumulates_and_resets():
    opt = cases.OPTION_SETS["fasta5"]
    e = Engine(opt)
    for seed in (1, 2, 3):
        e.process(synth.ont_like(40, 900 * seed, 40 + seed, p_chimera=0.1))
        assert_same(e.report_json(), twin(e, opt))
    e.reset()
    assert_same(e.report_json(), Engine(opt).report_json())
    e.process(synth.ont_like(30, 700, 44))
    assert_same(e.report_json(), twin(e, opt))


@pytest.mark.skipif(EMULATED, reason="millions of cycles: minutes under the emulator")
def test_report_reads_past_2_21_cycles():
    """three reads of 2-3 Mb: 11 curves of more than 2^21 values per Stats block"""
    rng = np.random.default_rng(21)
    reads = []
    for L in (2_300_000, 2_950_000, 2_150_000):
        s = synth.BASES[rng.integers(0, 4, L)].tobytes()
        q = (rng.integers(3, 45, L).astype(np.uint8) + 33).tobytes()
        reads.append((synth.ADAPTER_START.encode() + s, b"5" * len(synth.ADAPTER_START) + q))
    opt = cases.OPTION_SETS["cut_polyx_cplx"]
    e = Engine(opt)
    e.process(pack_reads(reads))
    text = e.report_json()
    rep = json.loads(text)
    assert rep["read_before_filtering"]["total_cycles"] > 1 << 21 and rep["read_after_filtering"]["total_cycles"] > 1 << 21
    assert_same(text, twin(e, opt))


def test_two_phase_contract():
    opt = cases.OPTION_SETS["default_se"]
    e = Engine(opt)
    e.process(synth.ont_like(60, 1500, 5))
    e.set_timing(True)
    lib = e.lib
    info = abi.FplReportInfo(C.sizeof(abi.FplReportInfo), 0, b"0.4.1", b"cmd")
    n = C.c_int64(-1)
    assert lib.fpl_report_json(e.h, C.byref(info), None, 0, C.byref(n)) == 1
    size = n.value
    assert size > 100000
    buf = np.full(size + 8, 0xAB, dtype=np.uint8)
    n.value = -1
    assert lib.fpl_report_json(e.h, C.byref(info), buf.ctypes.data, size - 1, C.byref(n)) == 1
    assert n.value == size and (buf == 0xAB).all()                   # too short: nothing written
    assert lib.fpl_report_json(e.h, C.byref(info), buf.ctypes.data, size + 8, C.byref(n)) == 0
    text = buf[:size].tobytes()
    assert (buf[size:] == 0xAB).all()
    assert text == e.report_json(command="cmd") == twin(e, opt, command="cmd")
    kt = e.kernel_times()
    e.sync()
    assert kt["k_report(sizes)"][1] == 1 and kt["k_report(text)"][1] == 1 and kt["k_report(cycles)"][1] == 1
    e.process(synth.ont_like(20, 800, 6))                            # a later call changes the accumulators
    assert lib.fpl_report_json(e.h, C.byref(info), None, 0, C.byref(n)) == 1
    after = e.report_json(command="cmd")
    assert after != text and after == twin(e, opt, command="cmd")
    bad = abi.FplReportInfo(C.sizeof(abi.FplReportInfo) + 4, 0, b"0.4.1", b"cmd")
    assert lib.fpl_report_json(e.h, C.byref(bad), None, 0, C.byref(n)) < 0
    assert b"struct_size" in lib.fpl_last_error()
    with pytest.raises(FplError):
        e._check(lib.fpl_report_json(e.h, C.byref(abi.FplReportInfo(C.sizeof(abi.FplReportInfo), 0, None, b"")), None, 0,
                                     C.byref(n)))


def run_reference(opt, batch, tmp_path, fasta=()):
    fq, js = str(tmp_path / "in.fq"), str(tmp_path / "ref.json")
    synth.to_fastq(batch, fq)
    extra = []
    if fasta:
        fa = str(tmp_path / "adapters.fa")
        with open(fa, "w") as f:        # headers chosen so that std::map order == list order (src/options.cpp:50-59)
            for i, s in enumerate(fasta):
                f.write(f">a{i:03d}\n{s}\n")
        extra = ["-a", fa]
    cmd = [REF_BIN, "-i", fq, "-o", str(tmp_path / "out.fq"), "-j", js, "-h", str(tmp_path / "r.html"), "-w", "3"]
    r = subprocess.run(cmd + opt.cli_flags() + extra, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    return open(js, "rb").read()


@pytest.mark.skipif(not os.path.exists(REF_BIN), reason="oracle/_ref/fastplong_ref not built")
@pytest.mark.parametrize("kind", ["fasta64", "rna"])
def test_report_matches_reference_binary(kind, tmp_path):
    if kind == "fasta64":
        opt = cases.OPTION_SETS["fasta64_polyx"]
        batch = cases.hifi_fasta64_batch(64, n=300, mean=2500)
    else:
        opt = cases.RNA_SETS["rna_reads_dna_adapters"]    # the CLI accepts A/T/C/G adapters only; it sets isRNA from the reads
        batch = cases.rna_batch(65, n=300)
    ref = run_reference(opt, batch, tmp_path, opt.adapter_fasta)
    e = Engine(opt)
    e.process(batch)
    got = e.report_json(is_rna=kind == "rna")
    assert_same(report_twin.without_command(got), report_twin.without_command(ref))
