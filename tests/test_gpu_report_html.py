"""fpl_report_html / Engine.report_html on the device: the reference's HTML report byte for byte, held to the plain-Python twin
(tests/report_html_twin.py) built from the library's accumulators and the ORACLE's records and output-read lists:
  - every option set, every --mask/--break set, RNA; empty reads and medians below 33; all reads failing; a fresh context;
  - accumulation over calls and fpl_reset; FASTQ text input; a call split into tiles and into upload pieces;
  - reads past 300 cycles (down-sampled curves), reads past 2^21 cycles and the N50 wrap (not under the emulator);
  - the two-phase contract, the error cases, kernel names and launch counts, and capture off changing nothing."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import cases
import report_html_twin
from fastplong_b200 import Options, abi, pack_reads, synth
from fastplong_b200.binding import Engine, FplError
from oracle_lib import OracleEngine, compare_results, compare_stats

pytestmark = pytest.mark.gpu

EMULATED = os.environ.get("FPL_EMULATE", "") not in ("", "0")
TIME = "2026-10-16      12:00:00"
EXT_NAMES = set(cases.MASK_BREAK_SETS)


def is_ext(opt):
    o = opt.to_abi()[0]
    return bool(o.mask_enabled or o.break_enabled)


class Twin:
    """the oracle run next to the library: the lists Stats::statRead would build, call after call"""

    def __init__(self, opt):
        self.opt, self.o, self.pre, self.post = opt, OracleEngine(opt), [], []

    def process(self, batch):
        res = self.o.process(batch)
        pre, post = report_html_twin.read_lists(batch.lens, res, self.o.segments() if is_ext(self.opt) else None)
        self.pre += pre
        self.post += post
        return res

    def reset(self):
        self.pre, self.post = [], []

    def text(self, e, **kw):
        kw.setdefault("time_text", TIME)
        return report_html_twin.report(e.stats(0), e.stats(1), e.counters(), self.opt, self.pre, self.post, **kw)


def engine(opt):
    e = Engine(opt)
    e.keep_read_lists(True)
    return e


def assert_same(got, want):
    if got != want:
        i = next((i for i in range(min(len(got), len(want))) if got[i] != want[i]), min(len(got), len(want)))
        raise AssertionError(f"reports differ at byte {i} of {len(got)} / {len(want)}:\n"
                             f"library: {got[max(0, i - 160):i + 60]!r}\ntwin:    {want[max(0, i - 160):i + 60]!r}")


def run_both(opt, batches, **kw):
    e, t = engine(opt), Twin(opt)
    for b in batches:
        compare_results(e.process(b), t.process(b), "records")
    assert_same(e.report_html(time_text=TIME, **kw), t.text(e, **kw))
    return e, t


def option_set_batch(name, seed):
    if name.startswith("long_adapter_"):
        return cases.long_adapter_batch(int(name.rsplit("_", 1)[1]), seed, n=60)
    if name == "fasta5":
        return pack_reads(cases.planted_fasta_reads(seed, n=80))
    if name == "fasta64_polyx":
        return cases.hifi_fasta64_batch(seed, n=80, mean=1500)
    return synth.ont_like(80, 1500, seed, p_chimera=0.08, p_polya=0.08, q_mean=17.0)


@pytest.mark.parametrize("name", sorted(cases.OPTION_SETS))
def test_html_equals_twin(name):
    run_both(cases.OPTION_SETS[name], [option_set_batch(name, 300 + len(name))], command=f"fastplong {name}")


@pytest.mark.parametrize("name", sorted(cases.MASK_BREAK_SETS))
def test_html_equals_twin_mask_break(name):
    run_both(cases.MASK_BREAK_SETS[name], [cases.blocky_quality_batch(500 + len(name), n=80)])


@pytest.mark.parametrize("name", sorted(cases.RNA_SETS))
def test_html_equals_twin_rna(name):
    e, _ = run_both(cases.RNA_SETS[name], [cases.rna_batch(70 + len(name), n=80)], is_rna=True)
    assert b"<td style='color:#333333'>UU</td>" in e.report_html(time_text=TIME, is_rna=True)


def test_empty_reads_and_low_medians():
    """quirk 1 (empty reads in the list, 0 in the density tail) and medians below '!' + 33 (negative x)"""
    reads = [(b"", b""), (b"ACGTACGTAC" * 30, b"\x1e" * 300), (b"", b""), (b"ACGT" * 100, b"(" * 400), (b"GATTACA" * 50, b"I" * 350)]
    batch = pack_reads(reads * 6)
    opt = Options(length_required=10)
    e, _ = run_both(opt, [batch], title="my run")
    text = e.report_html(time_text=TIME, title="my run")
    assert b"var density={x:[-3,-3,-3,-3,-3,-3,7," in text and b">my run</a>" in text
    dens = text.split(b"var density={x:[")[1].split(b"]")[0].split(b",")
    assert len(dens) == 30 and dens[-12:] == [b"0"] * 12


def test_all_reads_failing_and_no_reads():
    opt = Options(start_adapter=synth.ADAPTER_START, length_required=1_000_000, length_limit=2_000_000, low_complexity_filter=True)
    e, _ = run_both(opt, [synth.ont_like(50, 1200, 8)])
    text = e.report_html(time_text=TIME)
    assert b"reads too long:" in text and b"reads with low complexity:" in text
    fresh, tw = engine(opt), Twin(opt)
    text = fresh.report_html(time_text=TIME)
    assert_same(text, tw.text(fresh))
    assert b"reads passed filters:</td><td class='col2'>0 (-nan%)" in text


def test_accumulates_resets_and_reads_fastq():
    opt = cases.OPTION_SETS["fasta5"]
    e, t = engine(opt), Twin(opt)
    for seed in (1, 2, 3):
        b = synth.ont_like(40, 900 * seed, 40 + seed, p_chimera=0.1)
        e.process(b)
        t.process(b)
        assert_same(e.report_html(time_text=TIME), t.text(e))
    e.reset()
    t.reset()
    assert_same(e.report_html(time_text=TIME), t.text(e))
    b = synth.ont_like(30, 700, 44)
    text = b"".join(b"@r%d\n" % i + b.read(i)[0] + b"\n+\n" + b.read(i)[1] + b"\n" for i in range(b.n_reads))
    recs, res, used = e.process_fastq(text)
    compare_results(res, t.process(b), "fastq records")
    assert_same(e.report_html(time_text=TIME), t.text(e))


def _run_env(env, code):
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, env={**os.environ, **env}, timeout=1800,
                       cwd=os.path.dirname(os.path.abspath(__file__)))
    assert r.returncode == 0, r.stderr.decode()[-3000:]
    return r.stdout


TILE_CODE = """
import sys, hashlib, numpy as np
sys.path.insert(0, '..')
import cases
from fastplong_b200 import synth
from fastplong_b200.binding import Engine
e = Engine(cases.OPTION_SETS['cut_polyx_cplx']); e.keep_read_lists(True)
b = synth.ont_like(3000, 1500, 77, p_chimera=0.1)
e.process(b)
sys.stdout.write(hashlib.md5(e.report_html(time_text='t')).hexdigest())
"""


def test_tiles_and_upload_pieces_give_one_call_s_lists():
    one = _run_env({"FPL_TILE_MBASES": "0", "FPL_PIECE_MB": "0"}, TILE_CODE)
    assert _run_env({"FPL_PIECE_MB": "1"}, TILE_CODE) == one
    dev = TILE_CODE.replace("e.process(b)", "import torch; d = [torch.from_numpy(x).cuda() for x in (b.seq, b.qual, b.offsets, b.lens)]\n"
                            "e.process_device(*(t.data_ptr() for t in d), b.n_reads, b.n_bytes); e.sync()")
    if not EMULATED:
        assert _run_env({"FPL_TILE_MBASES": "1"}, dev) == one


def test_long_reads_are_down_sampled():
    rng = np.random.default_rng(5)
    reads = []
    for L in (350, 2000, 7777):
        s = synth.BASES[rng.integers(0, 4, L)].tobytes()
        reads.append((s, (rng.integers(3, 45, L).astype(np.uint8) + 33).tobytes()))
    e, _ = run_both(cases.OPTION_SETS["cut_polyx_cplx"], [pack_reads(reads * 3)])
    assert b",type:'log'" in e.report_html(time_text=TIME)


@pytest.mark.skipif(EMULATED, reason="millions of cycles: minutes under the emulator")
def test_reads_past_2_21_cycles():
    rng = np.random.default_rng(21)
    reads = []
    for L in (2_300_000, 2_950_000, 2_150_000):
        s = synth.BASES[rng.integers(0, 4, L)].tobytes()
        reads.append((synth.ADAPTER_START.encode() + s, b"5" * len(synth.ADAPTER_START) + (rng.integers(3, 45, L).astype(np.uint8) + 33).tobytes()))
    run_both(cases.OPTION_SETS["cut_polyx_cplx"], [pack_reads(reads)])


@pytest.mark.skipif(EMULATED, reason="2 Gb of reads: minutes under the emulator")
def test_n50_int_product_wraps():
    """2048 reads of 2^20 bases: one length holds 2^31 bases, its int * int product wraps to INT_MIN in the reference"""
    L = 1 << 20
    s = (b"ACGT" * (L // 4))
    q = b"5" * L
    reads = [(s, q)] * 2048 + [(s[:1000], q[:1000])] * 3
    opt = Options(disable_adapter_trimming=True)
    e, t = engine(opt), Twin(opt)
    b = pack_reads(reads)
    e.process(b)
    t.process(b)
    text = e.report_html(time_text=TIME)
    assert_same(text, t.text(e))
    assert report_html_twin.length_stats(t.pre, int(e.stats(0)[16 * e.cycles + abi.STATS_LENSUM]))[3] == 0


def test_two_phase_contract_errors_and_kernels():
    opt = cases.OPTION_SETS["default_se"]
    e, t = engine(opt), Twin(opt)
    b = synth.ont_like(60, 1500, 5)
    e.process(b)
    t.process(b)
    e.set_timing(True)
    lib = e.lib
    mk = lambda size=C.sizeof(abi.FplReportHtmlInfo), v=b"0.4.1", cmd=b"cmd", title=b"fastplong report", tt=TIME.encode(): \
        abi.FplReportHtmlInfo(size, 0, v, cmd, title, tt)  # noqa: E731
    info = mk()
    n = C.c_int64(-1)
    assert lib.fpl_report_html(e.h, C.byref(info), None, 0, C.byref(n)) == 1
    size = n.value
    buf = np.full(size + 8, 0xAB, dtype=np.uint8)
    assert lib.fpl_report_html(e.h, C.byref(info), buf.ctypes.data, size - 1, C.byref(n)) == 1
    assert n.value == size and (buf == 0xAB).all()
    assert lib.fpl_report_html(e.h, C.byref(info), buf.ctypes.data, size + 8, C.byref(n)) == 0
    assert (buf[size:] == 0xAB).all() and buf[:size].tobytes() == t.text(e, command="cmd")
    kt = e.kernel_times()
    for k in ("k_html(cycles)", "k_html(group hist)", "k_html(group scatter)", "k_html(sizes)", "k_html(text)"):
        assert kt[k][1] >= 1, k
    assert kt["k_html(lengths)"][1] == 2 and kt["k_html(values)"][1] == 2 and kt["k_html(sums)"][1] == 2
    assert lib.fpl_report_html(e.h, C.byref(mk(size=C.sizeof(abi.FplReportHtmlInfo) + 8)), None, 0, C.byref(n)) < 0
    assert b"struct_size" in lib.fpl_last_error()
    for bad in (mk(v=None), mk(cmd=None), mk(title=None), mk(tt=None)):
        assert lib.fpl_report_html(e.h, C.byref(bad), None, 0, C.byref(n)) < 0
    # one capture launch per call; a later call invalidates the text
    e.set_timing(True)
    b2 = synth.ont_like(20, 800, 6)
    e.process(b2)
    t.process(b2)
    assert e.kernel_times()["k_html(capture)"][1] == 1
    assert_same(e.report_html(time_text=TIME), t.text(e))
    # capture switched off for one call: refused until fpl_reset
    e.keep_read_lists(False)
    e.process(b2)
    e.keep_read_lists(True)
    with pytest.raises(FplError, match="capture"):
        e.report_html(time_text=TIME)
    e.reset()
    assert e.report_html(time_text=TIME)
    late = Engine(opt)
    late.process(b2)
    late.keep_read_lists(True)
    late.process(b2)
    with pytest.raises(FplError, match="capture"):
        late.report_html()


@pytest.mark.parametrize("name", ["cut_polyx_cplx", "mask_and_break"])
def test_capture_off_changes_nothing(name):
    opt = cases.OPTION_SETS.get(name) or cases.MASK_BREAK_SETS[name]
    b = cases.blocky_quality_batch(9, n=80) if name in EXT_NAMES else synth.ont_like(80, 1500, 9, p_chimera=0.1)
    on, off = engine(opt), Engine(opt)
    off.set_timing(True)
    r_on, r_off = on.process(b), off.process(b)
    compare_results(r_on, r_off, "records")
    for w in (0, 1):
        compare_stats(on.stats(w), off.stats(w), f"stats{w}")
    compare_stats(on.counters(), off.counters(), "counters")
    assert off.kernel_times()["k_html(capture)"][1] == 0
    assert on.report_json() == off.report_json()


import html_golden  # noqa: E402
import json  # noqa: E402

GOLDEN = json.load(open(html_golden.FIXTURE))


@pytest.mark.parametrize("name", sorted(GOLDEN))
def test_html_matches_golden_reference_run(name):
    """the library's report, masked (time text, footer command, quirk-1 tail), has the md5 of the reference binary's -w 1 -h report"""
    g = GOLDEN[name]
    opt, batch = html_golden.run_input(name)
    if html_golden.input_md5(batch) != g["input_md5"]:
        pytest.skip("numpy generator produced a different synthetic input than when the fixture was made")
    e = engine(opt)
    e.set_timing(True)
    e.process(batch)
    e.sync()
    assert e.kernel_times()["k_html(capture)"][1] == 1
    before = e.launch_count
    text = e.report_html(command="fastplong -i in.fq", title=html_golden.TITLE.get(name, "fastplong report"),
                         time_text=html_golden.TIME, is_rna=name in html_golden.IS_RNA)
    assert html_golden.masked_md5(text, g["empty"]) == g["html_md5"]
    # launches of one report: cycles + 2 bins, per block hist/scan/scatter (cub not counted) and 3 length kernels,
    # 2 values + 2 sums, sizes, frame + text
    kt = e.kernel_times()
    assert e.launch_count - before == 1 + 2 + 2 * 2 + 2 * 3 + 2 + 2 + 1 + 2
    assert kt["k_html(group hist)"][1] == 2 and kt["k_html(group scatter)"][1] == 2 and kt["k_html(text)"][1] == 1


def test_launch_count_of_an_empty_report():
    e = engine(cases.OPTION_SETS["default_se"])
    before = e.launch_count
    e.report_html(time_text=TIME)
    assert e.launch_count - before == 1 + 4 + 1          # k_report_cycles, 2 k_html_lenprod + 2 k_html_lensearch, k_report_frame
