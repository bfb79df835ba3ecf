"""The plain-Python twin of the HTML report (tests/report_html_twin.py) held to the reference binary, without a GPU:
  - the golden runs (tests/golden/html_golden.json: default, cut+polyX, --mask, --break, both, RNA, a 64-entry adapter FASTA,
    -y with --length_limit, reads of <= 300 cycles, empty reads with medians below 33 and -R): the twin's text, built from the
    oracle's accumulators and records, has the md5 of the reference's own masked -h report;
  - the same runs against fresh reference runs byte for byte (where oracle/_ref/fastplong_ref is built), so a mismatch shows
    where;
  - the twin's number formatting (std::to_string, ostream <<, HtmlReporter::formatNumber / getPercents) against the C library
    on the edge values: 999, 1000, 1001, 10^6, 0 / 0, and the k-mer colour boundaries 0.3 and 3.0."""
import ctypes as C
import json
import os

import pytest

import html_golden
import report_html_twin
from oracle_lib import REF_BIN, OracleEngine

GOLDEN = json.load(open(html_golden.FIXTURE))


def twin_text(name, command=""):
    opt, batch = html_golden.run_input(name)
    o = OracleEngine(opt)
    res = o.process(batch)
    ext = opt.to_abi()[0].mask_enabled or opt.to_abi()[0].break_enabled
    pre, post = report_html_twin.read_lists(batch.lens, res, o.segments() if ext else None)
    cyc = max(int(batch.lens.max()), 1)
    text = report_html_twin.report(o.stats(0, cyc), o.stats(1, cyc), o.counters(), opt, pre, post, command=command,
                                   title=html_golden.TITLE.get(name, "fastplong report"), time_text=html_golden.TIME,
                                   is_rna=name in html_golden.IS_RNA)
    return text, html_golden.empties(pre, post), html_golden.input_md5(batch)


@pytest.mark.parametrize("name", sorted(GOLDEN))
def test_twin_matches_golden_reference_report(name):
    text, empty, md5_in = twin_text(name, command="fastplong -i in.fq")
    g = GOLDEN[name]
    if md5_in != g["input_md5"]:
        pytest.skip("numpy generator produced a different synthetic input than when the fixture was made")
    assert empty == g["empty"]
    assert html_golden.masked_md5(text, empty) == g["html_md5"]


@pytest.mark.skipif(not os.path.exists(REF_BIN), reason="oracle/_ref/fastplong_ref not built")
@pytest.mark.parametrize("name", ["quirks", "mask_break", "rna", "cplx_limit", "short"])
def test_twin_equals_fresh_reference_run(name, tmp_path):
    text, empty, _ = twin_text(name)
    ref = html_golden.mask(html_golden.run_reference(REF_BIN, name, str(tmp_path)), empty)
    got = html_golden.mask(text, empty)
    if got != ref:
        i = next((i for i in range(min(len(got), len(ref))) if got[i] != ref[i]), min(len(got), len(ref)))
        raise AssertionError(f"differ at byte {i}:\ntwin: {got[max(0, i - 150):i + 60]!r}\nref:  {ref[max(0, i - 150):i + 60]!r}")


_libc = C.CDLL(None)


def c_fmt(fmt, v):
    buf = C.create_string_buffer(400)
    _libc.snprintf(buf, 400, fmt.encode(), C.c_double(v))
    return buf.value.decode()


def test_number_text_matches_the_c_library():
    nan = float("inf") - float("inf")
    vals = [0.0, 999.0, 1000.0, 1001.0, 1e6, 999.9995, 1000.0000001, 2.5e-7, 123456789.0, float("inf"), -float("inf"),
            report_html_twin.div(0.0, 0.0), nan, 0.3, 3.0, 100.0 / 3.0]
    for v in vals:
        assert report_html_twin.f_str(v) == c_fmt("%f", v), v
        assert report_html_twin.g_str(v) == c_fmt("%g", v), v
    # HtmlReporter::formatNumber: strictly above 1000 divides
    assert report_html_twin.format_number(999) == "999" and report_html_twin.format_number(1000) == "1000"
    assert report_html_twin.format_number(1001) == "1.001000 K"
    assert report_html_twin.format_number(10 ** 6) == "1000.000000 K" and report_html_twin.format_number(10 ** 6 + 1) == "1.000001 M"
    assert report_html_twin.get_percents(5, 0) == "0.0" and report_html_twin.get_percents(0, 7) == "0.000000"
    # x86's 0.0 / 0.0 is the negative default NaN: glibc prints "-nan", as the reference's summary does with no reads
    assert report_html_twin.f_str(report_html_twin.div(0.0 * 100.0, 0.0)) == "-nan"


def _kmer_cell(bases, val):
    """the background colour the twin gives a 5-mer with `val` hits in a block of `bases` bases"""
    s = {"bases": bases, "kmer": [val] * 1024}
    text = report_html_twin._kmer("x", s, False)
    return text.split("<td style='background:#", 1)[1][:6], text.split("\n", 6)[5]


def test_kmer_colour_boundaries():
    mean = 1024.0                                 # (bases + 1) / mKmerBufLen (2048) = 1024
    bases = 2048 * 1024 - 1
    for prop, colour in ((0.3, None), (0.3 + 1e-3, "c4c4c4"), (3.0, "c4c4c4"), (3.0 + 1e-3, None), (0.0, "0000ff")):
        val = int(round(prop * mean))
        got, _ = _kmer_cell(bases, val)
        p = val / mean
        if p <= 0.3:
            f = p * 2.0
            b = int(255 - 256 * f)
            want = "%02x%02x%02x" % (int(b * f), int(255 * f), b)
        elif p > 3.0:
            f = 2.0 / p
            r = int(255 - 128 * f)
            want = "%02x%02x%02x" % (r, int(128 * f), int(r * f))
        else:
            want = "c4c4c4"
        assert got == want and (colour is None or got == colour), (prop, got, want)
