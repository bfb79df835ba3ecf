"""The JSON report (fpl_report_json) without a GPU:
  1. the kernels' own value and formatting functions (report_value, fmt_g6 in fpl_stats.cu), cut out of the source and built for
     the host, against libc's snprintf("%.6g") of the same (double)a / (double)b over every small fraction, every quality-mean
     ratio, every tie at the sixth digit, the neighbours of every carry point and a million random int64 pairs;
  2. the plain-Python report (tests/report_twin.py) pinned to the unmodified reference's own reports (the golden runs)."""
import ctypes as C
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

import cases
from device_helpers import CSRC, ROOT, SHIMS, extract
from fastplong_b200 import abi, synth
from oracle_lib import OracleEngine
import report_twin

GOLDEN = os.path.join(ROOT, "tests", "golden")

HARNESS = r"""
#include <math.h>
#include <stdio.h>
static int in_domain(double v) { const double a = fabs(v); return v == 0 || (a >= 0x1p-64 && a < 1e6); }
// 1 if fmt_g6(v) != snprintf("%.6g", v); the first mismatch is described in bad
static int differs(double v, char* bad, int badlen) {
    char got[32], want[40];
    const int n = fmt_g6(v, got);
    got[n] = 0;
    snprintf(want, sizeof(want), "%.6g", v);
    if (n <= 12 && strcmp(got, want) == 0) return 0;
    if (!bad[0]) snprintf(bad, badlen, "%.17g: fmt_g6 '%s', printf '%s'", v, got, want);
    return 1;
}
extern "C" {
int h_fmt(double v, char* out) { const int n = fmt_g6(v, out); out[n] = 0; return n; }
double h_value(const unsigned long long* blk, long long C, long long c, int curve, int is_rna) {
    return report_value(blk, C, c, curve, is_rna);
}
// (double)a[i] / (double)b[i] for every pair in the domain; *checked = how many were
long long h_pairs(const long long* a, const long long* b, long long n, long long* checked, char* bad, int badlen) {
    long long miss = 0, k = 0;
    for (long long i = 0; i < n; i++) {
        const double v = (double)a[i] / (double)b[i];
        if (!in_domain(v)) continue;
        k++;
        miss += differs(v, bad, badlen);
    }
    *checked = k;
    return miss;
}
long long h_values(const double* v, long long n, long long* checked, char* bad, int badlen) {
    long long miss = 0, k = 0;
    for (long long i = 0; i < n; i++) {
        if (!in_domain(v[i])) continue;
        k++;
        miss += differs(v[i], bad, badlen);
    }
    *checked = k;
    return miss;
}
// every a / b with 1 <= b <= bmax, a in [lo * b, hi * b]
long long h_fractions(int bmax, int lo, int hi, long long* checked, char* bad, int badlen) {
    long long miss = 0, k = 0;
    for (long long b = 1; b <= bmax; b++)
        for (long long a = lo * b; a <= hi * b; a++) { k++; miss += differs((double)a / (double)b, bad, badlen); }
    *checked = k;
    return miss;
}
// every odd m / 2^k with exactly seven significant digits (m * 5^k in [10^6, 10^7)) below 10^6: a tie at the sixth digit
long long h_ties(long long* checked, char* bad, int badlen) {
    long long miss = 0, n = 0, p5 = 1;
    for (int k = 1; k <= 10; k++) {
        p5 *= 5;
        for (long long m = (1000000 + p5 - 1) / p5 | 1; m * p5 < 10000000; m += 2) {
            const double v = (double)m / (double)(1ll << k);
            if (v >= 1e6) break;
            n++;
            miss += differs(v, bad, badlen) + differs(-v, bad, badlen);
        }
    }
    *checked = n;
    return miss;
}
// the 2 * span + 1 doubles around each 10^k and 9.999995 * 10^k (the carry points) inside the domain
long long h_carries(int span, long long* checked, char* bad, int badlen) {
    long long miss = 0, n = 0;
    for (int e = -20; e <= 5; e++)
        for (int which = 0; which < 2; which++) {
            char s[32];
            snprintf(s, sizeof(s), which ? "9.999995e%d" : "1e%d", e);
            double v = strtod(s, nullptr);
            for (int i = 0; i < span; i++) v = nextafter(v, 0.0);
            for (int i = 0; i <= 2 * span; i++, v = nextafter(v, 1e300)) {
                if (!in_domain(v)) continue;
                n++;
                miss += differs(v, bad, badlen);
            }
        }
    *checked = n;
    return miss;
}
}
"""

_lib = None


def formatter():
    global _lib
    if _lib is not None:
        return _lib
    path = os.path.join(CSRC, "fpl_stats.cu")
    src = "\n".join([SHIMS, "#include <stdlib.h>",
                     "static inline int __clzll(long long x) { return x ? __builtin_clzll((unsigned long long)x) : 64; }",
                     extract(path, "report_value", "func"), extract(path, "fmt_g6", "func"), HARNESS])
    so = f"/tmp/fpl_report_fmt_{hashlib.md5(src.encode()).hexdigest()[:12]}.so"
    if not os.path.exists(so):
        cpp = so[:-3] + ".cpp"
        open(cpp, "w").write(src)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-w", "-I", os.path.join(ROOT, "include"),
                               "-o", so, cpp])
    lib = C.CDLL(so)
    lib.h_fmt.argtypes = [C.c_double, C.c_char_p]
    lib.h_value.argtypes = [C.c_void_p, C.c_longlong, C.c_longlong, C.c_int, C.c_int]
    lib.h_value.restype = C.c_double
    lib.h_pairs.argtypes = [C.c_void_p, C.c_void_p, C.c_longlong, C.POINTER(C.c_longlong), C.c_char_p, C.c_int]
    lib.h_values.argtypes = [C.c_void_p, C.c_longlong, C.POINTER(C.c_longlong), C.c_char_p, C.c_int]
    lib.h_fractions.argtypes = [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_longlong), C.c_char_p, C.c_int]
    lib.h_ties.argtypes = [C.POINTER(C.c_longlong), C.c_char_p, C.c_int]
    lib.h_carries.argtypes = [C.c_int, C.POINTER(C.c_longlong), C.c_char_p, C.c_int]
    for f in (lib.h_pairs, lib.h_values, lib.h_fractions, lib.h_ties, lib.h_carries):
        f.restype = C.c_longlong
    _lib = lib
    return lib


def run(fn, *args):
    """-> (mismatches, values checked, first mismatch)"""
    n, bad = C.c_longlong(), C.create_string_buffer(256)
    miss = fn(*args, C.byref(n), bad, 256)
    return miss, n.value, bad.value.decode()


def pairs(a, b):
    a, b = np.ascontiguousarray(a, dtype=np.int64), np.ascontiguousarray(b, dtype=np.int64)
    return run(formatter().h_pairs, a.ctypes.data, b.ctypes.data, len(a))


def test_formats_every_small_fraction():
    miss, n, bad = run(formatter().h_fractions, 2000, 0, 1)            # a / b, 0 <= a <= b <= 2000: the content curves
    assert n == sum(b + 1 for b in range(1, 2001)) and miss == 0, bad


def test_formats_every_quality_mean_ratio():
    miss, n, bad = run(formatter().h_fractions, 300, -33, 94)          # quality chars 0..127 minus 33, over up to 300 bases
    assert n == sum(127 * b + 1 for b in range(1, 301)) and miss == 0, bad


def test_formats_every_tie_at_the_sixth_digit():
    miss, n, bad = run(formatter().h_ties)
    assert n > 1_000_000 and miss == 0, bad
    lib = formatter()
    out = C.create_string_buffer(32)
    for v, want in ((65 / 64, "1.01562"), (123456.5, "123456"), (0.5, "0.5"), (1e-5, "1e-05"), (0.0001, "0.0001"),
                    (9.999995, "10"), (9.9999995e-05, "0.0001"), (1.1444091796875e-05, "1.14441e-05"), (0.0, "0"),
                    (-33.0, "-33"), (999999.5, "1e+06"), (2.0 ** -64, "5.42101e-20")):
        lib.h_fmt(v, out)
        assert out.value.decode() == want, (v, out.value, want)


def test_formats_the_neighbours_of_every_carry_point():
    miss, n, bad = run(formatter().h_carries, 64)
    assert n > 5000 and miss == 0, bad


def test_formats_ratios_of_large_integers():
    ks = np.arange(-40, 41, dtype=np.int64)
    big = np.concatenate([(1 << 53) + ks, (1 << 62) + ks, np.iinfo(np.int64).max - np.abs(ks)])
    small = np.concatenate([np.arange(1, 200), [1000003, 99991 * 7, 1 << 20, (1 << 31) - 1]]).astype(np.int64)
    a, b = np.meshgrid(big, np.concatenate([big, small]))
    miss, n, bad = pairs(a.ravel(), b.ravel())                         # ratios near 1 and up to 2^63
    assert n > 40000 and miss == 0, bad
    a, b = np.meshgrid(np.concatenate([small, -small]), big)           # down to 2^-63
    miss, n, bad = pairs(a.ravel(), b.ravel())
    assert n > 80000 and miss == 0, bad


def test_formats_random_int64_ratios():
    rng = np.random.default_rng(20261016)
    n = 1_300_000
    b = np.maximum(rng.integers(1, np.iinfo(np.int64).max, n, dtype=np.int64) >> rng.integers(0, 63, n), 1)
    r = rng.uniform(-64.0, np.log2(1e6), n)                            # |a / b| spread over the whole domain
    a = np.clip(b.astype(np.float64) * np.exp2(r), 0, 2.0 ** 62).astype(np.int64)
    a = (a + rng.integers(-1000, 1000, n)) * rng.choice([-1, 1], n)
    miss, checked, bad = pairs(a, b)
    assert checked >= 1_000_000 and miss == 0, bad
    vals = rng.uniform(-100, 100, 200_000) * np.exp2(rng.integers(-60, 13, 200_000).astype(np.float64))
    miss, checked, bad = run(formatter().h_values, np.ascontiguousarray(vals).ctypes.data, len(vals))
    assert checked > 150_000 and miss == 0, bad


def test_python_g_is_the_same_text():
    """the twin's premise: Python's '%g' prints what snprintf("%.6g") (hence fmt_g6) prints"""
    rng = np.random.default_rng(5)
    lib = formatter()
    out = C.create_string_buffer(32)
    vals = list(rng.integers(0, 5000, 20000) / rng.integers(1, 5000, 20000)) + [65 / 64, 123456.5, 9.999995, 9.9999995e-05]
    for v in vals:
        lib.h_fmt(float(v), out)
        assert out.value.decode() == "%g" % v, v


def test_report_values_are_the_reference_doubles():
    """report_value against numpy's float64 restatement (the twin's) on a random block, zero bins included"""
    rng = np.random.default_rng(9)
    Ccap, T = 64, 50
    blk = np.zeros(abi.stats_words(Ccap), dtype=np.int64)
    content = rng.integers(0, 1 << 40, (8, T)) * (rng.random((8, T)) < 0.7)
    content[:, -1] = 0
    content[1, -1] = 3                                                 # one bin only in the last cycle
    qual = content * rng.integers(-33, 94, (8, T)) + rng.integers(-5, 5, (8, T)) * (content > 0)
    blk[:8 * Ccap].reshape(8, Ccap)[:, :T] = content
    blk[8 * Ccap:16 * Ccap].reshape(8, Ccap)[:, :T] = qual
    lib = formatter()
    for is_rna in (0, 1):
        s = report_twin.summarize(blk)
        assert s["cycles"] == T
        t = "U" if is_rna else "T"
        want = ([s["quality"](ord(x) & 7) for x in ("A", t, "C", "G")] + [s["mean"]] +
                [s["content"](ord(x) & 7) for x in ("A", t, "C", "G", "N")] + [s["gc_curve"]])
        for k in range(11):
            got = np.array([lib.h_value(blk.ctypes.data, Ccap, c, k, is_rna) for c in range(T)])
            assert np.array_equal(got.view(np.int64), want[k].view(np.int64)), (is_rna, k)


def golden_input(name, g):
    if name.startswith("mb_"):
        opt, batch = cases.MASK_BREAK_SETS[g["options"]], cases.blocky_quality_batch(g["seed"], n=g["n_reads"])
    else:
        opt, batch = cases.OPTION_SETS[g["options"]], synth.ont_like(g["n_reads"], g["mean_len"], g["seed"], **g["synth_kwargs"])
    fq = b"".join(b"@read%d len=%d\n%s\n+\n%s\n" % (i, len(s), s, q) for i, (s, q) in
                  enumerate(batch.read(i) for i in range(batch.n_reads)))
    if hashlib.md5(fq).hexdigest() != g["input_md5"]:
        pytest.skip("numpy generator produced a different synthetic input than when the fixture was made")
    return opt, batch


GOLDEN_RUNS = ["c1_small", "cut_polyx", "loose", "mb_break", "mb_mask", "mb_both"]   # default_se, cut_polyx_cplx, loose_ed,
#                                                                                      break_default, mask_cplx, mask_and_break


@pytest.mark.parametrize("name", GOLDEN_RUNS)
def test_twin_reproduces_reference_report(name):
    """oracle accumulators -> the twin's text == the reference binary's JSON report minus its "command" line, byte for byte
    (curves, adapter map, polyX section, -N / -b post-filter Stats)"""
    g = json.load(open(os.path.join(GOLDEN, f"binary_{name}.json")))
    opt, batch = golden_input(name, g)
    o = OracleEngine(opt)
    o.process(batch)
    cyc = int(batch.lens.max())
    text = report_twin.report(o.stats(0, cyc), o.stats(1, cyc), o.counters(), opt, command="fastplong -i in.fq")
    assert hashlib.md5(report_twin.without_command(text)).hexdigest() == g["json_text_md5"]
    assert json.loads(text)["command"] == "fastplong -i in.fq"
