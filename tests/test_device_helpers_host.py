"""The kernels' own arithmetic helpers, cut out of the .cu sources and compiled for the host (tests/device_helpers.py), run
over input spaces the GPU tests can only sample: every byte value for the classifiers, random and adversarial pairs for the
bit-parallel edit distances against the oracle's textbook DP (itself pinned to the reference's edit_distance), the
one-sidedness and exactness of the search-mode filter, every tie of passFilter's integer forms against the reference's
double-precision forms."""
import ctypes as C

import numpy as np
import pytest

import device_helpers
from fastplong_b200 import Options, abi
from oracle_lib import OracleEngine


@pytest.fixture(scope="module")
def lib():
    return device_helpers.load()


@pytest.fixture(scope="module")
def orc():
    o = OracleEngine(Options())
    yield o
    o.close()


def _pairs(rng, n_cases, max_m, max_n, alphabet=b"ACGT"):
    """(text, pattern) pairs: unrelated, noisy copies, shifted copies, with N and odd bytes now and then"""
    al = np.frombuffer(alphabet, dtype=np.uint8)
    for k in range(n_cases):
        m = int(rng.integers(1, max_m + 1))
        pat = al[rng.integers(0, len(al), size=m)].copy()
        kind = k % 4
        if kind == 0:
            text = al[rng.integers(0, len(al), size=int(rng.integers(0, max_n + 1)))].copy()
        else:
            t = list(pat)
            for _ in range(int(rng.integers(0, 1 + m // 4))):
                op, p = rng.integers(0, 3), int(rng.integers(0, max(1, len(t))))
                if op == 0 and t:
                    t[p] = int(al[rng.integers(len(al))])
                elif op == 1:
                    t.insert(p, int(al[rng.integers(len(al))]))
                elif t:
                    del t[p]
            if kind == 3:
                t = list(al[rng.integers(0, len(al), size=int(rng.integers(0, 5)))]) + t
            text = np.array(t[:max_n], dtype=np.uint8)
        if k % 7 == 0 and len(text):
            text[int(rng.integers(len(text)))] = rng.choice([ord("N"), ord("U"), ord("a"), 0, 255])
        yield text.tobytes(), pat.tobytes()


@pytest.mark.parametrize("fn,max_m,max_n,cases", [("h_myers32", 32, 40, 4000), ("h_myers64", 64, 80, 2500), ("h_myers128", 128, 150, 1500),
                                                  ("h_myers_long", 1024, 400, 250)])
def test_bit_parallel_edit_distance_is_exact(lib, orc, fn, max_m, max_n, cases):
    """Myers32 / myers64 / myers128 / myers_long on the whole pattern and on sub-patterns [shift, shift + sub) — the form
    ed_adapter uses for the partial-adapter extension — equal the Levenshtein distance (src/editdistance.cpp:100-126)."""
    rng = np.random.default_rng(hash(fn) % 1000)
    f = getattr(lib, fn)
    for text, pat in _pairs(rng, cases, max_m, max_n):
        m = len(pat)
        assert f(text, len(text), pat, m, 0, m) == orc.edit_distance(text, pat), (fn, text, pat)
        shift = int(rng.integers(0, m))
        sub = int(rng.integers(1, m - shift + 1))
        if fn == "h_myers32" and shift + sub > 32:
            continue
        assert f(text, len(text), pat, m, shift, sub) == orc.edit_distance(text, pat[shift:shift + sub]), (fn, shift, sub, text, pat)
    for edge in (b"", b"A"):                       # empty text / pattern conventions
        assert f(edge, len(edge), b"ACGT", 4, 0, 4) == orc.edit_distance(edge, b"ACGT")
        assert f(b"ACGT", 4, b"ACGT", 4, 1, 0) == 4


def test_myers16_probe_distance_is_exact(lib, orc):
    rng = np.random.default_rng(16)
    for text, pat in _pairs(rng, 4000, 16, 16):
        if not text:
            continue
        assert lib.h_myers16(text, len(text), pat, len(pat)) == orc.edit_distance(text, pat), (text, pat)


@pytest.mark.parametrize("fn,m", [("h_search_scores", 16), ("h_search_scores", 30), ("h_search_scores64", 44), ("h_search_scores64", 64)])
def test_search_mode_filter_is_a_lower_bound_and_exact(lib, orc, fn, m):
    """SearchMyers (k_trim's pre-filters): the score after column e is the smallest distance of the pattern to ANY substring
    of the text ending at e.  So it bounds from below the distance of the 16-mer probe window ending at e and of every
    whole-adapter alignment ending there (a stage skipped because the bound exceeds the threshold could not have hit),
    and it is attained by some substring (the filter is as tight as a search can be)."""
    rng = np.random.default_rng(m)
    f = getattr(lib, fn)
    al = np.frombuffer(b"ACGT", dtype=np.uint8)
    for case in range(60):
        pat = al[rng.integers(0, 4, size=m)].tobytes()
        n = int(rng.integers(m, 200))
        text = bytearray(al[rng.integers(0, 4, size=n)].tobytes())
        if case % 2:                                # a noisy copy somewhere, as at a read end
            p = int(rng.integers(0, n - m + 1))
            noisy = bytearray(pat)
            for _ in range(int(rng.integers(0, 5))):
                noisy[int(rng.integers(m))] = int(al[rng.integers(4)])
            text[p:p + m] = noisy
        text = bytes(text)
        sg = (C.c_int * n)()
        f(text, n, pat, m, sg)
        for e in range(n):
            lo = max(0, e - m + 1)
            assert sg[e] <= orc.edit_distance(text[lo:e + 1], pat), (case, e)          # the window of pattern length
            for extra in (-3, -1, 1, 3, 8):                                             # other alignments ending at e
                s = e - m + 1 - extra
                if 0 <= s <= e + 1:
                    assert sg[e] <= orc.edit_distance(text[s:e + 1], pat), (case, e, extra)
        if case < 12:                               # exactness: the minimum over every start (the empty substring included)
            for e in range(0, n, 7):
                best = min(orc.edit_distance(text[s:e + 1], pat) for s in range(max(0, e + 1 - 2 * m), e + 2))
                assert sg[e] == best, (case, e)


def test_byte_classifiers_over_every_byte_value(lib):
    """is_acgt (window packing of k_trim), kmer_code (k_kmer_fix) and encode4 (k_cycle_stats: "not ACGTU" flag + 2-bit code
    per byte, four bytes per word, no carry between bytes) against their definitions, all 256 values in every byte lane;
    zero_bytes80 (word-wise N / unequal-neighbour counts of k_final) on random words."""
    code = {ord("A"): 0, ord("T"): 1, ord("U"): 1, ord("C"): 2, ord("G"): 3}           # Stats::base2val, src/stats.cpp:411-425
    rng = np.random.default_rng(4)
    for b in range(256):
        assert lib.h_is_acgt(b) == int(b in b"ACGT"), b
        assert lib.h_kmer_code(b) == code.get(b, 8), b
    nz, pc = C.c_uint32(), C.c_uint32()
    for lane in range(4):
        for b in range(256):
            for rep in range(6):
                others = rng.integers(0, 256, size=4) if rep else np.array([255, 255, 255, 255])
                bs = [int(x) for x in others]
                bs[lane] = b
                w = bs[0] | bs[1] << 8 | bs[2] << 16 | bs[3] << 24
                lib.h_encode4(w, C.byref(nz), C.byref(pc))
                for i in range(4):
                    assert ((nz.value >> (8 * i + 7)) & 1) == int(bs[i] not in code), (bs, i)
                assert nz.value & 0x7F7F7F7F == 0
                # codes c' = (b >> 1) & 3, oldest byte in the highest bit pair; T and U share a code, A / C / G / T differ
                assert pc.value == sum(((bs[i] >> 1) & 3) << (2 * (3 - i)) for i in range(4)), bs
    assert len({(ord(ch) >> 1) & 3 for ch in "ACGT"}) == 4 and (ord("T") >> 1) & 3 == (ord("U") >> 1) & 3
    for w in [0, 0xFFFFFFFF, 0x00FF00FF, 0x80808080, 0x01000100] + [int(x) for x in rng.integers(0, 1 << 32, size=3000)]:
        exp = sum(0x80 << (8 * i) for i in range(4) if (w >> (8 * i)) & 0xFF == 0)
        assert lib.h_zero_bytes80(w) == exp, hex(w)


def _reference_pass_filter(o, rlen, lowq, nn, totalq, diff):
    """Filter::passFilter's thresholds as the reference writes them, doubles included (src/filter.cpp:12-81; Python floats
    are C doubles, int / int true division is (double)a / (double)b)."""
    if rlen == 0:
        return abi.FAIL_LENGTH
    if o.qual_filter_enabled:
        if lowq > (o.unqualified_percent_limit * rlen / 100.0):
            return abi.FAIL_QUALITY
        if o.avg_qual_req > 0 and (abs(totalq) // rlen * (1 if totalq >= 0 else -1)) < o.avg_qual_req:   # C int division
            return abi.FAIL_QUALITY
        if nn * 100 > rlen * o.n_base_percent_limit:
            return abi.FAIL_N_BASE
        if o.n_base_limit != 1000000 and nn > o.n_base_limit:
            return abi.FAIL_N_BASE
    if o.length_filter_enabled:
        if rlen < o.length_required:
            return abi.FAIL_LENGTH
        if o.length_max > 0 and rlen > o.length_max:
            return abi.FAIL_TOO_LONG
    if o.complexity_enabled:
        if rlen <= 1:
            return abi.FAIL_COMPLEXITY
        if not (diff / (rlen - 1) >= o.complexity_threshold_pct / 100.0):
            return abi.FAIL_COMPLEXITY
    return abi.PASS_FILTER


def pass_filter_tie_space():
    """(fpl_options, rlen, lowq, nn, totalq, diff): for every read length up to 400 and every percentage 0..100, the count
    sitting exactly on each threshold and its two neighbours; the mean-quality ties; then random counts and lengths up to
    2 000 000."""
    def abi_opts(**kw):
        o, ad, keep = Options(disable_adapter_trimming=True, **kw).to_abi()
        return o

    lens = list(range(1, 401))
    for pct in range(0, 101):
        oc = abi_opts(low_complexity_filter=True, complexity_threshold=pct, length_required=0)
        ou = abi_opts(unqualified_percent_limit=pct, length_required=0)
        on = abi_opts(n_percent_limit=pct, length_required=0)
        for rlen in lens:
            edge = pct * (rlen - 1) // 100
            for d in (edge - 1, edge, edge + 1):
                if 0 <= d <= rlen - 1:
                    yield oc, rlen, 0, 0, 40 * rlen, d
            edge = pct * rlen // 100
            for k in (edge - 1, edge, edge + 1):
                if 0 <= k <= rlen:
                    yield ou, rlen, k, 0, 40 * rlen, 0
                    yield on, rlen, 0, k, 40 * rlen, 0
    for req in (0, 1, 7, 20, 40):       # a negative totalQual (bytes below '!') too: no --mean_qual check at 0
        o = abi_opts(mean_qual=req, length_required=0)
        for rlen in lens:
            for t in (req * rlen - 1, req * rlen, req * rlen + 1, (req + 1) * rlen - 1, -1, -rlen, -rlen - 1):
                yield o, rlen, 0, 0, t, 0
    rng = np.random.default_rng(9)
    for case in range(30000):
        o = abi_opts(low_complexity_filter=bool(rng.integers(2)), complexity_threshold=int(rng.integers(0, 101)),
                     unqualified_percent_limit=int(rng.integers(0, 101)), n_percent_limit=int(rng.integers(0, 101)),
                     n_base_limit=int(rng.choice([0, 5, 1000000])), mean_qual=int(rng.choice([0, 10, 25])),
                     length_required=int(rng.choice([0, 20, 1000])), length_limit=int(rng.choice([0, 500, 100000])),
                     disable_quality_filtering=bool(rng.integers(4) == 0), disable_length_filtering=bool(rng.integers(4) == 0)) if case % 50 == 0 else o
        rlen = int(rng.choice([rng.integers(0, 50), rng.integers(0, 5000), rng.integers(0, 2_000_000)]))
        lowq, nn = int(rng.integers(0, rlen + 1)), int(rng.integers(0, rlen // 4 + 1))
        yield o, rlen, lowq, nn, int(rng.integers(0, 60)) * rlen + int(rng.integers(0, rlen + 1)), int(rng.integers(0, max(1, rlen)))


def test_pass_filter_integer_forms_on_every_tie(lib):
    """k_final's pass_filter (integer products) against the reference's double forms over pass_filter_tie_space()."""
    for o, rlen, lowq, nn, totalq, diff in pass_filter_tie_space():
        got = lib.h_pass_filter(C.byref(o), rlen, lowq, nn, totalq, diff)
        assert got == _reference_pass_filter(o, rlen, lowq, nn, totalq, diff), (rlen, lowq, nn, totalq, diff)


# ---- helpers of the whole-read scan k_scan_jit v2 (cut out of the raw string NVRTC compiles) ----
def _words(bs):
    b = np.asarray(bs, dtype=np.uint8)
    return np.ascontiguousarray(b).view("<u4").copy()


def test_scan_bit_planes_and_byte_classes_over_every_byte_value():
    """plane<K>: bit 4n+j of plane K is bit K of byte j of word n, for ANY byte values.  The plane path's byte classes — the
    kernel's own lines — mark exactly the A / C / G / T / N bytes among the 0x40..0x5F range that takes that path (U, the IUPAC
    letters and the punctuation in that range are no adapter letter and no N), and the path test admits that range only."""
    lib = device_helpers.load_jit(30)
    rng = np.random.default_rng(12)
    out, path = np.zeros(5, dtype=np.uint32), C.c_int()
    for case in range(400):
        bs = rng.integers(0, 256, size=32).astype(np.uint8)
        w = _words(bs)
        lib.j_planes(w.ctypes.data, out.ctypes.data)
        for k in range(5):
            exp = 0
            for i in range(32):
                exp |= ((int(bs[i]) >> k) & 1) << i
            assert int(out[k]) == exp, (case, k)
    for b in range(256):
        for pos in (0, 5, 17, 31):
            bs = rng.integers(0x40, 0x60, size=32).astype(np.uint8)
            bs[pos] = b
            w = _words(bs)
            lib.j_classify(w.ctypes.data, out.ctypes.data, C.byref(path))
            assert path.value == int(0x40 <= b <= 0x5F), b
            if path.value:
                for k, ch in enumerate(b"ACGTN"):
                    exp = 0
                    for i in range(32):
                        exp |= int(bs[i] == ch) << i
                    assert int(out[k]) == exp, (b, chr(ch))


def test_scan_window_masks_and_zero_byte_tests():
    lib = device_helpers.load_jit(30)
    for n in range(16):
        assert lib.j_nibble_to_bytes(n) == sum(0xFF << (8 * k) for k in range(4) if (n >> k) & 1)
    for p_first in range(-70, 70):
        for n in range(-5, 100):
            exp = 0
            for i in range(32):
                exp |= int(0 <= p_first + i < n) << i
            assert lib.j_range_mask(p_first, n) == exp, (p_first, n)
    rng = np.random.default_rng(3)
    for d in [0, 0x7F7F7F7F, 0x80000000, 0x00010000] + [int(x) for x in rng.integers(0, 1 << 32, size=2000)]:
        exp = sum(0x80 << (8 * i) for i in range(4) if (d >> (8 * i)) & 0xFF)
        assert lib.j_nz7(d) == exp, hex(d)


@pytest.mark.parametrize("amax", [30, 45, 100, 128])
def test_scan_bit_sliced_count_comparison_is_exact(amax):
    """ge_mask: positions whose bit-sliced match count is >= the best so far, against the mask row of that value (the table
    the kernel keeps in shared memory: word b of row g = all ones iff bit b of g)."""
    lib = device_helpers.load_jit(amax)
    npl = lib.j_npl()
    rng = np.random.default_rng(amax)
    for case in range(300):
        counts = rng.integers(0, amax + 1, size=32)
        if case % 3 == 0:
            counts[:] = rng.integers(0, amax + 1)                       # ties everywhere
        c = np.zeros(npl, dtype=np.uint32)
        for i in range(32):
            for b in range(npl):
                c[b] |= np.uint32(((int(counts[i]) >> b) & 1) << i)
        for g in {0, 1, amax, int(counts.max()), int(counts.min()), int(rng.integers(0, amax + 1))}:
            row = np.array([0xFFFFFFFF if (g >> b) & 1 else 0 for b in range(8)], dtype=np.uint32)
            exp = 0
            for i in range(32):
                exp |= int(counts[i] >= g) << i
            assert lib.j_ge_mask(c.ctypes.data, row.ctypes.data) == exp, (case, g)


@pytest.mark.parametrize("fn", ["j_qual_words", "f_qual_words"])
def test_scan_quality_step_over_every_quality_byte(fn):
    """The byte-packed quality counts of the whole-read scans, the kernels' own lines: k_scan_jit adds x = q + (128 - Q) per
    byte with an unsigned and a signed dp4a ((accU - accS) >> 8 = #(q >= Q), accU - (KQ + 33) * n = sum(q - 33)); k_scan_fast
    counts bit 7 of (q | 0x80) - Q per byte.  Every q in 0..127 in every byte lane, the other lanes random, for every
    qualified char Q of -q 0..93 (33..126); then long runs of words at the extreme bytes, where the sums are largest."""
    lib = device_helpers.load_qual_step()
    f = getattr(lib, fn)
    ge, sm = C.c_int(), C.c_int()
    rng = np.random.default_rng(27)
    for Q in range(33, 127):
        for lane in range(4):
            bs = rng.integers(0, 128, size=(128, 4)).astype(np.uint8)
            bs[:, lane] = np.arange(128)
            for row in bs:
                w = np.ascontiguousarray(row).view("<u4").copy()
                f(w.ctypes.data, 1, Q, C.byref(ge), C.byref(sm))
                assert (ge.value, sm.value) == (int((row >= Q).sum()), int(row.astype(np.int64).sum()) - 33 * 4), (fn, Q, list(row))
        for b in (0, 1, 32, 33, Q - 1, Q, 126, 127):
            for n in (1, 8, 4096):
                w = np.full(n, b * 0x01010101, dtype=np.uint32)
                f(w.ctypes.data, n, Q, C.byref(ge), C.byref(sm))
                assert (ge.value, sm.value) == (4 * n * int(b >= Q), 4 * n * (b - 33)), (fn, Q, b, n)
