"""TEST INFRASTRUCTURE: the kernels' own arithmetic helpers, compiled for the HOST from the source text of the .cu files.

The bit-parallel edit distances (Myers32 / myers16 / myers64 / myers128 / myers_long), the search-mode lower-bound filter
(SearchMyers), the exact byte classifiers (is_acgt, encode4's ACGTU test, kmer_code), passFilter's integer forms (pass_filter,
and fpl_ext.cu's own copy pass_filter_ext) and the --mask / --break region walk (detect_regions, walk_break, the clamp of the mask
kernels) are plain integer C++ inside `__device__` functions.  This module cuts their definitions out of
fastplong_b200/csrc/*.cu / *.cuh by name, rewrites the two inline-PTX forms they use (`mad.lo.u32`) as C, and builds them
with g++ behind small shims (`__device__` -> nothing, `__ldg`, `__dp4a`, `uint4`) into /tmp — so that the CPU tests run the
very text the GPU runs, over input spaces the GPU tests can only sample (every byte value, ties of every threshold,
the one-sidedness of the filters).  Nothing here is shipped or used by the product path.
"""
import ctypes as C
import hashlib
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "fastplong_b200", "csrc")

SHIMS = r"""
#include <stdint.h>
#include <string.h>
#include <algorithm>
#include "fplgpu.h"
using std::min; using std::max;
#define __device__
#define __forceinline__ inline
#define __noinline__
#define __restrict__
struct uint4 { uint32_t x, y, z, w; };
template <class T> static inline T __ldg(const T* p) { return *p; }
static inline uint32_t __dp4a(uint32_t a, uint32_t b, uint32_t c) {
    for (int i = 0; i < 4; i++) c += ((a >> (8 * i)) & 0xFFu) * ((b >> (8 * i)) & 0xFFu);
    return c;
}
static inline int __dp4a(int a, int b, int c) {
    for (int i = 0; i < 4; i++) c += (int)(int8_t)((uint32_t)a >> (8 * i)) * (int)(int8_t)((uint32_t)b >> (8 * i));
    return c;
}
"""

HARNESS = r"""
// peq tables as fpl_create builds them (fpl_api.cu: bit j of word j >> 5 for the adapter's byte at j; 16-mer tables in
// one word; 64-bit words for the long form)
static void build_peq(const uint8_t* pat, int m, uint4* peq) {
    memset(peq, 0, sizeof(uint4) * 256);
    for (int j = 0; j < m && j < 128; j++) reinterpret_cast<uint32_t*>(&peq[pat[j]])[j >> 5] |= 1u << (j & 31);
}
extern "C" {
int h_myers32(const uint8_t* text, int n, const uint8_t* pat, int m, int shift, int sub) {
    uint4 peq[256]; build_peq(pat, m, peq);
    return myers32(text, n, peq, shift, sub);
}
int h_myers64(const uint8_t* text, int n, const uint8_t* pat, int m, int shift, int sub) {
    uint4 peq[256]; build_peq(pat, m, peq);
    return myers64(text, n, peq, shift, sub);
}
int h_myers128(const uint8_t* text, int n, const uint8_t* pat, int m, int shift, int sub) {
    uint4 peq[256]; build_peq(pat, m, peq);
    return myers128(text, n, peq, shift, sub);
}
int h_myers16(const uint8_t* text, int n, const uint8_t* pat, int m) {
    uint32_t t[256]; memset(t, 0, sizeof(t));
    for (int j = 0; j < m; j++) t[pat[j]] |= 1u << j;
    return myers16(text, n, t, m);
}
int h_myers_long(const uint8_t* text, int n, const uint8_t* pat, int m, int shift, int sub) {
    const int words = (m + 63) / 64;
    unsigned long long* peq = new unsigned long long[256 * (size_t)words]();
    for (int j = 0; j < m; j++) peq[(size_t)pat[j] * words + (j >> 6)] |= 1ull << (j & 63);
    const int d = myers_long(text, n, peq, words, shift, sub);
    delete[] peq;
    return d;
}
// search-mode pass over the text: sg[e] = SearchMyers' score after column e (pattern m <= 32 bits)
void h_search_scores(const uint8_t* text, int n, const uint8_t* pat, int m, int* sg) {
    uint32_t t[256]; memset(t, 0, sizeof(t));
    for (int j = 0; j < m; j++) t[pat[j]] |= 1u << j;
    SearchMyers<uint32_t> Q; Q.init(m);
    for (int e = 0; e < n; e++) { Q.column(t[text[e]]); sg[e] = Q.score; }
}
void h_search_scores64(const uint8_t* text, int n, const uint8_t* pat, int m, int* sg) {
    unsigned long long t[256]; memset(t, 0, sizeof(t));
    for (int j = 0; j < m; j++) t[pat[j]] |= 1ull << j;
    SearchMyers<unsigned long long> Q; Q.init(m);
    for (int e = 0; e < n; e++) { Q.column(t[text[e]]); sg[e] = Q.score; }
}
int h_pass_filter(const fpl_options* o, int rlen, int lowq, int nn, int totalq, int diff) {
    Counts c = {lowq, nn, totalq, diff};
    return pass_filter(*o, rlen, c);
}
int h_is_acgt(uint32_t b) { return is_acgt(b) ? 1 : 0; }
uint32_t h_kmer_code(uint32_t b) { return kmer_code(b); }
uint32_t h_zero_bytes80(uint32_t d) { return zero_bytes80(d); }
void h_encode4(uint32_t w, uint32_t* nz, uint32_t* pc) { encode4(w, 1u, *nz, *pc); }
}
"""

# (file, name, kind)
WANTED = [("fpl_device.cuh", "Myers32", "struct"), ("fpl_device.cuh", "myers_eq_top", "func"), ("fpl_device.cuh", "myers32", "func"),
          ("fpl_device.cuh", "myers_long", "func"), ("fpl_trim.cu", "peq_sub", "func"), ("fpl_trim.cu", "myers128", "func"),
          ("fpl_trim.cu", "myers64", "func"), ("fpl_trim.cu", "myers16", "func"), ("fpl_trim.cu", "is_acgt", "func"),
          ("fpl_trim.cu", "SearchMyers", "struct"), ("fpl_scan.cu", "Counts", "struct"), ("fpl_scan.cu", "pass_filter", "func"),
          ("fpl_scan.cu", "zero_bytes80", "func"), ("fpl_stats.cu", "kmer_code", "func"), ("fpl_stats.cu", "mad_u32", "func"),
          ("fpl_stats.cu", "encode4", "func")]


def _match_brace(text, i):
    depth = 0
    while True:
        ch = text[i]
        if ch == "{":
            depth += 1
        elif ch == "}":
            depth -= 1
            if depth == 0:
                return i
        i += 1


def extract(path, name, kind):
    """The definition of function / struct `name` in `path`, template header included."""
    text = open(path).read()
    if kind == "struct":
        m = re.search(r"^(template\s*<[^>\n]*>\s*\n)?struct\s+(?:__align__\(\d+\)\s+)?" + name + r"\s*\{", text, re.M)
    else:
        m = re.search(r"^(template\s*<[^>\n]*>\s*\n)?[A-Za-z_][^\n;{}()]*\b" + name + r"\s*\([^;{}]*\)\s*(?:const\s*)?\{", text, re.M)
    if not m:
        raise KeyError(f"{name} not found in {path}")
    end = _match_brace(text, m.end() - 1)
    body = text[m.start():end + 1]
    return body + (";" if kind == "struct" else "") + "\n"


def _asm_to_c(src):
    """mad.lo.u32 d, a, b, c  (operands %k or literals)  ->  d = a * b + c"""
    def repl(m):
        tmpl, outs, ins = m.group(1), m.group(2), m.group(3)
        ops = re.findall(r'"[^"]*"\s*\(([^()]*(?:\([^()]*\))?[^()]*)\)', outs) + re.findall(r'"r"\s*\(((?:[^()]|\([^()]*\))*)\)', ins)
        t = re.match(r"mad\.lo\.u32\s+(%\d+|\w+),\s*(%\d+|\w+),\s*(%\d+|\w+),\s*(%\d+|\w+);", tmpl)
        if not t:
            raise ValueError("inline PTX this harness does not know: " + tmpl)
        val = [("(uint32_t)(" + ops[int(x[1:])] + ")") if x.startswith("%") else x + "u" for x in t.groups()]
        return f"{ops[0]} = {val[1]} * {val[2]} + {val[3]};"
    return re.sub(r'asm\s*\(\s*"([^"]*)"\s*:\s*([^:;]*?)\s*:\s*(.*?)\);', repl, src)


def source():
    parts = [SHIMS]
    for fn, name, kind in WANTED:
        parts.append(f"// ---- {name} ({fn}) ----\n" + _asm_to_c(extract(os.path.join(CSRC, fn), name, kind)))
    parts.append(HARNESS)
    return "\n".join(parts)


# ---- the whole-read scan (k_scan_jit v2): its helpers live in a raw string that NVRTC compiles at fpl_create ----
JIT_WANTED = [("nz7", "func"), ("plane", "func"), ("nibble_to_bytes", "func"), ("range_mask", "func"), ("ge_mask", "func")]

JIT_HARNESS = r"""
extern "C" {
void j_planes(const uint32_t* w8, uint32_t* out5) {
    uint32_t w[8]; for (int i = 0; i < 8; i++) w[i] = w8[i];
    out5[0] = plane<0>(w); out5[1] = plane<1>(w); out5[2] = plane<2>(w); out5[3] = plane<3>(w); out5[4] = plane<4>(w);
}
// the byte classification of the plane path, the kernel's own lines: masks of A / C / G / T / N among the lane's 32 bytes and
// the test that sends a lane down that path at all
void j_classify(const uint32_t* w8, uint32_t* out5, int* plane_path) {
    uint32_t w[8]; for (int i = 0; i < 8; i++) w[i] = w8[i];
    uint32_t okacc = 0xFFFFFFFFu;
    for (int k = 0; k < 8; k++) okacc &= w[k] ^ 0xA0A0A0A0u;
    *plane_path = @@PLANE_TEST@@ ? 1 : 0;
    uint32_t MA, MC, MG, MT, NM;
    @@CLASSIFY@@
    out5[0] = MA; out5[1] = MC; out5[2] = MG; out5[3] = MT; out5[4] = NM;
}
uint32_t j_nibble_to_bytes(uint32_t n) { return nibble_to_bytes(n); }
uint32_t j_range_mask(int p_first, int n) { return range_mask(p_first, n); }
uint32_t j_nz7(uint32_t d) { return nz7(d); }
uint32_t j_ge_mask(const uint32_t* c, const uint32_t* row) {
    uint32_t cc[NPL]; for (int i = 0; i < NPL; i++) cc[i] = c[i];
    alignas(16) uint32_t r[8]; for (int i = 0; i < 8; i++) r[i] = row[i];
    return ge_mask(cc, r);
}
int j_npl() { return NPL; }
}
"""


def jit_source(amax):
    """Host translation unit with the helpers of k_scan_jit v2 for adapters of up to `amax` letters (NPL count planes)."""
    raw = open(os.path.join(CSRC, "fpl_scan_jit2_src.h")).read()
    text = raw[raw.index('R"JITSRC(') + len('R"JITSRC('):raw.rindex(')JITSRC"')]
    tmp = "/tmp/fpl_jit_text.cu"
    open(tmp, "w").write(text)
    parts = [SHIMS, _asm_to_c(extract(os.path.join(CSRC, "fpl_stats.cu"), "mad_u32", "func")),
             f"constexpr int NPL = {5 if amax <= 31 else 6 if amax <= 63 else 7 if amax <= 127 else 8};\n"]
    for name, kind in JIT_WANTED:
        parts.append(_asm_to_c(extract(tmp, name, kind)))
    m = re.search(r"if \(\((okacc \| 0x1F1F1F1Fu\) == 0xFFFFFFFFu)\) \{\s*\n(\s*const uint32_t B0 = plane<0>\(w\).*?NM = [^;]*;)", text, re.S)
    if not m:
        raise KeyError("the plane-path classification block of k_scan_jit was not found")
    parts.append(JIT_HARNESS.replace("@@PLANE_TEST@@", "((" + m.group(1) + ")").replace("@@CLASSIFY@@", m.group(2)))
    return "\n".join(parts)


_jit_libs = {}


def load_jit(amax=30):
    if amax in _jit_libs:
        return _jit_libs[amax]
    src = jit_source(amax)
    so = f"/tmp/fpl_jit_helpers_{hashlib.md5(src.encode()).hexdigest()[:12]}.so"
    if not os.path.exists(so):
        cpp = so[:-3] + ".cpp"
        open(cpp, "w").write(src)
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-w", "-I", os.path.join(ROOT, "include"), "-o", so, cpp])
    lib = C.CDLL(so)
    lib.j_planes.argtypes = [C.c_void_p, C.c_void_p]
    lib.j_classify.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_int)]
    lib.j_nibble_to_bytes.argtypes = lib.j_nz7.argtypes = [C.c_uint32]
    lib.j_nibble_to_bytes.restype = lib.j_nz7.restype = lib.j_range_mask.restype = lib.j_ge_mask.restype = C.c_uint32
    lib.j_range_mask.argtypes = [C.c_int, C.c_int]
    lib.j_ge_mask.argtypes = [C.c_void_p, C.c_void_p]
    _jit_libs[amax] = lib
    return lib


# ---- the byte-packed quality step of the whole-read scans: k_scan_jit v2 (x = q + KQ, unsigned and signed dp4a) and
# k_scan_fast ((q | 0x80) - Q per byte), the kernels' own lines ----
QUAL_HARNESS = r"""
extern "C" {
// k_scan_jit v2 over n quality words at qualified char FPL_QQ: #(q >= qualified) and sum(q - 33) as the kernel derives them
void j_qual_words(const uint32_t* q, int n, int FPL_QQ, int* ge_out, int* sum_out) {
    const uint32_t one = 1u;
    @@KQ@@
    uint32_t accU = 0;
    int accS = 0;
    for (int k = 0; k < n; k++) {
        @@STEP@@
    }
    const int nbytes = 4 * n;
    int ge = @@GE@@;
    int sumq = (int)accU;
    *ge_out = ge;
    *sum_out = @@SUM@@;
}
// k_scan_fast's word step over n words
void f_qual_words(const uint32_t* words, int n, int qualified_qual, int* ge_out, int* sum_out) {
    @@QQ4@@
    int lowq_ge = 0, totalq = 0;
    for (int k = 0; k < n; k++) {
        const uint32_t q = words[k];
        @@FSTEP@@
    }
    *ge_out = lowq_ge;
    *sum_out = totalq - 33 * 4 * n;
}
}
"""


def _one(pattern, text, what):
    m = re.search(pattern, text, re.S)
    if not m:
        raise KeyError(f"{what} not found")
    return m.group(1)


def qual_step_source():
    raw = open(os.path.join(CSRC, "fpl_scan_jit2_src.h")).read()
    fast = open(os.path.join(CSRC, "fpl_scan_fast.cu")).read()
    kq = _one(r"constexpr (uint32_t KQ = \(uint32_t\)\(128 - \(FPL_QQ & 0x7f\)\);)", raw, "KQ of k_scan_jit")
    step = _one(r"if \(interior\) \{\s*#pragma unroll\s*for \(int k = 0; k < 8; k\+\+\) \{\s*(const uint32_t x = mad_u32.*?accS\);)\s*\}", raw,
                "the interior quality step of k_scan_jit")
    ge = _one(r"int ge = (\(int\)\(\(accU - \(uint32_t\)accS\) >> 8\));", raw, "the count of k_scan_jit")
    sm = _one(r"sh32\[2\]\[wid\] = (sumq - \(int\)\(KQ \+ 33u\) \* nbytes);", raw, "the quality sum of k_scan_jit")
    qq4 = _one(r"(const uint32_t qq4 = \(uint32_t\)\(P\.opt\.qualified_qual & 0x7f\) \* 0x01010101u;)", fast, "qq4 of k_scan_fast")
    fstep = _one(r"\n\s*(totalq = \(int\)__dp4a\(q, 0x01010101u, \(unsigned\)totalq\);\s*lowq_ge \+= __popc\([^;]*;)", fast,
                 "the word step of k_scan_fast")
    h = (QUAL_HARNESS.replace("@@KQ@@", "const " + kq).replace("@@STEP@@", step).replace("@@GE@@", ge).replace("@@SUM@@", sm)
         .replace("@@QQ4@@", qq4.replace("P.opt.qualified_qual", "qualified_qual")).replace("@@FSTEP@@", fstep))
    return "\n".join([SHIMS, "static inline int __popc(uint32_t x) { return __builtin_popcount(x); }",
                      _asm_to_c(extract(os.path.join(CSRC, "fpl_stats.cu"), "mad_u32", "func")), h])


def load_qual_step():
    src = qual_step_source()
    so = f"/tmp/fpl_qual_step_{hashlib.md5(src.encode()).hexdigest()[:12]}.so"
    if not os.path.exists(so):
        cpp = so[:-3] + ".cpp"
        open(cpp, "w").write(src)
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-w", "-I", os.path.join(ROOT, "include"), "-o", so, cpp])
    lib = C.CDLL(so)
    for f in (lib.j_qual_words, lib.f_qual_words):
        f.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    return lib


# ---- the --mask / --break stage (fpl_ext.cu): its own passFilter copy, the region detection, the break walk and the clamp of
# maskRegionWithN, in a translation unit of their own (fpl_scan.cu has a `struct Counts` too) ----
EXT_WANTED = [("sq", "func"), ("detect_regions", "func"), ("walk_break", "func"), ("Counts", "struct"), ("pass_filter_ext", "func")]

EXT_HARNESS = r"""
extern "C" {
int e_pass_filter(const fpl_options* o, int rlen, int lowq, int nn, int totalq, int diff) {
    Counts c = {lowq, nn, totalq, diff};
    return pass_filter_ext(*o, rlen, c);
}
// n quality strings of l bytes each (stride l), window w, quality Q.  Per string i, with at most maxr regions / pieces:
//   nreg[i], reg[i][k] = (first, last)            detect_regions as it emits them
//   npc[i], pc[i][k] = (lo, len, break index)      walk_break (-1: no region, the read stays whole)
//   nmask[i], mreg[i][k] = (start, len)            k_ext_mask_count's count and k_ext_mask_emit's clamped regions
//   mseq[i][0..l)                                  'A' everywhere, 'N' where k_ext_mask_emit paints
void e_regions(const uint8_t* qs, int n, int l, int w, int Q, int maxr, int* nreg, int* reg, int* npc, int* pc, int* nmask,
               int* mreg, uint8_t* mseq) {
    for (int i = 0; i < n; i++) {
        const uint8_t* q = qs + (size_t)i * l;
        int k = 0;
        nreg[i] = detect_regions(q, l, w, Q, [&](int first, int last) {
            if (k < maxr) { reg[((size_t)i * maxr + k) * 2] = first; reg[((size_t)i * maxr + k) * 2 + 1] = last; }
            k++;
        });
        k = 0;
        npc[i] = walk_break(q, l, w, Q, [&](int plo, int plen, int bidx) {
            if (k < maxr) { int* p = pc + ((size_t)i * maxr + k) * 3; p[0] = plo; p[1] = plen; p[2] = bidx; }
            k++;
        });
        {   // k_ext_mask_count
            const int length = l;
            int n = 0;
            detect_regions(q, length, w, Q, [&](int first, int last) {
@@MASK_COUNT@@
            });
            nmask[i] = n;
        }
        {   // k_ext_mask_emit
            const int length = l;
            uint8_t* base = mseq + (size_t)i * l;
            memset(base, 'A', l);
            struct { int read, lo; } sg = {0, 0};
            fpl_region regs[64], *out = regs;
            detect_regions(q, length, w, Q, [&](int first, int last) {
@@MASK_EMIT@@
            });
            for (int k2 = 0; k2 < (int)(out - regs) && k2 < maxr; k2++) {
                mreg[((size_t)i * maxr + k2) * 2] = regs[k2].lo; mreg[((size_t)i * maxr + k2) * 2 + 1] = regs[k2].len;
            }
        }
    }
}
}
"""


def _mask_lambda(kernel_text, what):
    """the body of the region lambda a mask kernel hands to detect_regions"""
    return _one(r"detect_regions\(b\.qual[^\n]*\[&\]\(int first, int last\) \{\n(.*?)\n\s*\}\);", kernel_text, what)


def ext_source():
    path = os.path.join(CSRC, "fpl_ext.cu")
    parts = [SHIMS]
    for name, kind in EXT_WANTED:
        parts.append(f"// ---- {name} (fpl_ext.cu) ----\n" + extract(path, name, kind))
    count = _mask_lambda(extract(path, "k_ext_mask_count", "func"), "the region lambda of k_ext_mask_count")
    emit = _mask_lambda(extract(path, "k_ext_mask_emit", "func"), "the region lambda of k_ext_mask_emit")
    parts.append(EXT_HARNESS.replace("@@MASK_COUNT@@", count).replace("@@MASK_EMIT@@", emit))
    return "\n".join(parts)


_ext_lib = None


def load_ext():
    global _ext_lib
    if _ext_lib is not None:
        return _ext_lib
    src = ext_source()
    so = f"/tmp/fpl_ext_helpers_{hashlib.md5(src.encode()).hexdigest()[:12]}.so"
    if not os.path.exists(so):
        cpp = so[:-3] + ".cpp"
        open(cpp, "w").write(src)
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-w", "-I", os.path.join(ROOT, "include"), "-o", so, cpp])
    lib = C.CDLL(so)
    lib.e_pass_filter.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
    lib.e_regions.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 7
    _ext_lib = lib
    return lib


_lib = None


def load():
    global _lib
    if _lib is not None:
        return _lib
    src = source()
    tag = hashlib.md5(src.encode()).hexdigest()[:12]
    so = f"/tmp/fpl_device_helpers_{tag}.so"
    if not os.path.exists(so):
        cpp = so[:-3] + ".cpp"
        open(cpp, "w").write(src)
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-w", "-I", os.path.join(ROOT, "include"), "-o", so, cpp])
    lib = C.CDLL(so)
    for f in ("h_myers32", "h_myers64", "h_myers128", "h_myers_long"):
        getattr(lib, f).argtypes = [C.c_char_p, C.c_int, C.c_char_p, C.c_int, C.c_int, C.c_int]
    lib.h_myers16.argtypes = [C.c_char_p, C.c_int, C.c_char_p, C.c_int]
    lib.h_search_scores.argtypes = lib.h_search_scores64.argtypes = [C.c_char_p, C.c_int, C.c_char_p, C.c_int, C.c_void_p]
    lib.h_pass_filter.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
    lib.h_is_acgt.argtypes = lib.h_kmer_code.argtypes = lib.h_zero_bytes80.argtypes = [C.c_uint32]
    lib.h_kmer_code.restype = lib.h_zero_bytes80.restype = C.c_uint32
    lib.h_encode4.argtypes = [C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
    _lib = lib
    return lib
