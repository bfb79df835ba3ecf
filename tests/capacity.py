"""Batches on both sides of the kernels' fixed capacities, built from the constants as the sources define them.

The statistics and text kernels switch paths at fixed sizes: k_cycle_stats stages CS_STAGE segment descriptors at a time and
gives a CTA CS_GROUP segments (its packed counter count << 20 | sum(q) must not overflow); k_kmer_fix and k_read_qual keep
KF_LIST / RQ_LIST long items per block for the block-wide pass and hand the rest to one warp; the grid-stride kernels cap
their grids at multiples of FPL_NUM_SMS, so that past a size a warp loops over several reads and a block's shared
accumulators collect several reads before their flush.  `constants()` reads every one of these numbers (and the grid-cap
expressions) from the source text and fails loudly when one is not found: a retune moves the batches with it or breaks the
test, it never quietly stops reaching a path.  `shrunk_sources()` rewrites the `#define` lines, so that the emulated library
(tests/simt_emu.py) reaches the same paths at CPU-test sizes with the same batch builders.
"""
import os
import re

import numpy as np

from fastplong_b200 import Options, abi, pack_reads, synth
from oracle_lib import OracleEngine, compare_lists, compare_results, compare_stats

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "fastplong_b200", "csrc")
S, E = synth.ADAPTER_START, synth.ADAPTER_END

# name -> source file of its #define
DEFINES = {"FPL_NUM_SMS": "fpl_device.cuh", "CS_TILE": "fpl_stats.cu", "CS_GROUP": "fpl_stats.cu", "CS_STAGE": "fpl_stats.cu",
           "KF_WARPS": "fpl_stats.cu", "KF_LONG": "fpl_stats.cu", "KF_LIST": "fpl_stats.cu", "RQ_WARPS": "fpl_stats.cu",
           "RQ_LONG": "fpl_stats.cu", "RQ_LIST": "fpl_stats.cu"}
# kernel -> (source file, text in front of its grid-cap expression): grid = min(want, FPL_NUM_SMS * factor)
GRID_CAPS = {"k_kmer_fix": ("fpl_stats.cu", "void launch_kmer_fix("), "k_read_qual": ("fpl_stats.cu", "void launch_read_qual("),
             "k_fastq_pack": ("fpl_ingest.cu", "k_fastq_pack<<<"), "k_emit_copy": ("fpl_emit.cu", "k_emit_copy<<<")}


def _sources(texts=None):
    files = set(DEFINES.values()) | {f for f, _ in GRID_CAPS.values()}
    return {f: (texts or {}).get(f) or open(os.path.join(CSRC, f)).read() for f in files}


def _define_re(name):
    return re.compile(r"^(#define\s+" + name + r"\s+)(\([^()\n]*\)|[^\s/]+)", re.M)


def _value(expr):
    if not re.fullmatch(r"[0-9\s()*+-]+", expr):
        raise ValueError(f"not a constant expression: {expr!r}")
    return int(eval(expr))


def constants(texts=None):
    """{name: value} of DEFINES, plus "<kernel>_BLOCKS" (the grid cap) and "<kernel>_WARPS" (warps per block) of GRID_CAPS.
    texts: {file name: source text} replacing files of fastplong_b200/csrc (a shrunk build)."""
    src = _sources(texts)
    out = {}
    for name, fn in DEFINES.items():
        m = _define_re(name).findall(src[fn])
        if len(m) != 1:
            raise AssertionError(f"#define {name} not found exactly once in {fn}")
        out[name] = _value(m[0][1])
    for kern, (fn, anchor) in GRID_CAPS.items():
        text = src[fn]
        i = text.find(anchor)
        if i < 0:
            raise AssertionError(f"{anchor} not found in {fn}")
        j = text.index(">>>", text.index(kern + "<<<", i))
        m = re.search(r"want < FPL_NUM_SMS \* (\d+) \? want : FPL_NUM_SMS \* (\d+)", text[i:j])
        if not m or m.group(1) != m.group(2):
            raise AssertionError(f"the grid cap of {kern} (min(want, FPL_NUM_SMS * k)) not found in {fn}")
        out[kern + "_BLOCKS"] = out["FPL_NUM_SMS"] * int(m.group(1))
        launch = text[text.index(kern + "<<<", i):j + 3]
        threads = launch.split(",")[1].strip()
        threads = threads.replace("KF_WARPS", str(out["KF_WARPS"])).replace("RQ_WARPS", str(out["RQ_WARPS"]))
        out[kern + "_WARPS"] = _value(threads) // 32
    assert out["k_kmer_fix_WARPS"] == out["KF_WARPS"] and out["k_read_qual_WARPS"] == out["RQ_WARPS"]
    return out


def shrunk_sources(base=None, **values):
    """{file name: source text} with the #define of every given name set to its value; each must match exactly once.
    base: {file name: source text} to start from instead of the files (a mutant's)."""
    texts = dict(base or {})
    for name, v in values.items():
        fn = DEFINES[name]
        text = texts.get(fn) or open(os.path.join(CSRC, fn)).read()
        text, n = _define_re(name).subn(lambda m: m.group(1) + str(v), text)
        if n != 1:
            raise AssertionError(f"#define {name} matched {n} times in {fn}")
        texts[fn] = text
    return texts


# ---- comparison with the oracle (records, both Stats blocks, counters, -N/-b lists) ----
def compare_with_oracle(eng, opt, batch, what, oracle=None):
    """eng: a fresh binding.Engine (GPU or emulated).  Returns the oracle's records."""
    o = oracle or OracleEngine(opt)
    exp = o.process(batch)
    compare_results(eng.process(batch), exp, what)
    if opt.mask or opt.break_reads:
        compare_lists(eng.segments(), o.segments(), what + "/segments")
        compare_lists(eng.mask_regions(), o.mask_regions(), what + "/regions")
    cyc = max(1, int(batch.lens.max()) if batch.n_reads else 1)
    for w in (0, 1):
        compare_stats(eng.stats(w, cyc), o.stats(w, cyc), f"{what}/stats{w}")
    compare_stats(eng.counters(), o.counters(), what + "/counters")
    return exp


def passing_segments(res):
    n = res["n_segments"].astype(np.int64)
    k = np.arange(res["seg_result"].shape[1])[None, :]
    return int(((res["seg_result"] == abi.PASS_FILTER) & (k < n[:, None])).sum())


# ---- read makers ----
def _bases(rng, n):
    return synth.BASES[rng.integers(0, 4, size=n)].tobytes()


def _quals(rng, n, lo=1, hi=60):
    return (rng.integers(lo, hi + 1, size=n).astype(np.uint8) + 33).tobytes()


def _q(n, q):
    return bytes([33 + q]) * n


def _shuffled(rng, reads):
    order = rng.permutation(len(reads))
    return [reads[i] for i in order]


# ---- k_cycle_stats: staging rounds and groups ----
CS_SETS = {
    # post-filter Stats by the plain variant; trim_front = 3 moves every passing segment off its 16-byte boundary
    "plain": Options(start_adapter=S, end_adapter=E, trimming_extension=0, trim_front=3, trim_tail=2, disable_quality_filtering=True,
                     length_required=1),
    # --mask: the post-filter Stats over fpl_ext_run's segment list, by the 5-mer variant
    "mask": Options(start_adapter=S, end_adapter=E, trimming_extension=0, trim_front=3, trim_tail=2, disable_quality_filtering=True,
                    length_required=1, mask=True, mask_window_size=5, mask_mean_quality=12),
}


def cycle_counts(k):
    """the pre-filter segment counts around CS_STAGE and CS_GROUP"""
    st, gr = k["CS_STAGE"], k["CS_GROUP"]
    return sorted({st - 1, st, st + 1, 2 * st + 1, gr - 1, gr, gr + 1, 2 * gr + 1})


def _reach(k):
    """a length whose segment reaches the second 512-byte tile (len + 15 > CS_TILE), and one that does not"""
    return k["CS_TILE"] - 14, k["CS_TILE"] - 15


def cycle_stats_batch(k, count, kind, seed):
    """`count` reads (= pre-filter segments).  kind "ties": every read 40 bases (groups cut inside runs of equal length);
    "falloff": exactly CS_STAGE reads reach the second tile, the rest are shorter (the second tile's next staging round is
    empty: n == 0); "falloff_plus": CS_STAGE + 3 reach it (the next round stops at n < CS_STAGE).  The rest mix ties, lengths
    1..100 and empty reads."""
    rng = np.random.default_rng(seed)
    st = k["CS_STAGE"]
    far, near = _reach(k)
    n_long = {"ties": 0, "falloff": st, "falloff_plus": st + 3}[kind]
    assert n_long < count or kind == "ties"
    reads = []
    for i in range(count):
        if i < n_long:
            L = far + int(rng.integers(0, 60)) if i % 3 else far
        elif kind == "ties" or i % 2:
            L = 40
        else:
            L = (near, 0, 1, 5, int(rng.integers(1, 101)))[i % 5]
        reads.append((_bases(rng, L), _quals(rng, L)))
    return pack_reads(_shuffled(rng, reads))


def split_read(rng, la=241, lb=321, q=30):
    """a start adapter beyond the 200-base end windows: two passing parts"""
    s = _bases(rng, la) + S.encode() + _bases(rng, lb)
    return s, _quals(rng, len(s), q - 10, q + 10)


def post_count_batch(k, count, seed, n_split=8):
    """reads whose passing segments number exactly `count` under CS_SETS: n_split split reads (two parts each, the second
    at an arbitrary offset) and count - 2 * n_split reads of 40 bases (37 after the trims, starting 3 bytes into the slot)"""
    rng = np.random.default_rng(seed)
    reads = [split_read(rng, 241 + 7 * i, 321 + 5 * i) for i in range(n_split)]
    reads += [(_bases(rng, 40), _quals(rng, 40)) for _ in range(count - 2 * n_split)]
    return pack_reads(_shuffled(rng, reads))


def headroom_batch(k, mixed):
    """2 * CS_GROUP + 1 equal reads of 300 bases at quality byte 127: every column of group 0 holds count CS_GROUP and
    sum(q) = 127 * CS_GROUP, the largest the packed counter meets.  mixed: A and C in alternating columns (a second base
    bin) and one N per read, at a position that moves from read to read."""
    L, n = 300, 2 * k["CS_GROUP"] + 1
    reads = []
    for i in range(n):
        s = bytearray(b"A" * L)
        if mixed:
            s[1::2] = b"C" * (L // 2)
            s[(7 * i) % L] = ord("N")
        reads.append((bytes(s), b"\x7f" * L))
    return pack_reads(reads)


HEADROOM_OPT = Options(disable_adapter_trimming=True, disable_quality_filtering=True, length_required=0)


# ---- k_kmer_fix: long removed ranges per block ----
KF_OPT = Options(start_adapter=S, end_adapter=E, cut_front=True, cut_tail=True, cut_window_size=4, cut_mean_quality=20)


def kf_read(rng, k, n_long):
    """a read with `n_long` removed ranges longer than KF_LONG under KF_OPT: 0 a short good read; 1 a low-quality read the
    front cut drops whole; 2 low-quality head and tail around a good middle; 3 the same with a start and an end adapter
    KF_LONG bases apart in the middle (one split whose gap runs from one adapter to the other)"""
    h = k["KF_LONG"] + 40
    if n_long == 0:
        return _bases(rng, 20), _q(20, 30)
    if n_long == 1:
        return _bases(rng, k["KF_LONG"] + 100), _q(k["KF_LONG"] + 100, 2)
    head, tail = _bases(rng, h), _bases(rng, h)
    if n_long == 2:
        mid = _bases(rng, 300)
        return head + mid + tail, _q(h, 2) + _q(300, 30) + _q(h, 2)
    mid = _bases(rng, 400) + S.encode() + _bases(rng, k["KF_LONG"] + 40) + E.encode() + _bases(rng, 400)
    return head + mid + tail, _q(h, 2) + _q(len(mid), 30) + _q(h, 2)


def kf_block(rng, k, target):
    """KF_WARPS reads with `target` long removed ranges in all"""
    counts = [3] * (target // 3) + ([target % 3] if target % 3 else [])
    assert len(counts) <= k["KF_WARPS"], target
    counts += [0] * (k["KF_WARPS"] - len(counts))
    return [kf_read(rng, k, c) for c in rng.permutation(counts)]


def kf_targets(k):
    lst = k["KF_LIST"]
    return [lst, lst + 1, min(3 * k["KF_WARPS"], lst + lst // 2 + 2)]


def long_ranges(batch, res, kf_long):
    """per read: the removed ranges of k_kmer_fix (5-mer end positions outside every passing segment) longer than kf_long"""
    out = np.zeros(batch.n_reads, dtype=np.int64)
    for r in range(batch.n_reads):
        L = int(batch.lens[r])
        if L < 5:
            continue
        o = res[r]
        kept = [(int(o["seg_lo"][j]) + 4, int(o["seg_lo"][j]) + int(o["seg_len"][j])) for j in range(int(o["n_segments"]))
                if o["seg_result"][j] == abi.PASS_FILTER]
        frm = 4
        for j in range(len(kept) + 1):
            to = min(kept[j][0], L) if j < len(kept) else L
            out[r] += to - frm > kf_long
            if j < len(kept):
                frm = max(frm, max(to, kept[j][1]))
    return out


def kmer_fix_batch(k, seed):
    """blocks of KF_WARPS reads (while n_reads <= KF_WARPS * grid cap, block b owns reads 8b..8b+7) with exactly KF_LIST,
    KF_LIST + 1 and more long removed ranges, then two blocks of short reads"""
    rng = np.random.default_rng(seed)
    reads = []
    for t in kf_targets(k):
        reads += kf_block(rng, k, t)
    reads += [kf_read(rng, k, 0) for _ in range(2 * k["KF_WARPS"])]
    return pack_reads(reads)


def kmer_fix_loop_batch(k, seed):
    """more reads than the capped grid has warps: block 0's warps come back for reads KF_WARPS * cap + w, and those carry
    long ranges too (block 0 meets 2 * 3 * KF_WARPS of them over its two rounds)"""
    rng = np.random.default_rng(seed)
    per_round = k["KF_WARPS"] * k["k_kmer_fix_BLOCKS"]
    n = per_round + 3 * k["KF_WARPS"] + 5
    reads = [kf_read(rng, k, 0)] * n
    for i in list(range(k["KF_WARPS"])) + list(range(per_round, per_round + k["KF_WARPS"])):
        reads[i] = kf_read(rng, k, 3)
    return pack_reads(reads)


# ---- k_read_qual: the block-wide list of long reads and the grid stride ----
RQ_OPT = Options(start_adapter=S, end_adapter=E, cut_front=True, cut_tail=True, length_required=1)


def rq_indices(k, block, count):
    """the first `count` read indices block `block` visits: block * RQ_WARPS + w + j * (RQ_WARPS * grid cap)"""
    w, stride = k["RQ_WARPS"], k["RQ_WARPS"] * k["k_read_qual_BLOCKS"]
    return [block * w + i % w + (i // w) * stride for i in range(count)]


def read_qual_batch(k, seed):
    """RQ_LIST + 1 reads just over RQ_LONG at the indices block 0 visits (the last one goes to a lone warp), exactly RQ_LIST
    at block 1's; every other read empty or 1 base.  The long reads hold a start adapter in the middle (two passing parts:
    the segment histograms by subtraction and by direct count) and runs of low quality."""
    rng = np.random.default_rng(seed)
    lst, long_ = k["RQ_LIST"], k["RQ_LONG"]
    at = rq_indices(k, 0, lst + 1) + rq_indices(k, 1, lst)
    n = max(at) + 1 + 7
    tiny = [(b"", b""), (b"A", b"5"), (b"N", b"!"), (b"G", b"I")]
    reads = [tiny[i % 4] for i in range(n)]
    for j, i in enumerate(at):
        L = long_ + 1 + 37 * j
        a = int(rng.integers(L // 4, L // 2))
        s = bytearray(_bases(rng, L))
        s[a:a + len(S)] = S.encode()
        q = bytearray(_quals(rng, L, 5, 40))
        b0 = int(rng.integers(0, L - 200))
        q[b0:b0 + 150] = _q(150, 2)
        reads[i] = (bytes(s), bytes(q))
    return pack_reads(reads)


def stride_batch(k, seed):
    """more reads than k_read_qual's capped grid has warps (and so more than k_kmer_fix's): warps loop, and each block's
    shared histogram collects several reads before its flush; lengths 0..120 with every quality"""
    rng = np.random.default_rng(seed)
    n = k["RQ_WARPS"] * k["k_read_qual_BLOCKS"] * 4 // 3 + 11
    lens = rng.integers(0, 121, size=n)
    lens[::97] = 600
    return pack_reads([(_bases(rng, int(L)), _quals(rng, int(L), 1, 90)) for L in lens])


# ---- the FASTQ text path: more records than k_fastq_pack and k_emit_copy have warps ----
def text_batch(k, seed):
    rng = np.random.default_rng(seed)
    n = max(k["k_fastq_pack_BLOCKS"] * k["k_fastq_pack_WARPS"], k["k_emit_copy_BLOCKS"] * k["k_emit_copy_WARPS"]) + 1000
    lens = rng.integers(0, 50, size=n)
    lens[::50] = 400
    return pack_reads([(_bases(rng, int(L)), _quals(rng, int(L), 1, 93)) for L in lens])


def fastq_of(batch):
    """FASTQ text with names of varying length and '+' lines that sometimes repeat the name (as tests/test_gpu_emit.py)"""
    names, plus, parts = [], [], []
    for i in range(batch.n_reads):
        s, q = batch.read(i)
        nm = b"@read%d %s" % (i, b"x" * (i % 41))
        pl = b"+" if i % 3 else b"+read%d" % i
        names.append(nm)
        plus.append(pl)
        parts.append(nm + b"\n" + s + b"\n" + pl + b"\n" + q + b"\n")
    return b"".join(parts), names, plus


def check_text(eng, opt, batch, what):
    """fpl_process_fastq_host + fpl_emit_fastq_host against the oracle's records through the Python mirror of the writers"""
    from fastplong_b200 import hostside
    text, names, plus = fastq_of(batch)
    got = eng.process_fastq(text)
    assert got is not None, what
    recs, res, used = got
    assert used == len(text) and len(recs) == batch.n_reads, what
    o = OracleEngine(opt)
    ores = o.process(batch)
    compare_results(res, ores, what)
    exp_out, exp_failed = hostside.emit_fastq(batch, names, ores, strand=plus)
    out, failed = eng.emit_fastq(True)
    assert out == exp_out, f"{what}: --out text differs ({len(out)} bytes, expected {len(exp_out)})"
    assert failed == exp_failed, f"{what}: --failed_out text differs"
    cyc = max(1, int(batch.lens.max()))
    for w in (0, 1):
        compare_stats(eng.stats(w, cyc), o.stats(w, cyc), f"{what}/stats{w}")
    compare_stats(eng.counters(), o.counters(), what + "/counters")
