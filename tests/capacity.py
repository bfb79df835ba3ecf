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
           "RQ_LONG": "fpl_stats.cu", "RQ_LIST": "fpl_stats.cu", "HTML_CHUNK": "fpl_stats.h"}
# kernel -> (source file, text in front of its grid-cap expression): grid = min(want, FPL_NUM_SMS * factor), written out or as
# grid_for(n, FPL_NUM_SMS * factor)
GRID_CAPS = {"k_kmer_fix": ("fpl_stats.cu", "void launch_kmer_fix("), "k_read_qual": ("fpl_stats.cu", "void launch_read_qual("),
             "k_read_qual_exc": ("fpl_stats.cu", "void launch_read_qual_exc("),
             "k_fastq_pack": ("fpl_ingest.cu", "k_fastq_pack<<<"), "k_emit_copy": ("fpl_emit.cu", "k_emit_copy<<<"),
             "k_emit_batch_copy": ("fpl_emit.cu", "k_emit_batch_copy<<<"),
             "k_report_cycles": ("fpl_stats.cu", "void launch_report_cycles("),
             "k_html_capture": ("fpl_stats.cu", "void launch_html_capture("),
             "k_html_lenhist": ("fpl_stats.cu", "void launch_html_lenhist("),
             "k_html_bins": ("fpl_stats.cu", "void launch_html_bins("),
             "k_html_values": ("fpl_stats.cu", "void launch_html_values("),
             "k_merge_stats": ("fpl_stats.cu", "void launch_merge_stats(")}
CAP_RE = re.compile(r"want < FPL_NUM_SMS \* (\d+) \? want : FPL_NUM_SMS \* (\d+)"
                    r"|grid_for\([^()]*(?:\([^()]*\))?[^()]*, FPL_NUM_SMS \* (\d+)\)")


def _sources(texts=None):
    files = set(DEFINES.values()) | {f for f, _ in GRID_CAPS.values()}
    return {f: (texts or {}).get(f) or open(os.path.join(CSRC, f)).read() for f in files}


def _split_top(s):
    """the comma-separated arguments of s at bracket depth 0"""
    out, depth, cur = [], 0, ""
    for ch in s:
        depth += (ch in "([{") - (ch in ")]}")
        if ch == "," and depth == 0:
            out.append(cur.strip())
            cur = ""
        else:
            cur += ch
    return out + [cur.strip()]


def _cap_spans(src):
    """kernel -> (file, anchor, launch, end) of GRID_CAPS: where its anchor and its `kernel<<<` start, where the launch
    configuration ends"""
    out = {}
    for kern, (fn, anchor) in GRID_CAPS.items():
        text = src[fn]
        i = text.find(anchor)
        if i < 0:
            raise AssertionError(f"{anchor} not found in {fn}")
        k = text.find(kern + "<<<", i)
        if k < 0:
            raise AssertionError(f"no launch of {kern} behind {anchor} in {fn}")
        out[kern] = (fn, i, k, text.index(">>>", k))
    return out


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
    for kern, (fn, i, k, j) in _cap_spans(src).items():
        text = src[fn]
        caps = list(CAP_RE.finditer(text[i:j]))
        if len(caps) != 1 or (caps[0].group(1) and caps[0].group(1) != caps[0].group(2)):
            raise AssertionError(f"the grid cap of {kern} (min(want, FPL_NUM_SMS * k) or grid_for(n, FPL_NUM_SMS * k)) not found "
                                 f"exactly once in {fn}")
        out[kern + "_BLOCKS"] = out["FPL_NUM_SMS"] * int(caps[0].group(1) or caps[0].group(3))
        threads = _split_top(text[k + len(kern) + 3:j])[1]
        threads = threads.replace("KF_WARPS", str(out["KF_WARPS"])).replace("RQ_WARPS", str(out["RQ_WARPS"]))
        out[kern + "_WARPS"] = _value(threads) // 32
    assert out["k_kmer_fix_WARPS"] == out["KF_WARPS"] and out["k_read_qual_WARPS"] == out["k_read_qual_exc_WARPS"] == out["RQ_WARPS"]
    return out


def uncapped(texts=None):
    """(file, line) of every `FPL_NUM_SMS *` in fastplong_b200/csrc/*.cu outside the spans GRID_CAPS reads: a grid cap no
    capacity test knows of.  texts: {file name: source text} replacing files."""
    names = sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))
    src = {f: (texts or {}).get(f) or open(os.path.join(CSRC, f)).read() for f in set(names) | set(_sources(texts))}
    spans = _cap_spans(src).values()
    out = []
    for fn in names:
        for m in re.finditer(r"FPL_NUM_SMS\s*\*", src[fn]):
            if not any(f == fn and i <= m.start() < j for f, i, _, j in spans):
                out.append((fn, src[fn].count("\n", 0, m.start()) + 1))
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


# ---- which kernels made the quality histograms and the medians ----
# "scan": k_scan_jit counted them and k_read_qual_exc treated the reads k_final listed; "read_qual": k_read_qual did (every
# other scan kernel, -Q -L, and the pre-filter half of --mask/--break)
QUAL_TIMERS = {"scan": "k_read_qual(exceptions)", "read_qual": "k_read_qual(pre+post)"}


def quality_pass(eng):
    """"scan" or "read_qual", from the launches eng has timed: eng.set_timing(True) goes before its first process call"""
    kt = eng.kernel_times()
    ran = [name for name, timer in QUAL_TIMERS.items() if kt[timer][1] > 0]
    assert len(ran) == 1, f"quality passes that ran: {ran or 'none (is timing on?)'}"
    return ran[0]


# ---- comparison with the oracle (records, both Stats blocks, counters, -N/-b lists) ----
def compare_with_oracle(eng, opt, batch, what, oracle=None, qual_pass=None):
    """eng: a fresh binding.Engine (GPU or emulated).  qual_pass: the quality pass (quality_pass) that has to have run.
    Returns the oracle's records."""
    o = oracle or OracleEngine(opt)
    exp = o.process(batch)
    eng.set_timing(qual_pass is not None)
    compare_results(eng.process(batch), exp, what)
    if qual_pass is not None:
        got = quality_pass(eng)
        assert got == qual_pass, f"{what}: expected the {qual_pass} pass, got {got}"
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
# the quality pass each takes on the default (jit) scan: the length filter is on; --mask keeps k_read_qual
CS_PASS = {"plain": "scan", "mask": "read_qual"}


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


# ---- k_read_qual_exc: the list k_final makes of the reads whose one passing segment is not their window ----
END = 240          # adapters planted in the middle stay this far from both ends of the window (outside the end-trim windows)
EXC_KINDS = ("dead", "split", "left_fails", "right_fails", "none_pass", "gap_largest", "seg0_right", "fails", "cut_split")


def decided_read(rng, kind, L, wide=False):
    """one read of L bases whose segments k_final decides as `kind` under RQ_OPT (the split kinds want L >= 4 * END,
    "cut_split" 9 * END).  wide: quality bytes over all of 1..127 between two ends of 40 good bases."""
    s = bytearray(_bases(rng, L))
    q = bytearray(_quals(rng, L, 20, 40))
    if wide and L > 80:
        q[40:L - 40] = rng.integers(1, 128, size=L - 80).astype(np.uint8).tobytes()
    a = int(rng.integers(L // 3, max(L // 2, L // 3 + 1)))
    if kind in ("split", "left_fails", "right_fails", "none_pass"):   # a start adapter in the middle: two parts
        if kind == "none_pass":                  # ... which both fail the filter (N bases)
            s[::3] = b"N" * len(s[::3])
        s[a:a + len(S)] = S.encode()
        if kind == "left_fails":
            s[a // 4:a // 2] = b"N" * (a // 2 - a // 4)
        elif kind == "right_fails":
            b0, n = a + len(S), L - a - len(S)
            s[b0 + n // 4:b0 + n // 2] = b"N" * (n // 2 - n // 4)
    elif kind == "gap_largest":                  # both adapters far apart: the gap between them is the largest part
        s[END:END + len(S)] = S.encode()
        e = L - END - len(E)
        s[e:e + len(E)] = E.encode()
    elif kind == "seg0_right":                   # an end adapter within the trimming extension of the front: one, right part
        s[4:4 + len(E)] = E.encode()
    elif kind == "fails":                        # unsplit, the one segment fails the quality filter
        q[:] = rng.integers(1, 61, size=L).astype(np.uint8).tobytes() if wide else _quals(rng, L, 1, 12)
        e = min(40, L // 4)
        q[:e] = _q(e, 30)
        q[L - e:] = _q(e, 30)
    elif kind == "dead":                         # the quality cut drops it
        q[:] = rng.integers(1, 46, size=L).astype(np.uint8).tobytes() if wide else _q(L, 0)
    elif kind == "cut_head":                     # a long low-quality head that the front cut removes
        q[:L // 3] = _q(L // 3, 2)
    elif kind == "cut_split":                    # the cuts leave the middle third, and that window is split 1 : 2
        assert L >= 9 * END
        q[:L // 3] = _q(L // 3, 2)
        q[L - L // 3:] = _q(L // 3, 2)
        a = L // 3 + L // 9
        s[a:a + len(S)] = S.encode()
    else:
        assert kind == "plain", kind
    return bytes(s), bytes(q)


def listed(res):
    """per read (on the oracle's records): k_final puts it on k_read_qual_exc's list — every read but the ones whose one
    passing segment is the whole of their window"""
    split = (res["flags"] & abi.FLAG_MIDDLE_ADAPTER) != 0
    return split | (res["n_segments"] != 1) | (res["seg_result"][:, 0] != abi.PASS_FILTER)


def check_exc_kinds(batch, res, k):
    """the listed reads longer than RQ_LONG reach every kind of EXC_KINDS (on the oracle's records)"""
    r = res[listed(res) & (batch.lens > k["RQ_LONG"])]
    L = batch.lens[listed(res) & (batch.lens > k["RQ_LONG"])]
    flags, nseg, sr = r["flags"], r["n_segments"], r["seg_result"]
    split = (flags & abi.FLAG_MIDDLE_ADAPTER) != 0
    ok = (sr == abi.PASS_FILTER) & (np.arange(sr.shape[1])[None, :] < nseg[:, None])
    two = split & (nseg == 2)
    gap = r["seg_lo"][:, 1] - (r["seg_lo"][:, 0] + r["seg_len"][:, 0])
    # "cut_split": a window well inside the read, its smaller part counted directly and its larger one by subtraction
    window = r["seg_lo"][:, 1] + r["seg_len"][:, 1] - r["seg_lo"][:, 0]
    inside = two & ok.all(axis=1) & (r["seg_lo"][:, 0] > L // 4) & (window < L // 2)
    found = {"dead": (flags & abi.FLAG_DROPPED_BY_CUT) != 0, "split": two & ok.all(axis=1), "left_fails": two & ~ok[:, 0] & ok[:, 1],
             "right_fails": two & ok[:, 0] & ~ok[:, 1], "none_pass": two & ~ok.any(axis=1),
             "gap_largest": two & (gap > r["seg_len"].max(axis=1)), "seg0_right": (flags & abi.FLAG_SEG0_IS_RIGHT) != 0,
             "fails": ~split & (nseg == 1) & ~ok[:, 0],
             "cut_split": inside & (2 * r["seg_len"][:, 0] < window) & (2 * r["seg_len"][:, 1] >= window)}
    assert set(found) == set(EXC_KINDS)
    for kind, m in found.items():
        assert m.any(), f"no listed long read of kind {kind}"


def _long_len(k, j):
    return max(k["RQ_LONG"] + 1, 9 * END) + 37 * j


def exc_min_overflow(k):
    """the shortest list of long reads of which block 0 of k_read_qual_exc's capped grid meets RQ_LIST + 1, in any order"""
    w = k["RQ_WARPS"]
    return (k["RQ_LIST"] // w) * w * k["k_read_qual_exc_BLOCKS"] + k["RQ_LIST"] % w + 1


def exc_overflow_batch(k, seed):
    """every listed read is longer than RQ_LONG and the list is longer than exc_min_overflow: whatever its order, block 0
    meets more than RQ_LIST long reads and hands the rest to lone warps.  The reads that are not listed are short, and
    enough for the grid to reach its cap."""
    rng = np.random.default_rng(seed)
    n_long = exc_min_overflow(k) + 2 * len(EXC_KINDS)
    reads = [decided_read(rng, EXC_KINDS[j % len(EXC_KINDS)], _long_len(k, j)) for j in range(n_long)]
    reads += [decided_read(rng, "plain", int(rng.integers(50, 150))) for _ in range(k["RQ_WARPS"] * k["k_read_qual_exc_BLOCKS"] + 5)]
    return pack_reads(_shuffled(rng, reads))


def exc_kinds_batch(k, seed):
    """two reads longer than RQ_LONG of every kind of EXC_KINDS, a long and some short reads that are not listed, and short
    listed ones"""
    rng = np.random.default_rng(seed)
    reads = [decided_read(rng, kind, _long_len(k, j)) for j, kind in enumerate(EXC_KINDS + EXC_KINDS)]
    reads += [decided_read(rng, kind, _long_len(k, 3)) for kind in ("plain", "cut_head")]
    reads += [decided_read(rng, ("plain", "dead", "fails")[i % 3], int(rng.integers(50, 300))) for i in range(30)]
    return pack_reads(_shuffled(rng, reads))


LOOP_KINDS = ("dead", "fails", "split", "dead", "left_fails", "fails", "none_pass", "right_fails")


def exc_loop_batch(k, seed):
    """a list longer than k_read_qual_exc's capped grid has warps: warps loop, and each block takes many windows out of
    the post-filter sums before its one flush.  Mostly short listed reads with quality bytes over 1..127, one long read of
    every kind among them, and reads that are not listed."""
    rng = np.random.default_rng(seed)
    n = k["RQ_WARPS"] * k["k_read_qual_exc_BLOCKS"] * 9 // 8 + 11
    reads = []
    for i in range(n):
        kind = LOOP_KINDS[i % len(LOOP_KINDS)]
        L = int(rng.integers(20, 200)) if kind in ("dead", "fails") else 4 * END + int(rng.integers(0, 200))
        reads.append(decided_read(rng, kind, L, wide=True))
    reads += [decided_read(rng, "plain", int(rng.integers(50, 400)), wide=True) for _ in range(n // 8)]
    reads += [decided_read(rng, kind, _long_len(k, j), wide=j % 2 == 1) for j, kind in enumerate(EXC_KINDS)]
    return pack_reads(_shuffled(rng, reads))


def exc_list_batch(k, seed, every):
    """every: every read is listed (short ones of every kind, empty ones); otherwise none is (*n_exc == 0, every block of
    k_read_qual_exc idles)"""
    rng = np.random.default_rng(seed)
    reads = []
    for i in range(5 * k["RQ_WARPS"] + 3):
        if not every:
            reads.append(decided_read(rng, ("plain", "cut_head")[i % 2], int(rng.integers(50, 400))))
        elif i % 10 == 9:
            reads.append((b"", b""))
        else:
            kind = EXC_KINDS[i % len(EXC_KINDS)]
            reads.append(decided_read(rng, kind, 9 * END + i if kind not in ("dead", "fails") else 30 + i))
    return pack_reads(reads)


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


# ---- the report and merge kernels (fpl_report_json, fpl_report_html, fpl_merge_stats) ----
# every read passes whole: the post-filter list is the pre-filter one with a slot of no output read (bin 129) behind each read
REPORT_OPT = Options(disable_adapter_trimming=True, disable_quality_filtering=True, length_required=0)
# trimmed ends: the post-filter Stats have fewer cycles than the pre-filter ones
CURVE_OPT = Options(disable_adapter_trimming=True, disable_quality_filtering=True, length_required=1, trim_front=3, trim_tail=5)
# every read fails: a post-filter block without cycles
FAIL_OPT = Options(disable_adapter_trimming=True, disable_quality_filtering=True, length_required=1000)


def html_bins(entries):
    """k_html_hist's bin of each (length, median) entry: the median, 128 an empty read, 129 a slot without an output read"""
    return [129 if L < 0 else 128 if L == 0 else m & 127 for L, m in entries]


def post_slots(res):
    """the post-filter entries k_html_capture writes without --mask/--break: two slots per record"""
    out = []
    for r in res:
        for k in range(2):
            ok = k < int(r["n_segments"]) and r["seg_result"][k] == abi.PASS_FILTER
            out.append((int(r["seg_len"][k]), int(r["seg_median_qual"][k])) if ok else (-1, 0))
    return out


def warp_rounds(bins, chunk):
    """the 32-entry rounds of k_html_scatter: chunks of `chunk` entries, each cut into rounds from its start"""
    return [bins[lo:min(lo + 32, c + chunk, len(bins))] for c in range(0, len(bins), chunk)
            for lo in range(c, min(c + chunk, len(bins)), 32)]


def grouping_lengths(k):
    """pre-filter list lengths around one chunk and one block of k_html_hist / k_html_scatter, and one of 5 blocks and more whose
    chunk count is no multiple of 4"""
    ch = k["HTML_CHUNK"]
    return [ch - 1, ch, ch + 1, 4 * ch, 4 * ch + 1, 21 * ch + 17]


def _binned_read(rng, b, j):
    """occurrence j of bin b (0..128) as a read: median b (every quality byte b), a length of its own within the bin"""
    if b == 128:
        return b"", b""
    L = 1 + 2 * j + (b & 1)
    return _bases(rng, L), bytes([b]) * L


def grouping_batch(k, n, seed):
    """n reads whose entries fill bins 0..128 over every chunk and block (129 is the post-filter list's empty slots).  The first
    round of every other chunk c is, by c / 2 % 3: 0 one bin on all its lanes, 1 distinct bins, 2 medians 0 and 1 beside
    empty reads (bins 0 / 128 side by side; in the post-filter list 1 / 129).  Entries of one bin have distinct lengths, so a
    reordering within a bin changes the density plot's y list."""
    rng = np.random.default_rng(seed)
    ch = k["HTML_CHUNK"]
    bins = [(i * 53) % 129 for i in range(n)]
    for c in range(0, (n + ch - 1) // ch, 2):
        lo, hi, p = c * ch, min(c * ch + 32, (c + 1) * ch, n), c // 2 % 3
        for i in range(lo, hi):
            bins[i] = (7 * c) % 129 if p == 0 else (c + 5 * (i - lo)) % 129 if p == 1 else (0, 128, 1, 128)[(i - lo) % 4]
    seen = {}
    reads = []
    for b in bins:
        reads.append(_binned_read(rng, b, seen.get(b, 0)))
        seen[b] = seen.get(b, 0) + 1
    return pack_reads(reads)


def capture_cap_batch(k, seed):
    """more reads than k_html_capture's and k_html_lenhist's capped grids have threads (the lists past their caps), lengths
    0..12 with every median"""
    rng = np.random.default_rng(seed)
    n = max(k["k_html_capture_BLOCKS"], k["k_html_lenhist_BLOCKS"]) * 256 + 3 * 32 + 5
    return pack_reads([_binned_read(rng, int(b), int(rng.integers(0, 6))) for b in rng.integers(0, 129, size=n)])


# name -> (the reads' lengths, options): ties of Stats::calcLengthHistogram's strict > and its edges
LENGTH_CASES = {"median_tie": ([10, 20, 10, 20], REPORT_OPT),            # count at 10 = 2 = 4 / 2
                "n50_tie": ([50, 100, 50], REPORT_OPT),                  # 50 * 2 = 100 = 200 / 2
                "empty_only": ([0, 0, 0], REPORT_OPT), "single": ([37], REPORT_OPT), "one_length": ([25] * 6, REPORT_OPT),
                "post_empty": ([30, 45, 0], FAIL_OPT)}


def length_ties(lens):
    """(the running count meets half the entries exactly at a key, the running sum of length * count meets half the length
    sum exactly at a positive key)"""
    lens = [L for L in lens if L >= 0]
    keys, cnt, prod = sorted(set(lens)), 0, 0
    med = n50 = False
    for L in keys:
        cnt += lens.count(L)
        prod += L * lens.count(L)
        med |= cnt == len(lens) // 2
        n50 |= L > 0 and prod == sum(lens) // 2
    return med, n50


def length_batch(lens, seed):
    rng = np.random.default_rng(seed)
    return pack_reads([(_bases(rng, L), _quals(rng, L, 5, 40)) for L in lens])


def curve_totals(k):
    """longest reads (total cycles) on both sides of the 300-cycle down-sampling, none a multiple of 32, and one past the caps
    of k_report_cycles / k_html_bins (cap * 256 cycles) and k_html_values (11 * cycles > cap * 256); last, a read exactly as long
    as the library's first capacity (1024): the pre-filter block has no empty cycle, total_cycles == C"""
    past = max(k["k_report_cycles_BLOCKS"], k["k_html_bins_BLOCKS"]) * 256 + 37
    return [40, 41, 300, 301, max(past, k["k_html_values_BLOCKS"] * 256 // 11 + 37), 1024]


def curve_batch(total, seed):
    """reads of 1..total bases under CURVE_OPT, the longest exactly total"""
    rng = np.random.default_rng(seed)
    lens = [total, 1, 9] + [int(v) for v in rng.integers(1, total + 1, size=12)]
    return pack_reads([(_bases(rng, L), _quals(rng, L, 1, 60)) for L in lens])


def merge_sources(k, seed):
    """three batches for three contexts of three capacities (the library's first is 1024 cycles, it doubles): a longest read of
    exactly 1024 (rows == C), of 1500 and one past k_merge_stats' cap (2 * 16 * rows words > cap * 256 threads, and > 2048).
    Their read counts are no multiples of HTML_CHUNK: the merged lists' source boundaries fall inside chunks."""
    rng = np.random.default_rng(seed)
    ch = k["HTML_CHUNK"]
    longest = [1024, 1500, max(2100, k["k_merge_stats_BLOCKS"] * 256 // 32 + 101)]
    counts = [ch // 2 + 3, ch + 5, ch // 3 + 7]
    out = []
    for L, n in zip(longest, counts):
        lens = [L] + [int(v) for v in rng.integers(0, 200, size=n - 1)]
        out.append(pack_reads(_shuffled(rng, [(_bases(rng, x), _quals(rng, x, 1, 60)) for x in lens])))
    return out


REPORT_TIME = "2026-10-16      12:00:00"


def _same_text(got, want, what):
    if got != want:
        i = next((i for i in range(min(len(got), len(want))) if got[i] != want[i]), min(len(got), len(want)))
        raise AssertionError(f"{what}: differs at byte {i} of {len(got)} / {len(want)}:\n"
                             f"library: {got[max(0, i - 160):i + 60]!r}\ntwin:    {want[max(0, i - 160):i + 60]!r}")


def check_reports(eng, opt, lists, what):
    """the JSON and the HTML report of eng against the twins (tests/report_twin.py, tests/report_html_twin.py) over eng's own
    accumulators and the oracle's lists (pre, post)"""
    import report_html_twin
    import report_twin
    st = (eng.stats(0), eng.stats(1), eng.counters())
    _same_text(eng.report_json(), report_twin.report(*st, opt), what + "/json")
    _same_text(eng.report_html(time_text=REPORT_TIME), report_html_twin.report(*st, opt, *lists, time_text=REPORT_TIME), what + "/html")


def report_run(eng, opt, batches, what):
    """eng (fresh, lists kept) processes the batches; records, both Stats blocks and the counters against the oracle's over the
    same batches, both reports against the twins.  Returns (the oracle's records of the last batch, the oracle's lists)."""
    import report_html_twin
    eng.keep_read_lists(True)
    o = OracleEngine(opt)
    ext = opt.mask or opt.break_reads
    lists = ([], [])
    for j, b in enumerate(batches):
        res = o.process(b)
        compare_results(eng.process(b), res, f"{what}/{j}")
        pre, post = report_html_twin.read_lists(b.lens, res, o.segments() if ext else None)
        if ext:
            compare_lists(eng.segments(), o.segments(), f"{what}/{j}/segments")
        lists[0].extend(pre)
        lists[1].extend(post)
    cyc = max([1] + [int(b.lens.max()) for b in batches if b.n_reads])
    for w in (0, 1):
        compare_stats(eng.stats(w, cyc), o.stats(w, cyc), f"{what}/stats{w}")
    compare_stats(eng.counters(), o.counters(), what + "/counters")
    check_reports(eng, opt, lists, what)
    return res, lists


# the post-filter list is fpl_ext_run's list of output reads: --mask with a start adapter (a split read gives two), --break without
# adapters (a read of low quality only gives none)
MASK_OPT = Options(start_adapter=S, mask=True, disable_quality_filtering=True, length_required=0)
BREAK_OPT = Options(disable_adapter_trimming=True, break_reads=True, break_window_size=25, break_mean_quality=12,
                    disable_quality_filtering=True, length_required=0)


def segment_batch(k, seed, above):
    """above (MASK_OPT): split reads among short ones, more output reads than reads.  Otherwise (BREAK_OPT): more reads, and
    more output reads, than k_html_capture's capped grid has threads, every fifth read of low quality only (no output read)."""
    rng = np.random.default_rng(seed)
    if above:
        reads = [split_read(rng, 201 + 3 * i, 205 + 5 * i) for i in range(40)] + [(_bases(rng, 20 + i), _quals(rng, 20 + i)) for i in range(20)]
        return pack_reads(_shuffled(rng, reads))
    n = k["k_html_capture_BLOCKS"] * 256 * 5 // 4 + 100
    return pack_reads([(_bases(rng, 30), _q(30, 2)) if i % 5 == 4 else (_bases(rng, i % 13), _quals(rng, i % 13, 20, 60))
                       for i in range(n)])
