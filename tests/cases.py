"""Option sets and seeded inputs shared by the parity tests (oracle vs reference vs CUDA)."""
import numpy as np

from fastplong_b200 import Options, pack_reads, synth

S, E = synth.ADAPTER_START, synth.ADAPTER_END

FASTA5 = [  # a 5-entry adapter "FASTA" in std::map header order, incl. a 72-bp entry and one absent from reads
    "CTGTCTCTTATACACATCTCCGAGCCCACGAGAC",
    "AGATCGGAAGAGCACACGTCTGAACTCCAGTCACGGCTACATCTCGTATGCCGTCTTCTGCTTGAAAAAAGGGTTT",
    "GGTTCA",
    "TTTCTGTTGGTGCTGATATTGCT",
    "ACTTGCCTGTCGCTCTATCTTC",
]

def fasta64():
    """BASELINE.json configs[2]: a 64-entry adapter FASTA of random 20-44-mers in std::map (sorted header) order —
    the same set bench.py --workload c3 uses."""
    rng = np.random.default_rng(64)
    return sorted("".join("ACGT"[i] for i in rng.integers(0, 4, size=int(rng.integers(20, 45)))) for _ in range(64))


FASTA64 = fasta64()

OPTION_SETS = {
    "default_se": Options(start_adapter=S),
    "cut_polyx_cplx": Options(start_adapter=S, end_adapter=E, cut_front=True, cut_tail=True, cut_window_size=10,
                              trim_poly_x=True, low_complexity_filter=True),
    "trims_limits": Options(start_adapter=S, trim_front=5, trim_tail=7, mean_qual=10, n_base_limit=2,
                            length_limit=400, n_percent_limit=3, unqualified_percent_limit=30),
    "loose_ed": Options(start_adapter=S, distance_threshold=0.3, trimming_extension=4, cut_tail=True,
                        cut_tail_window_size=1, cut_tail_mean_quality=25),
    "fasta5": Options(start_adapter=S, adapter_fasta=FASTA5, trim_poly_x=True, poly_x_min_len=8),
    "fasta64_polyx": Options(start_adapter=S, end_adapter=E, adapter_fasta=FASTA64, trim_poly_x=True),
    "literal_auto": Options(start_adapter="auto", end_adapter="auto", cut_front=True, cut_front_window_size=7,
                            cut_front_mean_quality=15),
    "no_adapter_no_filters": Options(disable_adapter_trimming=True, disable_quality_filtering=True,
                                     disable_length_filtering=True),
    "empty_adapters": Options(start_adapter="", end_adapter="", disable_quality_filtering=True),
    "strict_ed0": Options(start_adapter=S, distance_threshold=0.0, trimming_extension=0, qualified_quality_phred=20,
                          length_required=100),
    "end_only_wide_window": Options(start_adapter="", end_adapter=E, cut_front=True, cut_tail=True,
                                    cut_window_size=100, cut_mean_quality=12, trim_tail=3),
}


def _rand_adapter(n, seed):
    rng = np.random.default_rng(seed)
    return "".join("ACGT"[i] for i in rng.integers(0, 4, size=n))


# -s/-e adapters of every word-count class of the scan kernels (halo 1..4 words, 5..8 counter planes) and, beyond 128 bp,
# of the multi-word paths (generic k_scan, myers_long); 641 is where the reference's own edit_distance changes method
LONG_ADAPTERS = {n: (_rand_adapter(n, 100 + n), _rand_adapter(max(4, n - 3), 200 + n)) for n in (31, 32, 33, 45, 64, 65, 96, 97, 127, 128, 129, 200, 300, 641, 1024)}
for _n, (_s, _e) in LONG_ADAPTERS.items():
    OPTION_SETS[f"long_adapter_{_n}"] = Options(start_adapter=_s, end_adapter=_e, low_complexity_filter=(_n % 2 == 0))


def long_adapter_batch(n_adapter, seed, n=160):
    """Reads with the long adapters planted at the ends and in the middle (chimeras), noisy."""
    s, e = LONG_ADAPTERS[n_adapter]
    return synth.ont_like(n, 1500, seed, adapter_start=s, adapter_end=e, p_chimera=0.15, p_n=0.002)


def planted_fasta_reads(seed, n=120):
    """Reads with FASTA5 entries planted at either end (noisy), for the fasta5 option set."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        L = int(rng.integers(60, 900))
        s = bytearray(synth.BASES[rng.integers(0, 4, size=L)].tobytes())
        for side in (0, 1):
            if rng.random() < 0.6:
                a = FASTA5[int(rng.integers(len(FASTA5)))].encode()
                if side == 1:
                    a = a[: int(rng.integers(max(6, len(a) // 2), len(a) + 1))]
                else:
                    a = a[len(a) - int(rng.integers(max(6, len(a) // 2), len(a) + 1)):]
                a = synth._noisy(rng, a, 0.06)
                k = int(rng.integers(0, 12))
                if len(a) + k < L:
                    if side == 0:
                        s[k:k + len(a)] = a
                    else:
                        s[L - k - len(a):L - k] = a
        q = (np.rint(rng.normal(20, 8, size=L)).clip(1, 50).astype(np.uint8) + 33).tobytes()
        out.append((bytes(s), q))
    return out


def hifi_fasta64_batch(seed, n=200, mean=2500):
    """configs[2]-shaped reads: HiFi-like qualities, poly-A/T tails, entries of FASTA64 planted in front of the reads."""
    return synth.ont_like(n, mean, seed, q_mean=33.0, q_sd=6.0, q_clip=60, p_polya=0.1, planted=FASTA64[:6] + FASTA64[40:43],
                          p_planted=0.4, p_chimera=0.03)


def adversarial_batch(seed):
    return pack_reads(synth.adversarial_reads(seed) + planted_fasta_reads(seed + 1000))


def ont_batch(seed, n=300, mean=2000, **kw):
    return synth.ont_like(n, mean, seed, **kw)


# ---- RNA reads (direct-RNA ONT: U instead of T).  The reference handles them on the same path: Stats::base2val maps U to
# T's code (src/stats.cpp:411-425), 'U' & 7 is its own content bin (5), adapters are compared byte-wise (so a DNA adapter
# never matches an RNA read), polyX counts A/T/C/G only (src/polyx.cpp:28-45), and the evaluator prints the detected end
# adapter with U (src/evaluator.cpp:245).  No other batch here holds a U inside a valid 5-mer. ----
def to_rna(text):
    return text.replace("T", "U")


RNA_SETS = {
    "rna_adapters": Options(start_adapter=to_rna(S), end_adapter=to_rna(E), cut_front=True, cut_tail=True, cut_window_size=10,
                            trim_poly_x=True, low_complexity_filter=True),
    "rna_reads_dna_adapters": Options(start_adapter=S, end_adapter=E, trim_poly_x=True, poly_x_min_len=8),
    "rna_mixed_adapter_fasta": Options(start_adapter=to_rna(S), end_adapter=E, adapter_fasta=[to_rna(FASTA5[0]), FASTA5[3], to_rna(FASTA5[4])],
                                       cut_tail=True),
}


def rna_batch(seed, n=200, mean=1500, mixed=False):
    """ont_like reads with every T turned into U (planted adapters, poly-T tails and slot padding included); mixed=True
    keeps T in every third read — a file the reference BINARY refuses ("contains both U and T") but its operators take."""
    from fastplong_b200 import PackedBatch
    b = synth.ont_like(n, mean, seed, p_chimera=0.1, p_polya=0.2, planted=[FASTA5[0], FASTA5[4]], p_planted=0.3)
    seq = b.seq.copy()
    for i in range(b.n_reads):
        if mixed and i % 3 == 0:
            continue
        o, L = int(b.offsets[i]), int(b.lens[i])
        v = seq[o:o + L]
        v[v == ord("T")] = ord("U")
    return PackedBatch(seq, b.qual, b.offsets, b.lens)


# ---- crafted boundary cases: every one of them is a single-token mutant of the oracle that the batches above did not
# tell apart from the reference (mutation run over oracle/fpl_oracle.c, DESIGN §5) ----
def _q(n, q):
    return bytes([33 + q]) * n


def _rb(rng, n):
    return synth.BASES[rng.integers(0, 4, size=n)].tobytes()


def edge_cases():
    """name -> (Options, PackedBatch)"""
    rng = np.random.default_rng(2718)
    out = {}
    # (a) more adapter events on one read than the record's four inline slots (FPL_INLINE_EVENTS): three FASTA entries
    # stacked at each end plus -s / -e; the event table and n_events keep counting
    fa = sorted(_rand_adapter(n, 300 + n) for n in (22, 26, 30, 34))
    s_ad, e_ad = _rand_adapter(28, 401), _rand_adapter(28, 402)
    reads = []
    for k in range(12):
        head = s_ad + "".join(fa[(k + j) % 4] for j in range(3))
        tail = "".join(fa[(k + j + 1) % 4] for j in range(3)) + e_ad
        body = _rb(rng, 300 + 17 * k)
        reads.append((head.encode() + body + tail.encode(), _q(len(head) + len(body) + len(tail), 25)))
    out["many_events"] = (Options(start_adapter=s_ad, end_adapter=e_ad, adapter_fasta=fa, trimming_extension=0), pack_reads(reads))
    # (b) global trims that eat the whole read exactly (Filter::trimAndCut, src/filter.cpp:137-157), with and without cuts
    lens = [10, 11, 12, 13, 14, 16, 17, 18, 30]
    reads = [(_rb(rng, n), _q(n, 30)) for n in lens for _ in range(2)]
    for name, kw in (("trims_eat_read", {}), ("trims_eat_read_cut_front", dict(cut_front=True, cut_window_size=4)),
                     ("trims_eat_read_cut_tail", dict(cut_tail=True, cut_window_size=1))):
        out[name] = (Options(disable_adapter_trimming=True, trim_front=5, trim_tail=7, length_required=0, **kw), pack_reads(reads))
    # (c) cut_front alone with a tail trim: no window qualifies / only the last one does (the scan stops one window short
    # of the end, src/filter.cpp:170-180); the same from the other side
    reads = []
    for n in (40, 41, 57, 80):
        reads.append((_rb(rng, n), _q(n, 3)))                                        # nothing qualifies
        reads.append((_rb(rng, n), _q(n - 12, 3) + _q(12, 35)))                      # good bases only at the very end
        reads.append((_rb(rng, n), _q(12, 35) + _q(n - 12, 3)))                      # ... only at the very start
        reads.append((_rb(rng, n), _q(n - 9, 3) + _q(6, 35) + _q(3, 3)))             # the last full window before the tail trim
    out["cut_front_tail_trim"] = (Options(disable_adapter_trimming=True, cut_front=True, cut_window_size=6, cut_mean_quality=20,
                                          trim_tail=3, length_required=0), pack_reads(reads))
    out["cut_tail_front_trim"] = (Options(disable_adapter_trimming=True, cut_tail=True, cut_window_size=6, cut_mean_quality=20,
                                          trim_front=3, length_required=0), pack_reads(reads))
    # (d) polyX: N inside the run counts for every base (src/polyx.cpp:40-45), for each of A/T/C/G; the stop rule at
    # pos == 8 with a long minimum length (:54)
    reads = []
    for base in b"ATCG":
        for k in (12, 20, 33):
            run = bytearray([base]) * k
            for p in rng.integers(1, k - 1, size=3):
                run[int(p)] = ord("N")
            body = _rb(rng, 120)
            reads.append((body + bytes(run), _q(120 + k, 30)))
            reads.append((body + bytes(run[:8]) + b"ACGT"[:1] + bytes(run[8:]), _q(121 + k, 30)))
        reads.append((_rb(rng, 100) + bytes([base]) * 8 + b"CAGT" + bytes([base]) * 9, _q(121, 30)))
    for ml in (5, 10, 20):
        out[f"polyx_with_n_min{ml}"] = (Options(disable_adapter_trimming=True, trim_poly_x=True, poly_x_min_len=ml), pack_reads(reads))
    # polyX stop rule around pos == 8 (:54): two mismatches among the last nine bases stop the walk (9 - 7 > 9 / 8) although
    # the run behind them would have been long enough to trim (`pos >= 8` vs `pos > 8` turns out to be an equivalent mutant:
    # the mismatch count cannot fall, so the walk stops one base later at the latest and neither stop reaches the minimum)
    reads = []
    for base, other in ((b"T", b"CG"), (b"A", b"CT"), (b"G", b"AT"), (b"C", b"GA")):
        tail = base * 26 + other[1:2] + base * 3 + other[0:1] + base * 3                 # reading from the end: 3, x, 3, y, 26
        reads.append((_rb(rng, 150) + tail, _q(150 + len(tail), 30)))
        tail = base * 26 + other[1:2] + base * 4 + other[0:1] + base * 3                 # the second mismatch one position later
        reads.append((_rb(rng, 150) + tail, _q(150 + len(tail), 30)))
    for ml in (9, 12):
        out[f"polyx_stop_at_8_min{ml}"] = (Options(disable_adapter_trimming=True, trim_poly_x=True, poly_x_min_len=ml), pack_reads(reads))
    # findMiddleAdapters with the end adapter at position 0 of the trimmed read (src/adaptertrimmer.cpp:19: `>= 0`): the
    # start trim removes a leading start adapter and leaves the read beginning with an end adapter; a second start adapter
    # sits further in
    reads = []
    for k in range(6):
        body1, body2 = _rb(rng, 320 + 11 * k), _rb(rng, 400)
        reads.append((S.encode() + E.encode() + body1 + S.encode() + body2, _q(30 + 30 + len(body1) + 30 + 400, 30)))
        reads.append((S.encode() + E.encode() + body1 + body2, _q(30 + 30 + len(body1) + 400, 30)))
    out["middle_end_adapter_at_0"] = (Options(start_adapter=S, end_adapter=E, trimming_extension=0), pack_reads(reads))
    out["middle_end_adapter_at_0_ext"] = (Options(start_adapter=S, end_adapter=E), pack_reads(reads))
    # (e) quality filter without the length filter (-L) and the other way round: the counts are taken when EITHER is on
    # (src/filter.cpp:23), the thresholds of each only when it is on; reads that fail on low-quality share, mean, N share, N count
    reads = []
    for k in range(6):
        n = 200 + 10 * k
        reads.append((_rb(rng, n), _q(n // 2, 5) + _q(n - n // 2, 30)))              # 50 % unqualified
        reads.append((_rb(rng, n), _q(n, 9)))                                        # low mean
        s = bytearray(_rb(rng, n))
        s[10:10 + n // 8] = b"N" * (n // 8)
        reads.append((bytes(s), _q(n, 30)))                                          # 12 % N
        reads.append((_rb(rng, 12), _q(12, 30)))                                     # short
    for name, kw in (("qual_filter_without_length_filter", dict(disable_length_filtering=True)),
                     ("length_filter_without_qual_filter", dict(disable_quality_filtering=True)),
                     ("neither_filter_but_complexity", dict(disable_length_filtering=True, disable_quality_filtering=True,
                                                            low_complexity_filter=True))):
        out[name] = (Options(disable_adapter_trimming=True, mean_qual=12, n_base_limit=20, **kw), pack_reads(reads))
    # reads of one and two bases under the complexity filter without the length filter: `rlen <= 1` fails complexity in the
    # reference (src/filter.cpp:70); the kernels' integer form would pass such a read without its own guard (0 >= pct * 0) — a
    # mutant of k_final's pass_filter that the emulated battery did not catch (tools/mutate_kernels.py)
    reads = [(b"A", _q(1, 30)), (b"AC", _q(2, 30)), (b"AA", _q(2, 30)), (b"ACG", _q(3, 30)), (b"G", _q(1, 30))]
    for pct in (0, 30, 100):
        out[f"complexity_on_tiny_reads_{pct}"] = (Options(disable_adapter_trimming=True, disable_length_filtering=True, low_complexity_filter=True,
                                                         complexity_threshold=pct), pack_reads(reads))
    # the same ties on the two sides of a SPLIT read (a start adapter in the middle, beyond the 200-base end windows): k_final
    # recounts the smaller parts of [A | gap | B] byte-wise at their ragged ends and takes the largest by subtraction; a mutant of
    # that recount's neighbour-byte pick survived the battery (tools/mutate_kernels.py).  Low-complexity two-letter sides with
    # exactly (len - 1) * 30 % unequal neighbours, one fewer, one more; side lengths that move the ragged ends through a word
    def two_letter(L, d, a=b"A", c=b"C"):        # (every flip moves on through a cycle of letters that starts with a, c)
        cycle = [a, c] + [x for x in (b"G", b"T", b"A", b"C") if x not in (a, c)]
        flips = set(int(x) for x in rng.choice(L - 1, size=d, replace=False))
        out_, k = bytearray(), 0
        for i in range(L):
            out_ += cycle[k % 4]
            if i in flips:
                k += 1
        return bytes(out_)
    reads = []
    for la in (241, 251, 261, 271):
        for lb in (321, 331):
            for da, db in ((0, 0), (-1, 0), (0, -1), (1, 1)):
                sA = two_letter(la, (la - 1) * 3 // 10 + da)
                sB = two_letter(lb, (lb - 1) * 3 // 10 + db, b"G", b"T")
                reads.append((sA + S.encode() + sB, _q(la + 30 + lb, 30)))
    out["split_read_complexity_ties"] = (Options(start_adapter=S, end_adapter=E, trimming_extension=0, low_complexity_filter=True,
                                                 complexity_threshold=30, length_required=10), pack_reads(reads))
    # (f) ties of the integer-valued comparisons: mean quality == requirement (integer division, src/filter.cpp:33),
    # complexity == threshold and one transition either side (:75-78), unqualified share and N share == limit (:31, :35)
    reads = []
    for n in (20, 21, 50):
        for q in (9, 10, 11):
            reads.append((_rb(rng, n), _q(n, q)))
        reads.append((_rb(rng, n), _q(n // 2, 10) + _q(n - n // 2, 11)))             # floor(mean) == 10
        reads.append((_rb(rng, n), _q(n // 2, 9) + _q(n - n // 2, 10)))              # floor(mean) == 9
    for L, d in ((11, 3), (11, 2), (11, 4), (21, 6), (21, 5), (21, 7), (101, 30), (101, 29), (101, 31), (41, 12), (41, 11)):
        s = bytearray(b"A" * L)                                                      # exactly d positions with seq[i] != seq[i+1]
        cur, flips = ord("A"), set(int(x) for x in rng.choice(L - 1, size=d, replace=False))
        for i in range(L):
            s[i] = cur
            if i in flips:
                cur = ord("C") if cur == ord("A") else ord("A")
        reads.append((bytes(s), _q(L, 30)))
    for n, low, nn in ((20, 8, 2), (20, 9, 3), (50, 20, 5), (50, 21, 6), (100, 40, 10), (100, 41, 11)):
        s = bytearray(_rb(rng, n))
        s[:nn] = b"N" * nn
        reads.append((bytes(s), _q(low, 5) + _q(n - low, 30)))                       # low == 40 % / nn == 10 % and one more
    for n in (9, 10, 11, 199, 200, 201):                                             # length_required / length_limit and one either side
        reads.append((_rb(rng, n), _q(n, 30)))
    out["filter_ties"] = (Options(disable_adapter_trimming=True, mean_qual=10, qualified_quality_phred=8, low_complexity_filter=True,
                                  complexity_threshold=30, length_required=10, length_limit=200), pack_reads(reads))
    return out


# ---- option values at the ends of what the reference's CLI accepts (src/options.cpp:validate): the longest windows, a distance
# threshold of 1, extensions and trims larger than most reads, 4-bp adapters, 200 FASTA entries, filters at 0 and 100 % ----
def _extreme_sets():
    rng = np.random.default_rng(5)
    fa = sorted("".join("ACGT"[i] for i in rng.integers(0, 4, size=int(rng.integers(6, 60)))) for _ in range(200))
    return {
        "window1000": Options(start_adapter=S, end_adapter=E, cut_front=True, cut_tail=True, cut_window_size=1000, cut_mean_quality=18),
        "window999_q36": Options(disable_adapter_trimming=True, cut_front=True, cut_tail=True, cut_window_size=999, cut_mean_quality=36),
        "ext100": Options(start_adapter=S, end_adapter=E, trimming_extension=100),
        "ed1": Options(start_adapter=S, end_adapter=E, distance_threshold=1.0),
        "polyx_min50": Options(start_adapter=S, trim_poly_x=True, poly_x_min_len=50),
        "polyx_min1": Options(start_adapter=S, trim_poly_x=True, poly_x_min_len=1),
        "front_tail_big": Options(start_adapter=S, trim_front=300, trim_tail=400, length_required=0),
        "adapters_4bp": Options(start_adapter="ACGT", end_adapter="TTGCA"),
        "fasta_200_entries": Options(start_adapter=S, end_adapter=E, adapter_fasta=fa),
        "complexity100": Options(start_adapter=S, low_complexity_filter=True, complexity_threshold=100),
        "complexity0": Options(start_adapter=S, low_complexity_filter=True, complexity_threshold=0),
        "qual_phred0_limits0": Options(start_adapter=S, qualified_quality_phred=0, unqualified_percent_limit=0, n_base_limit=0, n_percent_limit=0),
        "mask_break_w5_q30": Options(start_adapter=S, mask=True, mask_window_size=5, mask_mean_quality=30, break_reads=True,
                                     break_window_size=5, break_mean_quality=30),
        **QUALITY_SETS,
    }


# ---- the whole quality-byte range: bytes 1..127 (a 0 byte cannot reach the reference, which builds its reads from C strings)
# and the quality options at the ends of what src/options.cpp:validate accepts: -q 0..93, --mean_qual 0..93, the cut
# qualities 1..30 (the help text says 1~36; the validator is what holds).  validate does not check the --mask / --break
# qualities at all (the help text says 5~30): they run here at 1 and 93, the ends of the phred range a 7-bit byte can reach.
QUALITY_SETS = {
    "q93": Options(start_adapter=S, qualified_quality_phred=93, unqualified_percent_limit=60),
    "q0": Options(start_adapter=S, end_adapter=E, qualified_quality_phred=0, unqualified_percent_limit=0),
    "mean_qual93": Options(start_adapter=S, mean_qual=93, unqualified_percent_limit=100),
    "mean_qual1": Options(start_adapter=S, mean_qual=1, low_complexity_filter=True),
    "cut_q1_w4": Options(start_adapter=S, cut_front=True, cut_tail=True, cut_window_size=4, cut_mean_quality=1),
    "cut_q30_w1": Options(disable_adapter_trimming=True, cut_front=True, cut_tail=True, cut_window_size=1, cut_mean_quality=30,
                          length_required=1),
    "cut_front_q1_tail_q30": Options(start_adapter=S, end_adapter=E, cut_front=True, cut_tail=True, cut_front_window_size=10,
                                     cut_front_mean_quality=1, cut_tail_window_size=5, cut_tail_mean_quality=30),
    "mask_q1_break_q93": Options(start_adapter=S, mask=True, mask_window_size=5, mask_mean_quality=1, break_reads=True,
                                 break_window_size=10, break_mean_quality=93),
    "mask_q93_break_q1": Options(start_adapter=S, mask=True, mask_window_size=10, mask_mean_quality=93, break_reads=True,
                                 break_window_size=5, break_mean_quality=1),
    "mask_q20_w4": Options(start_adapter=S, mask=True, mask_window_size=4, mask_mean_quality=20, length_required=1),
}


def _window_on(rng, w, total):
    """w quality bytes in 1..127 whose sum is exactly `total` (w <= total <= 127 * w), some of them below 33"""
    q = rng.integers(1, 128, size=w)
    while q.sum() != total:
        i = int(rng.integers(w))
        step = int(np.sign(total - q.sum()))
        if 1 <= q[i] + step <= 127:
            q[i] += step
    return bytes(q.astype(np.uint8))


def quality_domain_batch(seed, n_random=60):
    """Reads whose quality bytes cover 1..127: long runs below 33 ('!' is 33), runs of 127, reads whose qualities are all below
    33 (a negative totalQual, Stats' quality sums going down), windows whose raw byte sum is exactly (33 + M) * w of a cut /
    mask / break window (and one more and one less) for the M and w of QUALITY_SETS and the defaults, and reads of bytes drawn
    uniformly from 1..127.  Start / end adapters and N now and then."""
    rng = np.random.default_rng(seed)
    reads = []

    def seq(n):
        s = bytearray(_rb(rng, n))
        for p in rng.integers(0, n, size=n // 200):
            s[int(p)] = ord("N")
        if n > 120 and rng.random() < 0.4:
            s[:30] = S.encode()
        if n > 120 and rng.random() < 0.3:
            s[n - 30:] = E.encode()
        return bytes(s)

    def uniform(n, lo=1, hi=127):
        return bytes(rng.integers(lo, hi + 1, size=n).astype(np.uint8))

    for k in range(12):                                           # runs below 33 and runs of 127 inside ordinary reads
        n = int(rng.integers(200, 1500))
        q = bytearray(uniform(n, 33 + 5, 33 + 40))
        for _ in range(3):
            a, m = int(rng.integers(0, n)), int(rng.integers(20, 300))
            q[a:a + m] = uniform(len(q[a:a + m]), 1, 32) if k % 2 else b"\x7f" * len(q[a:a + m])
        reads.append((seq(n), bytes(q)))
    for n in (1, 2, 5, 31, 32, 33, 100, 700):                     # every byte below 33: totalQual < 0
        reads.append((seq(n), uniform(n, 1, 32)))
        reads.append((seq(n), b"\x01" * n))
        reads.append((seq(n), b"\x7f" * n))
    for M in (1, 10, 15, 20, 30, 93):                             # windows exactly on the threshold, one above, one below
        for w in (1, 4, 5, 10):
            for d in (-1, 0, 1):
                total = (33 + M) * w + d
                if not w <= total <= 127 * w:
                    continue
                win = _window_on(rng, w, total)
                low, good = uniform(40, 1, 20), uniform(60, 33 + M, 127)
                reads.append((seq(100 + w), low + win + good))                # a front cut starts here or not
                reads.append((seq(100 + w), good + win + low))                # a tail cut ends here or not
                reads.append((seq(100 + 3 * w), good[:50] + win * 3 + good[:50]))   # mask / break windows in the middle
    for _ in range(n_random):
        n = int(rng.integers(50, 2000))
        reads.append((seq(n), uniform(n)))
    return pack_reads(reads)


EXTREME_SETS = _extreme_sets()


# ---- --mask / --break (SURVEY §8f row 3) ----
MASK_BREAK_SETS = {
    "break_default": Options(start_adapter=S, break_reads=True),
    "break_w20": Options(start_adapter=S, break_reads=True, break_window_size=20, break_mean_quality=16),
    "mask_default": Options(start_adapter=S, mask=True),
    "mask_cplx": Options(start_adapter=S, mask=True, mask_window_size=10, mask_mean_quality=17, low_complexity_filter=True,
                         n_percent_limit=20),
    "mask_and_break": Options(start_adapter=S, mask=True, mask_window_size=12, mask_mean_quality=15, break_reads=True,
                              break_window_size=30, break_mean_quality=14, cut_front=True, cut_tail=True,
                              n_base_limit=50, n_percent_limit=5),
    "break_no_adapter": Options(disable_adapter_trimming=True, break_reads=True, break_window_size=25,
                                break_mean_quality=12, disable_quality_filtering=True),
}

# the option sets that run on quality_domain_batch: QUALITY_SETS and sets of every other kind (adapters with the complexity
# filter, the global trims with --mean_qual, a one-base tail window, --mask with --break and the cuts)
QUALITY_DOMAIN_SETS = dict(QUALITY_SETS, **{n: OPTION_SETS[n] for n in ("default_se", "cut_polyx_cplx", "trims_limits", "loose_ed")},
                           mask_and_break=MASK_BREAK_SETS["mask_and_break"])


def blocky_quality_batch(seed, n=150):
    """Reads whose quality alternates between good (~Q30) and bad (~Q5) stretches of random length, some with
    adapters and chimeras: --break cuts them into several pieces, --mask paints the bad stretches."""
    rng = np.random.default_rng(seed)
    b = synth.ont_like(n, 1200, seed, p_chimera=0.1, q_mean=30.0, q_sd=3.0)
    q = b.qual.copy()
    for i in range(b.n_reads):
        o, L = int(b.offsets[i]), int(b.lens[i])
        pos = int(rng.integers(0, 300))
        while pos < L:
            bad = int(rng.integers(5, 260))
            q[o + pos:o + min(L, pos + bad)] = (np.rint(rng.normal(5, 2, size=min(L, pos + bad) - pos)).clip(1, 40).astype(np.uint8) + 33)
            pos += bad + int(rng.integers(20, 900))
    from fastplong_b200 import PackedBatch
    return PackedBatch(b.seq, q, b.offsets, b.lens)


# ---- randomised option sets x batches (tools/fuzz_*.py, test_*random*): the draw order is part of the contract, a
# (seed, index) pair names the same case everywhere ----
def random_option_kwargs(rng):
    def rand_adapter(lo=6, hi=45):
        return ''.join(rng.choice('ACGT') for _ in range(rng.randint(lo, hi)))
    kw = {}
    mode = rng.random()
    if mode < 0.15: kw['disable_adapter_trimming'] = True
    else:
        if rng.random() < 0.8: kw['start_adapter'] = rng.choice([synth.ADAPTER_START, rand_adapter()])
        if rng.random() < 0.8: kw['end_adapter'] = rng.choice([synth.ADAPTER_END, rand_adapter()])
        if rng.random() < 0.2: kw['adapter_fasta'] = [rand_adapter(8, 40) for _ in range(rng.randint(1, 4))]
        if rng.random() < 0.3: kw['distance_threshold'] = rng.choice([0.1, 0.2, 0.3, 0.4])
        if rng.random() < 0.3: kw['trimming_extension'] = rng.choice([0, 3, 10, 25])
    if rng.random() < 0.4: kw['cut_front'] = True
    if rng.random() < 0.4: kw['cut_tail'] = True
    if rng.random() < 0.4: kw['cut_window_size'] = rng.choice([1, 4, 10, 30]); kw['cut_mean_quality'] = rng.choice([10, 15, 20, 30])
    if rng.random() < 0.3: kw['trim_front'] = rng.choice([0, 1, 5, 40])
    if rng.random() < 0.3: kw['trim_tail'] = rng.choice([0, 1, 5, 40])
    if rng.random() < 0.3: kw['trim_poly_x'] = True; kw['poly_x_min_len'] = rng.choice([5, 10, 20])
    if rng.random() < 0.2: kw['disable_quality_filtering'] = True
    if rng.random() < 0.3: kw['qualified_quality_phred'] = rng.choice([5, 15, 25])
    if rng.random() < 0.3: kw['mean_qual'] = rng.choice([0, 8, 15])
    if rng.random() < 0.3: kw['n_base_limit'] = rng.choice([0, 2, 50])
    if rng.random() < 0.3: kw['n_percent_limit'] = rng.choice([1, 10, 50])
    if rng.random() < 0.3: kw['length_required'] = rng.choice([0, 15, 100, 1000])
    if rng.random() < 0.2: kw['length_limit'] = rng.choice([0, 500, 5000])
    if rng.random() < 0.3: kw['low_complexity_filter'] = True; kw['complexity_threshold'] = rng.choice([10, 30, 60])
    if rng.random() < 0.2: kw['mask'] = True; kw['mask_window_size'] = rng.choice([5, 10, 50]); kw['mask_mean_quality'] = rng.choice([8, 12, 20])
    if rng.random() < 0.2: kw['break_reads'] = True; kw['break_window_size'] = rng.choice([10, 30, 100]); kw['break_mean_quality'] = rng.choice([8, 12, 20])
    return kw


def random_case(rng):
    """-> (Options, batch, description)"""
    kw = random_option_kwargs(rng)
    opt = Options(**kw)
    kind = rng.random()
    seed = rng.randint(1, 10**6)
    if kind < 0.4: batch = adversarial_batch(seed)
    elif kind < 0.7: batch = blocky_quality_batch(seed, n=40)
    else: batch = ont_batch(seed, n=40, mean=1500, p_chimera=0.1, p_polya=0.1)
    return opt, batch, f"{kw} kind={kind:.3f} seed={seed}"


# ---- two more randomised families for tools/fuzz_gpu_vs_oracle.py (own draw order; random_case above is untouched) ----
def random_case_many_adapters(rng):
    """6-40 FASTA adapters of 8-70 bp (all three pre-filter widths: <= 32, <= 64, unfiltered), some planted at the read
    ends: the many-adapter pre-filter of k_trim and its re-filtering after a trim."""
    def rand_adapter(lo, hi):
        return ''.join(rng.choice('ACGT') for _ in range(rng.randint(lo, hi)))
    fasta = sorted(rand_adapter(8, rng.choice([20, 32, 44, 70])) for _ in range(rng.randint(6, 40)))
    kw = dict(adapter_fasta=fasta)
    if rng.random() < 0.7: kw['start_adapter'] = rng.choice([synth.ADAPTER_START, rand_adapter(6, 45)])
    if rng.random() < 0.7: kw['end_adapter'] = rng.choice([synth.ADAPTER_END, rand_adapter(6, 45)])
    if rng.random() < 0.3: kw['distance_threshold'] = rng.choice([0.1, 0.2, 0.3, 0.4])
    if rng.random() < 0.3: kw['trimming_extension'] = rng.choice([0, 3, 10, 25])
    if rng.random() < 0.3: kw['trim_poly_x'] = True
    if rng.random() < 0.3: kw['cut_front'] = True; kw['cut_tail'] = True
    seed = rng.randint(1, 10**6)
    planted = [fasta[rng.randrange(len(fasta))] for _ in range(rng.randint(1, 5))]
    batch = synth.ont_like(60, 1200, seed, planted=planted, p_planted=0.5, p_chimera=0.05, p_polya=0.1,
                           q_mean=rng.choice([17.0, 33.0]))
    return Options(**kw), batch, f"many {len(fasta)} adapters {kw.keys()} seed={seed}"


def random_case_long_reads(rng):
    """A few very long reads (up to ~400 kb) with chimeric inserts and every filter combination: the block-cooperative
    quality histogram (> 96 kb), the shared long ranges of k_kmer_fix, k_final's part counting, long Stats blocks."""
    kw = {}
    if rng.random() < 0.85:
        kw['start_adapter'] = synth.ADAPTER_START; kw['end_adapter'] = synth.ADAPTER_END
    else:
        kw['disable_adapter_trimming'] = True
    if rng.random() < 0.3: kw['disable_quality_filtering'] = True
    if rng.random() < 0.3: kw['disable_length_filtering'] = True
    if rng.random() < 0.4: kw['low_complexity_filter'] = True; kw['complexity_threshold'] = rng.choice([10, 30, 60])
    if rng.random() < 0.3: kw['qualified_quality_phred'] = rng.choice([5, 15, 25])
    if rng.random() < 0.3: kw['unqualified_percent_limit'] = rng.choice([10, 30, 60])
    if rng.random() < 0.3: kw['length_limit'] = rng.choice([0, 50000, 200000])
    if rng.random() < 0.3: kw['cut_front'] = True; kw['cut_tail'] = True
    if rng.random() < 0.3: kw['distance_threshold'] = rng.choice([0.25, 0.35, 0.45])     # loose: spurious middle hits, big gaps
    seed = rng.randint(1, 10**6)
    batch = synth.ont_like(rng.randint(3, 8), rng.choice([60000, 150000]), seed, p_chimera=0.6, q_mean=rng.choice([12.0, 18.0, 30.0]))
    return Options(**kw), batch, f"long {kw} seed={seed}"


# ---- --mask / --break at the edges of fpl_ext.cu: pieces on the length limits, filter ties counted on the masked copy, region
# walks that start at base 0 / end on the last base, more output reads than the record's two inline slots ----
# The reference's rolling sum holds w - 1 bytes (Filter::detectLowQualityRegions, SURVEY A.8): a window is low unless its bytes
# average about (33 + Q) * w / (w - 1), and after the first region the sum restarts from 0, so a later region ends only where a
# window of very low bytes is followed by one of high bytes.  The quality palette below is built around that.
MASK_BREAK_EDGE_SETS = {
    # pieces of length_required / length_limit and one either side; --mean_qual with bytes below '!'
    "break_lengths_mean": Options(disable_adapter_trimming=True, break_reads=True, break_window_size=4, break_mean_quality=10,
                                  length_required=6, length_limit=14, mean_qual=20, unqualified_percent_limit=100,
                                  n_percent_limit=100),
    # -n and the N share on the masked copy, -u with bytes exactly on -q
    "mask_n_limits": Options(disable_adapter_trimming=True, mask=True, mask_window_size=3, mask_mean_quality=12, n_base_limit=4,
                             n_percent_limit=30, qualified_quality_phred=20, unqualified_percent_limit=50, length_required=1),
    # both stages, -y ties on the masked copy and on 1- / 2-base pieces, the N share
    "mask_break_cplx": Options(disable_adapter_trimming=True, mask=True, mask_window_size=2, mask_mean_quality=20, break_reads=True,
                               break_window_size=3, break_mean_quality=8, low_complexity_filter=True, complexity_threshold=50,
                               length_required=0, n_percent_limit=50),
    # -q 0 / -u 0 under --break
    "break_q0_u0": Options(disable_adapter_trimming=True, break_reads=True, break_window_size=5, break_mean_quality=12,
                           qualified_quality_phred=0, unqualified_percent_limit=0, length_required=1),
    # complexity with neither the quality nor the length filter (no counts taken), one-base windows
    "cplx_only_w1": Options(disable_adapter_trimming=True, mask=True, mask_window_size=1, mask_mean_quality=30, break_reads=True,
                            break_window_size=6, break_mean_quality=8, disable_quality_filtering=True,
                            disable_length_filtering=True, low_complexity_filter=True, complexity_threshold=40),
    # the quality filter without the length filter (the counts are taken when either is on), one-base break windows (regions of
    # one base: first == last)
    "break_w1_qual_only": Options(disable_adapter_trimming=True, break_reads=True, break_window_size=1, break_mean_quality=20,
                                  disable_length_filtering=True, unqualified_percent_limit=30, n_percent_limit=20),
    # split reads (a start adapter in the middle) broken on either side
    "split_break_mask": Options(start_adapter=S, end_adapter=E, trimming_extension=0, mask=True, mask_window_size=6,
                                mask_mean_quality=18, break_reads=True, break_window_size=8, break_mean_quality=10,
                                length_required=5, low_complexity_filter=True, complexity_threshold=30),
}


def mask_break_edge_batch(seed=11, n=700):
    """Short reads (mostly 1..90 bases) whose qualities are blocks of high (73, 127), very low (1..5, below '!'), low-but-printable
    (34..40) and near-threshold bytes, windows of the sets above at both ends of a read, whole reads of high bytes (no region) and
    of low bytes (vanishing reads), sequences of two letters with runs of N (complexity and N ties, masked N next to N), long reads
    (pieces over 32 bases), and split reads (a start adapter in the middle of 600 bases).  The read count is no multiple of 8."""
    rng = np.random.default_rng(seed)
    reads = []

    def qblock(k, kind):
        if kind == 0:
            return bytes([73]) * k
        if kind == 1:
            return bytes([127]) * k
        if kind == 2:
            return bytes(rng.integers(1, 6, size=k).astype(np.uint8))
        if kind == 3:
            return bytes(rng.integers(34, 41, size=k).astype(np.uint8))
        return bytes(rng.integers(40, 60, size=k).astype(np.uint8))

    def qual(L):
        q = b""
        while len(q) < L:
            q += qblock(int(rng.integers(1, 12)), int(rng.choice(5, p=[0.3, 0.2, 0.25, 0.15, 0.1])))
        return q[:L]

    def seq(L):
        a, c = rng.choice(list(b"ACGT"), size=2, replace=False)
        p = rng.choice([0.1, 0.3, 0.5, 0.7])
        s, cur = bytearray(), int(a)
        for _ in range(L):
            s.append(cur)
            if rng.random() < p:
                cur = int(c) if cur == int(a) else int(a)
        for _ in range(int(rng.integers(0, 3))):
            if L:
                at, k = int(rng.integers(0, L)), int(rng.integers(1, 4))
                s[at:at + k] = b"N" * len(s[at:at + k])
        return bytes(s)

    for k in range(n - 64):
        L = int(rng.integers(1, 91)) if k % 10 else int(rng.integers(1, 8))
        reads.append((seq(L), qual(L)))
    for L in (1, 2, 3, 5, 8, 13):
        reads.append((seq(L), bytes([127]) * L))                   # no region
        reads.append((seq(L), bytes([3]) * L))                     # low everywhere: vanishes
    for L in (3, 4):                                               # at most one window (no region): sums of q - 33 on a mean of
        for total in (20 * L, 20 * L - 1, 21 * L - 1, -L):         # 20 (the --mean_qual of the sets), below it, negative
            q = [33 + total // L] * L
            q[0] += total - L * (total // L)
            reads.append((seq(L), bytes(q)))
    for q in (b"4\x7f5\x7f54\x7f5\x7f55\x7f", b"\x7f\x7f54\x7f55\x7f5", b"\x7f55\x7f4\x7f55\x7f4"):   # -q 20 ('5'): the
        reads.append((seq(len(q)), q))                             # bytes on it decide -u 50 (no mask region at w 3, Q 12)
    for q in ((2, 60, 118), (3, 3, 60, 118), (2, 60, 2, 60, 118)):  # one-base windows: a rise of 58 ends a region at once
        reads.append((seq(len(q)), bytes(q)))
    for L, k in ((10, 3), (10, 4), (20, 6), (20, 5)):              # the N share on 30 % and above it, on unmasked bases
        sq = bytearray(seq(L).replace(b"N", b"A"))
        sq[1:2 * k:2] = b"N" * k
        reads.append((bytes(sq), bytes([127]) * L))
    for k in range(16):                                            # pieces over 32 bases: the warp loops
        L = int(rng.integers(100, 400))
        q = bytearray(bytes([127]) * L)
        for at in rng.integers(0, L, size=3):
            q[int(at):int(at) + 12] = bytes([2]) * len(q[int(at):int(at) + 12])
        reads.append((seq(L), bytes(q)))
    for k in range(18):                                            # split reads, broken on the left, the right or both; a
        la, lb = 240 + 7 * k, 300 + 5 * k                          # region that ends near a side's end leaves a tail piece
        qa, qb = bytearray(bytes([73]) * la), bytearray(bytes([73]) * lb)
        t = 2 + k % 7
        if k % 3 != 1:
            qa[la - 30 - t:la - t] = bytes([2]) * 30
            qa[la - t:] = bytes([127]) * t
        if k % 3 != 0:
            qb[lb - 20 - t:lb - t] = bytes([2]) * 20
            qb[lb - t:] = bytes([127]) * t
        reads.append((seq(la) + S.encode() + seq(lb), bytes(qa) + bytes([73]) * len(S) + bytes(qb)))
    assert len(reads) % 8 and len(reads) % 256
    return pack_reads(reads)
