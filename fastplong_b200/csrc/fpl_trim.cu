// k_trim: the sequential, end-local part of processSingleEnd for one read per warp:
//   Filter::trimAndCut (src/filter.cpp:130-232) -> PolyX::trimPolyX (src/polyx.cpp:11-78) ->
//   AdapterTrimmer::trimBySequenceStart / trimBySequenceEnd for -s, -e and every FASTA adapter in order
//   (src/adaptertrimmer.cpp:42-57,168-302).
// Each stage is the parallel closed form of the reference's loop (SURVEY A.11): the 32 lanes evaluate 32
// candidate positions at once, a ballot / min-reduction picks what the sequential loop would have picked.
// Work is O(window) per read, not O(read length), except for degenerate quality cuts.
#include "fpl_device.cuh"

namespace {

__device__ __forceinline__ int sc(uint8_t b) { return (int)(signed char)b; }  // the reference reads `char`

// ---- Levenshtein distance, Myers/Hyyro bit-parallel, pattern = adapter bits [shift, shift+m) ----
// text = read bytes.  Equivalent to edit_distance() (src/editdistance.cpp:100-126): exact global distance.
__device__ __forceinline__ void peq_sub(const uint4* peq, uint8_t c, int shift, int m, unsigned long long& lo,
                                        unsigned long long& hi) {
    uint4 v = __ldg(&peq[c]);
    lo = ((unsigned long long)v.y << 32) | v.x;
    hi = ((unsigned long long)v.w << 32) | v.z;
    if (shift >= 64) { lo = hi >> (shift - 64); hi = 0; }
    else if (shift > 0) { lo = (lo >> shift) | (hi << (64 - shift)); hi >>= shift; }
    if (m < 64) { lo &= (1ull << m) - 1; hi = 0; }
    else if (m < 128) { hi &= (1ull << (m - 64)) - 1; }
}

__device__ int myers128(const uint8_t* text, int n, const uint4* peq, int shift, int m) {
    if (m == 0) return n;
    if (n == 0) return m;
    unsigned long long VPl, VPh, VNl = 0, VNh = 0;
    if (m < 64) { VPl = (1ull << m) - 1; VPh = 0; }
    else if (m == 64) { VPl = ~0ull; VPh = 0; }
    else if (m < 128) { VPl = ~0ull; VPh = (1ull << (m - 64)) - 1; }
    else { VPl = ~0ull; VPh = ~0ull; }
    const bool topHi = m > 64;
    const unsigned long long top = 1ull << ((m - 1) & 63);
    int score = m;
    for (int i = 0; i < n; i++) {
        unsigned long long El, Eh;
        peq_sub(peq, text[i], shift, m, El, Eh);
        unsigned long long Xvl = El | VNl, Xvh = Eh | VNh;
        // Xh = (((Eq & VP) + VP) ^ VP) | Eq, 128-bit add with carry
        unsigned long long al = El & VPl, ah = Eh & VPh;
        unsigned long long sl = al + VPl;
        unsigned long long carry = sl < al ? 1ull : 0ull;
        unsigned long long sh = ah + VPh + carry;
        unsigned long long Xhl = (sl ^ VPl) | El, Xhh = (sh ^ VPh) | Eh;
        unsigned long long HPl = VNl | ~(Xhl | VPl), HPh = VNh | ~(Xhh | VPh);
        unsigned long long HNl = VPl & Xhl, HNh = VPh & Xhh;
        unsigned long long hpTop = topHi ? HPh : HPl, hnTop = topHi ? HNh : HNl;
        if (hpTop & top) score++;
        else if (hnTop & top) score--;
        HPh = (HPh << 1) | (HPl >> 63); HPl = (HPl << 1) | 1ull;
        HNh = (HNh << 1) | (HNl >> 63); HNl = HNl << 1;
        VPl = HNl | ~(Xvl | HPl); VPh = HNh | ~(Xvh | HPh);
        VNl = HPl & Xvl; VNh = HPh & Xvh;
    }
    return score;
}

// Levenshtein distance for adapters of 33..64 bp: one 64-bit word (the same recurrence as myers128 without its high half)
__device__ int myers64(const uint8_t* text, int n, const uint4* peq, int shift, int m) {
    if (m == 0) return n;
    if (n == 0) return m;
    unsigned long long VP = m >= 64 ? ~0ull : ((1ull << m) - 1), VN = 0;
    const unsigned long long top = 1ull << (m - 1), mask = VP;
    int score = m;
    for (int i = 0; i < n; i++) {
        const uint4 v = __ldg(&peq[text[i]]);
        unsigned long long lo = ((unsigned long long)v.y << 32) | v.x, hi = ((unsigned long long)v.w << 32) | v.z;
        unsigned long long Eq = shift == 0 ? lo : shift >= 64 ? (hi >> (shift - 64)) : ((lo >> shift) | (hi << (64 - shift)));
        Eq &= mask;
        const unsigned long long Xv = Eq | VN;
        const unsigned long long Xh = (((Eq & VP) + VP) ^ VP) | Eq;
        unsigned long long HP = VN | ~(Xh | VP);
        unsigned long long HN = VP & Xh;
        if (HP & top) score++;
        else if (HN & top) score--;
        HP = (HP << 1) | 1ull; HN <<= 1;
        VP = HN | ~(Xv | HP);
        VN = HP & Xv;
    }
    return score;
}

// CLS: the size class of the adapters a kernel handles (decided at fpl_create): 0 = all <= 32 bp, 1 = all <= 64 bp, 2 = any.
// A kernel is compiled without the forms its class never needs, which would otherwise set its register budget.
template <int CLS>
__device__ __forceinline__ int ed_adapter(const DevParams& P, int aidx, const uint8_t* text, int n, int shift, int m, int alen) {
    const uint4* peq = P.peq + (size_t)aidx * 256;
    if (CLS == 0) return n <= 32 ? myers32_warp(text, n, peq, shift, m) : myers32(text, n, peq, shift, m);
    if (CLS == 1) {
        if (alen <= 32) return n <= 32 ? myers32_warp(text, n, peq, shift, m) : myers32(text, n, peq, shift, m);
        return myers64(text, n, peq, shift, m);
    }
    // every lane wants the same distance: for <= 32 text bytes lane i looks up the match mask of byte i once and the
    // recurrence runs on shuffled masks (no dependent loads inside the column loop)
    if (alen <= 32) return n <= 32 ? myers32_warp(text, n, peq, shift, m) : myers32(text, n, peq, shift, m);
    if (alen <= 128) return myers128(text, n, peq, shift, m);
    return myers_long(text, n, P.peq_long + (size_t)aidx * 256 * P.peq_words, P.peq_words, shift, m);
}

// 16-bit pattern variant for the probe loops (:202-216, :273-286); peq = the 256 match masks of the probe pattern.
// The score is m + (#columns whose top horizontal delta is +1) - (#columns where it is -1): the two counts are
// accumulated in units of `top` and the left shifts are multiplies, which keeps the logic pipe to 8 ops per column.
// (A warp-wide early exit on the lower bound score_i - (n - i) was measured and lost: the vote and the score
// reconstruction every four columns cost more than the columns they save.)
__device__ __forceinline__ int myers16(const uint8_t* text, int n, const uint32_t* peq, int m) {
    uint32_t VP = (1u << m) - 1u, VN = 0;
    const uint32_t top = 1u << (m - 1);
    uint32_t accP = 0, accN = 0;
#pragma unroll 4
    for (int i = 0; i < n; i++) {
        const uint32_t Eq = __ldg(&peq[text[i]]);
        const uint32_t Xv = Eq | VN;
        const uint32_t Xh = (((Eq & VP) + VP) ^ VP) | Eq;
        uint32_t HP = VN | ~(Xh | VP);
        uint32_t HN = VP & Xh;
        accP += HP & top;
        accN += HN & top;
        asm("mad.lo.u32 %0, %1, 2, 1;" : "=r"(HP) : "r"(HP));
        asm("mad.lo.u32 %0, %1, 2, 0;" : "=r"(HN) : "r"(HN));
        VP = HN | ~(Xv | HP);
        VN = HP & Xv;
    }
    return m + (int)(accP >> (m - 1)) - (int)(accN >> (m - 1));
}

__device__ __forceinline__ int hamming(const uint8_t* r, const uint8_t* a, int alen) {
    int mm = 0;
    for (int i = 0; i < alen; i++) mm += r[i] != __ldg(&a[i]);
    return mm;
}

// AdapterTrimmer::searchAdapter restricted to the two windowed modes (src/adaptertrimmer.cpp:84-134,156-165).
// left: first p with H<=T, else the LAST arg-min;  right: last p with H<=T, else the FIRST arg-min.
__device__ __forceinline__ bool is_acgt(uint32_t b) {   // exact: A 0x41, C 0x43, G 0x47, T 0x54
    return (b >> 5) == 2u && ((0x0010008Au >> (b & 31u)) & 1u);
}

template <int CLS>
__device__ int search_window(const DevParams& P, const uint8_t* rdata, int rlen, int aidx, int searchStart,
                             int searchLen, bool left, uint32_t* pk) {
    const int lane = lane_id();
    const int alen = P.alen[aidx];
    const uint8_t* adata = P.adapters + (size_t)aidx * FPL_MAX_ADAPTER_LEN;
    const int T = P.thr[alen];
    int searchEnd = rlen;
    if (searchLen > 0) searchEnd = min(rlen, searchLen + searchStart);
    if (searchStart + alen > rlen) return -1;
    int p0, p1;  // inclusive range of positions
    bool descending = false;
    if (left) { p0 = searchStart; p1 = searchEnd - alen - 1; }
    else if (searchEnd > alen) { p0 = searchStart; p1 = searchEnd - alen; descending = true; }
    else { p0 = searchStart; p1 = searchEnd - alen - 1; }  // generic mode, empty or tiny range
    unsigned accept = descending ? 0u : 0xFFFFFFFFu;
    unsigned best = 0xFFFFFFFFu;  // (H << 16) | tie-break key, minimised
    // Packed form of the window for ACGT-only adapters of <= 32 bp: 2-bit codes and "not ACGT" flags, 16 bases per
    // word, in shared memory (pk[0..17] codes, pk[18..35] flags); H(p) = popcount over the adapter's positions of
    // (code differs | base invalid), exactly the byte-wise count of src/adaptertrimmer.cpp:93-96.
    const uint4 ac = __ldg(reinterpret_cast<const uint4*>(P.acode) + aidx);
    const int nbytes = p1 - p0 + alen;
    const bool packed = (ac.z | ac.w) != 0u && nbytes <= 256 && p1 >= p0;
    if (packed) {
        uint32_t codes = 0, inv = 0;
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const int idx = 8 * lane + j;
            const uint32_t b = idx < nbytes ? rdata[p0 + idx] : 0u;
            codes |= ((b >> 1) & 3u) << (2 * j);
            inv |= (is_acgt(b) ? 0u : 1u) << (2 * j);
        }
        __syncwarp();
        reinterpret_cast<uint16_t*>(pk)[lane] = (uint16_t)codes;
        reinterpret_cast<uint16_t*>(pk + 18)[lane] = (uint16_t)inv;
        if (lane < 2) { pk[16 + lane] = 0; pk[34 + lane] = 0x55555555u; }
        __syncwarp();
    }
    for (int p = p0 + lane; p <= p1; p += 32) {
        int mm;
        if (packed) {
            const int q = p - p0, wi = q >> 4, sh = (q & 15) * 2;
            const uint32_t c0 = pk[wi], c1 = pk[wi + 1], c2 = pk[wi + 2];
            const uint32_t i0 = pk[18 + wi], i1 = pk[19 + wi], i2 = pk[20 + wi];
            const uint32_t dlo = __funnelshift_r(c0, c1, sh) ^ ac.x, dhi = __funnelshift_r(c1, c2, sh) ^ ac.y;
            const uint32_t mlo = (dlo | (dlo >> 1) | __funnelshift_r(i0, i1, sh)) & ac.z;
            const uint32_t mhi = (dhi | (dhi >> 1) | __funnelshift_r(i1, i2, sh)) & ac.w;
            mm = __popc(mlo) + __popc(mhi);
        } else {
            mm = hamming(rdata + p, adata, alen);
        }
        unsigned rel = (unsigned)(p - p0);
        if (mm <= T) accept = descending ? max(accept, rel + 1u) : min(accept, rel);
        // ascending loops keep the last minimum (<=), the descending loop also uses <= and so keeps the smallest p;
        // the generic loop (<) keeps the smallest p
        unsigned key = (left ? (0xFFFFu - rel) : rel);
        best = min(best, ((unsigned)mm << 16) | key);
    }
    accept = descending ? __reduce_max_sync(0xffffffffu, accept) : __reduce_min_sync(0xffffffffu, accept);
    best = __reduce_min_sync(0xffffffffu, best);
    if (descending) { if (accept != 0u) return p0 + (int)accept - 1; }
    else if (accept != 0xFFFFFFFFu && (left)) return p0 + (int)accept;
    if (best == 0xFFFFFFFFu) return -1;
    unsigned key = best & 0xFFFFu;
    int pos = p0 + (int)(left ? (0xFFFFu - key) : key);
    int ed = ed_adapter<CLS>(P, aidx, rdata + pos, alen, 0, alen, alen);
    return ed <= T ? pos : -1;
}

template <typename W>
struct SearchMyers {                      // pattern in the low m bits; standard Myers/Hyyro search recurrence
    W VP, VN, top;
    int score, best;
    __device__ __forceinline__ void init(int m) {
        VP = m >= (int)(8 * sizeof(W)) ? ~(W)0 : (((W)1 << m) - 1);
        VN = 0; top = (W)1 << (m - 1); score = m; best = m;
    }
    __device__ __forceinline__ void column(W Eq) {
        const W Xv = Eq | VN;
        const W Xh = (((Eq & VP) + VP) ^ VP) | Eq;
        W HP = VN | ~(Xh | VP);
        W HN = VP & Xh;
        score += (HP & top) ? 1 : 0;
        score -= (HN & top) ? 1 : 0;
        HP <<= 1; HN <<= 1;                // search mode: the horizontal delta entering row 0 is 0
        VP = HN | ~(Xv | HP);
        VN = HP & Xv;
        best = min(best, score);
    }
};


// The probe loops (src/adaptertrimmer.cpp:202-216, 273-286) take the Levenshtein distance of up to 184 sixteen-mers of
// the end window to the adapter's 16-mer and use only those within thr(16).  Which positions CAN be within it is decided
// first, by one search-mode pass per lane over its ~6 positions (+ 15 columns of run-in): sg(e), the best distance of any
// window substring ending at e, bounds ED(window[e-15..e], 16-mer) from below.  Only those candidates get the exact
// distance; the rest could never have been hits, so the loops' results are unchanged.
// Start side: probe p is rdata[p .. p+plen); end side: probe p is rdata[rlen-plen-p .. rlen-p).
// Returns the number of candidates, their positions (ascending) in list[].  All 32 lanes.
__device__ int probe_candidates(const uint8_t* rdata, int rlen, int np, int plen, const uint32_t* t16, int T16, bool endside,
                                uint8_t* list) {
    const int lane = lane_id();
    if (np <= 0) return 0;
    const int CH = (np + 31) >> 5;
    const int p0 = lane * CH, p1 = min(np, p0 + CH);
    uint32_t cb = 0;
    if (p0 < np) {
        // text columns in read order; ends e of this lane's probes: start side e = p + plen - 1, end side e = rlen - 1 - p
        const int e_lo = endside ? rlen - p1 : p0 + plen - 1;
        const int e_hi = endside ? rlen - 1 - p0 : p1 - 1 + plen - 1;
        // (keeping the four bases' masks in registers and unrolling the columns costs 24 registers and lost; the two
        //  dependent L1 loads per column stay)
        SearchMyers<uint32_t> Q;
        Q.init(plen);
        for (int j = e_lo - (plen - 1); j <= e_hi; j++) {
            Q.column(__ldg(&t16[rdata[j]]));
            if (j >= e_lo && Q.score <= T16) cb |= 1u << ((endside ? rlen - 1 - j : j - (plen - 1)) - p0);
        }
    }
    // compact the candidate positions, ascending, into list[]
    const int cnt = __popc(cb);
    const int before = warp_incl_scan(cnt) - cnt;
    const int total = __shfl_sync(0xffffffffu, before + cnt, 31);
    __syncwarp();
    int k = before;
    for (uint32_t m = cb; m; m &= m - 1) list[k++] = (uint8_t)(p0 + __ffs(m) - 1);
    __syncwarp();
    return total;
}

struct Win { int lo, len; };

__device__ __forceinline__ void trim_front(Win& w, int n) {  // Read::trimFront, src/read.cpp:69-73
    n = min(w.len - 1, n);
    if (n < 0) { w.lo += w.len; w.len = 0; return; }
    w.lo += n; w.len -= n;
}
__device__ __forceinline__ void resize_(Win& w, int n) {     // Read::resize, src/read.cpp:62-67
    if (n > w.len || n < 0) return;
    w.len = n;
}

struct EventSink {
    fpl_read_result* out;
    unsigned long long* table;  // device event count table
    int n;
    __device__ __forceinline__ void add(int idx, int side, int cmplen) {
        if (lane_id() == 0) {
            if (n < FPL_INLINE_EVENTS) out->events[n] = FPL_EVENT(idx, side, cmplen);
            atomicAdd(&table[((size_t)idx * 2 + side) * (FPL_MAX_ADAPTER_LEN + 1) + cmplen], 1ull);
        }
        n++;
    }
};

// AdapterTrimmer::trimBySequenceStart (src/adaptertrimmer.cpp:168-236)
// tryWindow / tryProbes: false when the caller's pre-filter has proved that stage cannot hit (the stage then returns what
// it would have returned: nothing found)
template <int CLS>
__device__ int trim_start(const DevParams& P, const uint8_t* seq, Win& w, int aidx, EventSink& ev, uint8_t* scratch,
                          bool tryWindow = true, bool tryProbes = true) {
    const int lane = lane_id();
    const int alen = P.alen[aidx], ext = P.opt.trimming_extension;
    const uint8_t* rdata = seq + w.lo;
    const int rlen = w.len;
    if (rlen < FPL_PATTERN_LEN) return 0;
    const int plen = min(FPL_PATTERN_LEN, alen);
    int mpos = tryWindow ? search_window<CLS>(P, rdata, rlen, aidx, 0, FPL_WINDOW, false, reinterpret_cast<uint32_t*>(scratch)) : -1;
    if (mpos >= 0) {
        mpos = min(mpos + ext, rlen - alen);
        ev.add(aidx, 0, alen);
        trim_front(w, mpos + alen);
        return mpos + alen;
    }
    // probe: best (smallest ed, earliest p) 16-mer hit of the adapter's last plen chars (:202-216)
    const int np = min(rlen - plen, FPL_WINDOW - plen);
    const int T16 = P.thr[plen];
    unsigned best = 0xFFFFFFFFu;
    const uint32_t* t16 = P.peq16 + (size_t)aidx * 512 + 256;   // last plen chars
    if (!tryProbes) return 0;
    const int ncand = probe_candidates(rdata, rlen, np, plen, t16, T16, false, scratch);
    for (int c0 = 0; c0 < ncand; c0 += 32) {
        if (c0 + lane < ncand) {
            const int p = scratch[c0 + lane];
            const int ed = myers16(rdata + p, plen, t16, plen);
            if (ed <= T16) best = min(best, ((unsigned)ed << 16) | (unsigned)p);
        }
    }
    best = __reduce_min_sync(0xffffffffu, best);
    if (best != 0xFFFFFFFFu) {
        int pos = (int)(best & 0xFFFFu);
        int cmplen = min(pos + plen, alen);
        int ed = ed_adapter<CLS>(P, aidx, rdata + pos + plen - cmplen, cmplen, alen - cmplen, cmplen, alen);
        if (ed <= P.thr[cmplen]) {
            pos = min(pos + ext, rlen - alen);
            ev.add(aidx, 0, cmplen);
            trim_front(w, pos + plen);
            return pos + plen;
        }
    }
    return 0;
}

// AdapterTrimmer::trimBySequenceEnd (src/adaptertrimmer.cpp:238-302)
template <int CLS>
__device__ int trim_end(const DevParams& P, const uint8_t* seq, Win& w, int aidx, EventSink& ev, uint8_t* scratch,
                        bool tryWindow = true, bool tryProbes = true) {
    const int lane = lane_id();
    const int alen = P.alen[aidx], ext = P.opt.trimming_extension;
    const uint8_t* rdata = seq + w.lo;
    const int rlen = w.len;
    if (rlen < FPL_PATTERN_LEN) return 0;
    const int plen = min(FPL_PATTERN_LEN, alen);
    const int searchStart = max(0, rlen - FPL_WINDOW);
    int mpos = tryWindow ? search_window<CLS>(P, rdata, rlen, aidx, searchStart, FPL_WINDOW, true, reinterpret_cast<uint32_t*>(scratch)) : -1;
    if (mpos >= 0) {
        mpos = max(0, mpos - ext);
        ev.add(aidx, 1, alen);
        resize_(w, mpos);
        return rlen - mpos;
    }
    // probe from the tail with the "last best, stop at the first worse hit" rule (:273-286), 32 positions per step:
    // the distances of a step in parallel, then the sequential rule in closed form (SURVEY A.11) — walk the hits in
    // order, stop at the first hit whose distance exceeds the previous hit's, keep the hit before it.  The reference
    // stops probing there and so do we: with an adapter near the end that is the first or second step.
    const int np = min(rlen - plen, FPL_WINDOW - plen);
    const int T16 = P.thr[plen];
    const uint32_t* t16 = P.peq16 + (size_t)aidx * 512;         // first plen chars
    int pos = -1, carryE = -1, carryPos = -1;
    bool done = false;
    if (!tryProbes) return 0;
    const int ncand = probe_candidates(rdata, rlen, np, plen, t16, T16, true, scratch);
    for (int c0 = 0; c0 < ncand && !done; c0 += 32) {
        const bool have = c0 + lane < ncand;
        const int p = have ? scratch[c0 + lane] : 0;
        int e = 255;
        if (have) {
            const int ed = myers16(rdata + rlen - plen - p, plen, t16, plen);
            e = ed <= T16 ? ed : 255;
        }
        const bool hit = e != 255;
        const unsigned m = __ballot_sync(0xffffffffu, hit);
        const unsigned lower = m & ((1u << lane) - 1u);
        const int src = lower ? 31 - __clz(lower) : -1;
        int pe = __shfl_sync(0xffffffffu, e, src >= 0 ? src : 0);
        if (src < 0) pe = carryE;
        const unsigned bm = __ballot_sync(0xffffffffu, hit && pe >= 0 && e > pe);
        if (bm) {
            const int bl = __ffs(bm) - 1;
            const unsigned lowerb = m & ((1u << bl) - 1u);
            pos = lowerb ? scratch[c0 + 31 - __clz(lowerb)] : carryPos;
            done = true;
        } else if (m) {
            const int last = 31 - __clz(m);
            carryE = __shfl_sync(0xffffffffu, e, last);
            carryPos = scratch[c0 + last];
        }
    }
    if (!done) pos = carryPos;
    __syncwarp();
    if (pos > 0) {
        int cmplen = min(pos + plen, alen);
        int ed = ed_adapter<CLS>(P, aidx, rdata + rlen - plen - pos, cmplen, 0, cmplen, alen);
        if (ed <= P.thr[cmplen]) {
            pos = min(pos + ext, rlen - plen);
            ev.add(aidx, 1, cmplen);
            resize_(w, rlen - plen - pos);
            return pos + plen;
        }
    }
    return 0;
}


// ------------------------------------------------------------------------------------------------------------------
// Pre-filter for trimByMultiSequences (src/adaptertrimmer.cpp:42-57) with many FASTA adapters (BASELINE configs[2]: 64).
// For every adapter the reference runs trimBySequenceStart and trimBySequenceEnd: a Hamming search of the 200-base end
// window plus one Levenshtein verification, then up to 184 sixteen-mer Levenshtein probes — and on a read without that
// adapter all of it finds nothing.  "Finds nothing" is decided here for 32 (adapter, side) pairs at a time, one per lane,
// by two approximate-matching passes of Myers' bit-vector algorithm in SEARCH mode over the window (text = the window,
// free start): sg(e) = min over s of ED(window[s..e], pattern) is a lower bound of the distance of EVERY alignment the
// exact code evaluates that ends at e — ED(read[p..p+alen), adapter) in searchAdapter, which also bounds the Hamming
// distance from below, and ED(read[p..p+16), 16-mer) in the probe loops.  If sg never reaches thr(alen) for the whole
// adapter nor thr(16) for the probe 16-mer, neither stage can return a hit and the pair is skipped; otherwise the exact
// code runs as before.  The filter only ever says "maybe" too often, never "no" wrongly: results are unchanged.
// ------------------------------------------------------------------------------------------------------------------
#define PF_WIN FPL_WINDOW
#define PF_WORDS ((2 * FPL_MAX_ADAPTERS + 31) / 32)

// maybe-bits of the (adapter, side) pairs of all FASTA adapters for the window w: bit 2 * (k - 2) + side.  The pairs are
// walked in P.pf_order (adapters grouped by width class), 32 per round, one per lane.
// head / tail: the warp's staging buffers (PF_WIN bytes each); bits: one bit per pair (zeroed by the caller).  All 32 lanes.
template <typename W>
__device__ void prefilter_round(const DevParams& P, const uint8_t* head, const uint8_t* tail, int hw, int base, int nitems,
                                uint32_t* bits) {
    const int lane = lane_id();
    const int item = base + lane;
    const bool active = item < nitems;
    const int k = active ? __ldg(&P.pf_order[item >> 1]) : 2, side = item & 1;
    const int alen = active ? P.alen[k] : 1;
    const bool filterable = active && alen >= 1 && alen <= (int)(8 * sizeof(W));
    const int plen = min(FPL_PATTERN_LEN, alen);
    const uint4* peq = P.peq + (size_t)k * 256;
    auto eq_of = [&](uint32_t ch) -> W {
        const uint4 v = __ldg(&peq[ch]);
        if (sizeof(W) == 8) return (W)(((unsigned long long)v.y << 32) | v.x);
        return (W)v.x;
    };
    W eA = 0, eC = 0, eG = 0, eT = 0;
    if (filterable) { eA = eq_of('A'); eC = eq_of('C'); eG = eq_of('G'); eT = eq_of('T'); }
    // the probe pattern: the adapter's LAST plen chars on the start side, its FIRST plen chars on the end side
    // (an adapter wider than W is not filtered — both verdicts are "maybe" — so its columns run on a 1-bit dummy pattern:
    //  shifting by alen - 1 or alen - plen >= the word width would be undefined; found by UBSan on the emulated build)
    const int sh16 = (filterable && side == 0) ? alen - plen : 0;
    const uint32_t m16 = plen >= 32 ? 0xFFFFFFFFu : ((1u << plen) - 1u);
    SearchMyers<W> F;
    SearchMyers<uint32_t> Q;
    F.init(filterable ? alen : 1); Q.init(max(plen, 1));
    const uint8_t* text = side == 0 ? head : tail;
    for (int j = 0; j < hw; j++) {
        const uint32_t b = text[j];
        const uint32_t code = (b >> 1) & 3u;                 // A 0, C 1, T 2, G 3 — for exact A/C/G/T bytes
        W Eq;
        if (is_acgt(b)) Eq = code == 0 ? eA : code == 1 ? eC : code == 2 ? eT : eG;
        else Eq = filterable ? eq_of(b) : 0;                 // N, lower case, IUPAC: the table knows
        F.column(Eq);
        Q.column((uint32_t)(Eq >> sh16) & m16);
    }
    // bitsF: the window stage (Hamming search + verification) can hit; bitsQ: a probe can
    const bool mF = active && (!filterable || F.best <= P.thr[alen]);
    const bool mQ = active && (!filterable || Q.best <= P.thr[plen]);
    const int bit = 2 * (k - 2) + side;
    if (mF) atomicOr(&bits[bit >> 5], 1u << (bit & 31));
    if (mQ) atomicOr(&bits[PF_WORDS + (bit >> 5)], 1u << (bit & 31));
}

template <int CLS>
__device__ void prefilter(const DevParams& P, const uint8_t* seq, const Win& w, uint8_t* head, uint8_t* tail, uint32_t* bits) {
    const int lane = lane_id();
    const int nitems = 2 * (P.n_adapters - 2);
    const int hw = min(w.len, PF_WIN);
    __syncwarp();
    for (int j = lane; j < hw; j += 32) { head[j] = seq[w.lo + j]; tail[j] = seq[w.lo + w.len - hw + j]; }
    for (int i = lane; i * 32 < nitems; i += 32) { bits[i] = 0; bits[PF_WORDS + i] = 0; }
    __syncwarp();
    for (int base = 0; base < nitems; base += 32) {
        // one width per round: 64-bit vectors only if an adapter of this round needs them (the order groups them)
        const int it = base + lane;
        const bool wide = __any_sync(0xffffffffu, it < nitems && P.alen[__ldg(&P.pf_order[(it < nitems ? it : 0) >> 1])] > 32);
        if (CLS > 0 && wide) prefilter_round<unsigned long long>(P, head, tail, hw, base, nitems, bits);
        else prefilter_round<uint32_t>(P, head, tail, hw, base, nitems, bits);
    }
    __syncwarp();
}

// first s in [s_lo, s_hi) whose w-wide quality window sum reaches `need`; s_hi if none (filter.cpp:171-181)
__device__ int first_good_window_fwd(const uint8_t* qual, int s_lo, int s_hi, int w, int need) {
    const int lane = lane_id();
    for (int s0 = s_lo; s0 < s_hi; s0 += 32) {
        int s = s0 + lane;
        int sum = 0;
        if (s < s_hi)
            for (int j = 0; j < w; j++) sum += sc(qual[s + j]);
        unsigned m = __ballot_sync(0xffffffffu, s < s_hi && sum >= need);
        if (m) return s0 + __ffs(m) - 1;
    }
    return s_hi;
}
// largest t in (t_lo, t_hi] whose window qual[t-w+1..t] reaches `need`; t_lo if none (filter.cpp:203-212)
__device__ int first_good_window_bwd(const uint8_t* qual, int t_hi, int t_lo, int w, int need) {
    const int lane = lane_id();
    for (int t0 = t_hi; t0 > t_lo; t0 -= 32) {
        int t = t0 - lane;
        int sum = 0;
        if (t > t_lo)
            for (int j = 0; j < w; j++) sum += sc(qual[t - j]);
        unsigned m = __ballot_sync(0xffffffffu, t > t_lo && sum >= need);
        if (m) return t0 - (__ffs(m) - 1);
    }
    return t_lo;
}

// Filter::trimAndCut: returns false if the read is dropped (NULL)
__device__ bool trim_and_cut(const DevParams& P, const uint8_t* seq, const uint8_t* qual, int l, Win& w) {
    const fpl_options& o = P.opt;
    const int lane = lane_id();
    int front = o.trim_front, tail = o.trim_tail;
    const bool cf = o.cut_front_enabled, ct = o.cut_tail_enabled;
    w.lo = 0; w.len = l;
    if (front == 0 && tail == 0 && !cf && !ct) return true;
    int rlen = l - front - tail;
    if (rlen < 0) return false;
    if (front == 0 && !cf && !ct) { resize_(w, rlen); return true; }
    if (!cf && !ct) { w.lo = front; w.len = rlen; return true; }
    if (cf) {
        const int ws = o.cut_front_window;
        if (l - front - tail - ws <= 0) return false;
        int s = first_good_window_fwd(qual, front, l - tail - ws, ws, (33 + o.cut_front_quality) * ws);
        if (s > 0) s = s + ws - 1;
        // while (s < l && seq[s] == 'N') s++
        while (true) {
            int i = s + lane;
            unsigned m = __ballot_sync(0xffffffffu, !(i < l && seq[i] == 'N'));
            if (m) { s += __ffs(m) - 1; break; }
            s += 32;
        }
        front = s;
        rlen = l - front - tail;
    }
    if (ct) {
        const int ws = o.cut_tail_window;
        if (l - front - tail - ws <= 0) return false;
        int t = first_good_window_bwd(qual, l - tail - 1, front + ws - 1, ws, (33 + o.cut_tail_quality) * ws);
        if (t < l - 1) t = t - ws + 1;
        // while (t >= 0 && seq[t] == 'N') t--
        while (true) {
            int i = t - lane;
            unsigned m = __ballot_sync(0xffffffffu, !(i >= 0 && seq[i] == 'N'));
            if (m) { t -= __ffs(m) - 1; break; }
            t -= 32;
        }
        rlen = t - front + 1;
    }
    if (rlen <= 0 || front >= l - 1) return false;
    w.lo = front; w.len = rlen;
    return true;
}

// PolyX::trimPolyX closed form (SURVEY A.11): suffix counts by warp scan, first position where the stop rule fires.
__device__ void trim_polyx(const DevParams& P, const uint8_t* data, Win& w, fpl_read_result* out,
                           unsigned long long* counters) {
    const int lane = lane_id();
    const int rlen = w.len;
    const int compareReq = P.opt.polyx_min_len;
    int cA = 0, cT = 0, cC = 0, cG = 0;
    int pos = rlen;
    int nA = 0, nT = 0, nC = 0, nG = 0;
    bool found = false;
    for (int p0 = 0; p0 < rlen && !found; p0 += 32) {
        int p = p0 + lane;
        bool valid = p < rlen;
        uint8_t ch = valid ? data[rlen - p - 1] : 0;
        int a = (ch == 'A') | (ch == 'N'), t = (ch == 'T') | (ch == 'N');
        int c = (ch == 'C') | (ch == 'N'), g = (ch == 'G') | (ch == 'N');
        a = warp_incl_scan(a) + cA; t = warp_incl_scan(t) + cT;
        c = warp_incl_scan(c) + cC; g = warp_incl_scan(g) + cG;
        int cmp = p + 1;
        int allowed = min(5, cmp / 8);
        bool stop = valid && (cmp - a > allowed) && (cmp - t > allowed) && (cmp - c > allowed) && (cmp - g > allowed) &&
                    (p >= 8 || p + 1 >= compareReq - 1);
        unsigned m = __ballot_sync(0xffffffffu, stop);
        int src = m ? __ffs(m) - 1 : 31;
        nA = __shfl_sync(0xffffffffu, a, src); nT = __shfl_sync(0xffffffffu, t, src);
        nC = __shfl_sync(0xffffffffu, c, src); nG = __shfl_sync(0xffffffffu, g, src);
        if (m) { pos = p0 + src; found = true; }
        else { cA = nA; cT = nT; cC = nC; cG = nG; }
    }
    if (!found) { nA = cA; nT = cT; nC = cC; nG = cG; pos = rlen; }
    if (pos + 1 >= compareReq) {
        int poly = 0, mx = nA;
        if (nT > mx) { mx = nT; poly = 1; }
        if (nC > mx) { mx = nC; poly = 2; }
        if (nG > mx) { mx = nG; poly = 3; }
        const uint8_t polyBase = poly == 0 ? 'A' : poly == 1 ? 'T' : poly == 2 ? 'C' : 'G';
        // back off to the last matching base: first j >= max(0, rlen-pos-1) with data[j] == polyBase
        int j = max(0, rlen - pos - 1);
        int hit = -1;
        for (; j < rlen; j += 32) {
            int i = j + lane;
            unsigned m = __ballot_sync(0xffffffffu, i < rlen && data[i] == polyBase);
            if (m) { hit = j + __ffs(m) - 1; break; }
        }
        int newpos = hit >= 0 ? rlen - hit - 1 : -1;
        resize_(w, rlen - newpos - 1);
        if (lane == 0) {
            out->flags |= FPL_FLAG_POLYX;
            out->polyx_base = (uint8_t)poly;
            out->polyx_len = newpos + 1;
            atomicAdd(&counters[FPL_CNT_POLYX_READS + poly], 1ull);
            atomicAdd(&counters[FPL_CNT_POLYX_BASES + poly], (unsigned long long)(long long)(newpos + 1));
        }
    }
}

}  // namespace

#define TRIM_WARPS 4

// The end-local stages for -s / -e: trimAndCut, trimPolyX, trimBySequenceStart(-s), trimBySequenceEnd(-e).
template <int CLS>
__global__ void __launch_bounds__(TRIM_WARPS * 32)
k_trim(const __grid_constant__ DevParams P, DevBatch b, ReadState* __restrict__ st, fpl_read_result* __restrict__ res,
       unsigned long long* __restrict__ counters) {
    __shared__ __align__(16) uint8_t scratch_all[TRIM_WARPS][208];   // probe candidates / packed window (36 words)
    const int wid = threadIdx.x >> 5, lane = lane_id();
    const int64_t r = (int64_t)blockIdx.x * TRIM_WARPS + wid;
    if (r >= b.n_reads) return;
    uint8_t* scratch = scratch_all[wid];
    const int64_t off = b.offsets[r];
    const int L = b.lens[r];
    const uint8_t* seq = b.seq + off;
    const uint8_t* qual = b.qual + off;
    fpl_read_result* out = &res[r];
    if (lane == 0) {
        // zero the record; later kernels fill segments / medians
        uint4* o4 = reinterpret_cast<uint4*>(out);
        o4[0] = make_uint4(0, 0, 0, 0); o4[1] = o4[0]; o4[2] = o4[0]; o4[3] = o4[0];
    }
    __syncwarp();
    Win w;
    bool alive = trim_and_cut(P, seq, qual, L, w);
    if (alive && P.opt.polyx_enabled) trim_polyx(P, seq + w.lo, w, out, counters);
    int trimmed = 0;
    EventSink ev{out, counters + FPL_CNT_FIXED, 0};
    if (alive && P.opt.adapter_enabled) {
        if (P.alen[0] > 0) trimmed += trim_start<CLS>(P, seq, w, 0, ev, scratch);
        if (P.alen[1] > 0) trimmed += trim_end<CLS>(P, seq, w, 1, ev, scratch);
    }
    if (lane == 0) {
        ReadState s;
        s.lo = w.lo; s.len = w.len; s.alive = alive ? 1u : 0u; s.pad = 0;
        s.best[0] = ~0ull; s.best[1] = ~0ull;
        s.lowq = s.nn = s.totalq = s.diff = 0;
        // k_scan_jit with the quality histograms takes the read's length and where to add them from here (its
        // arguments are the adapters' scan's)
        s.reserved[0] = 0; s.reserved[1] = L;
        s.reserved[2] = (int32_t)(uint32_t)reinterpret_cast<uintptr_t>(P.qstripes);
        s.reserved[3] = (int32_t)(uint32_t)(reinterpret_cast<uintptr_t>(P.qstripes) >> 32);
        st[r] = s;
        if (!alive) out->flags |= FPL_FLAG_DROPPED_BY_CUT;
        else { out->trim_lo = w.lo; out->trim_len = w.len; }
        out->n_events = (uint16_t)ev.n;
        out->adapter_trimmed_bases = trimmed;
    }
}

// trimByMultiSequences (src/adaptertrimmer.cpp:42-57): the FASTA adapters in order, each on the read as the previous
// ones left it — a kernel of its own (launched only with --adapter_fasta) so that its 64-bit pre-filter does not set the
// register budget of the two-adapter path above.  Continues from the window, the event count and the trimmed-base count
// k_trim left in the read's state and record.
template <int CLS>
__global__ void __launch_bounds__(TRIM_WARPS * 32)
k_trim_fasta(const __grid_constant__ DevParams P, DevBatch b, ReadState* __restrict__ st, fpl_read_result* __restrict__ res,
             unsigned long long* __restrict__ counters) {
    __shared__ __align__(16) uint8_t scratch_all[TRIM_WARPS][208];
    __shared__ __align__(16) uint8_t pf_win[TRIM_WARPS][2][PF_WIN + 8];     // many-adapter pre-filter: end windows ...
    __shared__ uint32_t pf_bits[TRIM_WARPS][2 * PF_WORDS];   // ... and its maybe-bits: [window stage | probe stage]
    const int wid = threadIdx.x >> 5, lane = lane_id();
    const int64_t r = (int64_t)blockIdx.x * TRIM_WARPS + wid;
    if (r >= b.n_reads) return;
    if (!st[r].alive) return;
    uint8_t* scratch = scratch_all[wid];
    const uint8_t* seq = b.seq + b.offsets[r];
    fpl_read_result* out = &res[r];
    Win w;
    w.lo = st[r].lo; w.len = st[r].len;
    int trimmed = out->adapter_trimmed_bases;
    EventSink ev{out, counters + FPL_CNT_FIXED, (int)out->n_events};
    __syncwarp();
    // pairs the pre-filter rules out are skipped, and a trim (which moves the end windows) re-filters what is still to come
    uint32_t* bits = pf_bits[wid];
    const bool use_pf = P.n_adapters > 4 && w.len >= FPL_PATTERN_LEN;
    if (use_pf) prefilter<CLS>(P, seq, w, pf_win[wid][0], pf_win[wid][1], bits);
    for (int k = 2; k < P.n_adapters; k++) {
        const int i0 = 2 * (k - 2), i1 = i0 + 1;
        const bool f0 = !use_pf || (bits[i0 >> 5] >> (i0 & 31) & 1u), q0 = !use_pf || (bits[PF_WORDS + (i0 >> 5)] >> (i0 & 31) & 1u);
        if (f0 || q0) {
            const int t = trim_start<CLS>(P, seq, w, k, ev, scratch, f0, q0);
            trimmed += t;
            if (t && use_pf) prefilter<CLS>(P, seq, w, pf_win[wid][0], pf_win[wid][1], bits);
        }
        const bool f1 = !use_pf || (bits[i1 >> 5] >> (i1 & 31) & 1u), q1 = !use_pf || (bits[PF_WORDS + (i1 >> 5)] >> (i1 & 31) & 1u);
        if (f1 || q1) {
            const int t = trim_end<CLS>(P, seq, w, k, ev, scratch, f1, q1);
            trimmed += t;
            if (t && use_pf && k + 1 < P.n_adapters) prefilter<CLS>(P, seq, w, pf_win[wid][0], pf_win[wid][1], bits);
        }
    }
    __syncwarp();
    if (lane == 0) {
        st[r].lo = w.lo; st[r].len = w.len;
        out->trim_lo = w.lo; out->trim_len = w.len;
        out->n_events = (uint16_t)ev.n;
        out->adapter_trimmed_bases = trimmed;
    }
}

void launch_trim(const DevParams& P, const DevBatch& b, ReadState* st, fpl_read_result* res,
                 unsigned long long* counters, cudaStream_t stream) {
    if (b.n_reads == 0) return;
    unsigned grid = (unsigned)((b.n_reads + TRIM_WARPS - 1) / TRIM_WARPS);
    if (P.small_adapters == 0) k_trim<0><<<grid, TRIM_WARPS * 32, 0, stream>>>(P, b, st, res, counters);
    else if (P.small_adapters == 1) k_trim<1><<<grid, TRIM_WARPS * 32, 0, stream>>>(P, b, st, res, counters);
    else k_trim<2><<<grid, TRIM_WARPS * 32, 0, stream>>>(P, b, st, res, counters);
    if (P.opt.adapter_enabled && P.n_adapters > 2) {
        if (P.fasta_class == 0) k_trim_fasta<0><<<grid, TRIM_WARPS * 32, 0, stream>>>(P, b, st, res, counters);
        else if (P.fasta_class == 1) k_trim_fasta<1><<<grid, TRIM_WARPS * 32, 0, stream>>>(P, b, st, res, counters);
        else k_trim_fasta<2><<<grid, TRIM_WARPS * 32, 0, stream>>>(P, b, st, res, counters);
    }
}
