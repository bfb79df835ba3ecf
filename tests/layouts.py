"""Other layouts of the same reads: what include/fplgpu.h (fpl_batch) allows beyond pack_reads' 128-byte slots with zero
padding.  relayout() copies every read of a batch into a new pair of buffers — slots on any multiple of 16, in any memory
order, with free space between them and behind the last one — and fills every byte that does not belong to a read with
"poison".  The kernels must ignore those bytes, so a relaid batch has to give exactly what the canonical batch gives."""
import numpy as np

from fastplong_b200 import PackedBatch

POISONS = ("zero", "acgt", "adapter", "n_runs", "high", "u_lower", "stale")


def _fill(kind, n, rng, adapters, stale, where):
    """-> (seq bytes, qual bytes) for n poisoned bytes that start at buffer offset `where`"""
    if kind == "zero":
        return np.zeros(n, np.uint8), np.zeros(n, np.uint8)
    if kind == "acgt":                   # plausible bases of the highest quality
        return np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, n)], np.full(n, ord("I"), np.uint8)
    if kind == "n_runs":                 # N with quality 2: counts as N and as a low-quality base if it leaks
        return np.full(n, ord("N"), np.uint8), np.full(n, 33 + 2, np.uint8)
    if kind == "high":                   # bytes 0x80..0xFF: an index past any 128-entry table
        return rng.integers(0x80, 0x100, n).astype(np.uint8), rng.integers(0x80, 0x100, n).astype(np.uint8)
    if kind == "u_lower":                # U (a base of its own in Stats) and lower-case letters
        return np.frombuffer(b"UuacgtnU", np.uint8)[rng.integers(0, 8, n)], np.full(n, ord("I"), np.uint8)
    if kind == "stale":                  # the bytes of another batch at the same buffer positions, wrapped around
        idx = (where + np.arange(n)) % stale.n_bytes
        return stale.seq[idx].copy(), stale.qual[idx].copy()
    if kind == "adapter":
        # the option set's adapters running on from the end of the read in front and ending right at the start of the
        # next read, at quality 'I': a kernel that lets one leaked byte into a match window finds a better match
        a = adapters[int(rng.integers(len(adapters)))].encode() if adapters else b"ACGT"
        h = n // 2
        fwd = (a * (h // len(a) + 1))[:h]
        back = (a * ((n - h) // len(a) + 1))
        back = back[len(back) - (n - h):] if n - h else b""
        return np.frombuffer(fwd + back, np.uint8).copy(), np.full(n, ord("I"), np.uint8)
    raise ValueError(kind)


def relayout(batch, *, align=16, order="identity", gaps=0, poison="zero", tail=0, seed=0, adapters=(), stale=None):
    """The reads of `batch` in a new layout.
      align    every slot starts on a multiple of this (a multiple of 16)
      order    memory order of the slots: "identity", "reversed" or "shuffled" (read i keeps index i)
      gaps     up to this many free 16-byte units in front of each slot, drawn at random (0: slots touch)
      poison   what every byte outside the reads holds (POISONS); "adapter" uses `adapters`, "stale" the bytes of `stale`
      tail     poisoned bytes behind the end of the last read (n_bytes includes them)"""
    assert align % 16 == 0 and poison in POISONS
    rng = np.random.default_rng(seed)
    n = batch.n_reads
    lens = batch.lens.astype(np.int64)
    mem = {"identity": np.arange(n), "reversed": np.arange(n)[::-1], "shuffled": rng.permutation(n)}[order]
    offsets = np.zeros(n, np.int64)
    cur = 0
    for i in mem:
        cur += 16 * int(rng.integers(0, gaps + 1)) if gaps else 0
        cur = -(-cur // align) * align
        offsets[i] = cur
        cur += int(lens[i])
    total = cur + tail
    seq = np.empty(total, np.uint8)
    qual = np.empty(total, np.uint8)
    owned = np.zeros(total, bool)
    for i in range(n):
        o, L, s = int(offsets[i]), int(lens[i]), int(batch.offsets[i])
        seq[o:o + L] = batch.seq[s:s + L]
        qual[o:o + L] = batch.qual[s:s + L]
        owned[o:o + L] = True
    # every maximal run of bytes no read owns gets its own fill
    edges = np.flatnonzero(np.diff(np.concatenate([[True], owned, [True]])))
    for a, b in zip(edges[0::2], edges[1::2]):
        seq[a:b], qual[a:b] = _fill(poison, int(b - a), rng, list(adapters), stale, int(a))
    return PackedBatch(seq, qual, offsets, batch.lens.astype(np.int32).copy())


def adapters_of(opt):
    """The adapter strings an option set searches for (what "adapter" poison plants)."""
    out = [a for a in (opt.start_adapter, opt.end_adapter) if a and a != "auto"]
    return out + list(opt.adapter_fasta or ())


def end_of_reads(batch):
    """One past the last byte any read owns (0 for no reads)."""
    return int((batch.offsets + batch.lens).max()) if batch.n_reads else 0


def every_vector_end_batch(seed):
    """Reads of 1..40 bases and of every length = 0, 1, 15, 16, 17, 31, 32, 33 (mod 32) up to about 600: at 16-byte slots the
    read ends fall on every position of a 16- and a 32-byte vector, and a read's last vector holds the next read's first bytes."""
    from fastplong_b200 import pack_reads, synth
    rng = np.random.default_rng(seed)
    lens = list(range(1, 41)) + [32 * k + r for k in range(1, 19) for r in (0, 1, 15, 16, 17, 31, 32, 33)]
    reads = []
    for L in lens:
        s = bytearray(synth.BASES[rng.integers(0, 4, L)].tobytes())
        if L > 60 and rng.random() < 0.5:             # adapters at the ends so that the scans have something to find
            a = synth.ADAPTER_START.encode()
            s[:len(a)] = a
        if L > 60 and rng.random() < 0.4:
            e = synth.ADAPTER_END.encode()[: int(rng.integers(6, 31))]
            s[L - len(e):] = e
        if rng.random() < 0.2:
            s[int(rng.integers(0, L))] = ord("N")
        q = (np.rint(rng.normal(22, 9, L)).clip(1, 45).astype(np.uint8) + 33).tobytes()
        reads.append((bytes(s), q))
    order = rng.permutation(len(reads))
    return pack_reads([reads[i] for i in order])
