"""The fused k_cycle_stats pass: the pre-filter pass over whole reads also counts each read's slot-0 passing segment
[s, e) into the post-filter per-cycle counters when s < CS_REACH; the residual pass counts the other passing segments
(slot 1 of a split read, starts at or beyond the reach).  Everything is compared with the oracle: records, both Stats
blocks (per-cycle counters and 5-mers), counters.

Covered: post starts s = 0, 1, 15, 16, 17, CS_REACH - 1 and CS_REACH; segments ending inside tile 0, in the tile that
holds s, exactly on a tile boundary and one byte past it; split reads; reads that fail or lose their segment to the quality
cut; batches past CS_STAGE and CS_GROUP at the largest count of the packed counter and of both 16-bit halves of the 5-mer
tables (poly-A: the low half, poly-C: both).

Runs on the GPU and, with FPL_EMULATE=1, on the emulated library (tests/test_capacity_shrunk_fused.py runs the same
cases on the shrunk builds)."""
import os
import re

import numpy as np
import pytest

import capacity
from fastplong_b200 import Options, pack_reads, synth

pytestmark = pytest.mark.gpu

K = capacity.constants()


def reach():
    """CS_REACH as fpl_stats.cu defines it: 16 * CS_PROWW - CS_TILE - 16"""
    text = open(os.path.join(capacity.CSRC, "fpl_stats.cu")).read()
    assert re.search(r"^#define CS_REACH \(16 \* CS_PROWW - CS_TILE - 16\)", text, re.M)
    return 16 * int(re.search(r"^#define CS_PROWW (\d+)", text, re.M).group(1)) - K["CS_TILE"] - 16


def engine(opt):
    from fastplong_b200.binding import Engine
    return Engine(opt)


STARTS = sorted({0, 1, 15, 16, 17, reach() - 1, reach()})


def trim_opt(s, tail=2):
    return Options(disable_adapter_trimming=True, disable_quality_filtering=True, length_required=1, trim_front=s,
                   trim_tail=tail)


def start_batch(s, seed):
    """reads whose segment [s, L - 2) ends inside tile 0, in the tile holding s, on a tile boundary and one past it, far
    behind; too short for a segment; with N bases and every quality byte"""
    rng = np.random.default_rng(seed)
    T = K["CS_TILE"]
    ends = {s + 1, s + 7, (s // T + 1) * T - 1, T, T + 1, 2 * T, 2 * T + 1, 3 * T - 5, s + T + 3, 4 * T + 77}
    lens = sorted({e + 2 for e in ends if e > s} | {0, 1, s, s + 2})
    reads = []
    for L in lens:
        for rep in range(3):
            seq = bytearray(capacity._bases(rng, L))
            if rep == 1 and L:
                seq[int(rng.integers(0, L))] = ord("N")
            qual = (rng.integers(0, 94, size=L).astype(np.uint8) + 33).tobytes()
            reads.append((bytes(seq), qual))
    return pack_reads(capacity._shuffled(rng, reads))


@pytest.mark.parametrize("s", STARTS)
def test_post_start(s):
    opt = trim_opt(s)
    capacity.compare_with_oracle(engine(opt), opt, start_batch(s, 100 + s), f"start{s}")


def test_split_reads_and_quality_cut():
    """split reads (slot 1 goes to the residual pass) next to single segments; heads cut by the quality window at
    lengths on both sides of the reach; reads the cut or the filters fail"""
    rng = np.random.default_rng(7)
    r = reach()
    reads = [capacity.split_read(rng, 241 + 13 * i, 321 + 11 * i) for i in range(12)]
    for i, head in enumerate([0, 1, 16, 17, r - 30, r - 1, r, r + 40, 900]):
        L = head + 300 + 37 * i
        q = capacity._q(head, 3) + capacity._quals(rng, L - head, 25, 60)
        reads.append((capacity._bases(rng, L), q))
    reads += [(capacity._bases(rng, 700), capacity._q(700, 2)) for _ in range(3)]          # cut away entirely
    reads += [(capacity._bases(rng, 40), capacity._quals(rng, 40)) for _ in range(20)]
    batch = pack_reads(capacity._shuffled(rng, reads))
    opt = Options(start_adapter=synth.ADAPTER_START, end_adapter=synth.ADAPTER_END, cut_front=True, cut_tail=True,
                  cut_window_size=4, cut_mean_quality=20, length_required=30)
    exp = capacity.compare_with_oracle(engine(opt), opt, batch, "split+cut")
    assert (exp["n_segments"] == 2).sum() >= 10


HEADROOM_OPT = Options(disable_adapter_trimming=True, disable_quality_filtering=True, length_required=0, trim_front=17)


def headroom_batch(k, base):
    """2 * CS_GROUP + 1 equal homopolymer reads of 300 bases at quality byte 127, segment starting at 17: every post column
    of group 0 holds count CS_GROUP and sum(q) = 127 * CS_GROUP; every lane's 5-mer word 16 * CS_GROUP in its low half
    (poly-A) or in both halves (poly-C)"""
    L, n = 300, 2 * k["CS_GROUP"] + 1
    return pack_reads([(base.encode() * L, b"\x7f" * L)] * n)


def post_list_batch(k, count):
    """`count` reads with segments starting at 5, ending on both sides of the second tile"""
    rng = np.random.default_rng(count)
    far, near = capacity._reach(k)
    return pack_reads([(capacity._bases(rng, L), capacity._quals(rng, L)) for L in
                       [far + 7 + int(rng.integers(0, 60)) if i % 2 else near + 7 for i in range(count)]])


@pytest.mark.parametrize("base", ["A", "C"])
def test_headroom_past_group(base):
    batch = headroom_batch(K, base)
    if os.environ.get("FPL_EMULATE", "") not in ("", "0") and batch.n_reads > 10000:
        pytest.skip("too slow for the emulator")
    capacity.compare_with_oracle(engine(HEADROOM_OPT), HEADROOM_OPT, batch, f"headroom/{base}")


@pytest.mark.parametrize("count", capacity.cycle_counts(K))
def test_post_list_past_stage_and_group(count):
    if os.environ.get("FPL_EMULATE", "") not in ("", "0") and count > 10000:
        pytest.skip("too slow for the emulator")
    opt = trim_opt(5)
    capacity.compare_with_oracle(engine(opt), opt, post_list_batch(K, count), f"post_list{count}")
