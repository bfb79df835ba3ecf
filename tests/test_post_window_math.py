"""The index arithmetic of the fused k_cycle_stats pass (fastplong_b200/csrc/fpl_stats.cu), checked on the CPU: the post-filter
window (count1ff / count_post_masked: immediate 4*((m & 15)*CS_PROWW + (m >> 4)), m = J + T, on top of the post lane base
4*(lane + (CS_REACH - s) >> 4)) is injective per bin, free of bank conflicts for every post start s < CS_REACH, every
segment misalignment and every bin mix, and its flush maps every word back to the post-filter cycle p - s of the byte; the
dp4a weight of the post bin stride fits a byte; the split 16-bit 5-mer words give back both codes."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = open(os.path.join(ROOT, "fastplong_b200", "csrc", "fpl_stats.cu")).read()


def define(name):
    m = re.search(r"#define\s+%s\s+(.+?)\s*(//.*)?$" % name, SRC, re.M)
    assert m, name
    return m.group(1)


TILE = int(define("CS_TILE"))
PROWW = int(define("CS_PROWW"))
PBINW = eval(define("CS_PBINW").replace("CS_PROWW", str(PROWW)))
REACH = eval(define("CS_REACH").replace("CS_PROWW", str(PROWW)).replace("CS_TILE", str(TILE)))


def post_word(lane, j, sh, s):
    """the word of byte j of `lane`'s vector for a segment at address & 15 == sh whose post part starts s into the read"""
    d = REACH - s
    t = (15 - sh) + (d & 15)
    m = j + t
    return (m & 15) * PROWW + (m >> 4) + lane + (d >> 4)


def test_constants():
    assert PBINW % 32 == 0 and PBINW * 4 // 16 <= 255 and PBINW * 4 % 16 == 0
    assert 16 * PROWW >= TILE + 15 + REACH and REACH % 16 == 0 and REACH > 0


def test_mapping_is_injective_and_flush_inverts_it():
    t0 = 3 * TILE                                   # any tile: the flush is relative to t0
    for sh in range(16):
        for s in range(REACH):
            seen = {}
            for lane in range(32):
                for j in range(16):
                    w = post_word(lane, j, sh, s)
                    assert 0 <= w < PBINW, (sh, s, lane, j)
                    pre_cycle = t0 + 16 * lane + j - sh
                    assert seen.setdefault(w, pre_cycle) == pre_cycle
                    # the flush: word p -> post cycle t0 - 15 - CS_REACH + 16*(p % PROWW) + p // PROWW
                    assert t0 - 15 - REACH + 16 * (w % PROWW) + w // PROWW == pre_cycle - s


def test_no_bank_conflicts_for_any_start_misalignment_or_bin_mix():
    for sh in (0, 1, 7, 15):
        for s in range(REACH):
            for j in range(16):
                for bins in ([0] * 32, list(range(8)) * 4, [7, 0] * 16, [3, 5, 1, 6] * 8):
                    banks = {(b * PBINW + post_word(lane, j, sh, s)) % 32 for lane, b in enumerate(bins)}
                    assert len(banks) == 32, (sh, s, j)


def test_split_kmer_words_give_back_both_codes():
    """word [code >> 1][lane]: the low half counts codes 2w and 2w + 1, the high half code 2w + 1 (bit 1 of the newest
    base's byte); at 16 * CS_GROUP 5-mers per lane the low half does not carry into the high one"""
    group = int(define("CS_GROUP"))
    assert 16 * group <= 0xFFFF
    for ch, low_bit in {"A": 0, "C": 1, "T": 0, "U": 0, "G": 1}.items():     # c' = (byte >> 1) & 3: A 0, C 1, T/U 2, G 3
        assert (ord(ch) >> 1) & 1 == ((ord(ch) >> 1) & 3) & 1 == low_bit
    for n_even, n_odd in ((0, 0), (5, 3), (16 * group, 0), (0, 16 * group), (16 * group - 7, 7)):
        v = n_even * 1 + n_odd * 0x10001
        assert v < 1 << 32
        assert (v >> 16, (v & 0xFFFF) - (v >> 16)) == (n_odd, n_even)
