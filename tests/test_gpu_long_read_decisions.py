"""Long reads of every segment-decision shape on k_read_qual's block-wide path.  k_final decides each read's segments
(adapter verification, split, filter); k_read_qual reads them back from the records to build the post-filter quality
histograms.  A read longer than RQ_LONG goes on its block's list and the whole block streams it after the block barrier;
past RQ_LIST such reads the warp that meets it streams it alone.  These batches put long reads of every decision shape on
those paths, next to reads that trimAndCut drops, and compare records, both Stats blocks and the counters with the oracle:
  - split reads whose two parts both pass, whose gap is the largest part, whose only segment is the right part (slot 0 is
    the right side), and whose left part fails the filter;
  - long and short reads dropped by the quality cut in the same block as the long list;
  - the same batch under --mask/--break, where k_read_qual counts the pre-filter Stats only.
k_read_qual makes the post-filter histograms where k_scan_jit does not count them: the cases run with FPL_NO_JIT=1
(k_scan_fast) for that, and on the default scan too, where k_read_qual_exc treats the same reads from k_final's list (in
the list's order: the placement below means nothing there).  Every case asserts which of the two ran.

Runs on the GPU and, with FPL_EMULATE=1, on the emulated library (tests/test_capacity_shrunk_long_reads.py runs the same
cases on the shrunk build)."""
import numpy as np
import pytest

import capacity
import cases
from fastplong_b200 import Options, abi, pack_reads

pytestmark = pytest.mark.gpu

S, E = capacity.S, capacity.E
OPT = Options(start_adapter=S, end_adapter=E, cut_front=True, cut_tail=True, length_required=1)
EXT_OPT = cases.MASK_BREAK_SETS["mask_and_break"]
KINDS = ("split", "gap_largest", "seg0_right", "left_fails", "dead", "plain")
END = capacity.END


def long_decision_batch(k, seed):
    """RQ_LIST + 1 long reads at the indices block 0 of k_read_qual visits (the last one goes to a lone warp) and len(KINDS)
    at block 1's, cycling through KINDS; every other read short: dropped by the cut, empty, or one base"""
    rng = np.random.default_rng(seed)
    at = capacity.rq_indices(k, 0, k["RQ_LIST"] + 1) + capacity.rq_indices(k, 1, len(KINDS))
    n = max(at) + 1 + 5
    short = min(120, k["RQ_LONG"])
    reads = []
    for i in range(n):
        if i % 3 == 0:
            reads.append((capacity._bases(rng, short), capacity._q(short, 0)))
        else:
            reads.append(((b"", b""), (b"A", b"5"))[i % 3 - 1])
    for j, i in enumerate(at):
        L = max(k["RQ_LONG"] + 1, 4 * END) + 37 * j
        reads[i] = capacity.decided_read(rng, KINDS[j % len(KINDS)], L)
    return pack_reads(reads), at


def check_shapes(batch, at, res):
    """the long reads reach every decision shape (on the oracle's records)"""
    long_ = [i for i in at if batch.lens[i] > 0]
    r = res[long_]
    nseg, flags = r["n_segments"], r["flags"]
    assert ((flags & abi.FLAG_MIDDLE_ADAPTER) != 0).sum() >= 4
    assert ((flags & abi.FLAG_SEG0_IS_RIGHT) != 0).any()
    assert ((flags & abi.FLAG_DROPPED_BY_CUT) != 0).any()
    two = r[nseg == 2]
    gap = two["seg_lo"][:, 1] - (two["seg_lo"][:, 0] + two["seg_len"][:, 0])
    assert (gap > two["seg_len"].max(axis=1)).any()
    assert ((two["seg_result"][:, 0] != abi.PASS_FILTER) & (two["seg_result"][:, 1] == abi.PASS_FILTER)).any()


def run_cases(make_engine, scans, k, what):
    """make_engine(opt, scan); scans: {scan: the quality pass OPT takes with it}"""
    batch, at = long_decision_batch(k, 11)
    for scan, qual_pass in scans.items():
        res = capacity.compare_with_oracle(make_engine(OPT, scan), OPT, batch, f"{what}/decisions/{scan}", qual_pass=qual_pass)
        check_shapes(batch, at, res)
        # short reads dropped by the cut share block 0 with the long list
        dropped = np.flatnonzero(res["flags"] & abi.FLAG_DROPPED_BY_CUT)
        assert (dropped < k["RQ_WARPS"]).any() and (batch.lens[dropped] <= k["RQ_LONG"]).any()
        capacity.compare_with_oracle(make_engine(EXT_OPT, scan), EXT_OPT, batch, f"{what}/mask_break/{scan}", qual_pass="read_qual")


def test_long_read_decisions():
    from test_gpu_capacity import SCANS, engine
    run_cases(engine, {scan: qual_pass for scan, (_, qual_pass) in SCANS.items()}, capacity.constants(), "gpu")
