"""The batch-layout contract of include/fplgpu.h (fpl_batch): the same reads laid out in any way the ABI allows — slots on any
multiple of 16 down to 16-byte slots whose last vector holds the next read's first bytes, any memory order, gaps, poisoned bytes
between and behind the slots, a piecewise upload, a device batch with only FPL_TAIL_PAD behind its last vector, one submission split
into several calls — give the records, both Stats blocks, the counters and the -N/-b lists the oracle gives on the canonical
pack_reads layout.  The oracle reads only the reads' own bytes, so it is the reference for every layout (tests/layouts.py).
Runs on the GPU and, with FPL_EMULATE=1, on the emulated library."""
import os

import numpy as np
import pytest

import cases
import layouts
from fastplong_b200 import PackedBatch, abi, pack_reads, synth
from fastplong_b200.abi import RESULT_DTYPE
from oracle_lib import OracleEngine, compare_lists, compare_results, compare_stats

pytestmark = pytest.mark.gpu

EMULATE = os.environ.get("FPL_EMULATE", "") not in ("", "0")

# one option set per kernel variant that reads the batch: (options, environment of fpl_create, batch of its own or None)
SETS = {
    "default_se": (cases.OPTION_SETS["default_se"], {}, None),                     # k_scan_jit
    "cut_polyx_cplx": (cases.OPTION_SETS["cut_polyx_cplx"], {}, None),             # k_scan_jit with complexity
    "fasta5": (cases.OPTION_SETS["fasta5"], {}, None),                             # k_trim_fasta
    "fasta64_polyx": (cases.OPTION_SETS["fasta64_polyx"], {}, None),
    "literal_auto": (cases.OPTION_SETS["literal_auto"], {}, None),                 # generic k_scan
    "long_adapter_129": (cases.OPTION_SETS["long_adapter_129"], {}, None),         # generic k_scan, myers_long
    "long_adapter_64_no_jit": (cases.OPTION_SETS["long_adapter_64"], {"FPL_NO_JIT": "1"}, None),   # k_scan_fast
    "mask_and_break": (cases.MASK_BREAK_SETS["mask_and_break"], {}, None),         # fpl_ext_run and the masked copy
    "mask_cplx": (cases.MASK_BREAK_SETS["mask_cplx"], {}, None),
    "trims_limits": (cases.OPTION_SETS["trims_limits"], {}, None),
    "filter_ties": (cases.edge_cases()["filter_ties"][0], {}, cases.edge_cases()["filter_ties"][1]),
}
LAYOUTS = [(16, p) for p in layouts.POISONS] + [(48, "adapter"), (128, "high"), (4096, "stale")]    # (slot alignment, poison)
ORDERS = ("identity", "reversed", "shuffled")


def make_engine(opt, env, monkeypatch):
    from fastplong_b200.binding import Engine
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    try:
        return Engine(opt)
    finally:
        for k in env:
            monkeypatch.delenv(k)


def compare_all(g, o, opt, res, exp, cyc, what):
    compare_results(res, exp, what)
    if opt.mask or opt.break_reads:
        compare_lists(g.segments(), o.segments(), what + "/segments")
        compare_lists(g.mask_regions(), o.mask_regions(), what + "/regions")
    for w in (0, 1):
        compare_stats(g.stats(w, cyc), o.stats(w, cyc), f"{what}/stats{w}")
    compare_stats(g.counters(), o.counters(), what + "/counters")


def check_layout(name, canon, relaid, what, monkeypatch):
    """A fresh context on the relaid batch against a fresh oracle on the canonical one"""
    opt, env, _ = SETS[name]
    g, o = make_engine(opt, env, monkeypatch), OracleEngine(opt)
    try:
        compare_all(g, o, opt, g.process(relaid), o.process(canon), max(1, int(canon.lens.max())), what)
    finally:
        g.close()


def stale_source(seed):
    return cases.ont_batch(seed, n=80, mean=1500, p_chimera=0.2, p_polya=0.2)


@pytest.mark.parametrize("name", sorted(SETS))
def test_every_poison_between_the_slots(name, monkeypatch):
    """fpl_process_host on the adversarial reads (or the set's own batch): every kind of poison at 16-byte slots, where a read's
    last vector holds its neighbour's bytes, and the wider slots under some of them; identity, reversed and shuffled memory
    order, with and without gaps"""
    opt, _, own = SETS[name]
    canon = own if own is not None else cases.adversarial_batch(3)
    for k, (align, poison) in enumerate(LAYOUTS):
        order = ORDERS[k % 3]
        relaid = layouts.relayout(canon, align=align, order=order, gaps=3 if k % 2 else 0, poison=poison, tail=48, seed=k,
                                  adapters=layouts.adapters_of(opt), stale=stale_source(k))
        check_layout(name, canon, relaid, f"{name}/{poison}/align{align}/{order}", monkeypatch)


RAGGED_SETS = ("default_se", "cut_polyx_cplx", "fasta5", "literal_auto", "long_adapter_64_no_jit", "mask_and_break", "trims_limits")


@pytest.mark.parametrize("name", RAGGED_SETS)
@pytest.mark.parametrize("poison", ["adapter", "high", "n_runs"])
def test_read_ends_at_every_vector_position(name, poison, monkeypatch):
    """Reads of 1..40 bases and of every length = 0, 1, 15, 16, 17, 31, 32, 33 (mod 32), on touching 16-byte slots: every
    window, count and 5-mer mask at a read's end sees the next read's bytes in the same vector, and the last read ends at n_bytes"""
    opt = SETS[name][0]
    canon = layouts.every_vector_end_batch(7)
    relaid = layouts.relayout(canon, align=16, poison=poison, tail=0, seed=1, adapters=layouts.adapters_of(opt))
    check_layout(name, canon, relaid, f"{name}/vector-ends/{poison}", monkeypatch)


@pytest.mark.parametrize("poison,align", [("acgt", 16), ("high", 48), ("u_lower", 16)])
def test_split_read_complexity_ties(poison, align):
    """k_final recounts the ragged ends of the parts of a split read byte-wise: at 16-byte slots those ends sit next to poison"""
    from fastplong_b200.binding import Engine
    opt, canon = cases.edge_cases()["split_read_complexity_ties"]
    relaid = layouts.relayout(canon, align=align, order="shuffled", poison=poison, seed=3)
    g, o = Engine(opt), OracleEngine(opt)
    compare_all(g, o, opt, g.process(relaid), o.process(canon), int(canon.lens.max()), f"split-ties/{poison}")
    g.close()


@pytest.mark.parametrize("name", ["cut_polyx_cplx", "mask_and_break", "long_adapter_64_no_jit"])
def test_reads_longer_than_96_kb(name, monkeypatch):
    """The block-wide k_read_qual path and the long removed ranges of k_kmer_fix, at 16- and 4096-byte slots"""
    canon = synth.ont_like(4, 110000, 31, p_chimera=0.7, p_n=0.001)
    canon = pack_reads([canon.read(i) for i in range(canon.n_reads)] + [(b"ACGTN" * 7, b"I" * 35)])
    for align, poison in ((16, "high"), (4096, "acgt")):
        relaid = layouts.relayout(canon, align=align, order="reversed", poison=poison, seed=align)
        check_layout(name, canon, relaid, f"{name}/long/{align}", monkeypatch)


@pytest.mark.parametrize("piece_mb,order", [(None, "identity"), ("1", "identity"), ("1", "shuffled"), ("0", "identity")])
@pytest.mark.parametrize("name", ["cut_polyx_cplx", "mask_and_break"])
def test_piecewise_upload(name, piece_mb, order, monkeypatch):
    """fpl_process_host uploads in FPL_PIECE_MB pieces and starts a piece's kernels when it has arrived.  A ~6 MB batch at
    16-byte slots, after a batch of the same size on the same context: the bytes just past a piece and in the padding are the
    earlier batch's (on the device and in the host buffers alike).  A shuffled order takes the one-piece path."""
    opt, env, _ = SETS[name]
    env = dict(env, **({"FPL_PIECE_MB": piece_mb} if piece_mb is not None else {}))
    first = synth.ont_like(700, 8000, 41, p_chimera=0.05)
    canon = synth.ont_like(700, 8000, 42, p_chimera=0.1, p_polya=0.1)
    first_relaid = layouts.relayout(first, align=16, poison="acgt", tail=4096, seed=1)
    relaid = layouts.relayout(canon, align=16, order=order, gaps=1, poison="stale", tail=16, seed=2, stale=first_relaid)
    assert relaid.n_bytes > (5 << 20)
    g, o = make_engine(opt, env, monkeypatch), OracleEngine(opt)
    try:
        compare_results(g.process(first_relaid), o.process(first), name + "/first")
        launches = g.launch_count
        res = g.process(relaid)
        exp = o.process(canon)
        compare_all(g, o, opt, res, exp, int(max(first.lens.max(), canon.lens.max())), f"{name}/pieces{piece_mb}/{order}")
        per_call = g.launch_count - launches
    finally:
        g.close()
    g1 = make_engine(opt, dict(env, FPL_PIECE_MB="0"), monkeypatch)
    try:
        before = g1.launch_count
        g1.process(relaid)
        one_piece = g1.launch_count - before
    finally:
        g1.close()
    if piece_mb == "1" and order == "identity" and not (opt.mask or opt.break_reads):
        assert per_call > one_piece        # the kernels did run piece by piece
    else:
        assert per_call == one_piece


def device_buffers(batch, n_bytes, pad_poison=None):
    """seq, qual, offsets, lens on the device (torch CPU tensors under FPL_EMULATE=1: the emulated library's device memory is
    host memory), the byte buffers exactly FPL_BATCH_BYTES(n_bytes) long, filled from `batch` (whose arrays must cover that)"""
    import torch
    dev = torch.device("cpu" if EMULATE else "cuda:0")
    size = abi.batch_bytes(n_bytes)
    assert batch.n_bytes >= size
    out = [torch.from_numpy(batch.seq[:size].copy()).to(dev), torch.from_numpy(batch.qual[:size].copy()).to(dev),
           torch.from_numpy(batch.offsets.astype(np.int64)).to(dev), torch.from_numpy(batch.lens.astype(np.int32)).to(dev)]
    if dev.type == "cuda":
        torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("tiling", [None, "1"])
@pytest.mark.parametrize("name", ["default_se", "cut_polyx_cplx", "fasta64_polyx", "long_adapter_129", "long_adapter_64_no_jit",
                                  "mask_and_break", "mask_cplx", "filter_ties"])
def test_device_batch_with_the_documented_tail(name, tiling, monkeypatch):
    """fpl_process_device on buffers that end FPL_TAIL_PAD bytes behind the last read's vector, the tail and the padding
    poisoned, with and without read tiling; two layouts back to back on one context"""
    opt, env, own = SETS[name]
    if tiling:
        env = dict(env, FPL_TILE_MBASES=tiling)
    canon = own if own is not None else cases.adversarial_batch(4)
    g, o = make_engine(opt, env, monkeypatch), OracleEngine(opt)
    keep = []
    try:
        for k, (align, order, poison) in enumerate(((16, "identity", "adapter"), (48, "shuffled", "high"))):
            relaid = layouts.relayout(canon, align=align, order=order, gaps=2, poison=poison, tail=64, seed=k,
                                      adapters=layouts.adapters_of(opt))
            n_bytes = layouts.end_of_reads(relaid)
            seq, qual, offs, lens = device_buffers(relaid, n_bytes)
            keep.append((seq, qual, offs, lens))
            g.process_device(seq.data_ptr(), qual.data_ptr(), offs.data_ptr(), lens.data_ptr(), relaid.n_reads, n_bytes)
            g.sync()
            what = f"{name}/device/{align}/{order}/tiling{tiling}"
            compare_all(g, o, opt, g.fetch_results(canon.n_reads), o.process(canon), int(canon.lens.max()), what)
    finally:
        g.close()


def capacity_batches(seed):
    """Six batches whose longest read is 1024, 1025, 2048, 2049, 4096, 4097 bases: each raises the context's Stats capacity
    (1024 at creation, doubled as needed) exactly past a boundary or stops exactly at one"""
    rng = np.random.default_rng(seed)
    out = []
    for top in (1024, 1025, 2048, 2049, 4096, 4097):
        reads = []
        for L in [top] + [int(x) for x in rng.integers(1, top, 7)]:
            s = bytearray(synth.BASES[rng.integers(0, 4, L)].tobytes())
            if L > 100:
                s[L - 30:] = synth.ADAPTER_END.encode()
                s[L // 3:L // 3 + 30] = synth.ADAPTER_START.encode()
            reads.append((bytes(s), (np.rint(rng.normal(22, 8, L)).clip(1, 45).astype(np.uint8) + 33).tobytes()))
        out.append(pack_reads(reads))
    return out


@pytest.mark.parametrize("entry", ["host", "device"])
@pytest.mark.parametrize("name", ["cut_polyx_cplx", "mask_cplx"])
def test_one_submission_split_at_the_capacity_boundaries(name, entry, monkeypatch):
    """The same reads in six calls on one context equal one oracle pass over all of them: every call's records, and the Stats
    and counters accumulated across the capacity changes 1024 -> 2048 -> 4096 -> 8192.  fpl_process_device's calls go back to
    back without fpl_sync, each into its own results buffer, so the capacity grows while earlier calls may still be queued."""
    import torch
    opt, env, _ = SETS[name]
    canons = capacity_batches(11)
    g, o = make_engine(opt, env, monkeypatch), OracleEngine(opt)
    try:
        exps = [o.process(b) for b in canons]
        relaid = [layouts.relayout(b, align=16, order=("identity", "shuffled")[k % 2], poison="acgt", tail=32, seed=k)
                  for k, b in enumerate(canons)]
        if entry == "host":
            for k, b in enumerate(relaid):
                compare_results(g.process(b), exps[k], f"{name}/host/call{k}")
        else:
            keep, outs = [], []
            for b in relaid:
                n_bytes = layouts.end_of_reads(b)
                bufs = device_buffers(b, n_bytes)
                out = torch.zeros(b.n_reads * RESULT_DTYPE.itemsize, dtype=torch.uint8, device=bufs[0].device)
                keep.append(bufs)
                outs.append(out)
                g.process_device(*(t.data_ptr() for t in bufs), b.n_reads, n_bytes, results_ptr=out.data_ptr())
            g.sync()
            for k, out in enumerate(outs):
                compare_results(out.cpu().numpy().view(RESULT_DTYPE), exps[k], f"{name}/device/call{k}")
        assert g.cycles == 8192
        for w in (0, 1):
            compare_stats(g.stats(w, 4097), o.stats(w, 4097), f"{name}/{entry}/stats{w}")
        compare_stats(g.counters(), o.counters(), f"{name}/{entry}/counters")
    finally:
        g.close()


def test_offsets_must_be_multiples_of_16(monkeypatch):
    """Both entry points refuse a slot at offset 8 with a loud error and accept one at 16 (include/fplgpu.h, fpl_batch)"""
    import torch
    from fastplong_b200.binding import Engine, FplError
    opt = cases.OPTION_SETS["cut_polyx_cplx"]
    reads = [(b"ACGTTGCA", b"IIIIIIII"), (b"TTGACCAGTACGATCAG", b"I" * 17)]
    canon = pack_reads(reads)
    exp = OracleEngine(opt).process(canon)
    dev = torch.device("cpu" if EMULATE else "cuda:0")
    for off, ok in ((16, True), (8, False)):
        seq = np.zeros(off + 17 + 64, np.uint8)
        qual = np.zeros_like(seq)
        for o_, (s, q) in zip((0, off), reads):
            seq[o_:o_ + len(s)] = np.frombuffer(s, np.uint8)
            qual[o_:o_ + len(q)] = np.frombuffer(q, np.uint8)
        b = PackedBatch(seq, qual, np.array([0, off], np.int64), np.array([8, 17], np.int32))
        g = Engine(opt)
        if ok:
            compare_results(g.process(b), exp, "offset16/host")
        else:
            with pytest.raises(FplError, match="multiples of 16"):
                g.process(b)
        t = [torch.from_numpy(x).to(dev) for x in (b.seq, b.qual, b.offsets, b.lens)]
        for tiling in (None, "1"):
            gd = make_engine(opt, {"FPL_TILE_MBASES": tiling} if tiling else {}, monkeypatch)
            if ok:
                gd.process_device(*(x.data_ptr() for x in t), 2, b.n_bytes)
                gd.sync()
                compare_results(gd.fetch_results(2), exp, f"offset16/device/tiling{tiling}")
            else:
                with pytest.raises(FplError, match="multiple of 16"):
                    gd.process_device(*(x.data_ptr() for x in t), 2, b.n_bytes)
            gd.close()
        g.close()
