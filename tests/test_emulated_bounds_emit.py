"""How far fpl_emit_batch_device reads and writes outside its buffers, measured exactly on the EMULATED library as in
tests/test_emulated_bounds.py: the device batch fpl_process_device ran on ends right at FPL_BATCH_BYTES(n_bytes) in front of a
PROT_NONE page (or starts right behind one), and so do the `out` and `failed` batches the emit writes, each exactly
FPL_BATCH_BYTES(n_bytes) long.  The read that ends the input has an output read whose window runs to its last base: it ends
mid-vector, on a vector end, and past 96 kb.  Under -N the copy reads the bases from the library's masked copy of the sequence
buffer instead, which is NOT guarded here (an internal allocation with a doubling capacity); the -N cases guard the qualities,
the outputs, and check the masked bytes by value.  The copy's loads stay inside any window's 16-byte vectors by construction
(warp_copy in fpl_emit.cu: every load is an aligned word holding a byte of the window), which the unmasked cases measure.  An
access outside the guarded buffers ends the process with SIGSEGV, so every run is a subprocess (this file run as a script); the
runs also compare the emitted batches with the expected ones.

This instrument runs on the CPU only: nothing here makes a GPU touch memory it does not own."""
import ctypes as C
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

CASES = ("default_se", "cut_polyx_cplx", "mask_default", "mask_cplx", "break_default")
LAST_LENS = (149, 160, 100001)      # the read that ends the input: mid-vector, on a vector end, > 96 kb


def _host_view(ptr, n):
    import numpy as np
    return np.frombuffer((C.c_uint8 * n).from_address(ptr), dtype=np.uint8).copy() if n else np.zeros(0, np.uint8)


def worker(side):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    import numpy as np
    import cases
    import layouts
    import simt_emu
    from fastplong_b200 import abi, pack_reads, synth
    from oracle_lib import OracleEngine
    from test_emulated_bounds import _guarded
    from test_gpu_emit_batch import expected
    rng = np.random.default_rng(7)
    for name in CASES:
        opt = cases.OPTION_SETS.get(name) or cases.MASK_BREAK_SETS[name]
        for last in LAST_LENS:
            base = cases.adversarial_batch(3)
            s = synth.BASES[rng.integers(0, 4, last)].tobytes()
            q = (np.rint(rng.normal(30, 4, last)).clip(20, 45) + 33).astype(np.uint8)
            if opt.mask:
                q[last // 2:last // 2 + 40] = 33 + 3             # a stretch -N paints, well inside the read
            canon = pack_reads([base.read(i) for i in range(base.n_reads)] + [(s, q.tobytes())])
            b = layouts.relayout(canon, align=16, poison="acgt", tail=abi.TAIL_PAD + 16, seed=last)
            n_bytes = layouts.end_of_reads(b)
            size = abi.batch_bytes(n_bytes)
            print(f"case {name} last={last} side={side}", flush=True)
            bufs = []
            for arr in (b.seq, b.qual):
                p = _guarded(size, side)
                C.memmove(p, arr.ctypes.data, size)
                bufs.append(p)
            offs = b.offsets.astype(np.int64)
            lens = b.lens.astype(np.int32)
            e, o = simt_emu.EmuEngine(opt), OracleEngine(opt)
            e.process_device(bufs[0], bufs[1], offs.ctypes.data, lens.ctypes.data, b.n_reads, n_bytes)
            e.sync()
            ores = o.process(canon)
            exp = expected(opt, canon, o, ores)
            assert any(len(x["lens"]) and x["segs"]["read"][-1] == canon.n_reads - 1 and
                       x["segs"]["lo"][-1] + x["segs"]["len"][-1] == last for x in exp), "no output read ends with the last base"
            descs = [abi.FplOutBatch(), abi.FplOutBatch()]
            assert e.lib.fpl_emit_batch_device(e.h, C.byref(descs[0]), C.byref(descs[1])) in (0, 1)
            keep = []
            for d in descs:
                n, nb = int(d.n_reads), int(d.n_bytes)
                if not n:
                    continue
                d.seq, d.qual = _guarded(abi.batch_bytes(nb), side), _guarded(abi.batch_bytes(nb), side)
                idx = [np.zeros(n, np.int64), np.zeros(n, np.int32), np.zeros(n, abi.SEGMENT_DTYPE)]
                keep.append(idx)
                d.offsets, d.lens, d.segs = (a.ctypes.data for a in idx)
                d.cap_reads, d.cap_bytes = n, abi.batch_bytes(nb)
            assert e.lib.fpl_emit_batch_device(e.h, C.byref(descs[0]), C.byref(descs[1])) == 0, e.lib.fpl_last_error()
            e.sync()
            k = 0
            for d, x in zip(descs, exp):
                assert int(d.n_reads) == len(x["lens"]) and int(d.n_bytes) == x["n_bytes"], name
                if not d.n_reads:
                    continue
                got_off, got_len, got_segs = keep[k]
                k += 1
                nbb = abi.batch_bytes(int(d.n_bytes))
                assert np.array_equal(_host_view(d.seq, nbb), x["seq"]) and np.array_equal(_host_view(d.qual, nbb), x["qual"]), name
                assert np.array_equal(got_off, x["offsets"]) and np.array_equal(got_len, x["lens"]), name
                assert got_segs.tobytes() == x["segs"].tobytes(), name
            e.close()
    print("ok", flush=True)


@pytest.mark.parametrize("side", ["front", "back"])
def test_emit_stays_inside_the_documented_batches(side):
    p = subprocess.run([sys.executable, os.path.abspath(__file__), side], capture_output=True, text=True, timeout=1800, cwd=ROOT)
    assert p.returncode == 0, f"exit status {p.returncode} (-11: an access outside the buffers)\n{p.stdout[-1500:]}\n{p.stderr[-3000:]}"
    assert p.stdout.strip().endswith("ok")


if __name__ == "__main__":
    worker(sys.argv[1])
