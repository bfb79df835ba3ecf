"""How far the kernels read outside a device batch, measured exactly on the EMULATED library (tests/simt_emu.py), where device
memory is host memory: the seq and qual buffers of fpl_process_device are placed against a PROT_NONE page — offset 0 right behind
the front guard, or the last byte the batch may be read at (FPL_TAIL_PAD behind the end of the last read's 16-byte vector) right in
front of the back guard.  An access outside that range ends the process with SIGSEGV, so every run is a subprocess (this file run
as a script) and the test asserts its exit status.  The runs also compare with the oracle, so a read whose last vector is the last
of the buffer is checked for its results as well.

This instrument runs on the CPU only: nothing here makes a GPU touch memory it does not own."""
import ctypes as C
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


# every kernel variant that reads the batch: (option set, how fpl_create sets up the scan); the -N/-b sets read the masked copy
CASES = [("default_se", "jit"), ("cut_polyx_cplx", "jit"), ("fasta5", "jit"), ("fasta64_polyx", "jit"), ("literal_auto", "jit"),
         ("long_adapter_129", "jit"), ("long_adapter_64", "fast"), ("cut_polyx_cplx", "generic"), ("mask_and_break", "jit"),
         ("mask_cplx", "jit"), ("trims_limits", "jit"), ("filter_ties", "jit")]
LAST_LENS = (149, 160, 4097, 100001)      # the read that ends the buffer: mid-vector, on a vector end, past a scan tile, > 96 kb


def _option_set(name):
    import cases
    if name == "filter_ties":
        return cases.edge_cases()["filter_ties"]
    return cases.OPTION_SETS.get(name) or cases.MASK_BREAK_SETS[name], None


def _guarded(n, side):
    """n bytes of fresh memory that end right at a PROT_NONE page (side "back") or start right behind one ("front")"""
    libc = C.CDLL(None, use_errno=True)
    libc.mmap.restype = C.c_void_p
    libc.mmap.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_long]
    libc.mprotect.argtypes = [C.c_void_p, C.c_size_t, C.c_int]
    page = os.sysconf("SC_PAGE_SIZE")
    pages = (n + page - 1) // page
    base = libc.mmap(None, (pages + 2) * page, 3, 0x22, -1, 0)          # PROT_READ|WRITE, MAP_PRIVATE|ANONYMOUS
    assert base not in (None, C.c_void_p(-1).value)
    assert libc.mprotect(base, page, 0) == 0 and libc.mprotect(base + (pages + 1) * page, page, 0) == 0
    start = base + page if side == "front" else base + (pages + 1) * page - n
    assert start % 16 == 0
    return start


def worker(side, tail, tiled):
    """Every CASES entry on a batch whose buffers end `tail` bytes behind the last read's 16-byte vector (side "back"; with
    tail == FPL_TAIL_PAD that is FPL_BATCH_BYTES(n_bytes)), or start at a guard page (side "front"); exit status 0 iff no access
    left the buffers and every result matched the oracle."""
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    import numpy as np
    import cases
    import layouts
    import simt_emu
    from fastplong_b200 import Options, pack_reads, synth
    from fastplong_b200.abi import RESULT_DTYPE
    from oracle_lib import OracleEngine, compare_lists, compare_results, compare_stats
    if tiled:
        os.environ["FPL_TILE_MBASES"] = "1"
    rng = np.random.default_rng(5)
    for name, scan in CASES:
        opt, own_batch = _option_set(name)
        for last in LAST_LENS:
            base = own_batch if own_batch is not None else cases.adversarial_batch(3)
            s = bytearray(synth.BASES[rng.integers(0, 4, last)].tobytes())
            s[-30:] = synth.ADAPTER_END.encode()                       # the scans have a hit right at the buffer's end
            extra = (bytes(s), bytes((np.rint(rng.normal(25, 8, last)).clip(1, 45) + 33).astype(np.uint8)))
            canon = pack_reads([base.read(i) for i in range(base.n_reads)] + [extra])
            b = layouts.relayout(canon, align=16, poison="acgt", tail=tail + 16, seed=last)
            n_bytes = layouts.end_of_reads(b)
            size = (n_bytes + 15) // 16 * 16 + tail
            print(f"case {name}/{scan} last={last} side={side} tail={tail} tiled={tiled}", flush=True)
            bufs = []
            for arr in (b.seq, b.qual):
                p = _guarded(size, side)
                C.memmove(p, arr.ctypes.data, size)
                bufs.append(p)
            offs = b.offsets.astype(np.int64)
            lens = b.lens.astype(np.int32)
            e, o = simt_emu.EmuEngine(opt, scan=scan), OracleEngine(opt)
            e.process_device(bufs[0], bufs[1], offs.ctypes.data, lens.ctypes.data, b.n_reads, n_bytes)
            e.sync()
            what = f"{name}/{scan}/last{last}"
            compare_results(e.fetch_results(b.n_reads), o.process(canon), what)
            if opt.mask or opt.break_reads:
                compare_lists(e.segments(), o.segments(), what + "/segments")
                compare_lists(e.mask_regions(), o.mask_regions(), what + "/regions")
            cyc = int(canon.lens.max())
            for w in (0, 1):
                compare_stats(e.stats(w, cyc), o.stats(w, cyc), f"{what}/stats{w}")
            compare_stats(e.counters(), o.counters(), what + "/counters")
            e.close()
    print("ok", flush=True)


def run_worker(side, tail, tiled=False):
    return subprocess.run([sys.executable, os.path.abspath(__file__), side, str(tail), str(int(tiled))], capture_output=True,
                          text=True, timeout=1200, cwd=ROOT)


@pytest.mark.parametrize("tiled", [False, True])
@pytest.mark.parametrize("side", ["front", "back"])
def test_kernels_stay_inside_the_documented_batch(side, tiled):
    """fpl_process_device reads nothing in front of offset 0 and nothing beyond FPL_BATCH_BYTES(n_bytes), on every kernel
    variant, with and without read tiling.  (The bound is tight: with 16 bytes less, the 32-byte lane loads of the precompiled
    k_scan_fast leave the buffer.)"""
    from fastplong_b200 import abi
    p = run_worker(side, abi.TAIL_PAD, tiled)
    assert p.returncode == 0, f"exit status {p.returncode} (-11: an access outside the batch)\n{p.stdout[-1500:]}\n{p.stderr[-3000:]}"
    assert p.stdout.strip().endswith("ok")


if __name__ == "__main__":
    worker(sys.argv[1], int(sys.argv[2]), sys.argv[3] == "1")
