"""fpl_state_merge reads nothing outside [images[i], images[i] + n_bytes[i]), measured on the EMULATED library (tests/simt_emu.py)
with the instrument of tests/test_emulated_bounds.py: a state image placed flush against a PROT_NONE page — its last byte right in
front of the back guard, or its first right behind the front guard — is merged, and the same image truncated at every section
boundary, one byte short and into its header is refused, without an access to the guard page (that would end the process with
SIGSEGV, so the run is a subprocess: this file run as a script).  Runs on the CPU only."""
import ctypes as C
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def worker(side):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    import cases
    import simt_emu
    import test_gpu_state as S
    from test_emulated_bounds import _guarded
    from fastplong_b200 import synth
    opt = cases.MASK_BREAK_SETS["mask_and_break"]
    src = simt_emu.EmuEngine(opt)
    src.keep_read_lists(True)
    src.process(cases.blocky_quality_batch(7, n=30))
    img = src.export_state()
    dst = simt_emu.EmuEngine(opt)
    dst.keep_read_lists(True)
    dst.process(synth.ont_like(10, 800, 8))
    lib = dst.lib
    before = dst.export_state()
    cuts = sorted({n for at in S.sections(img) for n in (at, at - 1)} | {0, 8, S.HEADER // 2, len(img)})
    for n in cuts:
        if n > len(img):
            continue
        r = (n + 16) // 16 * 16               # _guarded places 16-byte multiples: the image ends at the back guard
        p = _guarded(r, side) + (r - n if side == "back" else 0)
        C.memmove(p, img, n)
        print(f"side={side} n={n} of {len(img)}", flush=True)
        rc = lib.fpl_state_merge(dst.h, (C.c_void_p * 1)(p), (C.c_int64 * 1)(n), 1)
        if n == len(img):
            assert rc == 0, lib.fpl_last_error().decode()
        else:
            assert rc < 0 and dst.export_state() == before, (n, lib.fpl_last_error().decode())
    want = simt_emu.EmuEngine(opt)
    want.keep_read_lists(True)
    want.process(synth.ont_like(10, 800, 8))
    want.merge(src)
    assert dst.export_state() == want.export_state()
    print("ok", flush=True)


def test_merge_reads_only_the_image():
    for side in ("back", "front"):
        p = subprocess.run([sys.executable, os.path.abspath(__file__), side], capture_output=True, text=True, timeout=1200, cwd=ROOT)
        assert p.returncode == 0, f"exit status {p.returncode} (-11: an access outside the image)\n{p.stdout[-1500:]}\n{p.stderr[-3000:]}"
        assert p.stdout.strip().endswith("ok")


if __name__ == "__main__":
    worker(sys.argv[1])
