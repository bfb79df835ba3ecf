"""Development aid: compile the k_scan_jit source (version 2 by default, `--v1` for the round-1 kernel) with NVRTC
(no GPU needed; `--no-qhist` without the quality histograms), print ptxas statistics and write the cubin to /tmp/scan_jit.cubin for cuobjdump."""
import ctypes
import os
import re
import sys
from cuda.bindings import nvrtc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
args = [a for a in sys.argv[1:] if not a.startswith("--")]
v1 = "--v1" in sys.argv
a0 = args[0] if len(args) > 0 else "AATGTACTTCGTTCAGTTACGTATTGCTAA"
a1 = args[1] if len(args) > 1 else "TTAGCAATACGTAACTGAACGAAGTACATT"
cplx = "true" if "--cplx" in sys.argv else "false"
qhist = "false" if "--no-qhist" in sys.argv else "true"
if v1:
    src = open(os.path.join(ROOT, "fastplong_b200/csrc/fpl_scan_jit_src.h")).read()
    body = re.search(r'R"JITSRC\((.*)\)JITSRC"', src, re.S).group(1)
else:
    lib = ctypes.CDLL(os.path.join(ROOT, "fastplong_b200/libfplgpu.so"))
    lib.fpl_jit_debug_source.restype = ctypes.c_char_p
    lib.fpl_jit_debug_source.argtypes = [ctypes.c_char_p, ctypes.c_char_p]
    body = lib.fpl_jit_debug_source(a0.encode(), a1.encode()).decode()
    open("/tmp/scan_jit_src.cu", "w").write(body)
defs = (f'#define FPL_A0 "{a0}"\n#define FPL_A1 "{a1}"\n#define FPL_ALEN0 {len(a0)}\n#define FPL_ALEN1 {len(a1)}\n'
        f'#define FPL_DO_ADAPTERS true\n#define FPL_DO_COUNTS true\n#define FPL_DO_CPLX {cplx}\n#define FPL_DO_QHIST {qhist}\n'
        f'#define FPL_QQ 48\n#define FPL_MINBLOCKS 8\n')
err, prog = nvrtc.nvrtcCreateProgram((defs + body).encode(), b"fpl_scan_jit.cu", 0, [], [])
opts = [b"--gpu-architecture=sm_90a", b"-std=c++17", b"-lineinfo", b"--ptxas-options=-v"]
err, = nvrtc.nvrtcCompileProgram(prog, len(opts), opts)
_, n = nvrtc.nvrtcGetProgramLogSize(prog)
log = b" " * n
nvrtc.nvrtcGetProgramLog(prog, log)
print(log.decode(errors="replace")[-3000:])
print("compile status", err)
if int(err) == 0:
    _, n = nvrtc.nvrtcGetCUBINSize(prog)
    cubin = b" " * n
    nvrtc.nvrtcGetCUBIN(prog, cubin)
    open("/tmp/scan_jit.cubin", "wb").write(cubin)
    print("cubin bytes", n)
