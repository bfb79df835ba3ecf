"""CPU-side check that the C-ABI library loads and exports every symbol include/fplgpu.h declares
(no compute calls without a GPU), and that the Python mirror of the structs matches the header."""
import ctypes as C
import os
import re

import pytest

from fastplong_b200 import abi, binding

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_functions():
    text = open(os.path.join(ROOT, "include", "fplgpu.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(fpl_[a-z_0-9]+)\s*\(", text)))


def test_header_functions_are_listed_in_binding():
    assert header_functions() == sorted(binding.EXPORTS)


@pytest.mark.skipif(not os.path.exists(binding.LIB_PATH), reason="libfplgpu.so not built (run __graft_entry__.build())")
def test_library_exports_every_declared_symbol():
    lib = C.CDLL(binding.LIB_PATH)
    for name in header_functions():
        assert hasattr(lib, name), name
    lib.fpl_abi_version.restype = C.c_int
    assert lib.fpl_abi_version() == abi.ABI_VERSION


def test_struct_mirror_sizes():
    assert C.sizeof(abi.FplOptions) == 144
    assert abi.RESULT_DTYPE.itemsize == 64
    hdr = open(os.path.join(ROOT, "include", "fplgpu.h")).read()
    assert int(re.search(r"#define FPL_MAX_ADAPTER_LEN (\d+)", hdr).group(1)) == abi.MAX_ADAPTER_LEN
    assert int(re.search(r"#define FPL_STATS_TAIL (\d+)", hdr).group(1)) == abi.STATS_TAIL
    assert int(re.search(r"#define FPL_CNT_FIXED (\d+)", hdr).group(1)) == abi.CNT_FIXED
    assert int(re.search(r"#define FPL_TAIL_PAD (\d+)", hdr).group(1)) == abi.TAIL_PAD
    # FPL_BATCH_BYTES(n) evaluated from its text (the int64_t casts dropped; every n here is >= 0) against abi.batch_bytes
    body = re.search(r"#define FPL_BATCH_BYTES\(n_bytes\) (.*)", hdr).group(1).replace("(int64_t)", "")
    for n in (0, 1, 15, 16, 17, 31, 32, 33, 149, 4097, 123456789):
        assert eval(body.replace("FPL_TAIL_PAD", str(abi.TAIL_PAD)), {"n_bytes": n}) == abi.batch_bytes(n), n
    assert [abi.batch_bytes(n) for n in (0, 1, 16, 17)] == [16, 32, 32, 48]


@pytest.mark.skipif(not os.path.exists(binding.LIB_PATH), reason="libfplgpu.so not built")
def test_create_fails_loudly_without_a_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from fastplong_b200 import Options
    with pytest.raises(binding.FplError):
        binding.Engine(Options())
