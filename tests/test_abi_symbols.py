"""CPU: the CUDA library builds for sm_90a, loads without a GPU and exports every symbol include/aie_b200.h
declares.  No compute call is made here."""
import os
import re
import subprocess

from ai_economist_b200 import _abi
from ai_economist_b200.build import CSRC, build_library

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "aie_b200.h")).read()
    return sorted(set(re.findall(r"\b(aie_[a-z_]+)\s*\(", src)))


def test_library_builds_and_exports_header_symbols():
    lib = build_library()
    L = _abi.load_library(lib)
    names = declared_symbols()
    assert set(names) == set(_abi.EXPORTED_SYMBOLS), (names, _abi.EXPORTED_SYMBOLS)
    for n in names:
        assert hasattr(L, n), n
    assert L.aie_abi_version() == _abi.ABI_VERSION


def test_library_is_sm_90a_with_tma_bulk_copies():
    lib = build_library()
    sass = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
    assert "arch = sm_90a" in sass
    assert "UBLKCP" in sass, "step/observe kernels must stage the env record with cp.async.bulk (UBLKCP)"


def test_create_without_gpu_fails_loudly():
    import ctypes as C
    import torch
    if torch.cuda.is_available():
        return
    L = _abi.load_library(build_library())
    from tests import golden_utils as gu
    z, meta, init = gu.load_fixture(gu.golden_files()[0])
    cfg = _abi.config_from_spec(meta["spec"])
    h = C.c_void_p()
    rc = L.aie_create(C.byref(cfg), 4, 0, C.byref(h))
    assert rc != 0 and b"no CPU fallback" in L.aie_last_error()
