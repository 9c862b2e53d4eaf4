"""CPU checks of the drop-in boundary: the C-ABI library builds, loads and exports every symbol the header declares;
the product fails loudly without a GPU (no CPU fallback)."""
import os
import re

import pytest

from tests.conftest import ROOT


def _header_symbols():
    src = open(os.path.join(ROOT, "include", "thewhisper_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(bw_[a-z0-9_]+)\s*\(", src)))


def test_library_builds_and_exports_header_symbols():
    from thewhisper_b200 import _lib, build

    build.build()
    lib = _lib.load()
    names = _header_symbols()
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/thewhisper_b200.h but not exported"
    assert sorted(_lib.SYMBOLS) == names, (sorted(set(names) ^ set(_lib.SYMBOLS)))
    assert lib.bw_abi_version() == 2


def test_no_cpu_fallback():
    import ctypes as C

    import torch

    from thewhisper_b200 import _lib

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    lib = _lib.load()
    cfg = _lib.bw_config(128, 2, 512, 2, 2, 128, 51866, 500, 448, 1, 1, 0, 448, 0)
    h = C.c_void_p()
    rc = lib.bw_engine_create(C.byref(cfg), C.byref(h))
    assert rc != 0 and b"no CUDA device" in lib.bw_last_error()
    from thewhisper_b200.engine import ModelDims, WhisperEngine

    with pytest.raises(_lib.BwError):
        WhisperEngine({}, ModelDims(128, 2, 512, 2, 2, 128, 51866))


def test_sass_is_hopper_native():
    """the built library must contain wgmma / TMA machine code (HGMMA, UTMALDG)"""
    import shutil
    import subprocess

    from thewhisper_b200 import _lib

    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not on PATH")
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    for mnem in ("HGMMA", "UTMALDG"):
        assert mnem in sass, mnem
    assert "HMMA.16816" not in sass  # no legacy mma.sync tensor path
