"""CPU check of the persistent decoder step's shared-memory plan (bw_op_mega_plan runs the launcher's plan code on the host):
at the benchmarked shapes the plan fits the H100's shared memory together with the kernel's static shared memory as
compiled, and keeps the double-buffered weight slabs where they fit."""
import ctypes as C
import re
import shutil
import subprocess

import pytest

OPTIN = 227 * 1024  # opt-in shared memory per block of an H100 (sm_90)
RESERVED = 1024     # shared memory the system reserves per block on sm_90 (cuobjdump's SHARED includes it)

# (name, Q, D, ffn, SMs, double-buffered): large-v3 / large-v3-turbo decoder dims (the same D and ffn) on H100 SXM (132 SMs),
# H100 PCIe (114 SMs) and a 148-SM part
CONFIGS = [
    ("large-v3-132-q1", 1, 1280, 5120, 132, True),
    ("large-v3-132-q2", 2, 1280, 5120, 132, False),
    ("large-v3-148-q1", 1, 1280, 5120, 148, True),
    ("large-v3-114-q1", 1, 1280, 5120, 114, False),
    ("large-v3-114-q2", 2, 1280, 5120, 114, False),
]


def _static_smem(lib_path):
    """largest static shared memory of the step kernel's instantiations in the built library"""
    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not on PATH")
    out = subprocess.run(["cuobjdump", "-res-usage", lib_path], capture_output=True, text=True).stdout
    sizes, fn = [], None
    for line in out.splitlines():
        if "Function" in line:
            fn = line
        elif fn and "decode_mega_kernel" in fn and "SHARED:" in line:
            sizes.append(int(re.search(r"SHARED:(\d+)", line).group(1)) - RESERVED)
    assert sizes, "decode_mega_kernel not found in the library"
    return max(sizes)


def _plan(lib, Q, D, ffn, sms, optin, static):
    out = (C.c_int64 * 2)()
    rc = lib.bw_op_mega_plan(Q, D, ffn, sms, optin, static, out)
    return rc, int(out[0]), int(out[1])


@pytest.mark.parametrize("cfg", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_mega_plan_fits(cfg):
    from thewhisper_b200 import _lib, build

    build.build()
    lib = _lib.load()
    static = _static_smem(_lib.LIB_PATH)
    _, Q, D, ffn, sms, dbuf = cfg
    rc, smem, p0_off = _plan(lib, Q, D, ffn, sms, OPTIN, static)
    assert rc == 0 and 0 < smem and smem + static <= OPTIN, (cfg, rc, smem, static)
    assert (p0_off > 0) == dbuf, (cfg, smem, p0_off)


def test_mega_plan_rejects_what_does_not_fit():
    from thewhisper_b200 import _lib

    lib = _lib.load()
    # 96 KB cannot hold the attention scratch, a 100 KB fc1 slab set and the LM head's slab stages
    rc, smem, _ = _plan(lib, 1, 1280, 5120, 132, 96 * 1024, 6 * 1024)
    assert rc == -3 and smem == 0
