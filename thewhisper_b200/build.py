"""In-tree build of the sm_90a (H100) shared library (explicit nvcc; no JIT cache, the .so travels with the repo).

    python -m thewhisper_b200.build            # builds thewhisper_b200/_C/libthewhisper_b200.so if stale
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT_DIR = os.path.join(HERE, "_C")
LIB = os.path.join(OUT_DIR, "libthewhisper_b200.so")
# compiled twice: 16-bit elements = bfloat16 (x.o) and, with -DBW_F16, = float16 (x_f16.o)
SOURCES_PER_DTYPE = ["api.cu", "gemm_tc.cu", "gemm_dec.cu", "attn_enc.cu", "logmel.cu", "decode.cu", "decode_stream.cu",
                     "decode_mega.cu", "decode_prefill.cu", "timestamps.cu"]
SOURCES_ONCE = ["abi.cu", "hostproc.cu", "host_decode.cu"]
HEADERS = ["common.cuh", "kernels.h", "decode.cuh", "decode_mega_common.cuh", "abi_rename.h", "abi_unrename.h",
           os.path.join("..", "..", "include", "thewhisper_b200.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _stale(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OUT_DIR, exist_ok=True)
    nvcc = _nvcc()
    # this file holds NVCC_FLAGS: objects built with other flags (another architecture) are stale too
    hdrs = [os.path.normpath(os.path.join(CSRC, h)) for h in HEADERS] + [os.path.abspath(__file__)]
    objs, jobs = [], []
    units = [(src, "", []) for src in SOURCES_ONCE + SOURCES_PER_DTYPE] + [(src, "_f16", ["-DBW_F16"]) for src in SOURCES_PER_DTYPE]
    for src, suffix, defs in units:
        s = os.path.join(CSRC, src)
        o = os.path.join(OUT_DIR, src.replace(".cu", suffix + ".o"))
        objs.append(o)
        if force or _stale(o, [s] + hdrs):
            jobs.append([nvcc] + NVCC_FLAGS + defs + (["-Xptxas", "-v"] if verbose else []) + ["-c", s, "-o", o])

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed: %s\n%s\n%s" % (" ".join(cmd), r.stdout, r.stderr))
        return r.stderr

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            for log in ex.map(run, jobs):
                if verbose and log:
                    print(log)
    if force or jobs or _stale(LIB, objs):
        run([nvcc, "-shared", "-o", LIB] + objs + ["-lcudart"])
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
