"""16-bit vs int8 decoder weights on the decoder step: C2 (large-v3, one 30 s chunk, Q = 1: the persistent step) and C3
(64 x 30 s chunks, greedy: Q = 64), the two formats alternating, `--runs` timed runs each, in one process.

    python tools/bench_decoder_weights.py [--runs 3] [--tokens 128] [--c3-audios 64]

Each run times `--tokens` greedy decoder steps with CUDA events (the encoder runs once per engine beforehand: its output and
the cross K/V are the same for both formats).  Prints one JSON line: per config and format the step time (median and spread
over the runs), tokens/s, the bytes one step must read (from the shapes, see step_bytes) and their share of the H100 SXM's
3.35 TB/s, the engine's kernels per step, the GPU name and power limit read in the same call.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("TRANSFORMERS_OFFLINE", "1")
os.environ.setdefault("HF_HUB_OFFLINE", "1")

from bench import CHUNK_S, PRESET, decode_bytes_per_step  # noqa: E402

HBM_BPS = 3.35e12  # H100 SXM data sheet


def step_bytes(dims, S: int, A: int, t_mean: float, fmt) -> float:
    """Bytes one decoder step reads: bench.decode_bytes_per_step (16-bit weights, cross K/V, self K/V), with the streamed
    weights at 1 byte each plus an fp32 scale per row for int8."""
    b = decode_bytes_per_step(dims, S, A, t_mean)
    if fmt == "int8":
        d, L, V, ffn = dims.d_model, dims.dec_layers, dims.vocab, dims.ffn
        n_w = L * (6 * d * d + 2 * d * ffn) + V * d
        rows = L * (3 * d + d + d + d + ffn + d) + V
        b += -1.0 * n_w + 4.0 * rows
    return b


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clk = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": clk}
    except Exception as ex:  # the numbers stand without it, but say so
        return {"error": repr(ex)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--tokens", type=int, default=128)
    ap.add_argument("--c3-audios", type=int, default=64)
    args = ap.parse_args()

    import torch

    from thewhisper_b200 import synthetic as S
    from thewhisper_b200.engine import DecodeOptions, ModelDims, WhisperEngine, pack_weights

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU")
    info = gpu_info()
    dev = torch.device("cuda:0")
    cfg = S.make_hf_config(PRESET)
    dims = ModelDims.from_hf_config(cfg)
    gcfg = S.make_generation_config(PRESET, eos_suppressed=True, suppress_timestamps=True)
    model = S.make_hf_model(PRESET, seed=0)
    sd = model.state_dict()
    pos = sd["model.encoder.embed_positions.weight"].float()
    weights = {fmt: pack_weights(sd, dims, pos, dev, torch.bfloat16, fmt) for fmt in (None, "int8")}
    del sd, model
    opts = DecodeOptions(eos_token=S.EOS, pad_token=S.EOS, suppress_tokens=list(gcfg.suppress_tokens),
                         begin_suppress_tokens=list(gcfg.begin_suppress_tokens))

    def engines(A):
        out = {}
        pcm = torch.from_numpy(np.stack([S.synth_audio(CHUNK_S, seed=1000 + i) for i in range(A)])).to(dev)
        for fmt, w in weights.items():
            eng = WhisperEngine(None, dims, chunk_length_s=CHUNK_S, max_audios=A, weights=w)
            eng.logmel_device(pcm, A)
            eng.encode(A)
            out[fmt or "16bit"] = eng
        torch.cuda.synchronize()
        return out

    def run(eng, A):
        prompt = np.array([[S.SOT, S.LANG_EN, S.TRANSCRIBE, S.NOTIMESTAMPS]] * A, dtype=np.int32)
        eng.decode_begin(prompt, A, 1, opts)
        eng.decode_run(prompt.shape[1] - 1)
        k0 = eng.decode_kernel_launches()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        eng.decode_run(args.tokens)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.tokens, (eng.decode_kernel_launches() - k0) / args.tokens

    result = {"gpu": info, "preset": PRESET, "tokens_per_run": args.tokens, "runs": args.runs, "configs": {}}
    for name, A in (("C2", 1), ("C3", args.c3_audios)):
        engs = engines(A)
        for e in engs.values():  # warm-up: graph capture, module load
            run(e, A)
        ms = {k: [] for k in engs}
        kern = {}
        for _ in range(args.runs):
            for k, e in engs.items():
                t, kern[k] = run(e, A)
                ms[k].append(t)
        cfg_out = {}
        for k in engs:
            med = float(np.median(ms[k]))
            b = step_bytes(dims, engs[k].S, A, 4 + args.tokens / 2, None if k == "16bit" else k)
            cfg_out[k] = {"step_ms": med, "step_ms_runs": ms[k], "tokens_per_sec": A * 1e3 / med, "bytes_per_step": b,
                          "hbm_share": b / (med * 1e-3) / HBM_BPS, "kernels_per_step": kern[k]}
        cfg_out["int8_speedup"] = cfg_out["16bit"]["step_ms"] / cfg_out["int8"]["step_ms"]
        result["configs"][name] = dict(audios=A, **cfg_out)
        for e in engs.values():
            e.close()
        del engs
        torch.cuda.empty_cache()
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
