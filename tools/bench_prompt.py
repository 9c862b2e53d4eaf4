"""Prompted decoding: the prompt's teacher-forced positions as one batched prefill pass (decode_prefill) vs step by step
(decode_run), large-v3 shape with random weights, the two alternating, `--runs` timed runs each, in one process.

    python tools/bench_prompt.py [--runs 3] [--plens 32,128,224]

Cells: prompt lengths (decoder input = random prompt tokens + SOT / language / task / notimestamps) x Q = 1, Q = 64 and 64 audios
x 5 beams, x 16-bit and int8 decoder weights.  Each run times, with CUDA events, decode_prefill(plen - 1) and
decode_run(plen - 1) after the same decode_begin.  Prints one JSON line: per cell both times (median and runs), the prefill's
kernel launches (from its pass count), the FLOPs and bytes it needs (from the shapes, see prefill_work) and its share of the
H100 SXM's peak by whichever bound applies, the first generated token's logits difference between the two paths in units of
their standard deviation, and the GPU name and power limit read in the same call.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("TRANSFORMERS_OFFLINE", "1")
os.environ.setdefault("HF_HUB_OFFLINE", "1")

from bench import CHUNK_S, PRESET  # noqa: E402
from tools.bench_decoder_weights import gpu_info  # noqa: E402

HBM_BPS = 3.35e12    # H100 SXM data sheet
DENSE_FLOPS = 989e12  # dense BF16 / FP16 tensor-core rate, same data sheet
PREFILL_ROWS = 4096   # rows of one prefill pass (api.cu PREFILL_ROWS)


def prefill_work(dims, S: int, A: int, G: int, n: int, w_bytes: float):
    """(FLOPs, bytes) of decode_prefill(n) over Q = A * G sequences: every layer's projections for Q * n rows (the last layer only
    its QKV projection), causal self-attention (QK^T and PV over t + 1 keys per row) and cross-attention over S keys; bytes = the
    decoder weights once per pass, the cross K/V of the A audios per pass, the self K/V rows written and read."""
    d, L, ffn = dims.d_model, dims.dec_layers, dims.ffn
    Q = A * G
    per = max(1, PREFILL_ROWS // Q)
    passes = -(-n // per)
    R = Q * n
    per_row_full = 2 * (3 * d * d + d * d + d * d + d * d + 2 * d * ffn)  # wqkv, wo, xwq, xwo, w1, w2
    flops = R * ((L - 1) * per_row_full + 2 * 3 * d * d)
    flops += (L - 1) * Q * 2 * 2 * d * (n * (n + 1) / 2)  # causal self-attention
    flops += (L - 1) * R * 2 * 2 * d * S                   # cross-attention
    w_elems = (L - 1) * (6 * d * d + 2 * d * ffn) + 3 * d * d
    byts = passes * (w_elems * w_bytes + (L - 1) * A * 2 * S * d * 2) + L * Q * n * 2 * d * 2 * 2
    launches = passes * (1 + 14 * (L - 1) + 3) + 1
    return flops, byts, launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--plens", default="32,128,224")
    args = ap.parse_args()
    plens = [int(x) for x in args.plens.split(",")]

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
    opts = DecodeOptions(eos_token=S.EOS, pad_token=S.EOS, suppress_tokens=list(gcfg.suppress_tokens),
                         begin_suppress_tokens=list(gcfg.begin_suppress_tokens))
    init = [S.SOT, S.LANG_EN, S.TRANSCRIBE, S.NOTIMESTAMPS]
    rng = np.random.default_rng(0)
    cells = [(1, 1), (64, 1), (64, 5)]
    result = {"gpu": info, "preset": PRESET, "runs": args.runs, "cells": []}
    for fmt in (None, "int8"):
        w = pack_weights(sd, dims, pos, dev, torch.bfloat16, fmt)
        eng = WhisperEngine(None, dims, chunk_length_s=CHUNK_S, max_audios=64, max_beams=5, weights=w)
        pcm = torch.from_numpy(np.stack([S.synth_audio(CHUNK_S, seed=1000 + i) for i in range(64)])).to(dev)
        eng.logmel_device(pcm, 64)
        eng.encode(64)
        torch.cuda.synchronize()
        for A, G in cells:
            for plen in plens:
                prompt = np.array([list(rng.integers(0, 50257, size=plen - len(init))) + init] * A, dtype=np.int32)
                prompts = np.repeat(prompt, G, axis=0)

                def one(prefill):
                    eng.decode_begin(prompts, A, G, opts)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    if prefill:
                        eng.decode_prefill(plen - 1)
                    else:
                        eng.decode_run(plen - 1)
                    e1.record()
                    torch.cuda.synchronize()
                    ms = e0.elapsed_time(e1)
                    eng.decode_run(1)
                    return ms, eng.logits().double().clone()

                one(True), one(False)  # warm-up: step-graph capture, module load, prefill scratch
                ms = {"prefill": [], "steps": []}
                for _ in range(args.runs):
                    t, lp = one(True)
                    ms["prefill"].append(t)
                    t, ls = one(False)
                    ms["steps"].append(t)
                dl = ((lp - ls).abs().max() / ls.std()).item()
                flops, byts, launches = prefill_work(dims, eng.S, A, G, plen - 1, 1.0 if fmt == "int8" else 2.0)
                tp = float(np.median(ms["prefill"]))
                ts = float(np.median(ms["steps"]))
                t_flops, t_bytes = flops / DENSE_FLOPS, byts / HBM_BPS
                result["cells"].append({
                    "weights": fmt or "16bit", "audios": A, "beams": G, "plen": plen, "prefill_ms": tp, "prefill_ms_runs": ms["prefill"],
                    "steps_ms": ts, "steps_ms_runs": ms["steps"], "speedup": ts / tp, "prefill_launches": launches,
                    "prefill_flops": flops, "prefill_bytes": byts, "bound": "compute" if t_flops > t_bytes else "hbm",
                    "peak_share": max(t_flops, t_bytes) / (tp * 1e-3), "first_logits_diff_sigma": dl})
                print(json.dumps(result["cells"][-1]), file=sys.stderr, flush=True)
        eng.close()
        del eng, w
        torch.cuda.empty_cache()
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
