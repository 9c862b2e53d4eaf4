"""Sequential long-form transcription at large-v3 shapes with random weights: 1 and 16 synthetic audios of 10 minutes, long form
(no chunk_length_s) with and without condition_on_prev_tokens, against chunked inference (chunk_length_s=30) on the same audio.

    python tools/bench_longform.py [--minutes 10] [--audios 1,16] [--max-new-tokens 0]

Per cell: wall time and audio seconds per second, windows encoded, decoder steps and prefill passes, the long log-mel kernel time
(CUDA events around engine.logmel_long of the group), step graphs captured, the time spent capturing and instantiating them, graphs
cached and evicted (the engine's own counters), and the GPU name and power limit read in the same call.  BW_STEP_GRAPHS=0 runs with
an unbounded step-graph cache.  Prints one JSON line.
Random weights do not produce speech-like text: the numbers show the schedule's cost (windows, graphs, steps), not a real
transcript's.  --max-new-tokens 0 keeps the generation config's budget.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("TRANSFORMERS_OFFLINE", "1")
os.environ.setdefault("HF_HUB_OFFLINE", "1")

from tools.bench_decoder_weights import gpu_info  # noqa: E402


def main():
    import torch

    from thewhisper_b200 import synthetic as S
    from thewhisper_b200.nvidia import ASRPipeline

    ap = argparse.ArgumentParser()
    ap.add_argument("--minutes", type=float, default=10.0)
    ap.add_argument("--audios", default="1,16")
    ap.add_argument("--max-new-tokens", type=int, default=0)
    args = ap.parse_args()
    counts = [int(x) for x in args.audios.split(",")]
    model = S.make_hf_model("large-v3", seed=0)
    pipe = ASRPipeline(model, feature_extractor=S.make_feature_extractor(30), tokenizer=S.make_tokenizer(), chunk_length_s=30,
                       device="cuda", torch_dtype=torch.float16, batch_size=max(counts))
    eng = pipe.engine
    mel_ms = []
    orig = eng.logmel_long

    def timed(pcm):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = orig(pcm)
        b.record()
        b.synchronize()
        mel_ms.append(a.elapsed_time(b))
        return out

    eng.logmel_long = timed
    gk = {"num_beams": 1, "language": "en", "task": "transcribe"}
    if args.max_new_tokens:
        gk["max_new_tokens"] = args.max_new_tokens
    cells = []
    warm = S.synth_audio(45.0, seed=1)
    pipe(warm, chunk_length_s=0, return_timestamps=True, generate_kwargs=dict(gk))  # module loads, first graphs
    for n in counts:
        audios = [S.synth_audio(args.minutes * 60, seed=100 + i) for i in range(n)]
        for mode, call in (("long", {"chunk_length_s": 0}), ("long_cond", {"chunk_length_s": 0, "cond": True}),
                           ("chunked30", {"chunk_length_s": 30})):
            kw = dict(gk, condition_on_prev_tokens=bool(call.get("cond")))
            before, g0 = dict(eng.stats), eng.graph_stats()
            mel_ms.clear()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pipe(list(audios), chunk_length_s=call["chunk_length_s"], batch_size=n, return_timestamps=True, generate_kwargs=kw)
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
            d = {k: eng.stats[k] - before[k] for k in eng.stats}
            g = eng.graph_stats()
            cells.append({"audios": n, "mode": mode, "wall_s": round(wall, 3), "audio_s_per_s": round(n * args.minutes * 60 / wall, 1),
                          "windows_encoded": d["chunks_encoded"], "decoder_steps": d["decode_steps"], "prefill_passes": d["prefill_passes"],
                          "logmel_long_ms": round(sum(mel_ms), 3), "step_graphs_captured": g["captured"] - g0["captured"],
                          "graph_capture_s": round(g["capture_s"] - g0["capture_s"], 3), "step_graphs_cached": g["cached"],
                          "step_graphs_evicted": g["evicted"] - g0["evicted"]})
            print(json.dumps(cells[-1]), file=sys.stderr, flush=True)
    print(json.dumps({"bench": "longform", "minutes": args.minutes, "gpu": gpu_info(), "cells": cells}), flush=True)


if __name__ == "__main__":
    main()
