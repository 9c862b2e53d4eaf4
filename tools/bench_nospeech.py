"""Cost of no-speech skipping at large-v3 shapes with random weights.

    python tools/bench_nospeech.py [--runs 3] [--tokens 128] [--minutes 10] [--audios 1,16] [--max-new-tokens 0] [--skip-step] [--skip-long]

1. Decoder step time with scores off and on (engine.decode_scores_enable), the two alternating `--runs` times, CUDA events around
   `--tokens` greedy steps after the init tokens: Q = 1 (the persistent step with its fused select, against the persistent step and
   select_kernel), Q = 2 (persistent + select_kernel both ways, with the timestamp rules), Q = 64 (the batched step) and 64 audios
   x 5 beams (beam steps, which synchronise with the host every step).
2. Long form on 10-minute audios with silent stretches, 1 and 16 at a time: without thresholds; with thresholds that skip every
   window (avg_logprob below 0 and no_speech_prob above 0: random weights model no speech); conditioned without thresholds; and
   conditioned with thresholds that skip nothing (no_speech_prob above 1), which pays for the scores and for the
   <|startoftranscript|> split on every window without changing the transcript.  Per cell: wall time, windows, windows skipped,
   decoder steps, and the forced steps the split adds (positions a conditioned window runs as steps instead of in the prefill).
Prints one JSON line with the GPU name, power limit and SM clock read in the same call.
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

SKIP_ALL = {"no_speech_threshold": 0.0, "logprob_threshold": 0.0, "temperature": 0.0}
KEEP_ALL = {"no_speech_threshold": 1.0, "logprob_threshold": 0.0, "temperature": 0.0}  # scores on, no window skipped


def step_cells(args, torch, S):
    from thewhisper_b200.engine import DecodeOptions, ModelDims, WhisperEngine, pack_weights

    dev = torch.device("cuda:0")
    model = S.make_hf_model("large-v3", seed=0)
    dims = ModelDims.from_hf_config(model.config)
    sd = model.state_dict()
    weights = pack_weights(sd, dims, sd["model.encoder.embed_positions.weight"].float(), dev, torch.float16)
    g = model.generation_config
    del sd, model
    init = [S.SOT, S.LANG_EN, S.TRANSCRIBE]
    out = []
    for name, A, G, ts in (("Q1", 1, 1, False), ("Q2_ts", 2, 1, True), ("Q64", 64, 1, False), ("Q64x5_beam", 64, 5, True)):
        eng = WhisperEngine(None, dims, chunk_length_s=30, max_audios=A, max_beams=G, weights=weights)
        pcm = torch.from_numpy(np.stack([S.synth_audio(30.0, seed=1000 + i) for i in range(A)])).to(dev)
        eng.logmel_device(pcm, A)
        eng.encode(A)
        opts = DecodeOptions(eos_token=S.EOS, pad_token=S.EOS, suppress_tokens=list(g.suppress_tokens) + [S.EOS],
                             begin_suppress_tokens=list(g.begin_suppress_tokens), timestamp_rules=ts,
                             max_initial_timestamp_index=50 if ts else -1)
        prompt = np.array([init + ([] if ts else [S.NOTIMESTAMPS])] * (A * G), dtype=np.int32)
        tokens = args.tokens if G == 1 else max(8, args.tokens // 8)

        def run(scores):
            eng.decode_begin(prompt, A, G, opts)
            if scores:
                eng.decode_scores_enable(0, S.NOSPEECH)
            eng.decode_run(prompt.shape[1] - 1)
            k0 = eng.decode_kernel_launches()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            if G == 1:
                eng.decode_run(tokens)
            else:
                run_scores = np.zeros(A * G, dtype=np.float32)
                for _ in range(tokens):  # candidate lists only: the step and its host round trip, no beam bookkeeping
                    eng.decode_beam_step(run_scores)
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / tokens, (eng.decode_kernel_launches() - k0) / tokens

        run(False), run(True)  # graph capture, module loads
        ms = {False: [], True: []}
        kern = {}
        for _ in range(args.runs):
            for sc in (False, True):
                t, kern[sc] = run(sc)
                ms[sc].append(t)
        off, on = float(np.median(ms[False])), float(np.median(ms[True]))
        out.append({"cell": name, "audios": A, "beams": G, "timestamp_rules": ts, "steps_timed": tokens,
                    "step_ms_off": off, "step_ms_on": on, "step_ms_off_runs": ms[False], "step_ms_on_runs": ms[True],
                    "extra_us_per_step": (on - off) * 1e3, "kernels_per_step_off": kern[False], "kernels_per_step_on": kern[True]})
        print(json.dumps(out[-1]), file=sys.stderr, flush=True)
        eng.close()
        del eng
        torch.cuda.empty_cache()
    return out


def long_cells(args, torch, S):
    from thewhisper_b200.nvidia import ASRPipeline

    counts = [int(x) for x in args.audios.split(",")]
    model = S.make_hf_model("large-v3", seed=0)
    pipe = ASRPipeline(model, feature_extractor=S.make_feature_extractor(30), tokenizer=S.make_tokenizer(), chunk_length_s=30,
                       device="cuda", torch_dtype=torch.float16, batch_size=max(counts))
    eng = pipe.engine
    gk = {"num_beams": 1, "language": "en", "task": "transcribe"}
    if args.max_new_tokens:
        gk["max_new_tokens"] = args.max_new_tokens
    pipe(S.synth_audio(45.0, seed=1), chunk_length_s=0, return_timestamps=True, generate_kwargs=dict(gk))  # module loads
    pipe(S.synth_audio(45.0, seed=1), chunk_length_s=0, return_timestamps=True, generate_kwargs=dict(gk, **SKIP_ALL))
    out = []

    def silent(sec, seed):
        a = S.synth_audio(sec, seed=seed)
        for k in range(0, int(sec), 120):  # a minute of silence every two minutes
            a[(k + 30) * 16000:(k + 90) * 16000] = 0.0
        return a

    for n in counts:
        audios = [silent(args.minutes * 60, 100 + i) for i in range(n)]
        for mode, kw in (("long", {}), ("long_skip_all", SKIP_ALL), ("long_cond", {"condition_on_prev_tokens": True}),
                         ("long_cond_scores", dict(KEEP_ALL, condition_on_prev_tokens=True))):
            before = dict(eng.stats)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pipe(list(audios), chunk_length_s=0, batch_size=n, return_timestamps=True, generate_kwargs=dict(gk, **kw))
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
            d = {k: eng.stats[k] - before[k] for k in eng.stats}
            ws = pipe.generator.window_stats
            out.append({"audios": n, "mode": mode, "wall_s": round(wall, 3), "windows": ws["windows"], "windows_skipped": ws["skipped"],
                        "conditioned_windows": ws["conditioned"], "decoder_steps": d["decode_steps"],
                        "sot_split_steps": d["sot_split_steps"], "prefill_passes": d["prefill_passes"]})
            print(json.dumps(out[-1]), file=sys.stderr, flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--tokens", type=int, default=128)
    ap.add_argument("--minutes", type=float, default=10.0)
    ap.add_argument("--audios", default="1,16")
    ap.add_argument("--max-new-tokens", type=int, default=0)
    ap.add_argument("--skip-step", action="store_true")
    ap.add_argument("--skip-long", action="store_true")
    args = ap.parse_args()

    import torch

    from thewhisper_b200 import synthetic as S

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU")
    result = {"bench": "nospeech", "gpu": gpu_info()}
    if not args.skip_step:
        result["step"] = step_cells(args, torch, S)
    if not args.skip_long:
        result["long"] = long_cells(args, torch, S)
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
