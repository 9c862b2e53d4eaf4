"""Mint golden vectors from the *real* reference (build container only).

    THESTAGE_REFERENCE=<checkout of TheStageAI/TheWhisper> python oracle/make_golden.py [--large]

Imports `thestage_speechkit` from that checkout (it does not travel with the tests), runs its own
`ASRPipeline` (HF branch) and its own `_find_longest_common_sequence` on deterministic synthetic
inputs, asserts that the restatement in oracle/hf_ref.py reproduces them output-for-output, and writes
small fixtures to tests/golden/.  This is what pins the oracle (task statement ③); the reference
itself ships no tests or golden vectors (SURVEY.md §4).
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")

from thewhisper_b200 import synthetic as S  # noqa: E402
from oracle import hf_ref  # noqa: E402


def _import_reference():
    import transformers  # noqa: F401  (must be imported before the reference, SURVEY.md §8c)
    ref = os.environ.get("THESTAGE_REFERENCE")
    if not ref or not os.path.isdir(os.path.join(ref, "thestage_speechkit")):
        raise SystemExit("make_golden.py: set THESTAGE_REFERENCE to a checkout of TheStageAI/TheWhisper "
                         f"(the directory that holds thestage_speechkit/); got {ref!r}")
    sys.path.insert(0, ref)
    import thestage_speechkit  # noqa: F401  (installs its LCS patch)
    from thestage_speechkit.nvidia import ASRPipeline
    from thestage_speechkit import _find_longest_common_sequence as ref_lcs
    return ASRPipeline, ref_lcs


def _ref_pipe(ASRPipeline, model, chunk_length_s):
    fe = S.make_feature_extractor(chunk_length_s)
    tok = S.make_tokenizer()
    pipe = ASRPipeline(model, feature_extractor=fe, tokenizer=tok, chunk_length_s=chunk_length_s,
                       device="cpu", batch_size=4)
    if chunk_length_s < 30:  # transformers>=5 shim (SURVEY.md §8c (i)); the reference predates it
        model.model.encoder.embed_positions.num_embeddings = model.config.max_source_positions
    return pipe, fe, tok


def golden_mel():
    out = {}
    for secs in (10, 15, 30):
        fe = S.make_feature_extractor(secs)
        m = hf_ref.logmel(fe, S.two_tone(secs))
        out[f"two_tone_{secs}s_stats"] = np.array([m.mean(), m.min(), m.max(), m[0, 0], m[10, 100], m[64, m.shape[1] // 2],
                                                   m[127, -1]], dtype=np.float64)
        out[f"two_tone_{secs}s_sub"] = m[:, ::25].copy()
    fe = S.make_feature_extractor(10)
    x = (np.random.RandomState(0).randn(160000) * 0.1).astype(np.float32)
    m = hf_ref.logmel(fe, x)
    out["noise_10s_sub"] = m[:, ::10].copy()
    out["noise_10s_stats"] = np.array([m.mean(), m.min(), m.max()], dtype=np.float64)
    # short (7.3 s) input in a 10 s window: exercises zero padding + attention mask
    x = S.synth_audio(7.3, seed=11)
    o = fe(x, sampling_rate=16000, return_tensors="np", return_attention_mask=True)
    out["speech_7p3s_sub"] = np.asarray(o["input_features"][0][:, ::10], dtype=np.float32)
    out["speech_7p3s_mask_sum"] = np.array([int(o["attention_mask"][0].sum())])
    bank = np.asarray(fe.mel_filters, dtype=np.float64)  # [201,128]
    out["mel_bank_sum_nnz"] = np.array([bank.sum(), (bank != 0).sum()], dtype=np.float64)
    out["mel_bank"] = bank.astype(np.float32)
    np.savez_compressed(os.path.join(GOLD, "logmel.npz"), **out)
    print("logmel.npz", {k: v.shape for k, v in out.items()})


def golden_lcs(ref_lcs):
    rng = np.random.RandomState(7)
    cases = []
    for c in range(40):
        nseq = rng.randint(2, 5)
        base = rng.randint(0, 30, size=rng.randint(20, 60)).tolist()
        seqs, pos = [], 0
        for s in range(nseq):
            ln = rng.randint(6, 20)
            piece = base[pos:pos + ln]
            if rng.rand() < 0.5 and len(piece) > 3:  # perturb so matches are imperfect
                piece = list(piece)
                piece[rng.randint(len(piece))] = int(rng.randint(30, 40))
            seqs.append(list(map(int, piece)))
            pos += max(1, ln - rng.randint(1, 6))
        with_ts = c % 2 == 1
        if with_ts:
            tss = []
            t = 0.0
            for s in seqs:
                ts = []
                tt = t + 0.003 * len(tss)  # distinct starts per sequence: (a,b)<=(a,None) would raise in REF
                for j in range(len(s)):
                    e = tt + 0.2
                    ts.append((round(tt, 3), None if (j == len(s) - 1 and rng.rand() < 0.5) else round(e, 3)))
                    tt = e
                tss.append(ts)
                t += 0.2 * max(1, len(s) - 3)
            a = ref_lcs([list(s) for s in seqs], [list(t) for t in tss])
            b = hf_ref.lcs_merge(seqs, tss)
            assert a[0] == b[0] and a[1] == b[1], (c, a, b)
            cases.append({"seqs": seqs, "ts": tss, "out": a[0], "out_ts": a[1]})
        else:
            a = ref_lcs([list(s) for s in seqs])
            b = hf_ref.lcs_merge(seqs)
            assert a == b, (c, a, b)
            cases.append({"seqs": seqs, "out": a})
    with open(os.path.join(GOLD, "lcs_cases.json"), "w") as f:
        json.dump(cases, f)
    print("lcs_cases.json", len(cases))


def _jsonable(o):
    if isinstance(o, dict):
        return {k: _jsonable(v) for k, v in o.items()}
    if isinstance(o, (list, tuple)):
        return [_jsonable(v) for v in o]
    if isinstance(o, (np.floating, float)):
        return float(o)
    if isinstance(o, (np.integer, int)):
        return int(o)
    return o


def golden_model(ASRPipeline, preset, tag, chunk_s, audio_s, n_tf=24, max_new=32, do_pipeline=True, gain=1.0):
    """Per-stage taps + end-to-end pipeline outputs of the real reference for one random checkpoint."""
    t0 = time.time()
    model = S.make_hf_model(preset, seed=0, layer_gain=gain)
    pipe, fe, tok = _ref_pipe(ASRPipeline, model, chunk_s)
    out = {}
    meta = {"preset": preset, "chunk_s": chunk_s, "seed": 0, "layer_gain": gain}
    audio = S.synth_audio(chunk_s, seed=1000)
    mel = hf_ref.logmel(fe, audio)
    enc = hf_ref.encoder_out(model, mel)
    out["enc_sub"] = enc[::max(1, enc.shape[0] // 50), ::max(1, enc.shape[1] // 64)].copy()
    out["enc_stats"] = np.array([enc.mean(), enc.std(), np.abs(enc).max()], dtype=np.float64)
    # teacher-forced logits over a random token sequence
    rng = np.random.RandomState(5)
    ids = [S.SOT, S.LANG_EN, S.TRANSCRIBE, S.NOTIMESTAMPS] + rng.randint(256, 50000, size=n_tf).tolist()
    lg = hf_ref.teacher_forced_logits(model, mel, ids)
    top = np.argsort(-lg, axis=1)[:, :8]
    out["tf_ids"] = np.array(ids, dtype=np.int64)
    out["tf_top_ids"] = top.astype(np.int64)
    out["tf_top_vals"] = np.take_along_axis(lg, top, axis=1).astype(np.float32)
    out["tf_lse"] = torch.logsumexp(torch.from_numpy(lg), dim=-1).numpy().astype(np.float32)
    out["tf_cols"] = lg[:, ::997].astype(np.float32)
    # free-running greedy, no timestamps, EOS free
    g = hf_ref.generate(model, mel[None], language="en", task="transcribe", max_new_tokens=max_new,
                        num_beams=1, do_sample=False)
    out["greedy_tokens"] = np.asarray(g[0] if not isinstance(g, dict) else g["sequences"][0], dtype=np.int64)
    if do_pipeline:
        long_audio = S.synth_audio(audio_s, seed=2000)
        gk = {"num_beams": 1, "do_sample": False, "language": "en", "task": "transcribe", "max_new_tokens": max_new}
        res = {}
        res["plain"] = pipe(long_audio.copy(), chunk_length_s=chunk_s - 1, batch_size=4, generate_kwargs=dict(gk))
        res["ts"] = pipe(long_audio.copy(), chunk_length_s=chunk_s - 1, batch_size=4, return_timestamps=True,
                         generate_kwargs=dict(gk))
        res["word"] = pipe(long_audio.copy(), chunk_length_s=chunk_s - 1, batch_size=4, return_timestamps="word",
                           generate_kwargs=dict(gk))
        gk5 = dict(gk, num_beams=5)
        res["beam5"] = pipe(long_audio.copy(), chunk_length_s=chunk_s - 1, batch_size=4, generate_kwargs=gk5)
        # word timestamps under beam search: cross-attention rows gathered along the winner's ancestry (beam_indices)
        res["word_beam5"] = pipe(long_audio.copy(), chunk_length_s=chunk_s - 1, batch_size=4, return_timestamps="word", generate_kwargs=gk5)
        # the restated glue must reproduce the reference exactly
        model2 = S.make_hf_model(preset, seed=0, layer_gain=gain)
        pipe2 = hf_ref.make_ref_pipeline(model2, S.make_feature_extractor(chunk_s), tok, chunk_length_s=chunk_s,
                                         device="cpu", batch_size=4)
        for key, kw in (("plain", {}), ("ts", {"return_timestamps": True}), ("word", {"return_timestamps": "word"})):
            r2 = pipe2(long_audio.copy(), chunk_length_s=chunk_s - 1, batch_size=4, generate_kwargs=dict(gk), **kw)
            assert _jsonable(r2) == _jsonable(res[key]), (key, r2, res[key])
        meta["pipeline"] = _jsonable(res)
        meta["audio_s"] = audio_s
    meta["seconds"] = time.time() - t0
    np.savez_compressed(os.path.join(GOLD, f"model_{tag}.npz"), **out)
    with open(os.path.join(GOLD, f"model_{tag}.json"), "w") as f:
        json.dump(meta, f, indent=1)
    print(f"model_{tag}: {time.time() - t0:.1f}s greedy={out['greedy_tokens'][:12]}")


STREAM_VOCAB = ["The", "quick,", "brown", "fox.", "It", "jumps", "over;", "lazy", "dogs!", "gonNA", ".", "-run", "and", "then",
                "stops?", "we", "wanNA", "go", "now:", "ok"]


class FakeWordBackend:
    """Deterministic stand-in for the ASR backend: one word per 0.4 s of absolute time, so re-transcriptions of a
    growing buffer agree with each other; used to pin the streaming state machine independently of any model."""

    def __init__(self):
        self.calls = []

    def transcribe(self, audio, buffer_start_time, sample_rate):
        dur = len(audio) / sample_rate
        self.calls.append(round(dur, 4))
        words = []
        k = int(np.ceil(buffer_start_time / 0.4 - 1e-9))
        while k * 0.4 + 0.3 <= buffer_start_time + dur:
            if k % 13 != 7:  # a pause now and then
                words.append({"text": (" " if k % 5 else "") + STREAM_VOCAB[k % len(STREAM_VOCAB)], "start": round(k * 0.4, 4),
                              "end": round(k * 0.4 + 0.3, 4)})
            k += 1
        return words


class FakeVad:
    def __call__(self, chunk, sr):
        return torch.tensor(1.0 if float(chunk.abs().mean()) > 0.01 else 0.0)

    def reset_states(self):
        pass


def stream_audio(seconds=40.0):
    x = S.synth_audio(seconds, seed=77, kind="noise")
    t = np.arange(len(x)) / 16000.0
    x[(t % 9.0) > 6.5] = 0.0  # 2.5 s of silence every 9 s
    return x


def golden_streaming():
    import importlib.machinery
    import types

    for name, attrs in (("sounddevice", ["InputStream"]), ("librosa", ["load", "resample"])):
        if name not in sys.modules:
            m = types.ModuleType(name)
            m.__spec__ = importlib.machinery.ModuleSpec(name, None)
            for a in attrs:
                setattr(m, a, None)
            sys.modules[name] = m
    from thestage_speechkit.streaming.streaming_pipeline import StreamingPipeline as RefStreaming

    out = {}
    audio = stream_audio()
    for tag, use_vad, step_s in (("novad_0p5", False, 0.5), ("novad_0p05", False, 0.05), ("vad_0p05", True, 0.05)):
        be = FakeWordBackend()
        if use_vad:
            orig = torch.hub.load
            torch.hub.load = lambda *a, **k: (FakeVad(), None)
        try:
            sp = RefStreaming(backend=be, use_vad=use_vad, chunk_length_s=15, min_process_chunk_s=0.5)
        finally:
            if use_vad:
                torch.hub.load = orig
        n = int(step_s * 16000)
        events = []
        for i in range(0, len(audio), n):
            c, u = sp(audio[i:i + n])
            if c or u:
                events.append([i // n, _jsonable(c), _jsonable(u)])
        out[tag] = {"step_s": step_s, "use_vad": use_vad, "backend_calls": be.calls, "events": events}
        print("streaming", tag, "calls", len(be.calls), "events", len(events), "max buffer", max(be.calls))
    with open(os.path.join(GOLD, "streaming.json"), "w") as f:
        json.dump(out, f)


def golden_decode_asr(ref_lcs):
    """Inputs and outputs of `WhisperTokenizer._decode_asr` with the REAL reference seam merge installed (the state `import thestage_speechkit`
    leaves the tokenizer module in): 2 x 240 random calls of oracle/decode_asr_cases.py, raised IndexErrors included."""
    from oracle import decode_asr_cases as DC

    rng = np.random.RandomState(20260923)
    cases = []
    n_raise = 0
    for kind in ("plain", "special"):  # only <|endoftext|> special (the synthetic tokenizer) / every control token special (released checkpoints)
        tok = DC.tokenizer_of(kind)
        n_kind = 0
        while n_kind < 240:
            case = DC.random_case(rng, tok)
            expect = DC.reference_result(case, tok, ref_lcs)
            again = DC.reference_result(case, tok, hf_ref.lcs_merge)  # the restated merge must not change anything
            assert expect == again, (case, expect, again)
            if "raises" in expect:
                n_raise += 1
                if n_raise > 24:
                    continue
            cases.append({"tokenizer": kind, "case": case, "expect": expect})
            n_kind += 1
    with open(os.path.join(GOLD, "decode_asr_cases.json"), "w") as f:
        json.dump(cases, f)
    print("decode_asr_cases.json", len(cases), "cases,", n_raise, "raising")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--large", action="store_true", help="also mint the large-v3-dims goldens (minutes)")
    ap.add_argument("--only", default="")
    a = ap.parse_args()
    os.makedirs(GOLD, exist_ok=True)
    ASRPipeline, ref_lcs = _import_reference()
    torch.set_num_threads(8)
    if a.only in ("", "mel"):
        golden_mel()
    if a.only in ("", "lcs"):
        golden_lcs(ref_lcs)
    if a.only in ("", "stream"):
        golden_streaming()
    if a.only in ("", "decode_asr"):
        golden_decode_asr(ref_lcs)
    if a.only in ("", "tiny"):
        golden_model(ASRPipeline, "tiny-test", "tiny10", chunk_s=10, audio_s=25.0, gain=8.0)
        golden_model(ASRPipeline, "small-test", "small30", chunk_s=30, audio_s=70.0, gain=8.0)
    if a.large:
        # the BASELINE.json configs C1 / C2 at their real dimensions.  layer_gain 4: with the plain HF init these sizes collapse to
        # one repeated token whatever the audio (gain 1 -> 29511 x 16); gain 4 gives varied, audio-dependent sequences
        golden_model(ASRPipeline, "large-v3-turbo", "turbo10", chunk_s=10, audio_s=10.0, n_tf=12, max_new=16,
                     do_pipeline=False, gain=4.0)
        golden_model(ASRPipeline, "large-v3", "large30", chunk_s=30, audio_s=30.0, n_tf=12, max_new=32,
                     do_pipeline=False, gain=4.0)


if __name__ == "__main__":
    main()
