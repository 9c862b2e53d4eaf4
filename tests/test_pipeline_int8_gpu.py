"""The public API with int8 decoder weights (ASRPipeline(decoder_weights="int8"), StreamingPipeline) on the golden tiny10 and
small30 checkpoints: greedy, segment and word timestamps, B = 1 vs B = 3 rows, beam candidates, a stream.

Greedy ids are held to the oracle (transformers) run on the SAME weights the engine computes with: the checkpoint with its
decoder matrices replaced by the dequantised s[n] * q[n, k] (the tie-aware replay of tests/parity_utils.py).  How far int8
lands from the unquantised checkpoint is measured and bounded separately, so that a loss of quantisation quality shows up."""
import copy
import json
import os

import numpy as np
import pytest
import torch

from tests.conftest import GOLD
from tests.parity_utils import DecodeRecorder, assert_oracle_greedy

pytestmark = pytest.mark.gpu

GK = {"num_beams": 1, "do_sample": False, "language": "en", "task": "transcribe", "max_new_tokens": 32}
# teacher-forced logits of the int8-dequantised checkpoint vs the unquantised one over the recorded greedy sequences:
# max |dlogit| / std(logits) and the count of teacher-forced positions whose arg-max differs, over the recorded greedy sequences
# (first two decode calls).  Measured on an H100 80GB HBM3 (700 W): tiny10 0.113 / 2, small30 0.218 / 7; bounds ~2-3x.
INT8_VS_FP = {"tiny10": (0.4, 5), "small30": (0.6, 20)}


def _dequantised(model):
    """The checkpoint with every decoder matrix the engine quantises replaced by s[n] * q[n, k] (fp32)."""
    from thewhisper_b200.engine import quantize_rows

    om = copy.deepcopy(model)
    sd = om.state_dict()
    names = ["model.decoder.embed_tokens.weight"]
    for i in range(om.config.decoder_layers):
        p = f"model.decoder.layers.{i}."
        names += [p + f"self_attn.{k}_proj.weight" for k in ("q", "k", "v")] + [p + "self_attn.out_proj.weight",
                  p + "encoder_attn.q_proj.weight", p + "encoder_attn.out_proj.weight", p + "fc1.weight", p + "fc2.weight"]
    with torch.no_grad():
        for n in names:
            if n.endswith(("k_proj.weight", "v_proj.weight")) and "self_attn" in n:
                continue  # fused with q below
            if n.endswith("self_attn.q_proj.weight"):
                b = n[: -len("q_proj.weight")]
                qkv = torch.cat([sd[b + "q_proj.weight"], sd[b + "k_proj.weight"], sd[b + "v_proj.weight"]], 0)
                q, s = quantize_rows(qkv)
                deq = (s[:, None].double() * q.double()).float()
                d = qkv.shape[1]
                for j, k in enumerate(("q", "k", "v")):
                    sd[b + f"{k}_proj.weight"].copy_(deq[j * d:(j + 1) * d])
                continue
            q, s = quantize_rows(sd[n])
            sd[n].copy_((s[:, None].double() * q.double()).float())
    return om  # (proj_out is tied to embed_tokens: the LM head reads the same dequantised rows)


def _setup(tag="tiny10", chunk_s=10, batch_size=4):
    from thewhisper_b200 import synthetic as S
    from thewhisper_b200.nvidia import ASRPipeline

    meta = json.load(open(os.path.join(GOLD, f"model_{tag}.json")))
    model = S.make_hf_model(meta["preset"], seed=meta["seed"], layer_gain=meta.get("layer_gain", 1.0))
    pipe = ASRPipeline(model, feature_extractor=S.make_feature_extractor(chunk_s), tokenizer=S.make_tokenizer(), chunk_length_s=chunk_s,
                       device="cuda", batch_size=batch_size, decoder_weights="int8")
    return meta, model, pipe


def _oracle(model, chunk_s):
    from oracle import hf_ref

    om = _dequantised(model).eval()
    hf_ref.interpolate_positions(om, chunk_s)
    return om


CASES = {"tiny10": (10, 9, 2000), "small30": (30, 29, 4242)}  # chunk_s, call chunk_length_s, audio seed


@pytest.mark.parametrize("tag", list(CASES))
def test_pipeline_int8_greedy_matches_dequantised_oracle(cuda, tag):
    from thewhisper_b200 import synthetic as S

    chunk_s, call_s, seed = CASES[tag]
    meta, model, pipe = _setup(tag, chunk_s)
    assert pipe.engine.decoder_weights == "int8"
    audio = S.synth_audio(min(meta.get("audio_s", 47.0), 47.0), seed=seed)
    rec = DecodeRecorder(pipe)
    out1 = pipe(audio.copy(), chunk_length_s=call_s, batch_size=1, generate_kwargs=dict(GK))
    out3 = pipe(audio.copy(), chunk_length_s=call_s, batch_size=3, generate_kwargs=dict(GK))
    assert out1["text"].split() and out3["text"].split()
    om = _oracle(model, chunk_s)
    near = assert_oracle_greedy(rec.records, om, max_near_ties=6)
    print(f"\n[int8 {tag} greedy] {sum(len(g) for r in rec.records for g in r['gen'])} ids, {near} near ties")

    # int8 vs the unquantised checkpoint on the same sequences: the cost of the quantisation itself
    from oracle import hf_ref

    fm = copy.deepcopy(model).eval()
    hf_ref.interpolate_positions(fm, chunk_s)
    worst, flips = 0.0, 0
    with torch.no_grad():
        for r in rec.records[:2]:
            for a in range(len(r["gen"])):
                ids = r["prompts"][a].tolist() + r["gen"][a].tolist()
                l8 = hf_ref.teacher_forced_logits(om, r["mel"][a], ids)
                lf = hf_ref.teacher_forced_logits(fm, r["mel"][a], ids)
                worst = max(worst, float(np.abs(l8 - lf).max() / lf.std()))
                flips += int((l8.argmax(-1) != lf.argmax(-1)).sum())
    b_lg, b_ids = INT8_VS_FP[tag]
    print(f"[int8 {tag}] vs the unquantised checkpoint: max |dlogit| / std {worst:.4f} (bound {b_lg}), "
          f"{flips} differing greedy ids (bound {b_ids})")
    assert worst < b_lg and flips <= b_ids


def _int8_engine(monkeypatch):
    """tests/test_model_gpu.py's engine factory with int8 decoder weights: its batch and beam tests run unchanged on them."""
    from tests import test_model_gpu as M

    orig = M._engine
    monkeypatch.setattr(M, "_engine", lambda model, chunk_s, **kw: orig(model, chunk_s, decoder_weights="int8", **kw))
    return M


@pytest.mark.parametrize("path", ["mega", "perop", "batched", "batched-xstream"])
def test_int8_batch_rows_agree(cuda, path, monkeypatch):
    """B = 3 audios decoded together give the tokens of the B = 1 runs, on every step path."""
    _int8_engine(monkeypatch).test_batch_rows_agree(cuda, path, monkeypatch)


@pytest.mark.parametrize("ts", [False, True], ids=["plain", "timestamps"])
@pytest.mark.parametrize("path", ["perop", "batched"])
def test_int8_beam_candidates_match_transformers(cuda, ts, path, monkeypatch):
    """Beam candidates (2G per sequence) against transformers' processors applied to the engine's own int8 logits."""
    _int8_engine(monkeypatch).test_beam_candidates_match_transformers(cuda, ts, path, monkeypatch)


def test_pipeline_int8_timestamps_beams_and_streaming(cuda):
    from thewhisper_b200 import synthetic as S
    from thewhisper_b200.streaming import StreamingPipeline

    meta, model, pipe = _setup()
    audio = S.synth_audio(meta["audio_s"], seed=2000)
    ref16 = json.load(open(os.path.join(GOLD, "model_tiny10.json")))["pipeline"]
    seg = pipe(audio.copy(), chunk_length_s=9, batch_size=4, return_timestamps=True, generate_kwargs=dict(GK))
    assert seg["chunks"] and all(c["timestamp"][0] is not None for c in seg["chunks"])
    starts = [c["timestamp"][0] for c in seg["chunks"]]
    assert starts == sorted(starts) and all(0.0 <= t <= meta["audio_s"] + 1 for t in starts)
    words = pipe(audio.copy(), chunk_length_s=9, batch_size=4, return_timestamps="word", generate_kwargs=dict(GK))
    ts = [c["timestamp"] for c in words["chunks"]]
    assert ts and all(a is not None and b is not None and a <= b for a, b in ts[:-1])
    assert all(x[0] <= y[0] + 1e-6 for x, y in zip(ts, ts[1:]))  # word starts never go backwards
    # the text agrees with the reference pipeline's word-mode text on a common prefix (quantisation may flip a near tie later)
    a, b = words["text"].split(), ref16["word"]["text"].split()
    n = 0
    while n < min(len(a), len(b)) and a[n] == b[n]:
        n += 1
    print(f"\n[int8 tiny10 words] common prefix with the 16-bit reference {n} of {len(b)} words")
    assert n >= min(2, len(b)), (a[:8], b[:8])
    beam = pipe(audio.copy(), chunk_length_s=9, batch_size=2, generate_kwargs=dict(GK, num_beams=5))
    assert beam["text"].split()
    print(f"\n[int8 tiny10] segments {len(seg['chunks'])}, words {len(ts)}, beam-5 words {len(beam['text'].split())}")

    sp = StreamingPipeline(model=model, chunk_length_s=10, feature_extractor=S.make_feature_extractor(10),
                           tokenizer=S.make_tokenizer(), use_vad=False, decoder_weights="int8")
    assert sp.backend.asr_pipeline.engine.decoder_weights == "int8"
    stream = S.synth_audio(12.0, seed=1)
    committed = []
    for i in range(0, len(stream), 8000):
        c, u = sp(stream[i:i + 8000])
        committed += c
    print(f"[int8 stream] {len(committed)} committed words, last uncommitted {len(u)}")
    assert committed or u
