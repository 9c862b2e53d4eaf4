"""The public drop-in API on the GPU (ASRPipeline / StreamingPipeline through the C-ABI engine) against the real
reference's pipeline outputs (tests/golden/model_tiny10.json, minted by oracle/make_golden.py) and against the oracle
pipeline run live on the CPU.

What is exact and what is not: the host logic of the pipeline is compared EXACTLY with the reference on the CPU
(tests/test_host_cpu.py, stand-in engine), and per-step greedy parity modulo oracle near-ties is asserted rigorously in
tests/test_model_gpu.py.  At pipeline level a random-weight checkpoint has top-1/top-2 margins below the bf16 logit
error at some of the ~100 decode steps of a multi-chunk input, and one flipped token changes the rest of that chunk.  So
here texts must agree on a common prefix (>= 10 words) and overall (difflib ratio >= 0.6); word timestamps (DTW over
bf16-fed attention scores) are compared on the common prefix with a one-frame (0.02 s) tolerance on >= 90% of the words
and 0.1 s on the rest."""
import difflib
import json
import os

import numpy as np
import pytest
import torch

from tests.conftest import GOLD
from tests.parity_utils import DecodeRecorder as _DecodeRecorder, assert_oracle_greedy as _assert_oracle_greedy

pytestmark = pytest.mark.gpu


def _pipe(chunk_s=10, batch_size=4, preset=None, gain=None, **kw):
    from thewhisper_b200 import synthetic as S
    from thewhisper_b200.nvidia import ASRPipeline

    meta = json.load(open(os.path.join(GOLD, "model_tiny10.json")))
    model = S.make_hf_model(preset or meta["preset"], seed=0, layer_gain=gain or meta["layer_gain"])
    pipe = ASRPipeline(model, feature_extractor=S.make_feature_extractor(chunk_s), tokenizer=S.make_tokenizer(),
                       chunk_length_s=chunk_s, device="cuda", batch_size=batch_size, **kw)
    return meta, model, pipe


GK = {"num_beams": 1, "do_sample": False, "language": "en", "task": "transcribe", "max_new_tokens": 32}


def _check_text(got: str, ref: str, min_prefix=10, min_ratio=0.6):
    """Bounds well below the measured agreement: the checkpoints are chaotic by
    construction (layer_gain 8), so one near-tie flip changes everything after it."""
    a, b = got.split(), ref.split()
    n = 0
    while n < min(len(a), len(b)) and a[n] == b[n]:
        n += 1
    ratio = difflib.SequenceMatcher(None, a, b).ratio()
    print(f"\n[text] common prefix {n} of {len(b)} words (bound {min(min_prefix, len(b))}), difflib ratio {ratio:.3f} (bound {min_ratio})")
    assert n >= min(min_prefix, len(b)), (n, a[:12], b[:12])
    assert ratio >= min_ratio, ratio
    return n


def _check_words(got, ref):
    n = 0
    while n < min(len(got), len(ref)) and got[n]["text"] == ref[n]["text"]:
        n += 1
    assert n >= min(10, len(ref)), (n, got[:3], ref[:3])
    got, ref = got[:n], ref[:n]
    close = 0
    for g, r in zip(got, ref):
        for a, b in zip(g["timestamp"], r["timestamp"]):
            assert (a is None) == (b is None)
            if a is not None:
                assert abs(a - b) <= 0.1 + 1e-6, (g, r)
        close += all((a is None and b is None) or abs(a - b) <= 0.02 + 1e-6 for a, b in zip(g["timestamp"], r["timestamp"]))
    print(f"\n[words] {n} common-prefix words, {close} with both times within one frame (bound {0.9 * len(ref):.0f})")
    assert close >= 0.9 * len(ref), (close, len(ref))


def test_pipeline_plain_and_segments_match_reference(cuda):
    from thewhisper_b200 import synthetic as S

    meta, model, pipe = _pipe()
    audio = S.synth_audio(meta["audio_s"], seed=2000)
    out = pipe(audio.copy(), chunk_length_s=9, batch_size=4, generate_kwargs=dict(GK))
    _check_text(out["text"], meta["pipeline"]["plain"]["text"], min_prefix=24, min_ratio=0.7)  # measured 72 of 88 words, 0.886
    plain = out["text"]
    out = pipe(audio.copy(), chunk_length_s=9, batch_size=4, return_timestamps=True, generate_kwargs=dict(GK))
    ref = meta["pipeline"]["ts"]
    _check_text(out["text"], ref["text"], min_prefix=2)
    assert len(out["chunks"]) >= 1 and all(len(c["timestamp"]) == 2 for c in out["chunks"])
    # list input + smaller batches than chunks: the engine must give the same answer as with batch 4 (same kernels)
    outs = pipe([audio.copy(), audio[:80000].copy()], chunk_length_s=9, batch_size=2, generate_kwargs=dict(GK))
    _check_text(outs[0]["text"], plain, min_prefix=30, min_ratio=0.75)  # measured 88 of 88, 1.000
    assert isinstance(outs[1]["text"], str) and len(outs[1]["text"]) > 0


def test_pipeline_word_timestamps_match_reference(cuda):
    from thewhisper_b200 import synthetic as S

    meta, model, pipe = _pipe()
    audio = S.synth_audio(meta["audio_s"], seed=2000)
    out = pipe(audio.copy(), chunk_length_s=9, batch_size=4, return_timestamps="word", generate_kwargs=dict(GK))
    ref = meta["pipeline"]["word"]
    _check_text(out["text"], ref["text"], min_prefix=2)
    _check_words(json.loads(json.dumps(out["chunks"], default=float)), ref["chunks"])


def test_pipeline_beam_search_matches_reference(cuda):
    from thewhisper_b200 import synthetic as S

    # beam search on a random checkpoint is chaotic (one flipped candidate changes the rest of a window): run it on the float16 build of
    # the engine, whose logits are much closer to the fp32 reference than bf16's -- the reference's own
    # streaming / benchmark dtype.  Per-step candidate parity is pinned rigorously in test_model_gpu.py::test_beam_candidates_*.
    meta, model, pipe = _pipe(torch_dtype=torch.float16)
    audio = S.synth_audio(meta["audio_s"], seed=2000)
    out = pipe(audio.copy(), chunk_length_s=9, batch_size=4, generate_kwargs=dict(GK, num_beams=5))
    _check_text(out["text"], meta["pipeline"]["beam5"]["text"], min_prefix=16, min_ratio=0.7)  # measured 48 of 48, 1.000 (fp16 engine)


def test_pipeline_unusual_chunk_length(cuda):
    """chunk_length_s = 12 (S = 600 encoder positions): the reference interpolates its positional table for any chunk length
    (REF asr_pipeline.py:15-27); the engine does the same table and its kernels take any S.  Tie-aware replay through the oracle."""
    from oracle import hf_ref
    from thewhisper_b200 import synthetic as S

    meta, model, pipe = _pipe(chunk_s=12, batch_size=2)
    rec = _DecodeRecorder(pipe)
    audio = S.synth_audio(20.0, seed=2100)
    out = pipe(audio.copy(), chunk_length_s=11, batch_size=2, generate_kwargs=dict(GK))
    assert isinstance(out["text"], str) and len(out["text"].split()) >= 3
    om = S.make_hf_model(meta["preset"], seed=0, layer_gain=meta["layer_gain"])
    hf_ref.interpolate_positions(om, 12)
    near = _assert_oracle_greedy(rec.records, om, max_near_ties=4)
    print(f"\n[chunk 12 s] {sum(len(g) for r in rec.records for g in r['gen'])} tokens replayed through the oracle, {near} near ties")


def test_pipeline_word_timestamps_under_beam_search(cuda):
    """return_timestamps="word" with num_beams=5: alignment scores are kept per sequence slot on the device and the timestamp kernels
    gather each step's row from the slot that was the winner's ancestor (bw_word_timestamps_gather).  The host logic is pinned
    exactly against the real reference on the CPU stand-in (tests/test_host_cpu.py); here the CUDA path must reproduce the reference's
    words on the common prefix with DTW times within a frame."""
    from thewhisper_b200 import synthetic as S

    meta, model, pipe = _pipe(torch_dtype=torch.float16)  # (float16 build: see test_pipeline_beam_search_matches_reference)
    if "word_beam5" not in meta["pipeline"]:
        pytest.skip("golden predates the word + beam case")
    audio = S.synth_audio(meta["audio_s"], seed=2000)
    out = pipe(audio.copy(), chunk_length_s=9, batch_size=4, return_timestamps="word", generate_kwargs=dict(GK, num_beams=5))
    ref = meta["pipeline"]["word_beam5"]
    _check_text(out["text"], ref["text"], min_prefix=10, min_ratio=0.7)  # measured 24 of 24, 1.000
    got, want = json.loads(json.dumps(out["chunks"], default=float)), ref["chunks"]
    n = 0
    while n < min(len(got), len(want)) and got[n]["text"] == want[n]["text"]:
        n += 1
    assert n >= 6, (n, got[:8], want[:8])
    close = sum(all((a is None and b is None) or (a is not None and b is not None and abs(a - b) <= 0.02 + 1e-6)
                    for a, b in zip(g["timestamp"], r["timestamp"])) for g, r in zip(got[:n], want[:n]))
    print(f"\n[word+beam] {n} common-prefix words, {close} with both times within one frame of the reference")
    assert close >= 0.8 * n, (close, n)


def test_pipeline_vs_live_oracle_small30(cuda):
    """30 s windows, 3-layer model, word timestamps, against the oracle run on the CPU in the same test.
    (1) rigorous and tie-aware: every decode call the pipeline made is replayed through the oracle by teacher forcing --
    each token is the oracle's processed arg-max modulo oracle near ties; (2) when no near tie occurred, text and word
    timestamps must match the oracle PIPELINE's output (a random-weight checkpoint has top-2 margins below the bf16
    logit error at some steps, and one flipped token changes the rest of its window, so (2) alone is box-dependent)."""
    from oracle import hf_ref
    from thewhisper_b200 import synthetic as S

    meta, model, pipe = _pipe(chunk_s=30, batch_size=2, preset="small-test", gain=8.0)
    rec = _DecodeRecorder(pipe)
    audio = S.synth_audio(47.0, seed=4242)
    gk = dict(GK, max_new_tokens=24)
    got = pipe(audio.copy(), chunk_length_s=29, batch_size=2, return_timestamps="word", generate_kwargs=dict(gk))
    om = S.make_hf_model("small-test", seed=0, layer_gain=8.0)
    assert len(rec.records) >= 1 and sum(len(g) for r in rec.records for g in r["gen"]) >= 8
    near = _assert_oracle_greedy(rec.records, om)
    ref_pipe = hf_ref.make_ref_pipeline(om, S.make_feature_extractor(30), S.make_tokenizer(), chunk_length_s=30, device="cpu", batch_size=2)
    ref = ref_pipe(audio.copy(), chunk_length_s=29, batch_size=2, return_timestamps="word", generate_kwargs=dict(gk))
    if near == 0:
        _check_text(got["text"], ref["text"], min_prefix=4)
        _check_words(json.loads(json.dumps(got["chunks"], default=float)), json.loads(json.dumps(ref["chunks"], default=float)))
    else:
        _check_text(got["text"], ref["text"], min_prefix=2, min_ratio=0.3)


def test_streaming_on_engine(cuda):
    """StreamingPipeline + StreamScheduler over the real engine: 3 streams batched per tick give each stream what it
    gets alone (same engine, batch 1)."""
    from thewhisper_b200 import synthetic as S
    from thewhisper_b200.streaming import LocalWhisperBackend, StreamingPipeline, StreamScheduler

    meta, model, pipe = _pipe(chunk_s=10, batch_size=3)
    be = LocalWhisperBackend(None, chunk_length_s=10, asr_pipeline=pipe, language="en")
    audios = [S.synth_audio(12.0, seed=s) for s in (1, 2, 3)]
    sched = StreamScheduler(be, 3, chunk_length_s=10, min_process_chunk_s=0.5)
    solo = [StreamingPipeline(backend=be, use_vad=False, chunk_length_s=10, min_process_chunk_s=0.5) for _ in range(3)]
    n = 8000
    same = total = 0
    for i in range(0, 12 * 16000, n):
        chunks = [a[i:i + n] for a in audios]
        got = sched.step(chunks)
        want = [s(c) for s, c in zip(solo, chunks)]
        # words must agree; times may differ by batch composition exactly as in the reference, whose token timestamps
        # normalise over however many decoder steps the *batch* ran (generation_whisper.py:343-345)
        for (gc, gu), (wc, wu) in zip(got, want):
            a = [w["text"] for w in gc + gu]
            b = [w["text"] for w in wc + wu]
            same += sum(x == y for x, y in zip(a, b))
            total += max(len(a), len(b))
    print(f"\n[scheduler vs solo streams] {same} of {total} words equal (bound {0.7 * total:.0f})")
    assert total > 0 and same >= 0.7 * total, (same, total)  # (near-tie flips between batch-3 and batch-1 kernels allowed)
    assert sched.backend_calls < sched.buffers_transcribed
