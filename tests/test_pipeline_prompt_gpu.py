"""ASRPipeline with generate_kwargs["prompt_ids"] on the GPU, in every mode (plain, segment and word timestamps, beam 5 on the
fp16 engine, int8 decoder weights, tiny10 and small30, two prompt lengths in one pipeline):
  * each decode call runs prompt + init tokens as its decoder input and its forced positions as one decode_prefill;
  * greedy modes: every recorded decode call replays through the transformers model run live on the CPU (the dequantised
    checkpoint for int8) with the prompt in its decoder ids, tie-aware: a token is accepted when it is the oracle's processed
    arg-max, or its processed score is within the bf16 logit tolerance of it (a near tie, counted);
  * beam 5: the transcript against the transformers pipeline run live on the CPU with the same generate_kwargs (per-step beam
    candidate parity is pinned in tests/test_model_gpu.py).
The host logic of the prompted path is compared exactly with transformers in tests/test_prompt_cpu.py."""
import json
import os

import numpy as np
import pytest
import torch

from tests.conftest import GOLD
from tests.test_pipeline_gpu import _check_text

pytestmark = pytest.mark.gpu

GK = {"num_beams": 1, "do_sample": False, "language": "en", "task": "transcribe", "max_new_tokens": 32}


class _Recorder:
    """parity_utils.DecodeRecorder for the prompted path (its _decode takes the prefill flag)."""

    def __init__(self, pipe):
        self.records = []
        gen, eng = pipe.generator, pipe.engine
        og, os_, od = gen.generate, eng.set_mel, gen._decode
        self._mel = None

        def generate(B, **kw):
            self._mel = kw["mel_f32"].float().cpu().numpy()[:B]
            return og(B, **kw)

        def set_mel(m):
            self._mel = m.float().cpu().numpy()
            return os_(m)

        def _decode(prompts, A, opts, max_new, num_beams, **kw):
            out = od(prompts, A, opts, max_new, num_beams, **kw)
            self.records.append({"mel": self._mel[:A].copy(), "prompts": np.array(prompts), "gen": [np.asarray(g) for g in out[0]],
                                 "eos_seen": list(out[2]), "opts": opts, "max_new": max_new})
            return out

        gen.generate, eng.set_mel, gen._decode = generate, set_mel, _decode


def _pipes(name, **kw):
    from oracle import hf_ref
    from thewhisper_b200 import synthetic as S
    from thewhisper_b200.nvidia import ASRPipeline

    meta = json.load(open(os.path.join(GOLD, f"model_{name}.json")))
    chunk = meta["chunk_s"]
    model = S.make_hf_model(meta["preset"], seed=0, layer_gain=meta["layer_gain"])
    pipe = ASRPipeline(model, feature_extractor=S.make_feature_extractor(chunk), tokenizer=S.make_tokenizer(), chunk_length_s=chunk,
                       device="cuda", batch_size=4, **kw)
    om = S.make_hf_model(meta["preset"], seed=0, layer_gain=meta["layer_gain"])
    if kw.get("decoder_weights") == "int8":
        from tests.test_pipeline_int8_gpu import _dequantised

        om = _dequantised(om)
    om.eval()
    ref = hf_ref.make_ref_pipeline(om, S.make_feature_extractor(chunk), S.make_tokenizer(), chunk_length_s=chunk)
    return meta, pipe, ref, om


def replay_greedy(records, om, max_near_ties):
    """Every recorded token must be the oracle's processed arg-max given the same decoder ids (teacher forcing through the HF
    model + oracle/whisper_ref.process_logits), or score within the bf16 logit tolerance of it; with timestamp rules, also the
    choice the rule makes when its own margin is inside the tolerance.  Returns the number of such near ties."""
    from oracle import hf_ref, whisper_ref

    near = 0
    for rec in records:
        o = rec["opts"]
        for a in range(len(rec["gen"])):
            prompt = rec["prompts"][a].tolist()
            gen = rec["gen"][a].tolist() + ([o.eos_token] if rec["eos_seen"][a] else [])
            if not gen:
                continue
            plen = len(prompt)
            lg = hf_ref.teacher_forced_logits(om, rec["mel"][a], prompt + gen)
            for i, tok in enumerate(gen):
                row = lg[plen - 1 + i]
                tol = 0.16 * float(row.std()) + 2e-3
                s, pre, rule_margin = whisper_ref.process_logits(
                    row, prompt + gen[:i], plen, suppress=list(o.suppress_tokens), begin_suppress=list(o.begin_suppress_tokens),
                    ts_rules=bool(o.timestamp_rules), ts_begin=o.timestamp_begin, no_ts=o.no_timestamps_token, eos=o.eos_token,
                    max_initial_ts=(o.max_initial_timestamp_index if o.max_initial_timestamp_index >= 0 else None), details=True)
                best = int(np.argmax(s))
                if tok == best:
                    continue
                ok = np.isfinite(s[tok]) and s[best] - s[tok] < tol
                if not ok and o.timestamp_rules and abs(rule_margin) < tol:
                    alt = pre.copy()
                    if rule_margin <= 0:  # the rule did not fire in the oracle; it may fire under bf16 noise
                        alt[: o.timestamp_begin] = -np.inf
                    ok = tok == int(np.argmax(alt))
                assert ok, (a, i, tok, best, float(s[best] - s[tok]), rule_margin, tol)
                near += 1
    assert near <= max_near_ties, near
    return near


CASES = [("tiny10", "plain", {}), ("tiny10", "ts", {}), ("tiny10", "word", {}), ("tiny10", "beam5", {"torch_dtype": torch.float16}),
         ("tiny10", "plain", {"decoder_weights": "int8"}), ("small30", "plain", {})]


@pytest.mark.parametrize("name,mode,kw", CASES, ids=[f"{n}-{m}-{'-'.join(map(str, k.values())) or 'bf16'}" for n, m, k in CASES])
def test_prompted_pipeline_matches_transformers(cuda, name, mode, kw):
    from thewhisper_b200 import synthetic as S

    meta, pipe, ref, om = _pipes(name, **kw)
    tok = S.make_tokenizer()
    prompt = torch.tensor(tok.get_prompt_ids(" Kubernetes, gRPC and Hopper"))
    audio = S.synth_audio(min(meta["audio_s"], 20.0), seed=2000)
    gk = dict(GK, num_beams=5 if mode == "beam5" else 1, prompt_ids=prompt)
    rk = {"ts": {"return_timestamps": True}, "word": {"return_timestamps": "word"}}.get(mode, {})
    rec = _Recorder(pipe)
    eng = pipe.engine
    calls, orun, opre = [], eng.decode_run, eng.decode_prefill
    eng.decode_run = lambda n: (calls.append(("run", n)), orun(n))[1]
    eng.decode_prefill = lambda n, *a: (calls.append(("prefill", n)), opre(n, *a))[1]
    got = pipe(audio.copy(), chunk_length_s=meta["chunk_s"] - 1, batch_size=4, generate_kwargs=dict(gk), **rk)
    assert rec.records
    # the prefill ran: one decode_prefill(plen - 1) per decode call, no decode_run over the forced positions
    for r in rec.records:
        plen = r["prompts"].shape[1]
        assert plen >= len(prompt) + 3 and (r["prompts"][:, : len(prompt)] == prompt.numpy()).all()
    plens = [r["prompts"].shape[1] for r in rec.records]
    assert [c for c in calls if c[0] == "prefill"] == [("prefill", p - 1) for p in plens], calls
    assert all(("run", p - 1) not in calls for p in plens if p - 1 != GK["max_new_tokens"]), calls
    if mode == "beam5":
        want = ref(audio.copy(), chunk_length_s=meta["chunk_s"] - 1, batch_size=4, generate_kwargs=dict(gk), **rk)
        _check_text(got["text"], want["text"], min_prefix=8, min_ratio=0.6)
    else:
        near = replay_greedy(rec.records, om, max_near_ties=4)
        print(f"\n[{name} {mode} {kw}] {len(rec.records)} decode calls replayed, {near} near ties")


def test_two_prompt_lengths_in_one_pipeline(cuda):
    """Each prompt length is a begin_index of its own, so a stale step graph would show as a wrong second transcript."""
    from thewhisper_b200 import synthetic as S

    meta, pipe, _, om = _pipes("tiny10")
    tok = S.make_tokenizer()
    audio = S.synth_audio(8.0, seed=7)
    for text in (" Hopper", " Kubernetes, gRPC, Hopper and a longer list of words to steer the spelling"):
        rec = _Recorder(pipe)
        pipe(audio.copy(), generate_kwargs=dict(GK, prompt_ids=torch.tensor(tok.get_prompt_ids(text))))
        replay_greedy(rec.records, om, max_near_ties=2)
