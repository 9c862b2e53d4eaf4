"""Prompted decoding (`generate_kwargs["prompt_ids"]`), host logic on the CPU stand-in engine against the transformers pipeline
run live on the same checkpoint with the same generate_kwargs: decoder input = prompt + init tokens, begin_index, timestamp rules,
the seek loop re-applying the prompt on every re-encoded window, token-timestamp layout, the prompt-length checks.  The stand-in
runs the prompt's forced positions as decode_run steps (what decode_prefill replaces on the GPU)."""
import json
import os

import numpy as np
import pytest
import torch

from tests.conftest import GOLD
from tests.test_host_cpu import _same

PROMPT_TEXT = " Kubernetes, gRPC and Hopper"


def _stub_cls():
    from oracle.engine_stub import StubEngine

    class PrefillStub(StubEngine):
        """The stand-in with the product engine's prefill entry: n teacher-forced decode_run steps."""

        def decode_prefill(self, n, max_rows_per_pass=0):
            self.prefill_calls = getattr(self, "prefill_calls", 0) + 1
            self.decode_run(n)

        def greedy(self, prompts, A, opts, max_new_tokens, poll_every=32, prefill=False):
            assert prefill and prompts.shape[1] > 4
            self.prefill_calls = getattr(self, "prefill_calls", 0) + 1
            return super().greedy(prompts, A, opts, max_new_tokens, poll_every)

    return PrefillStub


def _pipes(monkeypatch, batch_size=4):
    from oracle import hf_ref
    from thewhisper_b200 import synthetic as S
    import thewhisper_b200.nvidia.asr_pipeline as ap

    meta = json.load(open(os.path.join(GOLD, "model_tiny10.json")))
    model = S.make_hf_model(meta["preset"], seed=0, layer_gain=meta["layer_gain"])
    stub = _stub_cls()
    made = []

    def factory(state_dict, dims, chunk_length_s=30, device=None, max_audios=1, max_beams=1, alignment_heads=None, weights=None, **kw):
        made.append(stub(model, chunk_length_s=chunk_length_s, max_audios=max_audios, max_beams=max_beams, alignment_heads=alignment_heads))
        return made[-1]

    monkeypatch.setattr(ap, "WhisperEngine", factory)
    chunk = meta["chunk_s"]
    tok = S.make_tokenizer()
    ours = ap.ASRPipeline(model, feature_extractor=S.make_feature_extractor(chunk), tokenizer=tok, chunk_length_s=chunk, device="cuda",
                          batch_size=batch_size)
    ref_model = S.make_hf_model(meta["preset"], seed=0, layer_gain=meta["layer_gain"])
    ref = hf_ref.make_ref_pipeline(ref_model, S.make_feature_extractor(chunk), S.make_tokenizer(), chunk_length_s=chunk)
    return meta, ours, ref, tok, made


def _prompt(tok):
    return torch.tensor(tok.get_prompt_ids(PROMPT_TEXT))


def _norm(out):
    return json.loads(json.dumps(out, default=lambda o: float(o)))


@pytest.mark.parametrize("mode", ["plain", "ts", "word", "beam5", "word_beam5", "lang_none"])
def test_prompted_pipeline_matches_transformers(monkeypatch, mode):
    from thewhisper_b200 import synthetic as S

    meta, ours, ref, tok, made = _pipes(monkeypatch)
    audio = S.synth_audio(meta["audio_s"], seed=2000)
    gk = {"num_beams": 5 if "beam" in mode else 1, "do_sample": False, "language": None if mode == "lang_none" else "en",
          "task": "transcribe", "max_new_tokens": 32}
    kw = {"ts": {"return_timestamps": True}, "word": {"return_timestamps": "word"}, "word_beam5": {"return_timestamps": "word"}}.get(mode, {})
    got = ours(audio.copy(), chunk_length_s=meta["chunk_s"] - 1, batch_size=4, generate_kwargs=dict(gk, prompt_ids=_prompt(tok)), **kw)
    want = ref(audio.copy(), chunk_length_s=meta["chunk_s"] - 1, batch_size=4, generate_kwargs=dict(gk, prompt_ids=_prompt(tok)), **kw)
    assert _same(_norm(got), _norm(want)), (got, want)
    assert sum(getattr(e, "prefill_calls", 0) for e in made) > 0


def test_prompt_given_as_list_or_array(monkeypatch):
    from thewhisper_b200 import synthetic as S

    meta, ours, _, tok, _ = _pipes(monkeypatch)
    audio = S.synth_audio(6.0, seed=5)
    gk = {"language": "en", "task": "transcribe", "max_new_tokens": 16}
    p = _prompt(tok)
    outs = [ours(audio.copy(), generate_kwargs=dict(gk, prompt_ids=x)) for x in (p, p.numpy(), p.tolist())]
    assert outs[0] == outs[1] == outs[2]


def test_prompt_length_limits_like_transformers(monkeypatch):
    """A prompt near the 448-position limit decodes; one past it, or with max_new_tokens overflowing it, is the ValueError
    transformers raises."""
    from thewhisper_b200 import synthetic as S

    meta, ours, ref, tok, _ = _pipes(monkeypatch, batch_size=1)
    audio = S.synth_audio(4.0, seed=1)
    sop = tok.convert_tokens_to_ids("<|startofprev|>")
    gk = {"language": "en", "task": "transcribe"}
    near = torch.tensor([sop] + [220 + (i % 50) for i in range(440)])  # + 4 init tokens = 445
    got = ours(audio.copy(), generate_kwargs=dict(gk, prompt_ids=near))
    want = ref(audio.copy(), generate_kwargs=dict(gk, prompt_ids=near))
    assert _same(_norm(got), _norm(want)), (got, want)
    over = torch.tensor([sop] + [220] * 446)
    for p, extra in ((over, {}), (_prompt(tok), {"max_new_tokens": 440})):
        for pipe in (ours, ref):
            with pytest.raises(ValueError, match="exceeds the `max_target_positions`"):
                pipe(audio.copy(), generate_kwargs=dict(gk, prompt_ids=p, **extra))


def test_all_segments_is_not_implemented(monkeypatch):
    from thewhisper_b200 import synthetic as S

    meta, ours, _, tok, _ = _pipes(monkeypatch, batch_size=1)
    with pytest.raises(NotImplementedError, match="condition_on_prev_tokens"):
        ours(S.synth_audio(3.0, seed=1), generate_kwargs={"language": "en", "prompt_ids": _prompt(tok), "prompt_condition_type": "all-segments"})
