"""Sequential long-form transcription (input longer than the window, no chunk_length_s), host logic on the CPU stand-in engine
against transformers run live on the same checkpoint: the seek loop over each item's own frame count, language detection on the first
window, batch reduction, condition_on_prev_tokens (left-padded decoder inputs masked by a key start per row), prompt_ids with
first-segment / all-segments, word timestamps, beam search, and the errors.  Single items are compared with transformers' pipeline
(chunk_length_s=0); groups of three with model.generate on the feature extractor's padded batch (the transformers pipeline cannot
collate long inputs of different lengths).  The stand-in gets the engine's long-form entry points here: logmel_long through the
feature extractor, and the key start as the decoder attention mask transformers passes."""
import json
import os

import numpy as np
import pytest
import torch

from tests.conftest import GOLD
from tests.test_host_cpu import _same


def _stub_cls():
    from oracle.engine_stub import StubEngine

    class MaskedDecoder(torch.nn.Module):
        """The decoder with the key-start mask of the current decode: ids != pad with the pads on the left."""

        def __init__(self, dec, owner):
            super().__init__()
            self.dec = dec
            self.owner = [owner]

        def forward(self, input_ids=None, past_key_values=None, **kw):
            k0 = self.owner[0]._k0
            if k0 is not None:
                past = past_key_values.get_seq_length() if past_key_values is not None else 0
                m = torch.ones(input_ids.shape[0], past + input_ids.shape[1], dtype=torch.long)
                G = input_ids.shape[0] // len(k0)
                for r in range(input_ids.shape[0]):
                    m[r, : int(k0[r // G])] = 0
                kw["attention_mask"] = m
            return self.dec(input_ids=input_ids, past_key_values=past_key_values, **kw)

    class LongStub(StubEngine):
        def __init__(self, model, **kw):
            super().__init__(model, **kw)
            self._k0 = None
            self.key_starts = []
            self.prefill_calls = 0
            self.long_calls = 0
            if not isinstance(model.model.decoder, MaskedDecoder):
                model.model.decoder = MaskedDecoder(model.model.decoder, self)
            model.model.decoder.owner[0] = self

        def logmel_long(self, pcm):
            from transformers import WhisperFeatureExtractor

            self.long_calls += 1
            fe = WhisperFeatureExtractor(feature_size=self.dims.n_mels, chunk_length=self.n_samples // 16000)
            out = fe(list(pcm), sampling_rate=16000, truncation=False, padding="longest", return_tensors="np")
            return torch.from_numpy(np.asarray(out["input_features"], dtype=np.float32))

        def decode_begin(self, prompts, A, G, opts, begin_index=None, key_start=None):
            super().decode_begin(prompts, A, G, opts, begin_index)
            self._k0 = None if key_start is None else np.asarray(key_start)
            if key_start is not None:
                self.key_starts.append(np.asarray(key_start).copy())

        def decode_prefill(self, n, max_rows_per_pass=0):
            self.prefill_calls += 1
            self.decode_run(n)

        def greedy(self, prompts, A, opts, max_new_tokens, poll_every=32, prefill=False, key_start=None):
            self._k0 = None if key_start is None else np.asarray(key_start)
            if key_start is not None:
                self.key_starts.append(np.asarray(key_start).copy())
            self.prefill_calls += int(prefill)
            return super().greedy(prompts, A, opts, max_new_tokens, poll_every)

    return LongStub


META = json.load(open(os.path.join(GOLD, "model_tiny10.json")))


def _pipes(monkeypatch, batch_size=1, name="tiny10", edit=None):
    """Our pipeline on the stand-in and transformers' pipeline on the same checkpoint (edit(model): a change applied to both)."""
    from oracle import hf_ref
    from thewhisper_b200 import synthetic as S
    import thewhisper_b200.nvidia.asr_pipeline as ap

    meta = json.load(open(os.path.join(GOLD, f"model_{name}.json")))
    model = S.make_hf_model(meta["preset"], seed=0, layer_gain=meta["layer_gain"])
    if edit:
        edit(model)
    stub = _stub_cls()
    made = []

    def factory(state_dict, dims, chunk_length_s=30, device=None, max_audios=1, max_beams=1, alignment_heads=None, weights=None, **kw):
        made.append(stub(model, chunk_length_s=chunk_length_s, max_audios=max_audios, max_beams=max_beams, alignment_heads=alignment_heads))
        return made[-1]

    monkeypatch.setattr(ap, "WhisperEngine", factory)
    chunk = meta["chunk_s"]
    ours = ap.ASRPipeline(model, feature_extractor=S.make_feature_extractor(chunk), tokenizer=S.make_tokenizer(), chunk_length_s=chunk,
                          device="cuda", batch_size=batch_size)
    ref_model = S.make_hf_model(meta["preset"], seed=0, layer_gain=meta["layer_gain"])
    if edit:
        edit(ref_model)
    ref = hf_ref.make_ref_pipeline(ref_model, S.make_feature_extractor(chunk), S.make_tokenizer(), chunk_length_s=chunk)
    return ours, ref, ref_model, made


class Windows:
    """Records every window our generator decodes and classifies how it ends (the cases of _retrieve_segment)."""

    def __init__(self, pipe):
        self.kinds = {"single_ending": 0, "double_ending": 0, "no_pair": 0, "empty": 0}
        self.history_cut = 0
        self.outputs = []
        gen = pipe.generator
        tb = gen.timestamp_begin
        orig_decode, orig_generate = gen._decode, gen.generate

        def _decode(*a, **kw):
            out = orig_decode(*a, **kw)
            for seq in out[0]:
                seq = np.asarray(seq)
                is_ts = seq >= tb
                if len(seq) == 0:
                    self.kinds["empty"] += 1
                elif not (is_ts[:-1] & is_ts[1:]).any():
                    self.kinds["no_pair"] += 1
                elif is_ts[-2:].tolist() == [False, True]:
                    self.kinds["single_ending"] += 1
                else:
                    self.kinds["double_ending"] += 1
            return out

        def generate(*a, **kw):
            out = orig_generate(*a, **kw)
            self.history_cut += gen.window_stats["history_cut"]
            self.outputs.append(out)
            return out

        gen._decode = _decode
        gen.generate = generate


def _norm(out):
    return json.loads(json.dumps(out, default=lambda o: float(o)))


LENGTHS = (25.0, 37.3, 58.6)
GK = {"language": "en", "task": "transcribe", "num_beams": 1, "do_sample": False}
MODES = {
    "ts": ({"return_timestamps": True}, {}),
    "word": ({"return_timestamps": "word"}, {}),
    "beam5": ({"return_timestamps": True}, {"num_beams": 5, "max_new_tokens": 40}),
    "lang_none": ({"return_timestamps": True}, {"language": None}),
    "cond": ({"return_timestamps": True}, {"condition_on_prev_tokens": True}),
    "cond_word": ({"return_timestamps": "word"}, {"condition_on_prev_tokens": True}),
    "cond_beam5": ({"return_timestamps": True}, {"condition_on_prev_tokens": True, "num_beams": 5, "max_new_tokens": 40}),
    "prompt_first": ({"return_timestamps": True}, {"prompt_ids": "p"}),
    "prompt_first_cond": ({"return_timestamps": True}, {"prompt_ids": "p", "condition_on_prev_tokens": True}),
    "prompt_all": ({"return_timestamps": True}, {"prompt_ids": "p", "condition_on_prev_tokens": True,
                                                 "prompt_condition_type": "all-segments"}),
}


def _gk(mode, tok):
    kw, extra = MODES[mode]
    gk = dict(GK, **extra)
    if gk.get("prompt_ids") == "p":
        gk["prompt_ids"] = torch.tensor(tok.get_prompt_ids(" Kubernetes, gRPC and Hopper"))
    return kw, gk


@pytest.mark.parametrize("mode", list(MODES))
def test_single_item_matches_transformers_pipeline(monkeypatch, mode):
    from thewhisper_b200 import synthetic as S

    ours, ref, _, made = _pipes(monkeypatch)
    win = Windows(ours)
    kw, gk = _gk(mode, ours.tokenizer)
    seconds = LENGTHS[1:2] if "beam" in mode else LENGTHS
    for k, sec in enumerate(seconds):
        audio = S.synth_audio(sec, seed=3000 + k)
        got = ours(audio.copy(), chunk_length_s=0, generate_kwargs=dict(gk), **kw)
        want = ref(audio.copy(), chunk_length_s=0, generate_kwargs=dict(gk), **kw)
        assert _same(_norm(got), _norm(want)), (mode, sec, got, want)
    assert sum(e.long_calls for e in made) == len(seconds)
    if "cond" in mode or "all" in mode:
        assert sum(e.prefill_calls for e in made) > 0
    print(f"\n[long form {mode}] window endings {win.kinds}, histories cut at 223 tokens: {win.history_cut}")


def _hf_rows(out, pad, word):
    rows = []
    for j, segs in enumerate(out["segments"]):
        seq = out["sequences"][j].numpy()
        n = len(seq)
        while n > 0 and seq[n - 1] == pad:
            n -= 1
        r = {"sequence": seq[:n].tolist(),
             "segments": [(float(s["start"]), float(s["end"]), s["tokens"].tolist()) for s in segs]}
        if word:
            r["token_timestamps"] = [float(x) for x in torch.cat([s["token_timestamps"] for s in segs]).tolist()] if segs else []
        rows.append(r)
    return rows


def _our_rows(out, word):
    rows = []
    for j, segs in enumerate(out["segments"]):
        r = {"sequence": np.asarray(out["sequences"][j]).tolist(),
             "segments": [(float(s["start"]), float(s["end"]), np.asarray(s["tokens"]).tolist()) for s in segs]}
        if word:
            r["token_timestamps"] = [float(x) for x in out["token_timestamps"][j]]
        rows.append(r)
    return rows


def _check_group(ours, ref_model, win, audios, kw, gk):
    """ours on a group of inputs (the last generate call recorded by win) against transformers' generate on the feature
    extractor's padded batch with its attention mask."""
    from oracle import hf_ref

    ours(audios, chunk_length_s=0, batch_size=len(audios), generate_kwargs=dict(gk), **kw)
    word = kw["return_timestamps"] == "word"
    feats = ours.feature_extractor(audios, sampling_rate=16000, truncation=False, padding="longest", return_attention_mask=True,
                                   return_tensors="np")
    hk = dict(gk, return_token_timestamps=True) if word else dict(gk)
    want = hf_ref.generate(ref_model, feats["input_features"].astype(np.float32), np.asarray(feats["attention_mask"]),
                           return_timestamps=True, return_segments=True, **hk)
    got = _our_rows(win.outputs[-1], word)
    exp = _hf_rows(want, ref_model.generation_config.pad_token_id, word)
    assert _same(got, exp), (got, exp)


@pytest.mark.parametrize("mode", ["ts", "word", "lang_none", "cond", "cond_word", "cond_beam5", "prompt_first_cond", "prompt_all"])
def test_group_of_three_matches_transformers_generate(monkeypatch, mode):
    """Three inputs in one group, one of them shorter than the window: the features zero-padded to the longest item, each item's
    own frame count from the attention mask, rows dropping out of the batch as they finish."""
    from thewhisper_b200 import synthetic as S

    ours, _, ref_model, _ = _pipes(monkeypatch, batch_size=3)
    win = Windows(ours)
    kw, gk = _gk(mode, ours.tokenizer)
    _check_group(ours, ref_model, win, [S.synth_audio(sec, seed=4000 + k) for k, sec in enumerate((41.7, 7.3, 26.1))], kw, gk)
    if "cond" in mode or "all" in mode:
        assert ours.generator.window_stats["conditioned"] > 0


def test_longform_reaches_every_case(monkeypatch):
    """Inputs chosen so that, each compared with transformers, they reach every way a window can end, a conditioning history cut
    at 223 tokens, and a conditioned window whose rows are left-padded by different amounts (the key-start mask against
    transformers' decoder_attention_mask).  An empty window cannot occur with the timestamp rules on (their first step allows
    only timestamps), so long form never has one; the seek loop's empty-window branch is reached in short form without
    timestamps, on the checkpoint with EOS allowed first and made likely."""
    from thewhisper_b200 import synthetic as S

    seen = {"single_ending": 0, "double_ending": 0, "no_pair": 0, "empty": 0, "history_cut": 0, "left_padded_unequal": 0}

    def add(win):
        for k, v in win.kinds.items():
            seen[k] += v
        seen["history_cut"] += win.history_cut

    # rows of unequal histories: small30, whose output follows its audio, three items in one conditioned group
    ours, _, ref_model, made = _pipes(monkeypatch, batch_size=3, name="small30")
    win = Windows(ours)
    audios = [S.synth_audio(sec, seed=6000 + k) for k, sec in enumerate((93.0, 22.5, 66.6))]
    _check_group(ours, ref_model, win, audios, {"return_timestamps": True}, dict(GK, max_new_tokens=48, condition_on_prev_tokens=True))
    add(win)
    seen["left_padded_unequal"] += sum(len(set(k.tolist())) >= 2 and k.max() > 0 for e in made for k in e.key_starts)
    # a history longer than 223 tokens: a 240-token prompt is the first segment of every row's history
    ours, ref, _, _ = _pipes(monkeypatch)
    win = Windows(ours)
    sop = ours.tokenizer.convert_tokens_to_ids("<|startofprev|>")
    long_prompt = torch.tensor([sop] + [220 + (i % 50) for i in range(240)])
    cases = [(37.3, {"return_timestamps": True}, dict(GK, prompt_ids=long_prompt, condition_on_prev_tokens=True, max_new_tokens=24)),
             (37.3, {"return_timestamps": True}, dict(GK, max_new_tokens=6)),   # [ts, text, ts, ts, text, ts]: single ending
             (25.0, {"return_timestamps": True}, dict(GK, max_new_tokens=2))]   # [ts, text]: no timestamp pair
    for k, (sec, kw, gk) in enumerate(cases):
        audio = S.synth_audio(sec, seed=3000 + k)
        got = ours(audio.copy(), chunk_length_s=0, generate_kwargs=dict(gk), **kw)
        want = ref(audio.copy(), chunk_length_s=0, generate_kwargs=dict(gk), **kw)
        assert _same(_norm(got), _norm(want)), (k, got, want)
    add(win)

    # the empty window: EOS not begin-suppressed, and its (tied) output row twice that of the token this checkpoint emits first
    # (21363), so that EOS wins the first step -- the same checkpoint edit on both sides; no timestamps
    def eos_first(model):
        model.generation_config.begin_suppress_tokens = [220]
        E = model.model.decoder.embed_tokens.weight
        with torch.no_grad():
            E[model.generation_config.eos_token_id] = 2.0 * E[21363]

    ours, ref, _, _ = _pipes(monkeypatch, edit=eos_first)
    win = Windows(ours)
    audio = S.synth_audio(6.0, seed=5)
    got = ours(audio.copy(), generate_kwargs=dict(GK))
    want = ref(audio.copy(), generate_kwargs=dict(GK))
    assert _same(_norm(got), _norm(want)), (got, want)
    add(win)
    print(f"\n[long form] cases reached: {seen}")
    for k, v in seen.items():
        assert v > 0, (k, seen)


def test_just_past_the_window_encodes_its_own_features(monkeypatch):
    """Under 160 samples past the window the features are one window long (transformers' short form on the long-form
    features): they must reach the encoder, not whatever an earlier call left in the engine's mel buffer."""
    from thewhisper_b200 import synthetic as S

    ours, ref, _, made = _pipes(monkeypatch)
    n = made[-1].n_samples
    ours(S.synth_audio(6.0, seed=1), return_timestamps=True, generate_kwargs=dict(GK))
    audio = S.synth_audio((n + 80) / 16000, seed=2)
    assert len(audio) == n + 80
    got = ours(audio.copy(), chunk_length_s=0, return_timestamps=True, generate_kwargs=dict(GK))
    want = ref(audio.copy(), chunk_length_s=0, return_timestamps=True, generate_kwargs=dict(GK))
    feats = ours.feature_extractor(audio, sampling_rate=16000, truncation=False, padding="longest", return_tensors="np")["input_features"]
    assert feats.shape[-1] == made[-1].frames
    assert np.array_equal(made[-1].mel[:1].numpy(), feats.astype(np.float32))
    assert _same(_norm(got), _norm(want)), (got, want)


def test_longform_errors_like_transformers(monkeypatch):
    from thewhisper_b200 import synthetic as S

    ours, ref, _, _ = _pipes(monkeypatch)
    audio = S.synth_audio(23.0, seed=7)
    for pipe in (ours, ref):  # long form needs timestamps
        with pytest.raises(ValueError, match="requires the model to predict timestamp tokens"):
            pipe(audio.copy(), chunk_length_s=0, return_timestamps=False, generate_kwargs=dict(GK))
    for pipe in (ours, ref):
        with pytest.raises(ValueError, match="exceeds the `max_target_positions`"):
            pipe(audio.copy(), chunk_length_s=0, return_timestamps=True, generate_kwargs=dict(GK, max_new_tokens=446))
    for extra in ({"temperature": (0.0, 0.2)}, {"logprob_threshold": -1.0}, {"compression_ratio_threshold": 2.4},
                  {"no_speech_threshold": 0.6}, {"do_sample": True, "num_beams": 1}):
        name = next(iter(extra))
        with pytest.raises(NotImplementedError, match=name if name != "do_sample" else "sampling"):
            ours(audio.copy(), chunk_length_s=0, return_timestamps=True, generate_kwargs=dict(GK, **extra))
