"""No-speech skipping (no_speech_threshold with logprob_threshold at temperature 0), host logic on the CPU stand-in engine against
transformers run live on the same checkpoint, in the pattern of test_longform_cpu.py: single items against its pipeline, groups of
three against `model.generate`.  The stand-in records the three quantities the engine's select kernel writes -- the processed log-prob
of each selected token, the allowed mass (for beam search) and the no-speech probability -- from the same logits it selects with.

The checkpoint's tied-embedding row of <|nospeech|> is scaled (never an input token, so only that logit changes): the no-speech
probability then varies across windows, and the thresholds below reach skipped windows, windows kept for either reason, groups with
only some rows skipped, a skip on the first long-form window, two consecutive skips and a skip under conditioning.

Also here: float64 restatements of avg_logprob and no_speech_prob (`avg_logprob_ref`, `no_speech_prob_ref`), checked against
transformers' `_retrieve_avg_logprobs` and `WhisperNoSpeechDetection` on random logits."""
import json
import os

import numpy as np
import pytest
import torch

from tests.conftest import GOLD
from tests.test_host_cpu import _same
from tests.test_longform_cpu import GK, _hf_rows, _norm, _our_rows, _stub_cls


# ---------------------------------------------------------------------------------------------------------------------------
# float64 restatements
def _lse(x: np.ndarray) -> float:
    x = np.asarray(x, dtype=np.float64)
    m = x.max()
    return float(m + np.log(np.exp(x - m).sum())) if np.isfinite(m) else -np.inf


def processed_logprob_ref(raw: np.ndarray, processed: np.ndarray, tok: int) -> float:
    """log_softmax of the processed scores at tok = raw[tok] - logsumexp(raw logits the processors allow) (the processors only mask,
    and under beam search they act on log_softmax(raw), which shifts every logit alike)."""
    allowed = np.isfinite(np.asarray(processed, dtype=np.float64))
    return float(np.float64(raw[tok]) - _lse(np.asarray(raw, dtype=np.float64)[allowed]))


def allowed_mass_ref(raw: np.ndarray, processed: np.ndarray) -> float:
    """lmass = logsumexp(allowed raw logits) - logsumexp(raw logits)."""
    raw = np.asarray(raw, dtype=np.float64)
    return _lse(raw[np.isfinite(np.asarray(processed, dtype=np.float64))]) - _lse(raw)


def avg_logprob_ref(raw_steps, processed_steps, tokens, pad: int, eos: int, slots=None) -> float:
    """_retrieve_avg_logprobs over one row: raw_steps / processed_steps [steps, Q or 1, V] of every step of the decode, tokens the
    generated ids (trailing pads dropped, one kept when pad is EOS, as generate_with_fallback does), slots (beam search) the slot of
    the returned sequence's ancestor at each step (beam_indices), else row 0."""
    tokens = np.asarray(tokens, dtype=np.int64)
    if len(tokens) and tokens[-1] == pad:
        n = int((tokens == pad).sum()) - (1 if pad == eos else 0)
        if n:
            tokens = tokens[:-n]
    n = min(len(tokens), len(raw_steps))
    tokens = tokens[len(tokens) - n:] if len(raw_steps) < len(tokens) else tokens
    tot = 0.0
    for i in range(n):
        q = 0 if slots is None else int(slots[i])
        tot += processed_logprob_ref(raw_steps[i][q], processed_steps[i][q], int(tokens[i]))
    return tot / n


def no_speech_prob_ref(raw_row: np.ndarray, no_speech_token: int) -> float:
    """softmax of the raw logits of the step whose input is <|startoftranscript|>, at <|nospeech|>."""
    raw = np.asarray(raw_row, dtype=np.float64)
    return float(np.exp(raw[no_speech_token] - _lse(raw)))


# ---------------------------------------------------------------------------------------------------------------------------
# the stand-in with scores
class _Recorder:
    """Stands in for oracle.whisper_ref inside the stand-in's selection loops: records each (row length, raw, processed) it sees."""

    def __init__(self, ref):
        self.ref = ref
        self.calls = []

    def __getattr__(self, k):
        return getattr(self.ref, k)

    def process_logits(self, scores, seq, begin_index, **kw):
        s = self.ref.process_logits(scores, seq, begin_index, **kw)
        self.calls.append((len(seq), np.asarray(scores, dtype=np.float64).copy(), np.asarray(s, dtype=np.float64).copy()))
        return s


def _scores_stub_cls():
    import oracle.engine_stub as es

    LongStub = _stub_cls()

    class ScoresStub(LongStub):
        """lp / lmass / nsp as the engine's decode_scores returns them, from the logits the stand-in selects with."""

        def decode_begin(self, prompts, A, G, opts, begin_index=None, key_start=None):
            super().decode_begin(prompts, A, G, opts, begin_index, key_start)
            self._scores_on = False

        def decode_scores_enable(self, nospeech_pos=-1, nospeech_token=0):
            T, Q = self.dims.max_target_positions, self._A * self._G
            self._scores_on, self._ns = True, (int(nospeech_pos), int(nospeech_token))
            self._lp = np.zeros((Q, T), dtype=np.float32)
            self._lmass = np.zeros((Q, T), dtype=np.float32)
            self._nsp = np.zeros(Q, dtype=np.float32)

        def decode_scores(self):
            return self._lp.copy(), self._lmass.copy(), self._nsp.copy()

        @torch.no_grad()
        def _forced_nsp(self, prompts, G):
            """The no-speech probability at a forced position: the decoder over the whole input with the current key-start mask."""
            pos, tok = self._ns
            if pos < 0 or pos >= prompts.shape[1] - 1:
                return
            ids = torch.from_numpy(np.asarray(prompts)).long()
            enc = self.enc[: self._A].repeat_interleave(G, dim=0)
            out = self.model.model.decoder(input_ids=ids, encoder_hidden_states=enc)
            lg = self.model.proj_out(out.last_hidden_state[:, pos]).double().numpy()
            for q in range(ids.shape[0]):
                self._nsp[q] = no_speech_prob_ref(lg[q], tok)

        def teacher_force(self, plen, prefill, nospeech_pos=None):
            self.prefill_calls += int(prefill)
            if self._scores_on:
                self._forced_nsp(self._prompts, self._G)
            self.decode_run(plen - 1)

        def greedy(self, prompts, A, opts, max_new_tokens, poll_every=32, prefill=False, key_start=None, nospeech=None):
            if nospeech is None:
                return super().greedy(prompts, A, opts, max_new_tokens, poll_every, prefill, key_start)
            self.decode_begin(prompts, A, 1, opts, key_start=key_start)
            self.decode_scores_enable(*nospeech)
            self._k0 = None if key_start is None else np.asarray(key_start)
            self._forced_nsp(prompts, 1)
            rec, saved = _Recorder(es.whisper_ref), es.whisper_ref
            es.whisper_ref = rec
            try:
                gen, toks, done = super().greedy(prompts, A, opts, max_new_tokens, poll_every, prefill, key_start)
            finally:
                es.whisper_ref = saved
            plen = prompts.shape[1]
            pos, tok = self._ns
            fin = np.zeros(A, dtype=bool)
            for k, (n, raw, s) in enumerate(rec.calls):
                a = k % A
                t = int(toks[a, n])
                self._lmass[a, n] = allowed_mass_ref(raw, s)
                self._lp[a, n] = 0.0 if fin[a] else processed_logprob_ref(raw, s, t)
                fin[a] |= t == opts.eos_token
                if n - 1 == pos:
                    self._nsp[a] = no_speech_prob_ref(raw, tok)
            assert len(rec.calls) == A * done, (len(rec.calls), A, done)
            self.greedy_calls = getattr(self, "greedy_calls", 0) + 1
            return gen, toks, done

        def decode_beam_step(self, run_scores):
            rec, saved = _Recorder(es.whisper_ref), es.whisper_ref
            es.whisper_ref = rec
            try:
                cs, ct = super().decode_beam_step(run_scores)
            finally:
                es.whisper_ref = saved
            if self._scores_on:
                pos, tok = self._ns
                for q, (n, lp, s) in enumerate(rec.calls):
                    self._lmass[q, n] = allowed_mass_ref(lp, s)
                    if n - 1 == pos:
                        self._nsp[q] = float(np.exp(lp[tok]))
            return cs, ct

    return ScoresStub


def _scale_nospeech(factor):
    def edit(model):
        ns = model.generation_config.no_timestamps_token_id - 1
        with torch.no_grad():
            model.model.decoder.embed_tokens.weight[ns] *= factor
    return edit


# With the row scaled 100x this checkpoint's no_speech_prob is about 0.98 on every window (40x: under 0.01, "ns_low" below); with
# 24 new tokens its avg_logprob is about -8.6 on most windows and -8.0 on some, which logprob_threshold -8.3 tells apart by a wide
# margin
NS_FACTOR = 100.0
FACTORS = {"ns_low": 40.0}


def _pipes(monkeypatch, batch_size=1, name="tiny10", edit=_scale_nospeech(NS_FACTOR)):
    from oracle import hf_ref
    from thewhisper_b200 import synthetic as S
    import thewhisper_b200.nvidia.asr_pipeline as ap

    meta = json.load(open(os.path.join(GOLD, f"model_{name}.json")))
    model = S.make_hf_model(meta["preset"], seed=0, layer_gain=meta["layer_gain"])
    edit(model)
    stub = _scores_stub_cls()
    made = []

    def factory(state_dict, dims, chunk_length_s=30, device=None, max_audios=1, max_beams=1, alignment_heads=None, weights=None, **kw):
        made.append(stub(model, chunk_length_s=chunk_length_s, max_audios=max_audios, max_beams=max_beams, alignment_heads=alignment_heads))
        return made[-1]

    monkeypatch.setattr(ap, "WhisperEngine", factory)
    chunk = meta["chunk_s"]
    ours = ap.ASRPipeline(model, feature_extractor=S.make_feature_extractor(chunk), tokenizer=S.make_tokenizer(), chunk_length_s=chunk,
                          device="cuda", batch_size=batch_size)
    ref_model = S.make_hf_model(meta["preset"], seed=0, layer_gain=meta["layer_gain"])
    edit(ref_model)
    ref = hf_ref.make_ref_pipeline(ref_model, S.make_feature_extractor(chunk), S.make_tokenizer(), chunk_length_s=chunk)
    return ours, ref, ref_model, made


class Log:
    """Every window our generator decides: (avg_logprob, no_speech_prob, skipped) per row, one list per window, per generate call."""

    def __init__(self, pipe):
        self.calls = []
        gen = pipe.generator
        orig = gen.generate

        def generate(*a, **kw):
            out = orig(*a, **kw)
            self.calls.append({"log": [r for w in gen.window_log for r in w], "windows": list(gen.window_log), "out": out})
            return out

        gen.generate = generate


TH = {"no_speech_threshold": 0.5, "logprob_threshold": -8.3, "temperature": 0.0}  # (transformers needs the temperature set)
LENGTHS = (37.3, 25.0)
MODES = {
    "ts": ({"return_timestamps": True}, {}),
    "ns_low": ({"return_timestamps": True}, {}),
    "word": ({"return_timestamps": "word"}, {}),
    "beam5": ({"return_timestamps": True}, {"num_beams": 5, "max_new_tokens": 24}),
    "lang_none": ({"return_timestamps": True}, {"language": None}),
    "cond": ({"return_timestamps": True}, {"condition_on_prev_tokens": True}),
    "cond_beam5": ({"return_timestamps": True}, {"condition_on_prev_tokens": True, "num_beams": 5, "max_new_tokens": 24}),
    "prompt_first": ({"return_timestamps": True}, {"prompt_ids": "p"}),
    "prompt_all": ({"return_timestamps": True}, {"prompt_ids": "p", "condition_on_prev_tokens": True,
                                                 "prompt_condition_type": "all-segments"}),
}


def _gk(mode, tok, th=TH):
    kw, extra = MODES[mode]
    gk = dict(GK, max_new_tokens=24, **th)
    gk.update(extra)
    if gk.get("prompt_ids") == "p":
        gk["prompt_ids"] = torch.tensor(tok.get_prompt_ids(" Kubernetes, gRPC and Hopper"))
    return kw, gk


def _audio(sec, seed):
    """Synthetic speech with a silent stretch in its middle third (windows there are the no-speech candidates)."""
    from thewhisper_b200 import synthetic as S

    a = S.synth_audio(sec, seed=seed)
    n = len(a)
    a[n // 3: 2 * n // 3] *= 0.0
    return a


def _kinds(log, th=TH):
    """Which reasons each window's decision had."""
    out = {"skipped": 0, "kept_low_nsp": 0, "kept_high_logprob": 0}
    for avg, ns, skip in log:
        assert skip == (avg < th["logprob_threshold"] and ns > th["no_speech_threshold"])
        if skip:
            out["skipped"] += 1
        if ns <= th["no_speech_threshold"]:
            out["kept_low_nsp"] += 1
        if avg >= th["logprob_threshold"]:
            out["kept_high_logprob"] += 1
    return out


SEEN = {}


def _add(k, v=1):
    SEEN[k] = SEEN.get(k, 0) + v


@pytest.mark.parametrize("mode", list(MODES))
def test_single_item_matches_transformers_pipeline(monkeypatch, mode):
    ours, ref, _, made = _pipes(monkeypatch, edit=_scale_nospeech(FACTORS.get(mode, NS_FACTOR)))
    log = Log(ours)
    kw, gk = _gk(mode, ours.tokenizer)
    seconds = LENGTHS[1:2] if "beam" in mode else LENGTHS
    kinds = {"skipped": 0, "kept_low_nsp": 0, "kept_high_logprob": 0}
    for k, sec in enumerate(seconds):
        audio = _audio(sec, 3000 + k)
        got = ours(audio.copy(), chunk_length_s=0, generate_kwargs=dict(gk), **kw)
        want = ref(audio.copy(), chunk_length_s=0, generate_kwargs=dict(gk), **kw)
        assert _same(_norm(got), _norm(want)), (mode, sec, got, want)
        for c, v in _kinds(log.calls[-1]["log"]).items():
            kinds[c] += v
        skips = [s for _, _, s in log.calls[-1]["log"]]
        _add("first_window_skip", int(skips[0]))
        _add("consecutive_skips", int(any(a and b for a, b in zip(skips, skips[1:]))))
        if "cond" in mode or "all" in mode:
            _add("conditioned_skip", int(any(skips[1:])))
    print(f"\n[no-speech {mode}] {kinds}; windows {[(round(a, 3), round(n, 3), s) for c in log.calls for a, n, s in c['log']]}")
    for c, v in kinds.items():
        _add(c, v)


def _check_group(ours, ref_model, log, audios, kw, gk):
    from oracle import hf_ref

    ours(audios, chunk_length_s=0, batch_size=len(audios), generate_kwargs=dict(gk), **kw)
    word = kw["return_timestamps"] == "word"
    feats = ours.feature_extractor(audios, sampling_rate=16000, truncation=False, padding="longest", return_attention_mask=True,
                                   return_tensors="np")
    hk = dict(gk, return_token_timestamps=True) if word else dict(gk)
    want = hf_ref.generate(ref_model, feats["input_features"].astype(np.float32), np.asarray(feats["attention_mask"]),
                           return_timestamps=True, return_segments=True, **hk)
    got = _our_rows(log.calls[-1]["out"], word)
    exp = _hf_rows(want, ref_model.generation_config.pad_token_id, word)
    assert _same(got, exp), (got, exp)


@pytest.mark.parametrize("mode", ["ts", "word", "cond", "cond_beam5", "prompt_all"])
def test_group_of_three_matches_transformers_generate(monkeypatch, mode):
    """Three inputs in one long-form group: rows are skipped independently, and a conditioned row that was skipped keeps its history."""
    ours, _, ref_model, _ = _pipes(monkeypatch, batch_size=3)
    log = Log(ours)
    kw, gk = _gk(mode, ours.tokenizer)
    _check_group(ours, ref_model, log, [_audio(sec, 4000 + k) for k, sec in enumerate((41.7, 7.3, 26.1))], kw, gk)
    g = ours.generator
    logs = log.calls[-1]["log"]
    _add("partial_group", sum(any(s for *_, s in w) and not all(s for *_, s in w) for w in log.calls[-1]["windows"]))
    print(f"\n[no-speech group {mode}] {[(round(a, 3), round(n, 3), s) for a, n, s in logs]}, window stats {g.window_stats}")


def test_short_form_chunked_batches_match_transformers(monkeypatch):
    """chunk_length_s batches (short form, one window per chunk): a skipped chunk contributes no tokens, greedy and beam."""
    ours, ref, _, _ = _pipes(monkeypatch, batch_size=4)
    log = Log(ours)
    audio = _audio(41.0, 77)
    for extra in ({}, {"num_beams": 5}):
        for kw in ({"return_timestamps": True}, {}):
            gk = dict(GK, max_new_tokens=24, **extra, **TH)
            got = ours(audio.copy(), chunk_length_s=10, batch_size=4, generate_kwargs=dict(gk), **kw)
            want = ref(audio.copy(), chunk_length_s=10, batch_size=4, generate_kwargs=dict(gk), **kw)
            assert _same(_norm(got), _norm(want)), (extra, kw, got, want)
            for w in log.calls[-1]["windows"]:
                _add("partial_group", int(any(s for *_, s in w) and not all(s for *_, s in w)))
    print(f"\n[no-speech chunked] {[(round(a, 3), round(n, 3), s) for c in log.calls for a, n, s in c['log']]}")


def test_compression_ratio_threshold_is_accepted_and_ignored(monkeypatch):
    ours, ref, _, _ = _pipes(monkeypatch)
    audio = _audio(25.0, 3000)
    gk = dict(GK, max_new_tokens=24, **TH)
    a = ours(audio.copy(), chunk_length_s=0, return_timestamps=True, generate_kwargs=dict(gk))
    b = ours(audio.copy(), chunk_length_s=0, return_timestamps=True, generate_kwargs=dict(gk, compression_ratio_threshold=0.1))
    want = ref(audio.copy(), chunk_length_s=0, return_timestamps=True, generate_kwargs=dict(gk, compression_ratio_threshold=0.1))
    assert _same(_norm(a), _norm(b)) and _same(_norm(b), _norm(want))


def test_nospeech_reaches_every_case():
    """Runs after the tests above in this module (pytest keeps file order): every case the issue of no-speech skipping has was
    reached by a run that matched transformers."""
    need = ("skipped", "kept_low_nsp", "kept_high_logprob", "first_window_skip", "consecutive_skips", "conditioned_skip", "partial_group")
    print(f"\n[no-speech] cases reached: {SEEN}")
    if not SEEN:
        pytest.skip("run with the module's other tests")
    for k in need:
        assert SEEN.get(k, 0) > 0, (k, SEEN)


def test_thresholds_that_still_raise(monkeypatch):
    ours, _, _, _ = _pipes(monkeypatch)
    audio = _audio(23.0, 7)
    for extra, name in (({"no_speech_threshold": 0.6}, "no_speech_threshold"), ({"logprob_threshold": -1.0}, "logprob_threshold"),
                        ({"compression_ratio_threshold": 2.4}, "compression_ratio_threshold"),
                        ({"no_speech_threshold": 0.6, "compression_ratio_threshold": 2.4}, "compression_ratio_threshold"),
                        ({"logprob_threshold": -1.0, "compression_ratio_threshold": 2.4}, "logprob_threshold"),
                        (dict(TH, temperature=(0.0, 0.2)), "temperature"), (dict(TH, temperature=0.4), "temperature"),
                        (dict(TH, do_sample=True), "sampling")):
        with pytest.raises(NotImplementedError, match=name):
            ours(audio.copy(), chunk_length_s=0, return_timestamps=True, generate_kwargs=dict(GK, **extra))


# ---------------------------------------------------------------------------------------------------------------------------
# the restatements against transformers on random logits
def _ts_cfg():
    from transformers import GenerationConfig

    from thewhisper_b200 import synthetic as S

    return GenerationConfig(no_timestamps_token_id=S.NOTIMESTAMPS, eos_token_id=S.EOS, pad_token_id=S.EOS, max_initial_timestamp_index=50,
                            is_multilingual=True)


def _processors(begin_index, V, ts=True):
    from transformers.generation.logits_process import (SuppressTokensAtBeginLogitsProcessor, SuppressTokensLogitsProcessor,
                                                        WhisperTimeStampLogitsProcessor)

    from thewhisper_b200 import synthetic as S

    procs = [SuppressTokensLogitsProcessor([11, 13, S.STARTOFPREV]), SuppressTokensAtBeginLogitsProcessor([220, S.EOS], begin_index)]
    if ts:
        procs.append(WhisperTimeStampLogitsProcessor(_ts_cfg(), begin_index=begin_index))
    return procs


def _apply(procs, ids, scores):
    for p in procs:
        scores = p(ids, scores)
    return scores


@pytest.mark.parametrize("beam", [False, True])
def test_restatements_match_transformers(beam):
    """avg_logprob_ref / no_speech_prob_ref against _retrieve_avg_logprobs and WhisperNoSpeechDetection on random logits: steps
    that reach the begin-suppress step, forced timestamps (a row whose timestamp mass is planted above its best text), blocked
    timestamps, pad rows after EOS, and beam ancestry (scores of the returned sequence's ancestor slots)."""
    from transformers.generation.logits_process import WhisperNoSpeechDetection
    from transformers.models.whisper.generation_whisper import WhisperGenerationMixin

    from thewhisper_b200 import synthetic as S

    rng = np.random.default_rng(5 + beam)
    V, plen, steps = S.VOCAB, 3, 7
    Q = 4
    slots = rng.integers(0, Q, size=steps) if beam else None
    init = [S.SOT, S.LANG_EN, S.TRANSCRIBE]
    procs = _processors(plen, V)
    seqs = [list(init) for _ in range(Q)]
    raw_steps, proc_steps = [], []
    forced_seen = 0
    for t in range(steps):
        raw = torch.from_numpy(rng.normal(0, 3, (Q, V)).astype(np.float32))
        if t == 2:
            raw[0, S.TIMESTAMP_BEGIN:] += 6.0  # timestamp mass above the best text: the forcing rule
        ids = torch.tensor(seqs)
        x = torch.log_softmax(raw, -1) if beam else raw
        s = _apply(procs, ids, x.clone())
        forced_seen += int(bool(torch.isinf(s[:, :S.TIMESTAMP_BEGIN]).all(-1).any()) and t > 0)
        raw_steps.append(raw.numpy())
        proc_steps.append(s.numpy())
        nxt = s.argmax(-1).tolist()
        if beam:  # one returned sequence: every slot shares its history, its token comes from the ancestor slot of the step
            nxt = [nxt[int(slots[t])]] * Q
        if t == 4 and not beam:
            nxt[1] = S.EOS
        for q in range(Q):
            if len(seqs[q]) > plen and seqs[q][-1] == S.EOS:
                nxt[q] = S.EOS  # pad (= EOS) after EOS
            seqs[q].append(int(nxt[q]))
    assert forced_seen
    for q in range(Q):
        tokens = torch.tensor(seqs[q][plen:])
        sc = [torch.from_numpy(proc_steps[t][slots[t] if beam else q]) for t in range(steps)]
        t_hf = tokens
        if t_hf[-1] == S.EOS:
            n = int((t_hf == S.EOS).sum()) - 1
            if n:
                t_hf = t_hf[:-n]
        want = float(WhisperGenerationMixin._retrieve_avg_logprobs(sc, t_hf, 0.0))
        rows = [r[None, slots[t] if beam else q] for t, r in enumerate(raw_steps)]
        prs = [r[None, slots[t] if beam else q] for t, r in enumerate(proc_steps)]
        got = avg_logprob_ref(rows, prs, tokens.numpy(), S.EOS, S.EOS)
        assert abs(got - want) < 2e-5, (q, got, want)
    # no-speech probability: the first step's scores (begin_index 1), raw logits or log-probs
    det = WhisperNoSpeechDetection(no_speech_token=S.NOSPEECH, begin_index=1, scores_is_logprobs=beam)
    raw = torch.from_numpy(rng.normal(0, 3, (Q, V)).astype(np.float32))
    det(torch.zeros((Q, 1), dtype=torch.long), torch.log_softmax(raw, -1) if beam else raw)
    for q in range(Q):
        assert abs(no_speech_prob_ref(raw[q].numpy(), S.NOSPEECH) - float(det.no_speech_prob[q])) < 1e-6
