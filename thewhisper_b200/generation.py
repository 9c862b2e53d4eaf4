"""Host-side generation control for the engine: prompt tokens, the short-form `seek` loop, segment
extraction and token timestamps -- the integer/host half of WhisperGenerationMixin.generate
(TF/models/whisper/generation_whisper.py:383-968), restated without torch modules.  All arithmetic (encoder,
decoder steps, logits processors, argmax, DTW) runs in the CUDA engine; this module only sequences it.

What is covered (everything the reference's ASRPipeline / LocalWhisperBackend reach, SURVEY.md §3.2-3.4):
  * init tokens [SOT, lang, task, (notimestamps)] incl. language detection (:1455-1608, :1610-1673)
  * greedy decoding with EOS / max_new_tokens stopping, prompt + EOS stripping (:1042-1086)
  * return_timestamps: WhisperTimeStamp rules on the device, segment split on timestamp pairs and the re-encode
    `seek` loop for unfinished segments (:785-903, :1976-2073)
  * return_token_timestamps: per-token times from the alignment heads (:241-381) with HF's row bookkeeping
  * beam search (num_beams > 1) via thewhisper_b200.beam, incl. token timestamps along the winner's ancestry (beam_indices)
  * sequential long-form transcription (features longer than one window): the same seek loop over each item's own frame count
    (_retrieve_max_frames_and_seek), language detected once on the first window, batch reduction to the rows still active
  * condition_on_prev_tokens: [<|startofprev|> or the prompt (prompt_condition_type="all-segments"), last 223 tokens of the
    row's text] + init tokens, rows left-padded to the longest and the pads masked by a per-row key start in decoder
    self-attention (:1853-1915); the conditioning positions run as one batched prefill pass
  * no-speech skipping at temperature 0 (no_speech_threshold with logprob_threshold, _need_fallback's should_skip): avg_logprob from
    the processed log-probs the select kernel records, no_speech_prob from the raw logits of the step whose input is
    <|startoftranscript|> (WhisperNoSpeechDetection), in short and long form, greedy and beam
Not covered: temperature fallback and the compression-ratio threshold's fallback -- sampling is not part of the engine.
"""
from __future__ import annotations

import dataclasses
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from .engine import DecodeOptions, WhisperEngine

TASK_IDS = ("translate", "transcribe")


@dataclasses.dataclass
class GenerationSettings:
    """The subset of a Whisper generation_config.json the hot path needs."""
    decoder_start_token_id: int
    eos_token_id: int
    pad_token_id: int
    no_timestamps_token_id: int
    lang_to_id: Dict[str, int]
    task_to_id: Dict[str, int]
    suppress_tokens: Sequence[int] = ()
    begin_suppress_tokens: Sequence[int] = ()
    alignment_heads: Sequence[Sequence[int]] = ()
    max_initial_timestamp_index: Optional[int] = 50
    is_multilingual: bool = True
    max_length: int = 448
    median_filter_width: int = 7
    prev_sot_token_id: Optional[int] = None

    @staticmethod
    def from_hf(gc, config=None) -> "GenerationSettings":
        def lst(x):
            return list(x) if x is not None else []

        mi = getattr(gc, "max_initial_timestamp_index", None)
        return GenerationSettings(
            decoder_start_token_id=int(gc.decoder_start_token_id), eos_token_id=int(gc.eos_token_id if not isinstance(gc.eos_token_id, (list, tuple)) else gc.eos_token_id[0]),
            pad_token_id=int(gc.pad_token_id), no_timestamps_token_id=int(gc.no_timestamps_token_id),
            lang_to_id=dict(getattr(gc, "lang_to_id", {}) or {}), task_to_id=dict(getattr(gc, "task_to_id", {}) or {}),
            suppress_tokens=lst(getattr(gc, "suppress_tokens", None)), begin_suppress_tokens=lst(getattr(gc, "begin_suppress_tokens", None)),
            alignment_heads=[list(p) for p in (getattr(gc, "alignment_heads", None) or [])],
            max_initial_timestamp_index=mi, is_multilingual=bool(getattr(gc, "is_multilingual", True)),
            max_length=int(getattr(gc, "max_length", 448) or 448),
            median_filter_width=int(getattr(config, "median_filter_width", 7)) if config is not None else 7,
            prev_sot_token_id=(int(gc.prev_sot_token_id) if getattr(gc, "prev_sot_token_id", None) is not None else None))


def _language_token(language: str, st: GenerationSettings) -> int:
    from transformers.models.whisper.tokenization_whisper import TO_LANGUAGE_CODE  # a static name table

    language = language.lower()
    if language in st.lang_to_id:
        tok = language
    elif language in TO_LANGUAGE_CODE:
        tok = f"<|{TO_LANGUAGE_CODE[language]}|>"
    elif language in TO_LANGUAGE_CODE.values():
        tok = f"<|{language}|>"
    else:
        raise ValueError(f"Unsupported language: {language}.")
    if tok not in st.lang_to_id:
        raise ValueError(f"{tok} is not supported by this specific model as it is not in the `generation_config.lang_to_id`.")
    return st.lang_to_id[tok]


class WhisperGenerator:
    def __init__(self, engine: WhisperEngine, settings: GenerationSettings):
        self.eng = engine
        self.st = settings
        self.timestamp_begin = settings.no_timestamps_token_id + 1
        self.time_precision = 0.02

    # --------------------------------------------------------------------------------------------------------
    def _opts(self, return_timestamps: bool, record_alignment: bool, extra_suppress: Sequence[int] = ()) -> DecodeOptions:
        st = self.st
        return DecodeOptions(
            eos_token=st.eos_token_id, pad_token=st.pad_token_id,
            suppress_tokens=list(st.suppress_tokens) + list(extra_suppress), begin_suppress_tokens=list(st.begin_suppress_tokens),
            timestamp_rules=bool(return_timestamps), timestamp_begin=self.timestamp_begin,
            no_timestamps_token=st.no_timestamps_token_id,
            max_initial_timestamp_index=(st.max_initial_timestamp_index if (return_timestamps and st.max_initial_timestamp_index is not None) else -1),
            record_alignment=record_alignment)

    def detect_language(self, B: int) -> List[int]:
        """One decoder step from [SOT]; argmax over the language tokens (generation_whisper.py:1610-1673).
        The encoder output of the B audios must be resident."""
        st = self.st
        prompts = np.full((B, 1), st.decoder_start_token_id, dtype=np.int32)
        self.eng.decode_begin(prompts, B, 1, self._opts(False, False), begin_index=1)
        self.eng.decode_run(1)
        lg = self.eng.logits()[:B]
        ids = torch.tensor(sorted(st.lang_to_id.values()), device=lg.device, dtype=torch.long)
        best = lg[:, ids].argmax(-1)  # selection among V logits already computed by the engine
        return ids[best].tolist()

    def init_tokens(self, B: int, language, task, return_timestamps: bool) -> np.ndarray:
        st = self.st
        base = [st.decoder_start_token_id]
        if isinstance(language, (list, tuple)):
            if len(language) != B:
                raise ValueError(f"When passing a list of languages, the length of the list must match the batch size. "
                                 f"Expected length of {B}, but got {len(language)} languages.")
            lang_ids = [_language_token(l, st) for l in language]
        elif language is not None:
            lang_ids = [_language_token(language, st)] * B
        elif st.lang_to_id and st.is_multilingual:
            lang_ids = self.detect_language(B)
        else:
            lang_ids = None
        rows = []
        for i in range(B):
            r = list(base)
            if lang_ids is not None:
                r.append(lang_ids[i])
            if task is not None:
                if task not in TASK_IDS:
                    raise ValueError(f"The `{task}` task is not supported. The task should be one of `{TASK_IDS}`")
                r.append(st.task_to_id[task])
            elif language is not None and st.task_to_id:
                r.append(st.task_to_id["transcribe"])
            if not return_timestamps and r[-1] != st.no_timestamps_token_id:
                r.append(st.no_timestamps_token_id)
            rows.append(r)
        return np.asarray(rows, dtype=np.int32)

    # --------------------------------------------------------------------------------------------------------
    def _decode(self, prompts: np.ndarray, A: int, opts: DecodeOptions, max_new: int, num_beams: int, prefill: bool = False,
                key_start=None, n_init: Optional[int] = None):
        """-> (list of generated id arrays cut before EOS, n_steps HF would have run, eos_seen per row).  prefill: the
        teacher-forced positions run as one batched prefill pass (a prompt), not step by step.  key_start [A]: left-padded
        prompts, the positions below it are masked (engine.decode_begin).  n_init (no-speech skipping): the decode runs with scores,
        and self._window_scores = (avg_logprob [A], no_speech_prob [A]) of the window afterwards (_nospeech_stats)."""
        self._beam_indices = None
        self._window_scores = None
        plen = prompts.shape[1]
        kw = {"prefill": True} if prefill else {}
        if key_start is not None:
            kw["key_start"] = key_start
        if n_init is not None:  # the no-speech probability is read where <|startoftranscript|> is the input
            kw["nospeech"] = (plen - n_init, self.st.no_timestamps_token_id - 1)
        if num_beams > 1:
            from .beam import beam_search

            want_bidx = opts.record_alignment or n_init is not None  # which slot produced each token of the winner
            res = beam_search(self.eng, prompts, A, num_beams, opts, max_new, return_beam_indices=want_bidx, **kw)
            gen, steps, eos_seen = res[:3]
            if want_bidx:
                self._beam_indices = res[3]
            if n_init is not None:
                seqs = [self._hf_row(np.concatenate([g, [opts.eos_token]]) if e else g, opts) for g, e in zip(gen, eos_seen)]
                self._window_scores = self._nospeech_stats(seqs, plen, n_init, num_beams, tlp=res[4])
            return gen, steps, eos_seen
        gen, toks, done = self.eng.greedy(prompts, A, opts, max_new, **kw)
        first_eos = []
        for a in range(A):
            row = toks[a, plen:plen + done]
            w = np.where(row == opts.eos_token)[0]
            first_eos.append(int(w[0]) + 1 if len(w) else done)
        n_steps = min(done, max(first_eos)) if A else 0
        if n_init is not None:
            seqs = [self._hf_row(toks[a, plen:plen + n_steps], opts) for a in range(A)]
            self._window_scores = self._nospeech_stats(seqs, plen, n_init, 1)
        return gen, n_steps, [fe <= done and (toks[a, plen:plen + done] == opts.eos_token).any() for a, fe in enumerate(first_eos)]

    @staticmethod
    def _hf_row(row: np.ndarray, opts: DecodeOptions) -> np.ndarray:
        """The sequence transformers scores (generate_with_fallback): trailing pads dropped, one kept when pad is EOS."""
        row = np.asarray(row, dtype=np.int64)
        if len(row) and row[-1] == opts.pad_token:
            n = int((row == opts.pad_token).sum()) - (1 if opts.pad_token == opts.eos_token else 0)
            if n:
                row = row[:-n]
        return row

    def _nospeech_stats(self, seqs: List[np.ndarray], plen: int, n_init: int, G: int, tlp: Optional[np.ndarray] = None):
        """avg_logprob and no_speech_prob per row (_retrieve_avg_logprobs, WhisperNoSpeechDetection).  Greedy: the mean of the
        processed log-probs of the row's tokens.  Beam: along the winner's `beam_indices`, raw log-prob minus the slot's lmass at
        that step.  no_speech_prob is read at slot a * G, except when n_init == 1 under beam search: transformers then reads row a
        of its beam-expanded first-step scores, which is slot a."""
        lp, lmass, nsp = self.eng.decode_scores()
        A = len(seqs)
        avg = np.zeros(A, dtype=np.float64)
        for a, seq in enumerate(seqs):
            n = len(seq)
            if n == 0:
                continue
            if G > 1:
                slots = self._beam_indices[a, :n]
                vals = tlp[a, :n].astype(np.float64) - lmass[slots, plen + np.arange(n)]
            else:
                vals = lp[a, plen:plen + n].astype(np.float64)
            avg[a] = vals.sum() / n
        ns = nsp[np.arange(A)] if (G > 1 and n_init == 1) else nsp[np.arange(A) * G]
        return avg, ns.astype(np.float64)

    def _token_timestamps(self, A: int, plen: int, n_steps: int, num_frames: np.ndarray) -> List[np.ndarray]:
        """HF layout: zeros for the prompt, one time per generated position, last one duplicated (:375-379)."""
        bidx = getattr(self, "_beam_indices", None)
        if bidx is not None:
            # beam search (generation_whisper.py:265-301): the cross-attention row of step i comes from the sequence slot that was the
            # returned sequence's ancestor at that step (`beam_indices`); the length is the longest returned sequence of the batch;
            # steps beyond a shorter sequence's end (-1) read slot 0, exactly as the reference's masked_fill(…, 0) does
            n_valid = int((bidx != -1).sum(-1).max())
            T = n_valid - 1
            out = [np.zeros(plen + n_valid, dtype=np.float32) for _ in range(A)]
            if T >= 1 and A > 0:
                Tc = min(T, self.eng.max_align_steps)
                smap = np.where(bidx[:, 1:Tc + 1] >= 0, bidx[:, 1:Tc + 1], 0)  # row r <- the forward pass that consumed generated token r
                nfs = [max(1, min(int(num_frames[a]) // 2, self.eng.S)) for a in range(A)]
                jt = self.eng.word_timestamps_gather(smap, [Tc] * A, nfs, self.time_precision)
                for a in range(A):
                    out[a][plen:plen + Tc + 1] = jt[a, : Tc + 1]
            return out
        T = n_steps - 1
        out = [np.zeros(plen + n_steps, dtype=np.float32) for _ in range(A)]
        if T >= 1 and A > 0:  # all audios of the batch in one pass of the four timestamp kernels
            Tc = min(T, self.eng.max_align_steps)
            nfs = [max(1, min(int(num_frames[a]) // 2, self.eng.S)) for a in range(A)]
            jt = self.eng.word_timestamps_batch(list(range(A)), [Tc] * A, nfs, self.time_precision)
            for a in range(A):
                out[a][plen:plen + Tc + 1] = jt[a, : Tc + 1]
        return out

    def _split_segments(self, seq: np.ndarray, time_offset: float, seek_num_frames: int, idx_offset: int,
                        token_ts: Optional[np.ndarray]):
        """_retrieve_segment (generation_whisper.py:1976-2073) for one sequence: -> (segments, segment_offset frames)"""
        tb = self.timestamp_begin
        tp = self.time_precision
        is_ts = seq >= tb
        single_ending = is_ts[-2:].tolist() == [False, True]
        pair_idx = (np.where(is_ts[:-1] & is_ts[1:])[0] + 1).tolist()
        segs = []
        if len(pair_idx) > 0:
            slices = list(pair_idx)
            if single_ending:
                slices.append(len(seq))
            else:
                slices[-1] += 1
            last = 0
            for i, cur in enumerate(slices):
                is_last = i == len(slices) - 1
                sl = seq[last:cur]
                start_pos = int(sl[0]) - tb
                end_pos = int(sl[-1 if (not is_last or single_ending) else -2]) - tb
                s = {"start": time_offset + start_pos * tp, "end": time_offset + end_pos * tp, "tokens": sl,
                     "idxs": (idx_offset + last, idx_offset + cur)}
                if token_ts is not None:
                    s["token_timestamps"] = token_ts[idx_offset + last: idx_offset + cur] + time_offset
                segs.append(s)
                last = cur
            if single_ending:
                offset = seek_num_frames
            else:
                offset = (int(seq[last - 2]) - tb) * 2  # input_stride = 2 mel frames per encoder position
        else:
            ts_tokens = seq[is_ts]
            last_pos = float(int(seek_num_frames * 0.01 / tp))
            if len(ts_tokens) > 0 and int(ts_tokens[-1]) != tb:
                last_pos = float(int(ts_tokens[-1]) - tb)
            s = {"start": time_offset, "end": time_offset + last_pos * tp, "tokens": seq, "idxs": (idx_offset, idx_offset + len(seq))}
            if token_ts is not None:
                s["token_timestamps"] = token_ts[idx_offset: idx_offset + len(seq)] + time_offset
            segs.append(s)
            offset = seek_num_frames
        return segs, offset

    # --------------------------------------------------------------------------------------------------------
    def _max_new(self, plen: int, n_init: int, max_new_tokens: Optional[int]) -> int:
        """_set_max_new_tokens_and_length for a window whose decoder input is plen long (n_init of it init tokens): the length error,
        then the default budget, which grows by the conditioning tokens (prompt / previous text) up to max_target_positions."""
        st, mtp = self.st, self.eng.dims.max_target_positions
        if (max_new_tokens or 0) + plen > mtp:  # same check, same message as TF generation_whisper.py:1920-1930
            raise ValueError(
                f"The length of `decoder_input_ids`, including special start tokens, prompt tokens, and previous tokens, is {plen}, "
                f" and `max_new_tokens` is {max_new_tokens or 0}. Thus, the combined length of "
                f"`decoder_input_ids` and `max_new_tokens` is: {(max_new_tokens or 0) + plen}. This exceeds the "
                f"`max_target_positions` of the Whisper model: {mtp}. "
                "You should either reduce the length of your prompt, or reduce the value of `max_new_tokens`, "
                f"so that their combined length is less than {mtp}.")
        if max_new_tokens is not None:
            max_new = max_new_tokens
        elif plen > n_init:
            max_new = min(st.max_length + min(mtp // 2 - 1, plen - 1), mtp) - plen
        else:
            max_new = st.max_length - plen
        return min(max_new, mtp - plen)  # (only the max_length default can get past it)

    def _previous_tokens(self, segs: list, bos: Optional[np.ndarray]) -> np.ndarray:
        """One row of _pad_to_max_length(..., cut_off_length=max_target_positions // 2 - 1, skip_ending_double_timestamps=True)
        before the padding: the row's segment tokens (a segment ending on two timestamps loses the last), the last 223 of them,
        behind `bos` (<|startofprev|>, or the prompt with prompt_condition_type="all-segments")."""
        tb, cut = self.timestamp_begin, self.eng.dims.max_target_positions // 2 - 1
        parts = []
        for d in segs:
            t = np.asarray(d["tokens"], dtype=np.int64)
            parts.append(t[:-1] if len(t) > 2 and t[-2] >= tb else t)
        seq = np.concatenate(parts)[-cut:] if parts else np.zeros(0, dtype=np.int64)
        if bos is not None:
            seq = np.concatenate([bos.astype(np.int64), seq])
        return seq

    def generate(self, B: int, num_frames: Optional[np.ndarray] = None, mel_f32: Optional[torch.Tensor] = None,
                 return_timestamps: bool = False, return_token_timestamps: bool = False, language=None, task=None,
                 num_beams: int = 1, max_new_tokens: Optional[int] = None, extra_suppress: Sequence[int] = (),
                 encoded: bool = False, prompt_ids=None, prompt_condition_type: Optional[str] = None,
                 max_frames: Optional[np.ndarray] = None, condition_on_prev_tokens: bool = False,
                 no_speech_threshold: Optional[float] = None, logprob_threshold: Optional[float] = None):
        """Returns a dict with "sequences" (list of int arrays: generated ids, prompt and EOS stripped), optionally
        "token_timestamps" (list of float arrays aligned with sequences) and "segments".

        Short form (mel_f32 [B, n_mels, frames] of one window): the engine's mel buffer must hold the B chunks (engine.logmel /
        set_mel).  Long form (mel_f32 longer than the window, engine.logmel_long): transformers' sequential algorithm -- each
        window at `seek` is cut from mel_f32, encoded, decoded with the timestamp rules and split into segments, and `seek` moves to
        the end of the last complete segment; max_frames [B] are the items' own frame counts (attention mask), num_frames
        (token timestamps) default to them.  Long form requires timestamps (transformers' ValueError otherwise).
        prompt_ids (tensor, array or list of ids, e.g. from get_prompt_ids): decoded as prompt + init tokens on the first window
        (prompt_condition_type "first-segment") or on every window ("all-segments", needs condition_on_prev_tokens), as
        transformers' generate does (generation_whisper.py _prepare_decoder_input_ids).
        condition_on_prev_tokens: from the second window on, the decoder input of every row is [<|startofprev|> (or the prompt),
        last 223 tokens of its text so far] + init tokens, the rows left-padded to the longest; the pads are masked by a key start
        per row.  The conditioning positions run through the decoder in one batched prefill pass.
        no_speech_threshold with logprob_threshold (both or neither): a window of a row is skipped -- no tokens, no segment, `seek`
        moves by the window's frame count, the row's history is unchanged -- when its avg_logprob < logprob_threshold and its
        no_speech_prob > no_speech_threshold, as transformers decides it at one temperature (_need_fallback).  The decode then runs
        with scores (engine.decode_scores_enable); with a prompt or history the prefill stops before <|startoftranscript|>.
        self.window_stats["skipped"] counts skipped windows over all rows, and self.window_log holds per window the (avg_logprob, no_speech_prob,
        skipped) of each of its rows."""
        if (no_speech_threshold is None) != (logprob_threshold is None):
            raise ValueError("no_speech_threshold and logprob_threshold go together: set both or neither")
        nospeech = no_speech_threshold is not None
        eng, st = self.eng, self.st
        if prompt_condition_type not in (None, "first-segment", "all-segments"):
            raise ValueError(f"`prompt_condition_type={prompt_condition_type} does not exist. Make sure to set `prompt_condition_type` "
                             "to one of first-segment, all-segments")
        if prompt_condition_type == "all-segments" and not condition_on_prev_tokens:
            raise NotImplementedError("prompt_condition_type='all-segments' needs condition_on_prev_tokens=True")
        all_segments = prompt_condition_type == "all-segments"
        prompt = None
        if prompt_ids is not None:
            if isinstance(prompt_ids, torch.Tensor):
                prompt_ids = prompt_ids.detach().cpu().numpy()
            prompt = np.asarray(prompt_ids, dtype=np.int64).reshape(-1).astype(np.int32)
        F = eng.frames
        if mel_f32 is None:
            raise ValueError("generate needs the fp32 features (engine.logmel(..., return_f32=True)) for the seek loop")
        total_frames = int(mel_f32.shape[-1])
        long_form = total_frames > F
        if long_form:
            if not return_timestamps:  # _set_return_timestamps, same message
                raise ValueError(
                    "You have passed more than 3000 mel input features (> 30 seconds) which automatically "
                    "enables long-form generation which requires the model to predict timestamp tokens. Please "
                    "either pass `return_timestamps=True` or make sure to pass no more than 3000 mel input features.")
            return_timestamps = True
        if return_token_timestamps:
            return_timestamps = True
            if not eng.alignment_heads:
                raise ValueError("Model generation config has no `alignment_heads`, token-level timestamps not available.")
        max_frames = np.full(B, total_frames, dtype=np.int64) if max_frames is None else np.asarray(max_frames, dtype=np.int64)
        if num_frames is None:
            num_frames = max_frames if long_form else np.full(B, F, dtype=np.int64)
        num_frames = np.asarray(num_frames, dtype=np.int64)
        # the encoder output of mel_f32[:, :, :F] for all B rows is resident: short form (the engine's mel buffer), or long form
        # when the language is detected (once, on the first window, as transformers' detect_language reads it)
        resident = encoded
        if not long_form and not encoded:
            eng.encode(B)
            resident = True
        detect = not isinstance(language, (list, tuple)) and language is None and bool(st.lang_to_id) and st.is_multilingual
        if long_form and detect and not resident:
            eng.set_mel(mel_f32[:, :, :F])
            eng.encode(B)
            resident = True
        init_all = self.init_tokens(B, language, task, return_timestamps)
        n_init = init_all.shape[1]
        opts = self._opts(return_timestamps, return_token_timestamps, extra_suppress)
        if max_new_tokens is not None or prompt is not None:
            self._max_new(n_init + (len(prompt) if prompt is not None else 0), n_init, max_new_tokens)  # refused before any decode
        # _prepare_segments: with a first-segment prompt every row's history starts with the prompt (without <|startofprev|>)
        prev_sot = st.prev_sot_token_id if st.prev_sot_token_id is not None else (
            int(st.suppress_tokens[-2]) if len(st.suppress_tokens) >= 2 else None)
        segments: List[list] = [[] for _ in range(B)]
        n_hidden = 0
        if prompt is not None and not all_segments:
            p0 = prompt[1:] if st.prev_sot_token_id is not None and int(prompt[0]) == st.prev_sot_token_id else prompt
            segments = [[{"tokens": p0.astype(np.int64)}] for _ in range(B)]
            n_hidden = 1
        tb = self.timestamp_begin
        self.window_stats = {"windows": 0, "conditioned": 0, "left_padded": 0, "history_cut": 0, "skipped": 0}
        self.window_log = []

        seek = np.zeros(B, dtype=np.int64)
        first = True
        while (seek < max_frames).any():
            rows = [i for i in range(B) if seek[i] < max_frames[i]]
            A = len(rows)
            seek_num_frames = np.minimum(max_frames - seek, F)
            if not (first and A == B and resident and all(seek[i] == 0 and seek_num_frames[i] == F for i in rows)):
                # cut the remaining features of every active row, zero-pad to the window (:1831-1850), re-encode
                seg = torch.zeros((A, eng.dims.n_mels, F), dtype=torch.float32, device=mel_f32.device)
                for j, i in enumerate(rows):
                    n = int(seek_num_frames[i])
                    seg[j, :, :n] = mel_f32[i, :, int(seek[i]): int(seek[i]) + n]
                eng.set_mel(seg)
                eng.encode(A)
            first = False
            # decoder input (_prepare_decoder_input_ids): conditioning once row 0 has a history, else prompt + init, else init
            key_start = None
            if condition_on_prev_tokens and len(segments[0]) > 0:
                bos = prompt if (prompt is not None and all_segments) else (
                    np.asarray([prev_sot], dtype=np.int64) if prev_sot is not None else None)
                prev = [self._previous_tokens(segments[i], bos) for i in rows]
                width = max(len(p) for p in prev)
                ids = np.full((A, width), st.pad_token_id, dtype=np.int64)
                for j, p in enumerate(prev):
                    ids[j, width - len(p):] = p
                prompts = np.concatenate([ids, init_all[rows]], axis=1).astype(np.int32)
                valid = prompts != st.pad_token_id  # decoder_attention_mask; the pads sit on the left
                ks = valid.argmax(axis=1)
                if not all(valid[j, ks[j]:].all() for j in range(A)):
                    raise NotImplementedError("a conditioning token equals pad_token_id: the decoder mask would not be a key start")
                key_start = ks.astype(np.int32) if (ks > 0).any() else None
                self.window_stats["conditioned"] += 1
                self.window_stats["left_padded"] += int(key_start is not None)
                cut = eng.dims.max_target_positions // 2 - 1
                self.window_stats["history_cut"] += sum(
                    sum(len(d["tokens"]) - (1 if len(d["tokens"]) > 2 and d["tokens"][-2] >= tb else 0) for d in segments[i]) > cut
                    for i in rows)
            elif prompt is not None:
                prompts = np.concatenate([np.repeat(prompt[None, :], A, axis=0), init_all[rows]], axis=1)
            else:
                prompts = init_all[rows]
            plen = prompts.shape[1]
            max_new = self._max_new(plen, n_init, max_new_tokens)
            self.window_stats["windows"] += 1
            kw = {"prefill": True} if plen > n_init else {}
            if key_start is not None:
                kw["key_start"] = key_start
            if nospeech:
                kw["n_init"] = n_init
            gen, n_steps, _ = self._decode(prompts, A, opts, max_new, num_beams, **kw)
            skip = np.zeros(A, dtype=bool)
            if nospeech:
                avg_lp, ns_prob = self._window_scores
                skip = (avg_lp < logprob_threshold) & (ns_prob > no_speech_threshold)
                self.window_stats["skipped"] += int(skip.sum())
                self.window_log.append([(float(avg_lp[j]), float(ns_prob[j]), bool(skip[j])) for j in range(A)])
            tts = None
            if return_token_timestamps:
                tts = self._token_timestamps(A, plen, n_steps, (num_frames - seek)[rows])
            for j, i in enumerate(rows):
                if skip[j]:  # (generate_with_fallback's should_skip)
                    seek[i] += seek_num_frames[i]
                    continue
                seq = np.asarray(gen[j], dtype=np.int64)
                time_offset = float(seek[i]) * self.time_precision / 2.0  # (float64, as transformers computes it off the MPS device)
                if len(seq) == 0:  # (HF runs _retrieve_segment in every mode: timestamp ids are not masked without timestamps)
                    s = {"start": time_offset, "end": time_offset + int(seek_num_frames[i] * 0.01 / self.time_precision) * self.time_precision,
                         "tokens": seq, "idxs": (plen, plen + len(seq))}
                    if tts is not None:
                        s["token_timestamps"] = tts[j][plen: plen + len(seq)] + time_offset
                    segments[i].append(s)
                    seek[i] += seek_num_frames[i]
                    continue
                segs, off = self._split_segments(seq, time_offset, int(seek_num_frames[i]), plen, tts[j] if tts is not None else None)
                segments[i] += segs
                seek[i] += off
        segments = [segs[n_hidden:] for segs in segments]
        out = {"sequences": [np.concatenate([s["tokens"] for s in segs]) if segs else np.zeros(0, dtype=np.int64) for segs in segments],
               "segments": segments}
        if return_token_timestamps:
            out["token_timestamps"] = [np.concatenate([s["token_timestamps"] for s in segs]) if segs else np.zeros(0, dtype=np.float32)
                                       for segs in segments]
        return out
