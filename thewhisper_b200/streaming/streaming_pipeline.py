"""Streaming transcription on the engine: drop-in for `thestage_speechkit.streaming.StreamingPipeline`
(REF thestage_speechkit/streaming/streaming_pipeline.py:443-988) plus the multi-stream scheduler that replaces the
reference's one-stream-at-a-time design (SURVEY.md §2.1 row 3, §7 step 10).

Per stream the behaviour is the reference's: small chunks are accumulated (optionally VAD-gated, REF :640-738) until
`min_process_chunk_s`, the whole rolling buffer is re-transcribed with word timestamps (REF :740-776), the words are
cleaned up (REF :824-876), and once the buffer exceeds `chunk_length_s - 1 - min_process_chunk_s` seconds (or speech just
ended and it holds > 6 s) everything before a truncation point -- last sentence end older than 2 s, else last
comma, else longest pause, ... (REF :885-937) -- is committed and trimmed (REF :939-951).

What is new: `process_new_chunk` is split into `prepare()` (everything up to the backend call) and `complete(words)`
(everything after), so `StreamScheduler` can gather the ready buffers of many streams, run them through the engine as
ONE batch per tick, and hand each stream its words.  `StreamingPipeline.__call__` is still prepare -> backend -> complete
for a single stream.
"""
from __future__ import annotations

import zlib
from abc import ABC, abstractmethod
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np

Word = Dict[str, Any]


def _compression_ratio(text: str) -> float:
    raw = text.encode("utf-8")
    return len(raw) / len(zlib.compress(raw))


class TranscriptionBackend(ABC):
    """audio buffer -> [{"text", "start", "end"}] with absolute times in seconds (REF :51-64)."""

    @abstractmethod
    def transcribe(self, audio: np.ndarray, buffer_start_time: float, sample_rate: int) -> List[Word]: ...

    def transcribe_many(self, audios: Sequence[np.ndarray], buffer_start_times: Sequence[float], sample_rate: int) -> List[List[Word]]:
        return [self.transcribe(a, t, sample_rate) for a, t in zip(audios, buffer_start_times)]


def words_from_result(result: Dict[str, Any], audio_duration: float, buffer_start_time: float) -> List[Word]:
    """Pipeline output -> absolute-time words (REF :412-435): gibberish filter (zlib ratio > 2.2), open-ended last word
    capped to at most 1 s."""
    if _compression_ratio(result["text"]) > 2.2:
        return []
    out: List[Word] = []
    for ch in result["chunks"]:
        start, end = ch["timestamp"]
        if end is None:
            end = audio_duration if audio_duration - start < 1.0 else start + 1.0
        out.append({"text": ch["text"], "start": start + buffer_start_time, "end": end + buffer_start_time})
    return out


class LocalWhisperBackend(TranscriptionBackend):
    """REF :340-435 over the engine's ASRPipeline.  `platform` must be "nvidia"."""

    def __init__(self, model, model_size: str = "S", chunk_length_s: int = 10, platform: str = "nvidia", torch_dtype=None,
                 language: str = "en", feature_extractor=None, tokenizer=None, revision: str = "main", asr_pipeline=None,
                 batch_size: int = 1, device: str = "cuda", decoder_weights=None):
        if platform != "nvidia":
            raise ValueError(f"Invalid platform: {platform} (this build is the NVIDIA H100 engine)")
        self.chunk_length_s = chunk_length_s
        self.sample_rate = 16000
        self.device = device
        self.language = language
        if asr_pipeline is None:
            from ..nvidia import ASRPipeline

            asr_pipeline = ASRPipeline(model, model_size=model_size, chunk_length_s=chunk_length_s, torch_dtype=torch_dtype,
                                       device=device, feature_extractor=feature_extractor, tokenizer=tokenizer,
                                       revision=revision, batch_size=batch_size, decoder_weights=decoder_weights)
        self.asr_pipeline = asr_pipeline

    def _kwargs(self):
        return {"use_cache": True, "num_beams": 1, "do_sample": False, "max_new_tokens": 128, "language": self.language}

    def transcribe(self, audio, buffer_start_time, sample_rate):
        res = self.asr_pipeline(audio, return_timestamps="word", generate_kwargs=self._kwargs(), chunk_length_s=self.chunk_length_s)
        return words_from_result(res, len(audio) / sample_rate, buffer_start_time)

    def transcribe_many(self, audios, buffer_start_times, sample_rate):
        if not audios:
            return []
        res = self.asr_pipeline(list(audios), return_timestamps="word", generate_kwargs=self._kwargs(),
                                chunk_length_s=self.chunk_length_s, batch_size=len(audios))
        return [words_from_result(r, len(a) / sample_rate, t) for r, a, t in zip(res, audios, buffer_start_times)]


class StreamingPipeline:
    def __init__(self, model="", model_size: str = "S", chunk_length_s: int = 10, min_process_chunk_s: float = 0.5,
                 platform: str = "nvidia", torch_dtype=None, language: str = "en", feature_extractor=None, tokenizer=None,
                 backend: Optional[TranscriptionBackend] = None, use_remote_api: bool = False, api_url=None, api_auth_token=None,
                 api_model_name=None, api_lang_id=None, request_timeout_s=None, bytes_per_sample: int = 2,
                 sample_rate: int = 16000, revision="main", use_vad: bool = True, vad_threshold: float = 0.1,
                 vad_no_speech_chunks: int = 1, vad_prepend_chunks: int = 3, vad_model=None, decoder_weights=None):
        self.sample_rate = sample_rate
        self.chunk_length_s = chunk_length_s
        self.min_process_chunk_s = min_process_chunk_s
        self.window_size = chunk_length_s - 1
        if backend is None:
            if use_remote_api:
                raise NotImplementedError("the HTTP backends of the reference are outside this engine's scope (SURVEY.md §8 f2); "
                                          "inject a TranscriptionBackend instead")
            if not model:
                raise ValueError("model is required when using LocalWhisperBackend")
            backend = LocalWhisperBackend(model=model, model_size=model_size, chunk_length_s=chunk_length_s, platform=platform,
                                          torch_dtype=torch_dtype, language=language, feature_extractor=feature_extractor,
                                          tokenizer=tokenizer, revision=revision, decoder_weights=decoder_weights)
        self.backend = backend
        self.use_vad = use_vad
        self.vad_threshold = vad_threshold
        self._no_speech_threshold = vad_no_speech_chunks
        self._prepend_chunks = vad_prepend_chunks
        self.vad_model = vad_model
        if use_vad and vad_model is None:
            import torch  # Silero VAD as in the reference (REF :533-538); needs network access for torch.hub

            self.vad_model, _ = torch.hub.load(repo_or_dir="snakers4/silero-vad", model="silero_vad", trust_repo=True)
        self._reset_state()

    def _reset_state(self) -> None:
        self.current_audio_buffer: Optional[np.ndarray] = None
        self._pending_chunk: Optional[np.ndarray] = None
        self.buffer_start_time = 0.0
        self.current_time = 0.0
        self.audio_queue: List[np.ndarray] = []
        self.need_to_process = False
        self.history: List[List[Word]] = []
        self._last_committed_word: Optional[str] = None
        self._prev_speech_mode = False
        self._vad_history: List[bool] = []
        self._recent_chunks: List[np.ndarray] = []
        self._in_speech_mode = False
        self._vad_buffer = np.array([], dtype=np.float32)

    def clear(self) -> None:
        """Back to the initial state (REF :967-988)."""
        self._reset_state()
        if self.vad_model is not None and hasattr(self.vad_model, "reset_states"):
            self.vad_model.reset_states()

    # ---- ingest -----------------------------------------------------------------------------------------------------
    def _vad_has_speech(self, audio: np.ndarray) -> bool:
        """Silero expects exactly 512 samples per call and keeps state between calls (REF :589-622)."""
        if self.vad_model is None:
            return True
        import torch

        self._vad_buffer = np.concatenate([self._vad_buffer, audio.astype(np.float32)])
        speech = False
        while len(self._vad_buffer) >= 512:
            frame, self._vad_buffer = self._vad_buffer[:512], self._vad_buffer[512:]
            prob = self.vad_model(torch.from_numpy(frame), self.sample_rate).item()
            if prob > self.vad_threshold:
                speech = True
        return speech

    def _push_pending(self) -> None:
        self.audio_queue.append(self._pending_chunk)
        self.need_to_process = True
        self._pending_chunk = None

    def _append_pending(self, chunk: np.ndarray) -> None:
        self._pending_chunk = chunk if self._pending_chunk is None else np.concatenate([self._pending_chunk, chunk])

    def add_new_chunk(self, chunk: np.ndarray) -> None:
        if chunk is None or len(chunk) == 0:
            return
        if not self.use_vad or self.vad_model is None:
            self._append_pending(chunk)
        else:
            has_speech = self._vad_has_speech(chunk)
            self._recent_chunks.append(chunk)
            if len(self._recent_chunks) > self._prepend_chunks:
                self._recent_chunks.pop(0)
            self._vad_history.append(has_speech)
            if len(self._vad_history) > self._no_speech_threshold:
                self._vad_history.pop(0)
            if self._in_speech_mode:
                self._append_pending(chunk)
                recent = self._vad_history[-self._no_speech_threshold:]
                if len(self._vad_history) >= self._no_speech_threshold and not any(recent):
                    self._in_speech_mode = False  # speech -> silence: flush what was collected
                    if self._pending_chunk is not None and len(self._pending_chunk) > 0:
                        self._push_pending()
            elif has_speech:
                self._in_speech_mode = True  # silence -> speech: keep the pre-roll so the onset is not clipped
                pre = self._recent_chunks[:-1] if len(self._recent_chunks) > 1 else []
                self._pending_chunk = np.concatenate(pre) if pre else None
                self._append_pending(chunk)
        if self._pending_chunk is not None and len(self._pending_chunk) / self.sample_rate >= self.min_process_chunk_s:
            self._push_pending()

    # ---- the two halves of REF process_new_chunk (:740-822) ------------------------------------------------------------------
    def prepare(self) -> Optional[Tuple[np.ndarray, float]]:
        """Drain the queue into the rolling buffer.  Returns (buffer, buffer_start_time) when a transcription is due,
        None when there is nothing to do; `self._idle` says whether complete() must still run."""
        self._idle = True
        if len(self.audio_queue) == 0:
            return None
        chunk = np.concatenate(self.audio_queue)
        self.audio_queue = []
        self.current_time += len(chunk) / self.sample_rate
        self.current_audio_buffer = chunk if self.current_audio_buffer is None else np.concatenate([self.current_audio_buffer, chunk])
        if len(self.current_audio_buffer) < 2.0 * self.sample_rate:
            return None
        self._idle = False
        if self.need_to_process:
            return self.current_audio_buffer, self.buffer_start_time
        return None

    def complete(self, new_words: Optional[List[Word]]) -> Tuple[List[Word], List[Word]]:
        if self._idle:
            return [], []
        committed: List[Word] = []
        uncommitted: List[Word] = []
        if new_words is not None:
            words = self._postprocess_transcribtions(new_words)
            self.need_to_process = False
            uncommitted = words
            self.history.append(words)
        max_allowed = (self.window_size - self.min_process_chunk_s) * self.sample_rate
        must_trim = len(self.current_audio_buffer) > max_allowed
        cut: Optional[float] = None
        if self._prev_speech_mode and not self._in_speech_mode and len(self.current_audio_buffer) > 6 * self.sample_rate:
            must_trim = True
            cut = self.current_time
        self._prev_speech_mode = self._in_speech_mode
        if must_trim:
            final = self.history[-1] if self.history else []
            if cut is None:
                cut = self._get_truncation_time(final, True)
            if cut is not None:
                self._trim_audio_buffer(cut)
                committed = [w for w in final if w["start"] < cut]
                uncommitted = [w for w in final if w["start"] >= cut]
                if committed:
                    self._last_committed_word = committed[-1]["text"].strip()
        return committed, uncommitted

    def process_new_chunk(self) -> Tuple[List[Word], List[Word]]:
        job = self.prepare()
        words = None
        if job is not None:
            words = self.backend.transcribe(audio=job[0], buffer_start_time=job[1], sample_rate=self.sample_rate)
        return self.complete(words)

    def __call__(self, chunk: np.ndarray) -> Tuple[List[Word], List[Word]]:
        self.add_new_chunk(chunk)
        return self.process_new_chunk()

    # ---- text clean-up and commit policy ---------------------------------------------------------------------------
    def _postprocess_transcribtions(self, tokens: List[Word]) -> List[Word]:
        kept: List[Word] = []
        for tok in tokens:
            text = tok["text"]
            if text.strip() and all(c in " ." for c in text):
                if kept:  # a lone "." / " ..." is glued to the previous word
                    kept[-1]["text"] += text.strip()
            else:
                kept.append(tok)
        for tok in kept:
            if tok["text"] and not tok["text"].startswith(" "):
                tok["text"] = " " + tok["text"]
            if tok["text"].startswith(" -"):
                tok["text"] = tok["text"].replace(" -", "-")
            for bad, good in (("gonNA", "gonna"), ("gotTA", "gotta"), ("wanNA", "wanna")):
                tok["text"] = tok["text"].replace(bad, good)
        if len(kept) == 1 and kept[0]["text"].strip() in ("The.", "The", "I."):
            kept = []
        if self._last_committed_word is not None and kept:
            if kept[0]["text"].strip().lower() == self._last_committed_word.lower():
                kept = kept[1:]
        return kept

    def _get_truncation_time(self, final_words: List[Word], need_to_trim: bool = True) -> Optional[float]:
        sentence_i = comma_i = pause_i = None
        longest, prev_end = 0.0, 0.0
        horizon = self.current_time - 2.0
        for i, w in enumerate(final_words):
            text = w["text"].strip()
            if text.endswith((".", "?", "!")) and w["end"] < horizon:
                sentence_i = i
            if text.endswith((",", ";", ":")) and w["end"] < horizon:
                comma_i = i
            gap = w["start"] - prev_end
            if gap >= longest:
                longest, pause_i = gap, i - 1
            prev_end = w["end"]
        if sentence_i:  # (index 0 is falsy in the reference as well)
            return final_words[sentence_i]["end"]
        if comma_i:
            return final_words[comma_i]["end"]
        if not need_to_trim:
            return None
        if pause_i is not None and pause_i >= 0:
            return final_words[pause_i]["end"]
        if len(final_words) >= 2:
            return final_words[-2]["end"]
        if len(final_words) == 1:
            return final_words[0]["end"]
        return self.current_time - self.min_process_chunk_s * 2

    def _trim_audio_buffer(self, truncation_time: float) -> None:
        delta = truncation_time - self.buffer_start_time
        if delta > 0:
            self.current_audio_buffer = self.current_audio_buffer[int(delta * self.sample_rate):]
            self.buffer_start_time = truncation_time
            self.history = [h for h in ([w for w in el if w["start"] >= truncation_time] for el in self.history) if h]


class StreamScheduler:
    """Many streams on one engine: per tick every stream ingests its chunk, the buffers that are due are transcribed as
    one engine batch (`backend.transcribe_many`), and each stream completes with its own words.  Streams are sticky to
    their scheduler / GPU (per-stream buffers are host state, SURVEY.md §8e)."""

    def __init__(self, backend: TranscriptionBackend, n_streams: int, max_batch: Optional[int] = None, **stream_kwargs):
        self.backend = backend
        self.max_batch = max_batch or n_streams
        stream_kwargs.setdefault("use_vad", False)
        self.streams = [StreamingPipeline(backend=backend, **stream_kwargs) for _ in range(n_streams)]
        self.backend_calls = 0
        self.buffers_transcribed = 0

    def step(self, chunks: Sequence[Optional[np.ndarray]]) -> List[Tuple[List[Word], List[Word]]]:
        jobs: List[Tuple[int, np.ndarray, float]] = []
        for i, (s, c) in enumerate(zip(self.streams, chunks)):
            if c is not None:
                s.add_new_chunk(c)
            job = s.prepare()
            if job is not None:
                jobs.append((i, job[0], job[1]))
        words: Dict[int, List[Word]] = {}
        sr = self.streams[0].sample_rate if self.streams else 16000
        for b0 in range(0, len(jobs), self.max_batch):
            group = jobs[b0:b0 + self.max_batch]
            res = self.backend.transcribe_many([g[1] for g in group], [g[2] for g in group], sr)
            self.backend_calls += 1
            self.buffers_transcribed += len(group)
            for g, r in zip(group, res):
                words[g[0]] = r
        return [s.complete(words.get(i)) for i, s in enumerate(self.streams)]
