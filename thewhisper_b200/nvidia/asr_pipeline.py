"""Drop-in for `thestage_speechkit.nvidia.ASRPipeline` (REF thestage_speechkit/nvidia/asr_pipeline.py:30-92) on the
H100-native engine.

Same constructor and call surface (SURVEY.md §8b): `ASRPipeline(model, feature_extractor=None, tokenizer=None,
model_size=None, chunk_length_s=30, device="cuda", torch_dtype=None, batch_size=..., revision=...)` and
`pipe(audio | [audio...] | {"raw"|"array", "sampling_rate"} | path | bytes, chunk_length_s=..., stride_length_s=...,
return_timestamps=None|True|"word", return_language=..., batch_size=..., generate_kwargs={...})`
-> `{"text": str, "chunks": [{"text", "timestamp": (start, end)}]}`.
Without chunk_length_s, an input longer than the window is transcribed with Whisper's sequential long-form algorithm (as
transformers' pipeline does): inputs are grouped batch_size at a time, a group whose longest item fits the window takes the
one-window path, any other group the long-form seek loop of WhisperGenerator.generate (timestamps on; generate_kwargs
condition_on_prev_tokens / prompt_condition_type as in transformers).  generate_kwargs no_speech_threshold with logprob_threshold
skip the windows transformers skips at one temperature, in every mode (the item's text is "" in short form);
compression_ratio_threshold is accepted next to them and has no effect, as in transformers at one temperature.

Everything numeric below the call -- log-mel, encoder, decoder, logits rules, token selection, DTW -- runs in the CUDA
engine through the C-ABI.  What stays on the host is what the reference keeps on the host too: the window schedule of
chunked inference (TF/pipelines/automatic_speech_recognition.py:61-84,428-443) and the token -> text / chunks / words state
machine `WhisperTokenizer._decode_asr` (TF/models/whisper/tokenization_whisper.py:901-1150) with the reference's own seam merge
-- both native since round 2 (csrc/host_decode.cu behind hostproc.AsrDecoder: 123 -> 24 ms for 64 windows x 128 tokens in word
mode; `BW_HOST_DECODE=python` runs the installed tokenizer's instead, for comparison).
There is no CPU fallback: constructing the pipeline without a CUDA device raises.
"""
from __future__ import annotations

from typing import Any, Dict, List, Optional, Sequence, Union

import numpy as np
import torch

from ..engine import ModelDims, WhisperEngine, engine_dtype
from ..features import SAMPLE_RATE, long_form_frames, num_valid_frames, pad_or_trim
from ..generation import GenerationSettings, WhisperGenerator
from ..hostproc import AsrDecoder, chunk_windows, install_merge


class ASRPipeline:
    def __init__(self, model, feature_extractor=None, tokenizer=None, model_size: Optional[str] = None,
                 chunk_length_s: int = 30, device: str = "cuda", torch_dtype: Optional[torch.dtype] = None,
                 decoder_weights: Optional[str] = None, **kwargs):
        # decoder_weights="int8": the decoder matrices every step streams are held as int8 with an fp32 scale per row
        # (WhisperEngine / pack_weights); None keeps them in the engine's 16-bit type.  Independent of `model_size`.
        self.decoder_weights = decoder_weights
        revision = kwargs.pop("revision", "main")
        self.batch_size = int(kwargs.pop("batch_size", 1) or 1)
        self.max_beams = int(kwargs.pop("max_beams", 5))
        preloaded = kwargs.pop("weights", None)  # packed device weights (e.g. received by NCCL broadcast from rank 0)
        if isinstance(model, str):
            # weights come from a HF checkpoint; `model_size` ("S"/"XL") selected a TensorRT engine flavour in the
            # reference (REF :47-56) -- here there is one engine, so it is accepted and ignored.
            from transformers import WhisperFeatureExtractor, WhisperForConditionalGeneration, WhisperTokenizer

            name = model
            model = WhisperForConditionalGeneration.from_pretrained(name, revision=revision)
            if feature_extractor is None:
                feature_extractor = WhisperFeatureExtractor.from_pretrained(name, chunk_length=chunk_length_s)
            if tokenizer is None:
                tokenizer = WhisperTokenizer.from_pretrained(name)
        else:
            if feature_extractor is None:
                raise ValueError("feature_extractor must be provided when passing a model instance")
            if tokenizer is None:
                raise ValueError("tokenizer must be provided when passing a model instance")
        # the reference interpolates the positional table for ANY chunk length (REF asr_pipeline.py:15-27, :91-92); the kernels need a
        # whole number of encoder positions S = 1500 * c / 30 with 50 <= S <= 1500
        if not (1 <= chunk_length_s <= 30) or abs(1500 * chunk_length_s / 30 - round(1500 * chunk_length_s / 30)) > 1e-9:
            raise ValueError(f"chunk_length_s={chunk_length_s} is not supported: it must lie in 1..30 s and give a whole number of encoder "
                             f"positions (a multiple of 0.02 s)")
        self.chunk_length_s = chunk_length_s
        # torch_dtype picks the engine's 16-bit element type: float16 as the reference's streaming / benchmark paths pass it, else
        # bfloat16 (None / float32 = the reference's default fp32 model: the engine has no fp32-operand mode and says so once)
        self.torch_dtype = torch_dtype
        self.engine_dtype = engine_dtype(torch_dtype if torch_dtype is not None else getattr(model, "dtype", None))
        if torch_dtype in (None, torch.float32) and getattr(model, "dtype", torch.float32) == torch.float32:
            import warnings

            warnings.warn("thewhisper_b200: fp32 operands are not supported; running bfloat16 operands with fp32 accumulation "
                          "(pass torch_dtype=torch.float16 for the reference's fp16 mode)", stacklevel=2)
        self.tokenizer = tokenizer
        self.feature_extractor = feature_extractor
        self.config = model.config
        self.generation_config = model.generation_config
        self.settings = GenerationSettings.from_hf(model.generation_config, model.config)
        self.dims = ModelDims.from_hf_config(model.config)
        if self.dims.max_source_positions != 1500:  # an already patched model: undo, the engine interpolates itself
            self.dims.max_source_positions = 1500
        dev = device if isinstance(device, str) else str(device)
        if dev == "cuda":
            dev = f"cuda:{torch.cuda.current_device()}" if torch.cuda.is_available() else "cuda:0"
        self.device = dev
        self._state_dict = None if preloaded is not None else {k: v for k, v in model.state_dict().items()}
        self._weights = preloaded
        self.engine: Optional[WhisperEngine] = None
        self._build_engine(self.batch_size)
        install_merge()
        import os as _os

        # tokens -> text in the native library; the installed tokenizer's own state machine only on request
        self._asr_decode = None if _os.environ.get("BW_HOST_DECODE", "") == "python" else AsrDecoder(tokenizer)

    # ------------------------------------------------------------------------------------------------------------
    def _build_engine(self, capacity: int) -> None:
        if self.engine is not None:
            self._weights = self.engine.weights
            self.engine.close()
        self.engine = WhisperEngine(self._state_dict, self.dims, chunk_length_s=self.chunk_length_s, device=self.device,
                                    max_audios=capacity, max_beams=self.max_beams,
                                    alignment_heads=self.settings.alignment_heads, weights=self._weights, dtype=self.engine_dtype,
                                    decoder_weights=self.decoder_weights)
        self._weights = self.engine.weights
        self._state_dict = None if self._weights is not None else self._state_dict
        self.capacity = capacity
        self.generator = WhisperGenerator(self.engine, self.settings)

    # ------------------------------------------------------------------------------------------------------------
    @staticmethod
    def _to_array(inputs) -> np.ndarray:
        if isinstance(inputs, (str, bytes)):
            from transformers.pipelines.audio_utils import ffmpeg_read

            if isinstance(inputs, str):
                with open(inputs, "rb") as f:
                    inputs = f.read()
            inputs = ffmpeg_read(inputs, SAMPLE_RATE)
        if isinstance(inputs, dict):
            inputs = dict(inputs)
            if not ("sampling_rate" in inputs and ("raw" in inputs or "array" in inputs)):
                raise ValueError('When passing a dictionary to AutomaticSpeechRecognitionPipeline, the dict needs to contain a '
                                 '"raw" key containing the numpy array or torch tensor representing the audio and a "sampling_rate" key')
            arr = inputs.pop("raw", None)
            if arr is None:
                arr = inputs.pop("array")
            sr = inputs.pop("sampling_rate")
            if isinstance(arr, torch.Tensor):
                arr = arr.detach().cpu().numpy()
            if sr != SAMPLE_RATE:
                from torchaudio import functional as AF  # same dependency the reference path has for resampling

                arr = AF.resample(torch.from_numpy(np.asarray(arr, dtype=np.float32)), sr, SAMPLE_RATE).numpy()
            inputs = arr
        if isinstance(inputs, torch.Tensor):
            inputs = inputs.detach().cpu().numpy()
        if not isinstance(inputs, np.ndarray):
            raise TypeError(f"We expect a numpy ndarray or torch tensor as input, got `{type(inputs)}`")
        if inputs.ndim != 1:
            inputs = inputs.mean(axis=0)
        return np.asarray(inputs, dtype=np.float32)

    def _windows(self, audio: np.ndarray, chunk_length_s, stride_length_s):
        n_samples = self.engine.n_samples
        if chunk_length_s:
            if stride_length_s is None:
                stride_length_s = chunk_length_s / 6
            if isinstance(stride_length_s, (int, float)):
                stride_length_s = [stride_length_s, stride_length_s]
            chunk_len = int(round(chunk_length_s * SAMPLE_RATE))
            sl = int(round(stride_length_s[0] * SAMPLE_RATE))
            sr = int(round(stride_length_s[1] * SAMPLE_RATE))
            if chunk_len < sl + sr:
                raise ValueError("Chunk length must be superior to stride length")
            for start, end, stride, is_last in chunk_windows(audio.shape[0], chunk_len, sl, sr):
                yield audio[start:end], stride
        else:  # the whole input: one window, or sequential long-form transcription when it is longer
            yield audio, None

    # ------------------------------------------------------------------------------------------------------------
    def __call__(self, inputs, **kwargs):
        is_list = isinstance(inputs, (list, tuple))
        items = list(inputs) if is_list else [inputs]
        chunk_length_s = kwargs.pop("chunk_length_s", self.chunk_length_s)
        stride_length_s = kwargs.pop("stride_length_s", None)
        return_timestamps = kwargs.pop("return_timestamps", None)
        return_language = kwargs.pop("return_language", None)
        batch_size = int(kwargs.pop("batch_size", self.batch_size) or 1)
        generate_kwargs = dict(kwargs.pop("generate_kwargs", None) or {})
        if "max_new_tokens" in kwargs:
            generate_kwargs["max_new_tokens"] = kwargs.pop("max_new_tokens")
        if return_timestamps not in (None, False, True, "word"):
            raise ValueError("Whisper cannot return `char` timestamps, only word level or segment level timestamps. "
                             "Use `return_timestamps='word'` or `return_timestamps=True` respectively.")
        if generate_kwargs.get("do_sample"):
            raise NotImplementedError("sampling is not part of the engine (greedy / beam only)")
        temperature = generate_kwargs.get("temperature")
        if isinstance(temperature, (list, tuple)) or (temperature is not None and temperature > 0.0):
            raise NotImplementedError(f"temperature={temperature!r}: temperature fallback samples, and sampling is not part of the engine "
                                      "(greedy / beam only)")
        # no-speech skipping needs both thresholds; at one temperature compression_ratio_threshold only marks a fallback that
        # never runs, so next to them it is accepted and has no effect (as in transformers)
        no_speech = generate_kwargs.get("no_speech_threshold") is not None and generate_kwargs.get("logprob_threshold") is not None
        if not no_speech:
            for name in ("logprob_threshold", "compression_ratio_threshold", "no_speech_threshold"):
                if generate_kwargs.get(name) is not None:
                    raise NotImplementedError(f"{name} is not implemented: the engine has no temperature fallback, and no-speech "
                                              "skipping needs both no_speech_threshold and logprob_threshold")
        condition = bool(generate_kwargs.get("condition_on_prev_tokens") or False)
        num_beams = int(generate_kwargs.get("num_beams", 1) or 1)
        if num_beams > self.max_beams:
            raise ValueError(f"num_beams={num_beams} exceeds the engine's max_beams={self.max_beams}")
        if batch_size > self.capacity:
            self._build_engine(batch_size)

        # ---- window schedule over all inputs, flattened like PipelineChunkIterator (pt_utils.py:156-198)
        flat: List[dict] = []
        for idx, item in enumerate(items):
            audio = self._to_array(item)
            for chunk, stride in self._windows(audio, chunk_length_s, stride_length_s):
                flat.append({"input": idx, "audio": chunk, "stride": stride})
        per_input: List[List[dict]] = [[] for _ in items]
        n_samples = self.engine.n_samples
        import time as _time

        tm = {"windows_s": 0.0, "generate_s": 0.0, "decode_asr_s": 0.0}  # host wall clock per phase of this call (diagnostics)
        t_ph = _time.perf_counter()
        for b0 in range(0, len(flat), batch_size):
            group = flat[b0:b0 + batch_size]
            B = len(group)
            longest = max(len(g["audio"]) for g in group)
            if longest <= n_samples:  # one window per item
                pcm = np.stack([pad_or_trim(g["audio"], n_samples) for g in group])
                num_frames = np.asarray([num_valid_frames(len(g["audio"]), n_samples) for g in group], dtype=np.int64)
                mel = self.engine.logmel(pcm, return_f32=True)
                long_kw = {}
            else:  # sequential long form: features of the group zero-padded to its longest item, each item's own frame count
                pcm = np.stack([pad_or_trim(g["audio"], longest) for g in group])
                num_frames = np.asarray([long_form_frames(len(g["audio"]), longest) for g in group], dtype=np.int64)
                mel = self.engine.logmel_long(pcm)
                if mel.shape[-1] > self.engine.frames:
                    long_kw = {"max_frames": num_frames}
                else:  # under 160 samples past the window: still one window of features (transformers' short form), which
                    # generate encodes from the engine's mel buffer -- bw_logmel_long does not write it
                    self.engine.set_mel(mel)
                    long_kw = {}
            tm["windows_s"] += _time.perf_counter() - t_ph
            t_ph = _time.perf_counter()
            out = self.generator.generate(
                B, num_frames=num_frames, mel_f32=mel, return_timestamps=bool(return_timestamps),
                return_token_timestamps=(return_timestamps == "word"), language=generate_kwargs.get("language"),
                task=generate_kwargs.get("task"), num_beams=num_beams, max_new_tokens=generate_kwargs.get("max_new_tokens"),
                prompt_ids=generate_kwargs.get("prompt_ids"), prompt_condition_type=generate_kwargs.get("prompt_condition_type"),
                condition_on_prev_tokens=condition, no_speech_threshold=generate_kwargs.get("no_speech_threshold") if no_speech else None,
                logprob_threshold=generate_kwargs.get("logprob_threshold") if no_speech else None, **long_kw)
            for j, g in enumerate(group):
                o: Dict[str, Any] = {"tokens": np.asarray(out["sequences"][j], dtype=np.int64)[None, :]}
                if return_timestamps == "word":
                    o["token_timestamps"] = np.asarray(out["token_timestamps"][j], dtype=np.float32)[None, :]
                if g["stride"] is not None:
                    ln, sl, sr = g["stride"]
                    o["stride"] = (ln / SAMPLE_RATE, sl / SAMPLE_RATE, sr / SAMPLE_RATE)
                per_input[g["input"]].append(o)
            tm["generate_s"] += _time.perf_counter() - t_ph
            t_ph = _time.perf_counter()

        # ---- tokens -> text (+ chunks): string-side state machine of the installed tokenizer
        time_precision = self.feature_extractor.chunk_length / self.engine.S
        results = []
        for outs in per_input:
            decode = self._asr_decode if self._asr_decode is not None else self.tokenizer._decode_asr
            text, optional = decode(outs, return_timestamps=return_timestamps, return_language=return_language, time_precision=time_precision)
            results.append({"text": text, **optional})
        tm["decode_asr_s"] = _time.perf_counter() - t_ph
        self.last_timing = tm
        return results if is_list else results[0]
