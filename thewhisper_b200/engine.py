"""WhisperEngine: Python host object over the C-ABI engine (one per GPU / process).

It owns the device weights (torch tensors used purely as device-memory containers), binds them by name into the
native engine, and exposes the three stages of the hot path: log-mel, encode (+ cross-K/V), decode.
No arithmetic of the path happens in Python or in torch ops; torch is used for allocation, H2D/D2H copies and the
current stream handle only.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F

from . import _lib
from .features import HOP, mel_filter_bank


@dataclasses.dataclass
class ModelDims:
    d_model: int
    n_heads: int
    ffn: int
    enc_layers: int
    dec_layers: int
    n_mels: int
    vocab: int
    max_source_positions: int = 1500
    max_target_positions: int = 448

    @staticmethod
    def from_hf_config(cfg) -> "ModelDims":
        return ModelDims(cfg.d_model, cfg.encoder_attention_heads, cfg.encoder_ffn_dim, cfg.encoder_layers,
                         cfg.decoder_layers, cfg.num_mel_bins, cfg.vocab_size, cfg.max_source_positions,
                         cfg.max_target_positions)


@dataclasses.dataclass
class DecodeOptions:
    eos_token: int
    pad_token: int
    suppress_tokens: Sequence[int] = ()
    begin_suppress_tokens: Sequence[int] = ()
    timestamp_rules: bool = False
    timestamp_begin: int = 50365
    no_timestamps_token: int = 50364
    max_initial_timestamp_index: int = -1
    record_alignment: bool = False


def interpolate_positions(table: torch.Tensor, chunk_length_s: float) -> torch.Tensor:
    """Encoder positional table for chunk_length_s < 30: int(1500*c/30) rows by linear interpolation with
    align_corners=False, computed once at load time with torch exactly as the reference does
    (REF thestage_speechkit/nvidia/asr_pipeline.py:15-27; SURVEY.md §7 hard part 8)."""
    n_pos = int(1500 * (chunk_length_s / 30))
    t = table.detach().float().cpu()
    out = F.interpolate(t.t().unsqueeze(0), size=n_pos, mode="linear", align_corners=False)
    return out.squeeze(0).t().contiguous()


ENGINE_DTYPES = {torch.bfloat16: 0, torch.float16: 1}

# The decoder matrices every step streams: per layer (engine names) and the tied embedding / LM head.  With
# decoder_weights="int8" these are int8 codes with an fp32 scale per output row ("<name>.scale"); xwk / xwv stay 16-bit.
INT8_LAYER_KINDS = ("wqkv", "wo", "xwq", "xwo", "w1", "w2")
DECODER_WEIGHTS = (None, "int8")


def quantize_rows(W: torch.Tensor):
    """Per-row symmetric int8: s = amax(|w|, dim=1) / 127 (an all-zero row gets s = 1), q = clamp(round_half_even(w / s),
    -127, 127).  -> (q int8 [N, K], s fp32 [N]); the weight the kernels compute with is exactly s[n] * q[n, k]."""
    w = W.detach().float()
    s = w.abs().amax(dim=1) / 127.0
    s = torch.where(s == 0, torch.ones_like(s), s)
    q = torch.clamp(torch.round(w / s[:, None]), -127, 127).to(torch.int8)  # torch.round rounds half to even
    return q.contiguous(), s.contiguous()


def decoder_weights_of(weights: Dict[str, torch.Tensor]) -> Optional[str]:
    """The decoder-weight format of a packed weight dict: "int8" when it holds "dec.embed.scale", else None."""
    return "int8" if "dec.embed.scale" in weights else None


def engine_dtype(torch_dtype) -> torch.dtype:
    """The 16-bit element type the engine runs for a caller's `torch_dtype` (REF nvidia/asr_pipeline.py:39: None = the checkpoint's
    fp32): float16 -> float16 (what the reference's streaming and benchmark paths use), bfloat16 / None / float32 -> bfloat16.
    Accumulation, softmax, LayerNorm and the residual stream are fp32 in both; there is no fp32-operand mode."""
    return torch.float16 if torch_dtype == torch.float16 else torch.bfloat16


def pack_weights(sd: Dict[str, torch.Tensor], dims: ModelDims, enc_pos: torch.Tensor, device: torch.device,
                 dtype: torch.dtype = torch.bfloat16, decoder_weights: Optional[str] = None) -> Dict[str, torch.Tensor]:
    """HF WhisperForConditionalGeneration state_dict -> named device tensors in the engine's layouts
    (16-bit [out, in] matrices in `dtype`, fp32 vectors; q/k/v fused; conv kernels reordered to [co][tap][ci]).
    decoder_weights="int8": dec.embed and the decoder layers' wqkv / wo / xwq / xwo / w1 / w2 are packed as int8 codes plus
    "<name>.scale" (quantize_rows of the checkpoint's values, on the device), with no 16-bit copy."""
    if decoder_weights not in DECODER_WEIGHTS:
        raise ValueError(f"decoder_weights must be one of {DECODER_WEIGHTS}, got {decoder_weights!r}")
    D = dims.d_model
    out: Dict[str, torch.Tensor] = {}

    def mat(t):
        return t.detach().to(device=device, dtype=dtype).contiguous()

    def dmat(name, t):  # a matrix every decoder step streams
        if decoder_weights == "int8":
            out[name], out[name + ".scale"] = quantize_rows(t.detach().to(device=device))
        else:
            out[name] = mat(t)

    def vec(t):
        return t.detach().to(device=device, dtype=torch.float32).contiguous()

    e = "model.encoder."
    out["enc.conv1.w"] = mat(sd[e + "conv1.weight"].permute(0, 2, 1).reshape(D, -1))
    out["enc.conv1.b"] = vec(sd[e + "conv1.bias"])
    out["enc.conv2.w"] = mat(sd[e + "conv2.weight"].permute(0, 2, 1).reshape(D, -1))
    out["enc.conv2.b"] = vec(sd[e + "conv2.bias"])
    out["enc.pos"] = vec(enc_pos)
    out["enc.lnf.g"] = vec(sd[e + "layer_norm.weight"])
    out["enc.lnf.b"] = vec(sd[e + "layer_norm.bias"])
    zeros = torch.zeros(D)
    for i in range(dims.enc_layers):
        p, o = f"{e}layers.{i}.", f"enc.{i}."
        out[o + "ln1.g"] = vec(sd[p + "self_attn_layer_norm.weight"])
        out[o + "ln1.b"] = vec(sd[p + "self_attn_layer_norm.bias"])
        out[o + "wqkv"] = mat(torch.cat([sd[p + "self_attn.q_proj.weight"], sd[p + "self_attn.k_proj.weight"],
                                         sd[p + "self_attn.v_proj.weight"]], 0))
        out[o + "bqkv"] = vec(torch.cat([sd[p + "self_attn.q_proj.bias"].float().cpu(), zeros,
                                         sd[p + "self_attn.v_proj.bias"].float().cpu()], 0))
        out[o + "wo"] = mat(sd[p + "self_attn.out_proj.weight"])
        out[o + "bo"] = vec(sd[p + "self_attn.out_proj.bias"])
        out[o + "ln2.g"] = vec(sd[p + "final_layer_norm.weight"])
        out[o + "ln2.b"] = vec(sd[p + "final_layer_norm.bias"])
        out[o + "w1"] = mat(sd[p + "fc1.weight"])
        out[o + "b1"] = vec(sd[p + "fc1.bias"])
        out[o + "w2"] = mat(sd[p + "fc2.weight"])
        out[o + "b2"] = vec(sd[p + "fc2.bias"])
    d = "model.decoder."
    dmat("dec.embed", sd[d + "embed_tokens.weight"])
    out["dec.pos"] = vec(sd[d + "embed_positions.weight"])
    out["dec.lnf.g"] = vec(sd[d + "layer_norm.weight"])
    out["dec.lnf.b"] = vec(sd[d + "layer_norm.bias"])
    for i in range(dims.dec_layers):
        p, o = f"{d}layers.{i}.", f"dec.{i}."
        out[o + "ln1.g"] = vec(sd[p + "self_attn_layer_norm.weight"])
        out[o + "ln1.b"] = vec(sd[p + "self_attn_layer_norm.bias"])
        dmat(o + "wqkv", torch.cat([sd[p + "self_attn.q_proj.weight"], sd[p + "self_attn.k_proj.weight"],
                                    sd[p + "self_attn.v_proj.weight"]], 0))
        out[o + "bqkv"] = vec(torch.cat([sd[p + "self_attn.q_proj.bias"].float().cpu(), zeros,
                                         sd[p + "self_attn.v_proj.bias"].float().cpu()], 0))
        dmat(o + "wo", sd[p + "self_attn.out_proj.weight"])
        out[o + "bo"] = vec(sd[p + "self_attn.out_proj.bias"])
        out[o + "ln2.g"] = vec(sd[p + "encoder_attn_layer_norm.weight"])
        out[o + "ln2.b"] = vec(sd[p + "encoder_attn_layer_norm.bias"])
        dmat(o + "xwq", sd[p + "encoder_attn.q_proj.weight"])
        out[o + "xbq"] = vec(sd[p + "encoder_attn.q_proj.bias"])
        out[o + "xwk"] = mat(sd[p + "encoder_attn.k_proj.weight"])
        out[o + "xwv"] = mat(sd[p + "encoder_attn.v_proj.weight"])
        out[o + "xbv"] = vec(sd[p + "encoder_attn.v_proj.bias"])
        dmat(o + "xwo", sd[p + "encoder_attn.out_proj.weight"])
        out[o + "xbo"] = vec(sd[p + "encoder_attn.out_proj.bias"])
        out[o + "ln3.g"] = vec(sd[p + "final_layer_norm.weight"])
        out[o + "ln3.b"] = vec(sd[p + "final_layer_norm.bias"])
        dmat(o + "w1", sd[p + "fc1.weight"])
        out[o + "b1"] = vec(sd[p + "fc1.bias"])
        dmat(o + "w2", sd[p + "fc2.weight"])
        out[o + "b2"] = vec(sd[p + "fc2.bias"])
    return out


class WhisperEngine:
    """Native engine for one GPU.  `state_dict` is an HF Whisper checkpoint (container of weights only).
    decoder_weights="int8" stores the decoder matrices every step streams as int8 with a scale per row (see pack_weights);
    a preloaded `weights` dict carries its own format (decoder_weights_of)."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], dims: ModelDims, chunk_length_s: float = 30,
                 device: str = "cuda:0", max_audios: int = 1, max_beams: int = 1,
                 alignment_heads: Optional[Sequence[Sequence[int]]] = None, max_align_steps: int = 448,
                 weights: Optional[Dict[str, torch.Tensor]] = None, dtype: torch.dtype = torch.bfloat16,
                 decoder_weights: Optional[str] = None):
        if decoder_weights not in DECODER_WEIGHTS:
            raise ValueError(f"decoder_weights must be one of {DECODER_WEIGHTS}, got {decoder_weights!r}")
        self.lib = _lib.load()
        if not torch.cuda.is_available() or self.lib.bw_device_count() == 0:
            raise _lib.BwError("no CUDA device visible: thewhisper_b200 has no CPU fallback")
        self.device = torch.device(device)
        torch.cuda.set_device(self.device)
        self.dims = dataclasses.replace(dims)
        self.chunk_length_s = chunk_length_s
        S = int(1500 * (chunk_length_s / 30))
        self.S = S
        self.n_samples = S * 2 * HOP
        self.frames = 2 * S
        self.dims.max_source_positions = S
        self.max_audios, self.max_beams = max_audios, max_beams
        self.alignment_heads = [list(map(int, p)) for p in (alignment_heads or [])]
        if weights is None:
            table = state_dict["model.encoder.embed_positions.weight"]
            enc_pos = table.detach().float().cpu() if table.shape[0] == S else interpolate_positions(table, chunk_length_s)
            weights = pack_weights(state_dict, dims, enc_pos, self.device, dtype, decoder_weights)
        else:  # preloaded: the matrices decide (all 16-bit tensors share one type), "dec.embed.scale" the decoder format
            if decoder_weights is not None and decoder_weights_of(weights) != decoder_weights:
                raise _lib.BwError(f"decoder_weights={decoder_weights!r} but the preloaded weights hold "
                                   f"{decoder_weights_of(weights) or '16-bit'} decoder matrices")
            mats = {t.dtype for t in weights.values() if t.dtype in ENGINE_DTYPES}
            if len(mats) != 1:
                raise _lib.BwError(f"preloaded weights must hold matrices of exactly one 16-bit type, got {mats}")
            dtype = mats.pop()
        if dtype not in ENGINE_DTYPES:
            raise _lib.BwError(f"engine dtype must be torch.bfloat16 or torch.float16, got {dtype}")
        self.dtype = dtype
        self.decoder_weights = decoder_weights_of(weights)
        self.weights = weights  # keeps the device memory alive
        cfg = _lib.bw_config(dims.d_model, dims.n_heads, dims.ffn, dims.enc_layers, dims.dec_layers, dims.n_mels,
                             dims.vocab, S, dims.max_target_positions, max_audios, max_beams,
                             len(self.alignment_heads), min(max_align_steps, dims.max_target_positions), ENGINE_DTYPES[dtype])
        self.max_align_steps = cfg.max_align_steps
        h = C.c_void_p()
        _lib.check(self.lib.bw_engine_create(C.byref(cfg), C.byref(h)))
        self.h = h
        for name, t in weights.items():
            _lib.check(self.lib.bw_engine_set_tensor(self.h, name.encode(), C.c_void_p(t.data_ptr())))
        bank = np.ascontiguousarray(mel_filter_bank(dims.n_mels), dtype=np.float32)
        _lib.check(self.lib.bw_engine_set_mel_filters(self.h, bank.ctypes.data_as(C.c_void_p)))
        if self.alignment_heads:
            ah = np.asarray(self.alignment_heads, dtype=np.int32).reshape(-1)
            _lib.check(self.lib.bw_engine_set_alignment_heads(self.h, ah.ctypes.data_as(C.c_void_p), len(self.alignment_heads)))
        _lib.check(self.lib.bw_engine_finalize(self.h))
        self._pcm_dev = torch.empty((max_audios, self.n_samples), dtype=torch.float32, device=self.device)
        self._pcm_pin = torch.empty((max_audios, self.n_samples), dtype=torch.float32).pin_memory()
        self._tok_host = np.zeros((max_audios * max_beams, dims.max_target_positions), dtype=np.int32)
        self._keep = None
        self._keep_pcm = None
        # work counters (bench / diagnostics): the timestamp `seek` loop may encode and decode a chunk more than once
        # sot_split_steps: teacher-forced positions run as decoder steps instead of in the prefill, so that the no-speech probability
        # can be read at the <|startoftranscript|> position (teacher_force)
        self.stats = {"encode_calls": 0, "chunks_encoded": 0, "decode_steps": 0, "sequence_steps": 0, "prefill_passes": 0,
                      "sot_split_steps": 0}

    # ------------------------------------------------------------------------------------------
    def close(self):
        if getattr(self, "h", None):
            self.lib.bw_engine_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _stream(self) -> C.c_void_p:
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def buffer(self, name: str, dtype: torch.dtype, shape: Sequence[int]) -> torch.Tensor:
        """A *copy* of an internal device buffer (tests / taps)."""
        p, nbytes = C.c_void_p(), C.c_size_t()
        _lib.check(self.lib.bw_engine_buffer(self.h, name.encode(), C.byref(p), C.byref(nbytes)))
        n = int(np.prod(shape))
        itemsize = torch.empty((), dtype=dtype).element_size()
        assert n * itemsize <= nbytes.value, (name, n * itemsize, nbytes.value)
        out = torch.empty(n, dtype=dtype, device=self.device)
        torch.cuda.current_stream(self.device).synchronize()
        _lib.device_copy(out.data_ptr(), p.value, n * itemsize)
        return out.view(*shape)

    def write_buffer(self, name: str, src: torch.Tensor, offset_bytes: int = 0) -> None:
        """Overwrite (part of) an internal device buffer from a device tensor (op-level tests: e.g. alignment scores)."""
        p, nbytes = C.c_void_p(), C.c_size_t()
        _lib.check(self.lib.bw_engine_buffer(self.h, name.encode(), C.byref(p), C.byref(nbytes)))
        src = src.contiguous()
        n = src.numel() * src.element_size()
        assert offset_bytes + n <= nbytes.value, (name, offset_bytes, n, nbytes.value)
        torch.cuda.current_stream(self.device).synchronize()
        _lib.device_copy(p.value + offset_bytes, src.data_ptr(), n)

    # ------------------------------------------------------------------------------------------
    def logmel(self, pcm: np.ndarray, return_f32: bool = False) -> Optional[torch.Tensor]:
        """pcm: host float32 [B, n_samples] (already padded / truncated).  Pinned staging + async H2D."""
        B = pcm.shape[0]
        assert pcm.shape[1] == self.n_samples and B <= self.max_audios, (pcm.shape, self.n_samples)
        self._pcm_pin[:B].copy_(torch.from_numpy(np.ascontiguousarray(pcm, dtype=np.float32)))
        self._pcm_dev[:B].copy_(self._pcm_pin[:B], non_blocking=True)
        return self.logmel_device(self._pcm_dev, B, return_f32)

    def logmel_device(self, pcm_dev: torch.Tensor, B: int, return_f32: bool = False) -> Optional[torch.Tensor]:
        out = None
        if return_f32:
            out = torch.empty((B, self.dims.n_mels, self.frames), dtype=torch.float32, device=self.device)
        _lib.check(self.lib.bw_logmel(self.h, C.c_void_p(pcm_dev.data_ptr()), B, self.n_samples,
                                      C.c_void_p(out.data_ptr()) if out is not None else None, self._stream()))
        return out

    def logmel_long(self, pcm: np.ndarray) -> torch.Tensor:
        """Features of audio of any length: pcm host float32 [B, L], every row zero-padded to the longest, L >= 400 ->
        device fp32 [B, n_mels, L // 160] (the feature extractor's truncation=False, padding="longest" layout, clamp per row).
        The PCM staging and the feature buffer are allocated per call, sized to the group (184 MB of features per hour of audio at
        128 mels); when either allocation fails this raises before anything is launched.  The engine's mel buffer is untouched."""
        pcm = np.ascontiguousarray(pcm, dtype=np.float32)
        B, L = pcm.shape
        assert B <= self.max_audios, (B, self.max_audios)
        try:
            pcm_dev = torch.empty((B, L), dtype=torch.float32, device=self.device)
            out = torch.empty((B, self.dims.n_mels, L // HOP), dtype=torch.float32, device=self.device)
        except torch.cuda.OutOfMemoryError as err:
            raise _lib.BwError(f"logmel_long: cannot allocate the features of {B} x {L} samples "
                               f"({(B * L + B * self.dims.n_mels * (L // HOP)) * 4 / 2**20:.0f} MiB): {err}") from None
        pcm_dev.copy_(torch.from_numpy(pcm))
        _lib.check(self.lib.bw_logmel_long(self.h, C.c_void_p(pcm_dev.data_ptr()), B, L, C.c_void_p(out.data_ptr()), self._stream()))
        self._keep_pcm = pcm_dev  # the copy and the kernels are stream-ordered; the staging lives until the next call
        return out

    def set_mel(self, mel: torch.Tensor) -> None:
        """Load externally computed features [B, n_mels, frames] (device fp32) instead of running bw_logmel."""
        mel = mel.to(device=self.device, dtype=torch.float32).contiguous()
        assert mel.shape[1:] == (self.dims.n_mels, self.frames), mel.shape
        _lib.check(self.lib.bw_set_mel(self.h, C.c_void_p(mel.data_ptr()), mel.shape[0], self._stream()))
        self._keep = mel

    def encode(self, B: int) -> None:
        _lib.check(self.lib.bw_encode(self.h, B, self._stream()))
        self.stats["encode_calls"] += 1
        self.stats["chunks_encoded"] += B

    def encoder_output(self, B: int) -> torch.Tensor:
        return self.buffer("enc_out", self.dtype, (self.max_audios, self.S, self.dims.d_model))[:B].float()

    # ------------------------------------------------------------------------------------------
    def decode_begin(self, prompts: np.ndarray, A: int, G: int, opts: DecodeOptions, begin_index: Optional[int] = None,
                     key_start: Optional[Sequence[int]] = None) -> None:
        """key_start [A] (left-padded prompts): positions below key_start[a] are absent as keys for audio a's sequences."""
        prompts = np.ascontiguousarray(prompts, dtype=np.int32)
        assert prompts.shape[0] == A * G, (prompts.shape, A, G)
        plen = prompts.shape[1]
        sup = np.ascontiguousarray(list(opts.suppress_tokens), dtype=np.int32)
        bsup = np.ascontiguousarray(list(opts.begin_suppress_tokens), dtype=np.int32)
        o = _lib.bw_decode_opts()
        o.begin_index = plen if begin_index is None else begin_index
        o.eos_token, o.pad_token = opts.eos_token, opts.pad_token
        o.timestamp_rules = int(opts.timestamp_rules)
        o.timestamp_begin, o.no_timestamps_token = opts.timestamp_begin, opts.no_timestamps_token
        o.max_initial_timestamp_index = opts.max_initial_timestamp_index
        o.suppress_tokens = sup.ctypes.data_as(C.POINTER(C.c_int32))
        o.n_suppress = len(sup)
        o.begin_suppress_tokens = bsup.ctypes.data_as(C.POINTER(C.c_int32))
        o.n_begin_suppress = len(bsup)
        o.record_alignment = int(opts.record_alignment)
        if key_start is None:
            _lib.check(self.lib.bw_decode_begin(self.h, A, G, prompts.ctypes.data_as(C.c_void_p), plen, C.byref(o), self._stream()))
        else:
            ks = np.ascontiguousarray(key_start, dtype=np.int32)
            assert ks.shape == (A,), (ks.shape, A)
            _lib.check(self.lib.bw_decode_begin_key_start(self.h, A, G, prompts.ctypes.data_as(C.c_void_p), plen, C.byref(o),
                                                          ks.ctypes.data_as(C.c_void_p), self._stream()))
        self._Q = A * G
        self._A = A
        self._plen = plen

    def decode_run(self, n_steps: int) -> None:
        _lib.check(self.lib.bw_decode_run(self.h, n_steps, self._stream()))
        self.stats["decode_steps"] += n_steps
        self.stats["sequence_steps"] += n_steps * self._Q

    def decode_prefill(self, n_positions: int, max_rows_per_pass: int = 0) -> None:
        """Run the teacher-forced positions 0..n_positions-1 of every sequence in one batched pass (or several of at most
        max_rows_per_pass = sequences x positions rows; 0 = the engine's default): the state n_positions decode_run steps
        leave, except the logits.  Must directly follow decode_begin; n_positions <= begin_index - 1."""
        _lib.check(self.lib.bw_decode_prefill(self.h, n_positions, max_rows_per_pass, self._stream()))
        self.stats["prefill_passes"] += 1

    def decode_scores_enable(self, nospeech_pos: int = -1, nospeech_token: int = 0) -> None:
        """Scores for the decode just begun (before its first step or prefill): every step also records the processed log-prob of
        the token it selects and the allowed mass (see decode_scores); the step that consumes position nospeech_pos (-1 = none)
        records softmax(raw logits)[nospeech_token].  Token selection is unchanged."""
        _lib.check(self.lib.bw_decode_scores_enable(self.h, int(nospeech_pos), int(nospeech_token), self._stream()))

    def decode_scores(self):
        """-> (lp [Q, Tmax], lmass [Q, Tmax], nsp [Q]) float32 of the decode with scores on: lp[q, t] the log-softmax of the processed
        logits at the token selected at index t (0 for a finished row), lmass[q, t] = logsumexp(allowed logits) - logsumexp(raw logits)
        of that step (so a candidate's processed log-prob is its raw log-prob minus lmass), nsp[q] the no-speech probability."""
        Q, T = self._Q, self.dims.max_target_positions
        lp = np.empty((Q, T), dtype=np.float32)
        lmass = np.empty((Q, T), dtype=np.float32)
        nsp = np.empty(Q, dtype=np.float32)
        _lib.check(self.lib.bw_decode_read_scores(self.h, lp.ctypes.data_as(C.c_void_p), lmass.ctypes.data_as(C.c_void_p),
                                                  nsp.ctypes.data_as(C.c_void_p), self._stream()))
        return lp, lmass, nsp

    def teacher_force(self, plen: int, prefill: bool, nospeech_pos: Optional[int] = None) -> None:
        """Run the teacher-forced positions 0..plen-2 of the decode just begun: one batched prefill pass when `prefill`, else
        decoder steps.  nospeech_pos (scores on): the prefill stops before that position, and the positions from it on run as steps,
        because the prefill has no LM head and the no-speech probability is read from the step that consumes it."""
        split = plen - 1 if nospeech_pos is None else min(plen - 1, nospeech_pos)
        if prefill and split >= 1:
            self.decode_prefill(split)
            self.decode_run(plen - 1 - split)
            self.stats["sot_split_steps"] += plen - 1 - split
        else:
            self.decode_run(plen - 1)

    def graph_stats(self) -> Dict[str, float]:
        """The engine's step-graph cache: graphs captured, seconds spent capturing them, graphs cached now, graphs evicted."""
        out = (C.c_int64 * 4)()
        _lib.check(self.lib.bw_decode_graph_stats(self.h, out))
        return {"captured": int(out[0]), "capture_s": out[1] / 1e6, "cached": int(out[2]), "evicted": int(out[3])}

    def decode_kernel_launches(self) -> int:
        """Kernels launched by decode_run so far (counted from the captured step graphs)."""
        return int(self.lib.bw_decode_kernel_launches(self.h))

    def decode_read(self):
        """-> (tokens [Q, Tmax] int32, finished [Q] int32, pos)"""
        Q = self._Q
        fin = np.zeros(Q, dtype=np.int32)
        pos = C.c_int32(0)
        _lib.check(self.lib.bw_decode_read(self.h, self._tok_host.ctypes.data_as(C.c_void_p), fin.ctypes.data_as(C.c_void_p),
                                           C.byref(pos), self._stream()))
        return self._tok_host[:Q].copy(), fin, int(pos.value)

    def decode_reorder(self, parent: np.ndarray, next_token: np.ndarray) -> None:
        parent = np.ascontiguousarray(parent, dtype=np.int32)
        next_token = np.ascontiguousarray(next_token, dtype=np.int32)
        _lib.check(self.lib.bw_decode_reorder(self.h, parent.ctypes.data_as(C.c_void_p), next_token.ctypes.data_as(C.c_void_p),
                                              self._stream()))

    def decode_beam_step(self, run_scores: np.ndarray):
        """One decoder step in beam mode: -> (cand_scores [Q, 2G] float32, cand_tokens [Q, 2G] int32)."""
        Q, K = self._Q, 2 * (self._Q // max(1, self._A))
        run = np.ascontiguousarray(run_scores, dtype=np.float32)
        cs = np.empty((Q, K), dtype=np.float32)
        ct = np.empty((Q, K), dtype=np.int32)
        _lib.check(self.lib.bw_decode_beam_step(self.h, run.ctypes.data_as(C.c_void_p), cs.ctypes.data_as(C.c_void_p),
                                                ct.ctypes.data_as(C.c_void_p), self._stream()))
        self.stats["decode_steps"] += 1
        self.stats["sequence_steps"] += Q
        return cs, ct

    def logits(self) -> torch.Tensor:
        vp = (self.dims.vocab + 31) // 32 * 32  # row pitch of the engine's logits buffer (rows stay 16-byte aligned)
        return self.buffer("logits", torch.float32, (self.max_audios * self.max_beams, vp))[: self._Q, : self.dims.vocab]

    def greedy(self, prompts: np.ndarray, A: int, opts: DecodeOptions, max_new_tokens: int, poll_every: int = 32,
               prefill: bool = False, key_start: Optional[Sequence[int]] = None, nospeech: Optional[Sequence[int]] = None):
        """Greedy decode of A audios (their cross K/V must be resident from encode()).  Returns generated ids per
        audio (prompt stripped, cut at and excluding EOS) and the raw token matrix.  prefill: run the teacher-forced
        positions as one batched prefill pass instead of step by step.  key_start: see decode_begin.  nospeech = (position,
        token): scores on (decode_scores_enable, teacher_force); read them with decode_scores afterwards."""
        plen = prompts.shape[1]
        Tmax = self.dims.max_target_positions
        max_new = max(0, min(max_new_tokens, Tmax - plen))
        self.decode_begin(prompts, A, 1, opts, key_start=key_start)
        if nospeech is not None:
            self.decode_scores_enable(*nospeech)
        self.teacher_force(plen, prefill, None if nospeech is None else nospeech[0])
        done = 0
        toks = fin = None
        while done < max_new:
            n = min(poll_every, max_new - done)
            self.decode_run(n)
            done += n
            toks, fin, _ = self.decode_read()
            if fin.all():
                break
        if toks is None:
            toks, fin, _ = self.decode_read()
        out = []
        for a in range(A):
            row = toks[a, plen:plen + done]
            cut = np.where(row == opts.eos_token)[0]
            out.append(row[: cut[0]] if len(cut) else row)
        return out, toks, done

    def word_timestamps_batch(self, audios: Sequence[int], n_tokens: Sequence[int], num_frames: Sequence[int],
                              time_precision: float = 0.02) -> np.ndarray:
        """Token times of several audios in one pass -> [n, max(n_tokens) + 1] float32 (rows padded with zeros)."""
        n = len(audios)
        au = np.ascontiguousarray(audios, dtype=np.int32)
        nt = np.ascontiguousarray(n_tokens, dtype=np.int32)
        nf = np.ascontiguousarray(num_frames, dtype=np.int32)
        pitch = int(nt.max()) + 1
        out = np.zeros((n, pitch), dtype=np.float32)
        _lib.check(self.lib.bw_word_timestamps_batch(self.h, n, au.ctypes.data_as(C.c_void_p), nt.ctypes.data_as(C.c_void_p),
                                                     nf.ctypes.data_as(C.c_void_p), time_precision, out.ctypes.data_as(C.c_void_p),
                                                     pitch, self._stream()))
        return out

    def word_timestamps_gather(self, slot_map: np.ndarray, n_tokens: Sequence[int], num_frames: Sequence[int],
                               time_precision: float = 0.02) -> np.ndarray:
        """Beam search: row t of item i comes from sequence slot slot_map[i, t] (the returned sequence's ancestor at step t)."""
        sm = np.ascontiguousarray(slot_map, dtype=np.int32)
        n = sm.shape[0]
        nt = np.ascontiguousarray(n_tokens, dtype=np.int32)
        nf = np.ascontiguousarray(num_frames, dtype=np.int32)
        pitch = int(nt.max()) + 1
        out = np.zeros((n, pitch), dtype=np.float32)
        _lib.check(self.lib.bw_word_timestamps_gather(self.h, n, sm.ctypes.data_as(C.c_void_p), sm.shape[1], nt.ctypes.data_as(C.c_void_p),
                                                      nf.ctypes.data_as(C.c_void_p), time_precision, out.ctypes.data_as(C.c_void_p),
                                                      pitch, self._stream()))
        return out

    def word_timestamps(self, audio: int, n_tokens: int, num_frames: int, time_precision: float = 0.02) -> np.ndarray:
        out = np.zeros(n_tokens + 1, dtype=np.float32)
        _lib.check(self.lib.bw_word_timestamps(self.h, audio, n_tokens, num_frames, time_precision,
                                               out.ctypes.data_as(C.c_void_p), self._stream()))
        return out
