"""Synthetic inputs for an offline box: model configs, random checkpoints, a tokenizer with the
large-v3 id layout, and deterministic 16 kHz audio.

No checkpoint, tokenizer file or audio exists on disk and there is no network (SURVEY.md §8c/§8d),
so parity and throughput are measured on these.  Nothing here is arithmetic of the hot path: the
random checkpoint is only a *container of weights* handed to both the CUDA engine and the oracle.

Token id layout follows whisper-large-v3 (SURVEY.md §8 "Model constants"): EOS 50257, SOT 50258,
<|en|> 50259, translate 50359, transcribe 50360, startofprev 50362, nospeech 50363,
notimestamps 50364, <|0.00|> 50365 ... <|30.00|> 51865.
"""
from __future__ import annotations

import dataclasses
import math
from typing import Dict, List, Optional

import numpy as np
import torch

# ----------------------------------------------------------------------------------------------
# model dimension presets
# ----------------------------------------------------------------------------------------------

PRESETS: Dict[str, dict] = {
    # whisper-large-v3: d=1280 H=20 ffn=5120 32+32 layers, 128 mels, V=51866
    "large-v3": dict(d_model=1280, heads=20, ffn=5120, enc_layers=32, dec_layers=32, n_mels=128, vocab=51866),
    # whisper-large-v3-turbo: same encoder, 4 decoder layers
    "large-v3-turbo": dict(d_model=1280, heads=20, ffn=5120, enc_layers=32, dec_layers=4, n_mels=128, vocab=51866),
    # CI-speed shapes (same id layout, same head_dim=64 so the wgmma attention tiles are exercised)
    "tiny-test": dict(d_model=128, heads=2, ffn=512, enc_layers=2, dec_layers=2, n_mels=128, vocab=51866),
    "small-test": dict(d_model=256, heads=4, ffn=1024, enc_layers=3, dec_layers=3, n_mels=128, vocab=51866),
}

EOS = 50257
SOT = 50258
LANG_EN = 50259
TRANSLATE = 50359
TRANSCRIBE = 50360
STARTOFLM = 50361
STARTOFPREV = 50362
NOSPEECH = 50363
NOTIMESTAMPS = 50364
TIMESTAMP_BEGIN = 50365
VOCAB = 51866

# openai/whisper language order (first 100 entries = large-v3's language tokens 50259..50358)
LANG_CODES = (
    "en zh de es ru ko fr ja pt tr pl ca nl ar sv it id hi fi vi he uk el ms cs ro da hu ta no th ur hr bg lt la "
    "mi ml cy sk te fa lv bn sr az sl kn et mk br eu is hy ne mn bs kk sq sw gl mr pa si km sn yo so af oc ka be "
    "tg sd gu am yi lo uz fo ht ps tk nn mt sa lb my bo tl mg as tt haw ln ha ba jw su yue"
).split()
assert len(LANG_CODES) == 100

# a fixed, arbitrary alignment-head set (the published generation_config.json is not on disk; any
# fixed set is valid for the synthetic oracle, SURVEY.md §8). (layer, head) pairs, layer < dec_layers.
def default_alignment_heads(dec_layers: int, heads: int) -> List[List[int]]:
    want = [[7, 0], [10, 17], [12, 18], [13, 12], [16, 1], [17, 14], [19, 11], [21, 4], [24, 1], [25, 6]]
    out = [[l, h] for l, h in want if l < dec_layers and h < heads]
    if not out:  # small models: take the last layers' first heads
        out = [[max(dec_layers - 1, 0), 0], [max(dec_layers - 1, 0), min(1, heads - 1)]]
        if dec_layers > 1:
            out.append([dec_layers - 2, 0])
    # de-duplicate, keep order
    seen, res = set(), []
    for p in out:
        if tuple(p) not in seen:
            seen.add(tuple(p))
            res.append(p)
    return res


# non-speech symbols the real checkpoints suppress; here: a fixed pseudo-random set of text ids so
# the suppress path is exercised, plus the special ids HF always suppresses for whisper-large-v3.
def default_suppress_tokens() -> List[int]:
    rng = np.random.RandomState(1234)
    text = sorted(set(int(x) for x in rng.randint(1, 50000, size=80)))
    special = [50258, 50359, 50360, 50361, 50362, 50363]  # sot, translate, transcribe, startoflm, startofprev, nospeech
    return text + special


BEGIN_SUPPRESS = [220, EOS]


def make_hf_config(preset: str = "large-v3", max_source_positions: int = 1500):
    """transformers.WhisperConfig for a preset (container type only)."""
    from transformers import WhisperConfig

    p = PRESETS[preset]
    return WhisperConfig(
        vocab_size=p["vocab"],
        num_mel_bins=p["n_mels"],
        d_model=p["d_model"],
        encoder_layers=p["enc_layers"],
        decoder_layers=p["dec_layers"],
        encoder_attention_heads=p["heads"],
        decoder_attention_heads=p["heads"],
        encoder_ffn_dim=p["ffn"],
        decoder_ffn_dim=p["ffn"],
        max_source_positions=max_source_positions,
        max_target_positions=448,
        pad_token_id=EOS,
        bos_token_id=EOS,
        eos_token_id=EOS,
        decoder_start_token_id=SOT,
        activation_function="gelu",
        scale_embedding=False,
        dropout=0.0,
        attention_dropout=0.0,
        activation_dropout=0.0,
    )


def make_generation_config(preset: str = "large-v3", eos_suppressed: bool = False, suppress_timestamps: bool = False):
    from transformers import GenerationConfig

    p = PRESETS[preset]
    lang_to_id = {f"<|{c}|>": LANG_EN + i for i, c in enumerate(LANG_CODES)}
    sup = default_suppress_tokens()
    if eos_suppressed:
        sup = sorted(set(sup + [EOS]))
    if suppress_timestamps:
        # throughput runs: a random checkpoint emits timestamp ids at random even without timestamps, which would send the
        # (reference-faithful) seek loop into extra encode+decode passes; fixed-length runs mask them for every arm
        sup = sorted(set(sup) | set(range(TIMESTAMP_BEGIN, VOCAB)))
    g = GenerationConfig(
        max_length=448,
        pad_token_id=EOS,
        bos_token_id=EOS,
        eos_token_id=EOS,
        decoder_start_token_id=SOT,
        suppress_tokens=sup,
        begin_suppress_tokens=list(BEGIN_SUPPRESS),
    )
    g.no_timestamps_token_id = NOTIMESTAMPS
    g.is_multilingual = True
    g.lang_to_id = lang_to_id
    g.task_to_id = {"transcribe": TRANSCRIBE, "translate": TRANSLATE}
    g.alignment_heads = default_alignment_heads(p["dec_layers"], p["heads"])
    g.max_initial_timestamp_index = 50
    g.prev_sot_token_id = STARTOFPREV
    g.return_timestamps = False
    g.no_speech_threshold = None
    return g


def make_hf_model(preset: str = "large-v3", seed: int = 0, logit_scale: float = 1.0,
                  dtype: torch.dtype = torch.float32, round_to_bf16: bool = True, layer_gain: float = 1.0):
    """Random-weight HF WhisperForConditionalGeneration (HF init, std 0.02) used as the checkpoint.

    round_to_bf16: round every floating parameter to the nearest bf16 value (kept in `dtype`
    storage).  The checkpoint is then exactly representable in the engine's bf16 weight format, so
    the oracle (fp32 arithmetic) and the engine (bf16 storage, fp32 accumulate) see the *same*
    weights and only arithmetic differs.
    logit_scale: multiplies the tied embedding (LM head) to widen top-1/top-2 margins
    (SURVEY.md §7 hard part 1c).
    layer_gain: multiplies every 2-D weight inside encoder/decoder layers.  With the plain HF init
    the residual stream is dominated by the token embedding and greedy decoding collapses to one
    repeated token that ignores the audio (SURVEY.md §7 hard part 1); gain≈8 gives varied,
    audio-dependent sequences, which is what the parity fixtures use.
    """
    from transformers import WhisperForConditionalGeneration

    torch.manual_seed(seed)
    cfg = make_hf_config(preset)
    model = WhisperForConditionalGeneration(cfg)
    model.eval()
    with torch.no_grad():
        if logit_scale != 1.0:
            model.model.decoder.embed_tokens.weight.mul_(logit_scale)
        if layer_gain != 1.0:
            for name, prm in model.named_parameters():
                if "layers." in name and name.endswith("weight") and prm.dim() == 2:
                    prm.mul_(layer_gain)
        if round_to_bf16:
            for prm in model.parameters():
                prm.copy_(prm.to(torch.bfloat16).to(prm.dtype))
    model.generation_config = make_generation_config(preset)
    if dtype != torch.float32:
        model = model.to(dtype)
    return model


# ----------------------------------------------------------------------------------------------
# tokenizer
# ----------------------------------------------------------------------------------------------

def _bytes_to_unicode() -> Dict[int, str]:
    bs = list(range(ord("!"), ord("~") + 1)) + list(range(ord("¡"), ord("¬") + 1)) + list(range(ord("®"), ord("ÿ") + 1))
    cs = bs[:]
    n = 0
    for b in range(256):
        if b not in bs:
            bs.append(b)
            cs.append(256 + n)
            n += 1
    return dict(zip(bs, [chr(c) for c in cs]))


_TOKENIZER_CACHE = {}


def make_tokenizer():
    """WhisperTokenizer with 51 866 entries and the large-v3 special-id layout (SURVEY.md §8c recipe)."""
    if "tok" in _TOKENIZER_CACHE:
        return _TOKENIZER_CACHE["tok"]
    from tokenizers import AddedToken
    from transformers import WhisperTokenizer

    b2u = _bytes_to_unicode()
    vocab = {}
    for b in range(256):
        vocab[b2u[b]] = len(vocab)
    i = 0
    while len(vocab) < EOS:  # fillers: " w0", " w1", ... (Ġ = byte-level space)
        vocab[f"Ġw{i}"] = len(vocab)
        i += 1
    tok = WhisperTokenizer(vocab=vocab, merges=[], pad_token="<|endoftext|>")
    specials = ["<|endoftext|>", "<|startoftranscript|>"] + [f"<|{c}|>" for c in LANG_CODES] + [
        "<|translate|>", "<|transcribe|>", "<|startoflm|>", "<|startofprev|>", "<|nospeech|>", "<|notimestamps|>"]
    tok.add_tokens([AddedToken(s, special=True, normalized=False) for s in specials], special_tokens=True)
    tok.add_tokens([AddedToken("<|%.2f|>" % (k * 0.02), special=False, normalized=False) for k in range(1501)])
    assert len(tok) == VOCAB, len(tok)
    ids = tok.convert_tokens_to_ids(["<|endoftext|>", "<|startoftranscript|>", "<|en|>", "<|transcribe|>",
                                     "<|notimestamps|>", "<|0.00|>", "<|30.00|>"])
    assert ids == [EOS, SOT, LANG_EN, TRANSCRIBE, NOTIMESTAMPS, TIMESTAMP_BEGIN, VOCAB - 1], ids
    _TOKENIZER_CACHE["tok"] = tok
    return tok


def make_feature_extractor(chunk_length_s: int = 30, n_mels: int = 128):
    from transformers import WhisperFeatureExtractor

    return WhisperFeatureExtractor(feature_size=n_mels, chunk_length=chunk_length_s)


# ----------------------------------------------------------------------------------------------
# audio
# ----------------------------------------------------------------------------------------------

def two_tone(seconds: float, sr: int = 16000) -> np.ndarray:
    """RNG-free golden signal of SURVEY.md §8c: 0.5 sin(2π440t) + 0.25 sin(2π1000t), float32."""
    n = np.arange(int(round(seconds * sr)), dtype=np.float64)
    x = 0.5 * np.sin(2 * np.pi * 440.0 * n / sr) + 0.25 * np.sin(2 * np.pi * 1000.0 * n / sr)
    return x.astype(np.float32)


def synth_audio(seconds: float, seed: int, sr: int = 16000, kind: str = "speechlike") -> np.ndarray:
    """Deterministic synthetic audio, float32 in [-1, 1].

    kind="noise": 0.1·N(0,1) (SURVEY.md §8d).
    kind="speechlike": amplitude-modulated harmonic bursts + noise, so frames differ in energy and
    spectrum (more input dependence for parity runs than stationary noise).
    """
    n = int(round(seconds * sr))
    rng = np.random.RandomState(seed)
    if kind == "noise":
        x = 0.1 * rng.randn(n)
    else:
        t = np.arange(n, dtype=np.float64) / sr
        x = 0.02 * rng.randn(n)
        pos = 0.0
        while pos < seconds:
            dur = 0.08 + 0.3 * rng.rand()
            f0 = 90.0 + 200.0 * rng.rand()
            a = 0.05 + 0.3 * rng.rand()
            i0, i1 = int(pos * sr), min(n, int((pos + dur) * sr))
            if i1 > i0:
                tt = t[i0:i1] - pos
                env = np.sin(np.pi * tt / max(dur, 1e-3)) ** 2
                sig = np.zeros_like(tt)
                for k in range(1, 6):
                    sig += (1.0 / k) * np.sin(2 * np.pi * f0 * k * tt + rng.rand() * 6.28)
                x[i0:i1] += a * env * sig
            pos += dur + 0.15 * rng.rand()
    return np.clip(x, -1.0, 1.0).astype(np.float32)
