"""ORACLE (test infrastructure, never the product path).

CPU restatement of the reference's NVIDIA/HF hot path, i.e. what
`thestage_speechkit.nvidia.ASRPipeline(model_size=None)` computes
(REF = a checkout of TheStageAI/TheWhisper, TF = installed transformers 5.5.0; the reference pins 4.52.3):

  * REF/thestage_speechkit/nvidia/asr_pipeline.py:15-27   patch_hf_model      -> interpolate_positions()
  * REF/thestage_speechkit/nvidia/asr_pipeline.py:30-92   ASRPipeline         -> RefASRPipeline
  * REF/thestage_speechkit/__init__.py:5-139              LCS monkey patch    -> lcs_merge() / install_lcs()
  * TF/models/whisper/feature_extraction_whisper.py:135-164  log-mel          -> called, not restated here
    (an independent numpy restatement lives in oracle/whisper_ref.py)
  * TF/models/whisper/modeling_whisper.py, generation_whisper.py              -> called through the HF classes

The arithmetic lives in the third-party dependency `transformers` (un-vendored; present in this
image on both the build container and the GPU box), so this module *drives* it exactly the way the
reference does and restates only the reference's own glue.  It is pinned by
`oracle/make_golden.py`, which imports the real reference from such a checkout in the build
container, checks this restatement against it output-for-output, and writes `tests/golden/*.npz`.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this module.
"""
from __future__ import annotations

import contextlib
from typing import List, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F


# ----------------------------------------------------------------------------------------------
# reference glue, restated
# ----------------------------------------------------------------------------------------------

def interpolate_positions(model, chunk_length_s: float) -> None:
    """REF nvidia/asr_pipeline.py:15-27: shrink the encoder's sinusoid table to int(1500*c/30) rows by
    linear interpolation (align_corners=False).  Plus the one-line shim transformers>=5 needs
    (SURVEY.md §8c (i)): the encoder indexes arange(embed_positions.num_embeddings)."""
    n_pos = int(1500 * (chunk_length_s / 30))
    model.config.max_source_positions = n_pos
    table = model.model.encoder.embed_positions.weight  # [1500, d]
    shrunk = F.interpolate(table.t().unsqueeze(0), size=n_pos, mode="linear", align_corners=False)
    model.model.encoder.embed_positions.weight.data = shrunk.squeeze(0).t().contiguous()
    model.model.encoder.embed_positions.num_embeddings = n_pos  # 5.x shim


def lcs_merge(sequences: Sequence[Sequence[int]], token_timestamp_sequences=None):
    """REF thestage_speechkit/__init__.py:5-134, restated with plain loops.

    Slides the right sequence over the left one; for overlap offset i scores
    matches/i + i/10000, needs matches > 1; with timestamps a match additionally needs
    left_ts <= right_ts unless the left entry's end time is None (REF :75-78).  The seam is cut at
    the midpoints of the best overlap (REF :111-115)."""
    left = list(sequences[0])
    total: List[int] = []
    have_ts = bool(token_timestamp_sequences)
    if have_ts:
        left_ts = list(token_timestamp_sequences[0])
        total_ts: list = []
    for k in range(1, len(sequences)):
        right = list(sequences[k])
        nl, nr = len(left), len(right)
        best, best_idx = 0.0, (nl, nl, 0, 0)
        for i in range(1, nl + nr):
            l0, l1 = max(0, nl - i), min(nl, nl + nr - i)
            r0, r1 = max(0, i - nl), min(nr, i)
            if l1 - l0 != r1 - r0:
                raise RuntimeError("overlap windows of different size: bug in whisper decode_asr")
            m = 0
            for j in range(l1 - l0):
                if left[l0 + j] != right[r0 + j]:
                    continue
                if have_ts:
                    a = left_ts[l0 + j]
                    b = token_timestamp_sequences[k][r0 + j]
                    if not (a[1] is None or a <= b):
                        continue
                m += 1
            score = m / i + i / 10000.0
            if m > 1 and score > best:
                best, best_idx = score, (l0, l1, r0, r1)
        l0, l1, r0, r1 = best_idx
        lmid, rmid = (l0 + l1) // 2, (r0 + r1) // 2
        total.extend(left[:lmid])
        left = right[rmid:]
        if have_ts:
            total_ts.extend(left_ts[:lmid])
            left_ts = list(token_timestamp_sequences[k][rmid:])
    total.extend(left)
    if token_timestamp_sequences is None:
        return total
    if len(token_timestamp_sequences) > 0:
        total_ts.extend(left_ts)
        return total, total_ts
    return total, []


def install_lcs() -> None:
    """REF thestage_speechkit/__init__.py:137-139: rebind transformers' seam merge."""
    import transformers.models.whisper.tokenization_whisper as tw

    tw._find_longest_common_sequence = lcs_merge


def make_ref_pipeline(model, feature_extractor, tokenizer, chunk_length_s: int = 30, device: str = "cpu",
                      torch_dtype: Optional[torch.dtype] = None, **kw):
    """REF nvidia/asr_pipeline.py:30-92 for the model-instance branch (model_size=None):
    HF AutomaticSpeechRecognitionPipeline + position patch for chunk_length_s < 30 + LCS rebinding."""
    from transformers import AutomaticSpeechRecognitionPipeline

    if feature_extractor is None:
        raise ValueError("feature_extractor must be provided when passing a model instance")
    if tokenizer is None:
        raise ValueError("tokenizer must be provided when passing a model instance")
    install_lcs()
    pipe = AutomaticSpeechRecognitionPipeline(
        model, feature_extractor=feature_extractor, tokenizer=tokenizer, device=device,
        chunk_length_s=chunk_length_s, torch_dtype=torch_dtype, **kw)
    if chunk_length_s < 30 and model.config.max_source_positions == 1500:
        interpolate_positions(model, chunk_length_s)
    return pipe


# ----------------------------------------------------------------------------------------------
# stage taps used by the parity tests
# ----------------------------------------------------------------------------------------------

def logmel(feature_extractor, audio: np.ndarray) -> np.ndarray:
    """[n] float32 PCM -> [n_mels, frames] float32 through TF feature_extraction_whisper.py:189-342
    (zero-pad/truncate to chunk length, torch.stft path)."""
    out = feature_extractor(audio, sampling_rate=16000, return_tensors="np", return_attention_mask=True)
    return np.asarray(out["input_features"][0], dtype=np.float32)


@torch.no_grad()
def encoder_out(model, mel: np.ndarray) -> np.ndarray:
    """[n_mels, 2*S] -> [S, d] float32 (TF modeling_whisper.py:593-647)."""
    x = torch.from_numpy(mel)[None].to(model.dtype)
    return model.model.encoder(x).last_hidden_state[0].float().numpy()


@torch.no_grad()
def teacher_forced_logits(model, mel: np.ndarray, decoder_ids: Sequence[int]) -> np.ndarray:
    """logits [T, V] float32 for a fixed decoder token sequence (no processors)."""
    x = torch.from_numpy(mel)[None].to(model.dtype)
    ids = torch.tensor([list(decoder_ids)], dtype=torch.long)
    return model(input_features=x, decoder_input_ids=ids).logits[0].float().numpy()


@torch.no_grad()
def generate(model, mel_batch: np.ndarray, attention_mask: Optional[np.ndarray] = None, **generate_kwargs):
    """model.generate on [B, n_mels, frames] (TF generation_whisper.py:383-968)."""
    x = torch.from_numpy(mel_batch).to(model.dtype)
    am = None if attention_mask is None else torch.from_numpy(attention_mask)
    return model.generate(input_features=x, attention_mask=am, **generate_kwargs)


@contextlib.contextmanager
def threads(n: Optional[int]):
    old = torch.get_num_threads()
    if n:
        torch.set_num_threads(n)
    try:
        yield
    finally:
        torch.set_num_threads(old)
