"""ORACLE (test infrastructure, never the product path): plain numpy restatements of the integer / rule parts of the
hot path, each citing the reference-side code it follows (TF = transformers 5.5.0 as installed):

  logmel_np              TF/models/whisper/feature_extraction_whisper.py:135-164 + TF/audio_utils.py (slaney bank)
  process_logits         TF/generation/logits_process.py:1812-1862 (begin suppress), :1865-1902 (suppress),
                         :1995-2043 (WhisperTimeStampLogitsProcessor)
  select_greedy / beam_candidates
                         the masks of process_logits, the probability rule in float64, greedy argmax + pad / finished
                         (TF/generation/utils.py:2762-2797), one beam's top 2G (TF/generation/utils.py:3256-3257)
  median_filter / dtw / token_timestamps
                         TF/models/whisper/generation_whisper.py:43-61, :64-115, :331-379

Pinned by tests/test_oracle_cpu.py against the golden fixtures minted from the real reference
(oracle/make_golden.py) and against the installed transformers implementations.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np


# ------------------------------------------------------------------------------------------------------------------
def logmel_np(audio: np.ndarray, bank: np.ndarray, n_samples: int) -> np.ndarray:
    """float32 PCM -> [n_mels, n_samples/160] log-mel, float64 DFT (independent of torch.stft)."""
    x = np.zeros(n_samples, dtype=np.float64)
    n = min(len(audio), n_samples)
    x[:n] = np.asarray(audio[:n], dtype=np.float32)
    xp = np.pad(x, 200, mode="reflect")
    win = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(400) / 400)
    frames = n_samples // 160
    idx = np.arange(400)[None, :] + 160 * np.arange(frames)[:, None]
    spec = np.fft.rfft(xp[idx] * win[None, :], n=400, axis=1)
    power = (np.abs(spec) ** 2).astype(np.float32)  # [frames, 201]
    mel = bank.astype(np.float32).T @ power.T
    log_spec = np.log10(np.maximum(mel, 1e-10))
    log_spec = np.maximum(log_spec, log_spec.max() - 8.0)
    return ((log_spec + 4.0) / 4.0).astype(np.float32)


# ------------------------------------------------------------------------------------------------------------------
def process_logits(scores: np.ndarray, seq: Sequence[int], begin_index: int, *, suppress: Sequence[int] = (),
                   begin_suppress: Sequence[int] = (), ts_rules: bool = False, ts_begin: int = 50365, no_ts: int = 50364,
                   eos: int = 50257, max_initial_ts: Optional[int] = None, details: bool = False):
    """One row of logits through SuppressTokensAtBegin -> SuppressTokens -> WhisperTimeStamp; seq = all tokens so far.
    details=True returns (processed, processed-before-the-probability-rule, ts_logprob - max text logprob): the last rule
    (TF/generation/logits_process.py:2034-2041) is a discrete comparison, so tie-aware parity checks need its margin."""
    s = np.array(scores, dtype=np.float32, copy=True)
    if len(seq) == begin_index and len(begin_suppress):
        s[list(begin_suppress)] = -np.inf
    if len(suppress):
        s[list(suppress)] = -np.inf
    if not ts_rules:
        return (s, s.copy(), float("nan")) if details else s
    s[no_ts] = -np.inf
    sampled = list(seq[begin_index:])
    last_ts = len(sampled) >= 1 and sampled[-1] >= ts_begin
    penult_ts = len(sampled) < 2 or sampled[-2] >= ts_begin
    if last_ts:
        if penult_ts:
            s[ts_begin:] = -np.inf
        else:
            s[:eos] = -np.inf
    tss = [t for t in sampled if t >= ts_begin]
    if tss:
        last = tss[-1] if (last_ts and not penult_ts) else tss[-1] + 1
        s[ts_begin:last] = -np.inf
    if len(seq) == begin_index:
        s[:ts_begin] = -np.inf
        if max_initial_ts is not None:
            s[ts_begin + max_initial_ts + 1:] = -np.inf
    m = s.max()
    lse_all = m + np.log(np.exp(s - m).sum()) if np.isfinite(m) else -np.inf
    logp = s - lse_all
    ts_part = logp[ts_begin:]
    tm = ts_part.max()
    ts_lp = tm + np.log(np.exp(ts_part - tm).sum()) if np.isfinite(tm) else -np.inf
    pre = s.copy()
    rule_margin = float(ts_lp - logp[:ts_begin].max())
    if ts_lp > logp[:ts_begin].max():
        s[:ts_begin] = -np.inf
    return (s, pre, rule_margin) if details else s


# ------------------------------------------------------------------------------------------------------------------
# token selection of one decoder step (decode.cu select_kernel, decode_mega.cu's fused greedy select), on exact logits
# ------------------------------------------------------------------------------------------------------------------
def rule_masks(V: int, seq: Sequence[int], begin_index: int, opts) -> np.ndarray:
    """The ids process_logits masks before its probability rule, for history `seq` (bool [V]).  `opts` carries the fields
    of thewhisper_b200.engine.DecodeOptions; max_initial_timestamp_index < 0 means no limit."""
    mit = opts.max_initial_timestamp_index
    _, pre, _ = process_logits(np.zeros(V, dtype=np.float32), seq, begin_index, suppress=list(opts.suppress_tokens),
                               begin_suppress=list(opts.begin_suppress_tokens), ts_rules=bool(opts.timestamp_rules),
                               ts_begin=opts.timestamp_begin, no_ts=opts.no_timestamps_token, eos=opts.eos_token,
                               max_initial_ts=None if mit < 0 else mit, details=True)
    return np.isneginf(pre)


def _logsumexp(x: np.ndarray) -> float:
    m = x.max() if len(x) else -np.inf
    return float(m + np.log(np.exp(x - m).sum())) if np.isfinite(m) else -np.inf


def _processed(vals: np.ndarray, seq, begin_index, opts, mask, rule_shift):
    """float64 row with the masks applied and, under timestamp rules, the probability rule evaluated in float64:
    logsumexp(timestamps) > max(text) masks all text.  -> (row, rule margin or nan).  rule_shift is added to the
    timestamp side (tests use it to restate a wrong rule; -inf turns the rule off)."""
    if mask is None:
        mask = rule_masks(len(vals), seq, begin_index, opts)
    s = np.where(mask, -np.inf, vals)
    margin = float("nan")
    if opts.timestamp_rules:
        tb = opts.timestamp_begin
        margin = _logsumexp(s[tb:]) - float(s[:tb].max())
        if margin + rule_shift > 0:
            s[:tb] = -np.inf
    return s, margin


def _order(s: np.ndarray, larger_id_ties: bool) -> np.ndarray:
    ids = np.arange(len(s))
    return np.lexsort((-ids if larger_id_ties else ids, -s))  # value descending, ties by id


def select_greedy(row, seq, begin_index: int, finished: bool, opts, *, mask=None, rule_shift: float = 0.0,
                  larger_id_ties: bool = False):
    """Greedy step on one exact logit row -> (token, finished after the step, rule margin): the masks of process_logits,
    the probability rule in float64, the first maximum (ties to the smaller id), then a finished row takes pad and a row
    that chose eos becomes finished."""
    s, margin = _processed(np.asarray(row, dtype=np.float64), seq, begin_index, opts, mask, rule_shift)
    tok = int(_order(s, larger_id_ties)[0])
    if finished:
        return opts.pad_token, True, margin
    return tok, tok == opts.eos_token, margin


def beam_candidates(row, seq, begin_index: int, run: float, n: int, opts, *, mask=None, rule_shift: float = 0.0,
                    larger_id_ties: bool = False):
    """One sequence's best n continuations -> (scores float64 [n], ids [n], rule margin): log-softmax of the raw row in
    float64 (HF takes it before the processors), the masks and probability rule on it (the rule is shift-invariant), plus
    the running score `run`; ordered by (score descending, id ascending), missing entries (-inf, -1)."""
    x = np.asarray(row, dtype=np.float64)
    s, margin = _processed(x - _logsumexp(x), seq, begin_index, opts, mask, rule_shift)
    s = s + run
    top = _order(s, larger_id_ties)[:n]
    top = top[np.isfinite(s[top])]
    scores = np.full(n, -np.inf)
    ids = np.full(n, -1, dtype=np.int64)
    scores[:len(top)], ids[:len(top)] = s[top], top
    return scores, ids, margin


# ------------------------------------------------------------------------------------------------------------------
def median_filter(x: np.ndarray, width: int = 7) -> np.ndarray:
    pad = width // 2
    if x.shape[-1] <= pad:
        return x
    xp = np.pad(x, [(0, 0)] * (x.ndim - 1) + [(pad, pad)], mode="reflect")
    win = np.lib.stride_tricks.sliding_window_view(xp, width, axis=-1)
    return np.sort(win, axis=-1)[..., pad]


def dtw(matrix: np.ndarray):
    """generation_whisper.py:64-115 verbatim semantics: float32 cost cells, strict '<', else-branch = c2."""
    T, N = matrix.shape
    cost = np.ones((T + 1, N + 1), dtype=np.float32) * np.inf
    trace = -np.ones((T + 1, N + 1), dtype=np.float32)
    cost[0, 0] = 0
    for j in range(1, N + 1):
        for i in range(1, T + 1):
            c0, c1, c2 = cost[i - 1, j - 1], cost[i - 1, j], cost[i, j - 1]
            if c0 < c1 and c0 < c2:
                c, t = c0, 0
            elif c1 < c0 and c1 < c2:
                c, t = c1, 1
            else:
                c, t = c2, 2
            cost[i, j] = matrix[i - 1, j - 1] + c
            trace[i, j] = t
    i, j = T, N
    trace[0, :] = 2
    trace[:, 0] = 1
    ti, tj = [], []
    while i > 0 or j > 0:
        ti.append(i - 1)
        tj.append(j - 1)
        if trace[i, j] == 0:
            i -= 1
            j -= 1
        elif trace[i, j] == 1:
            i -= 1
        else:
            j -= 1
    return np.array(ti)[::-1], np.array(tj)[::-1]


def token_timestamps(weights: np.ndarray, num_frames_half: int, time_precision: float = 0.02, width: int = 7) -> np.ndarray:
    """weights [Ha, T, S] softmax probabilities of the alignment heads for the T generated positions (prompt rows
    already dropped) -> [T + 1] seconds (last duplicated), as generation_whisper.py:331-379."""
    w = np.asarray(weights, dtype=np.float32)[..., :num_frames_half]
    std = w.std(axis=-2, keepdims=True)
    mean = w.mean(axis=-2, keepdims=True)
    with np.errstate(divide="ignore", invalid="ignore"):
        w = (w - mean) / std
    w = median_filter(w, width)
    m = w.mean(axis=0)
    ti, tj = dtw(-m.astype(np.float64))
    jumps = np.pad(np.diff(ti), (1, 0), constant_values=1).astype(bool)
    jt = tj[jumps] * time_precision
    return np.concatenate([jt, jt[-1:]]).astype(np.float32)
