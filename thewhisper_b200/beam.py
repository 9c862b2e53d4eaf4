"""Beam search bookkeeping on the host (numpy), over the engine's per-step candidate lists.

The device does the heavy part of every step -- decoder forward for all A*G sequences with the cross K/V of an audio
shared by its G beams, log-softmax, the Whisper logits rules, and each sequence's 2*G best continuations
(bw_decode_beam_step) -- and KV "reordering" is a block-table permutation (bw_decode_reorder), not a copy of the cache
as in the reference path (TF/cache_utils.py:81-85, SURVEY.md K4/K8).  What remains here is the integer bookkeeping of
GenerationMixin._beam_search (TF/generation/utils.py:3076-3420): top-2G merge across beams (:2945-2997), running /
finished beam update (:3000-3072) and the early-stop heuristic (:2876-2943), with the defaults the reference uses
(length_penalty 1.0, early_stopping False, one EOS id).
"""
from __future__ import annotations

from typing import List

import numpy as np

NEG = np.float32(-1.0e9)


def _topk_desc(values: np.ndarray, k: int) -> np.ndarray:
    """indices of the k largest per row, ties -> smaller index (stable)."""
    order = np.argsort(-values, axis=1, kind="stable")
    return order[:, :k]


def beam_search(eng, prompts: np.ndarray, A: int, G: int, opts, max_new: int, length_penalty: float = 1.0, return_beam_indices: bool = False,
                prefill: bool = False, key_start=None, nospeech=None):
    """prompts [A, plen] (prefill: teacher-forced positions in one batched prefill pass).  Returns (generated ids per audio (best beam, cut before EOS), n_steps, eos_seen) and, on request, the
    `beam_indices` of the returned sequences as GenerationMixin._beam_search keeps them (TF generation/utils.py:2984-2997,3065-3070):
    entry t = the global sequence slot (audio * G + beam) whose forward pass produced generated token t, -1 beyond the sequence.
    nospeech = (position, token): scores on (engine.decode_scores_enable); the result then also holds, last, the returned sequences'
    raw log-probs per generated token [A, max_length - plen] (candidate score minus its parent's running score), which with the
    engine's lmass at the slots of `beam_indices` give the processed log-probs."""
    plen = prompts.shape[1]
    V = eng.dims.vocab
    Tmax = eng.dims.max_target_positions
    max_length = min(plen + max_new, Tmax)
    K = 2 * G
    rep = np.repeat(prompts, G, axis=0)
    if key_start is None:
        eng.decode_begin(rep, A, G, opts)
    else:  # left-padded prompts: one key start per audio, shared by its beams
        eng.decode_begin(rep, A, G, opts, key_start=key_start)
    if nospeech is not None:  # the prefill stops before the no-speech position (engine.teacher_force)
        eng.decode_scores_enable(*nospeech)
        eng.teacher_force(plen, prefill, nospeech[0])
    elif prefill and plen > 1:  # teacher-forced prompt positions
        eng.decode_prefill(plen - 1)
    else:
        eng.decode_run(plen - 1)

    pad = opts.pad_token
    # (the bookkeeping arrays are as long as this decode can get, not max_target_positions: every step gathers and concatenates
    # them -- at 64 audios x 5 beams that is the host's share of a step)
    Tmax = max_length
    running_seq = np.full((A, G, Tmax), pad, dtype=np.int32)  # (int32: these rows are gathered and concatenated every step)
    running_seq[:, :, :plen] = prompts[:, None, :]
    sequences = running_seq.copy()
    running_scores = np.zeros((A, G), dtype=np.float32)
    running_scores[:, 1:] = NEG
    beam_scores = np.full((A, G), NEG, dtype=np.float32)
    finished = np.zeros((A, G), dtype=bool)
    running_bidx = np.full((A, G, Tmax), -1, dtype=np.int32)
    bidx = running_bidx.copy()
    running_tlp = np.zeros((A, G, Tmax), dtype=np.float32)  # raw log-prob of each generated token (scores on)
    tlp = running_tlp.copy()
    unsat = np.ones((A, 1), dtype=bool)
    top_mask = np.arange(K) < G
    ar = np.arange(A)[:, None]  # row gathers below: x[ar, idx] picks whole [Tmax] rows (np.take_along_axis would build an [A, K, Tmax] index grid)
    cur_len = plen
    steps = 0
    while True:
        cs, ct = eng.decode_beam_step(running_scores.reshape(-1))  # [A*G, K] each
        steps += 1
        cs = cs.reshape(A, G * K).astype(np.float32)
        ct = ct.reshape(A, G * K).astype(np.int64)
        beam_of = np.repeat(np.arange(G), K)[None, :].repeat(A, 0)
        # merge: order by score desc, ties by flat index beam*V + token (torch.topk over [G*V] picks the first)
        flat = beam_of * V + np.where(ct >= 0, ct, V - 1)
        key = np.lexsort((flat, -cs), axis=1)[:, :K]
        top_scores = np.take_along_axis(cs, key, 1)
        top_beam = np.take_along_axis(beam_of, key, 1)
        top_tok = np.take_along_axis(ct, key, 1)
        top_tok = np.where(top_tok >= 0, top_tok, pad)
        top_seq = running_seq[ar, top_beam]  # [A, K, Tmax] (a copy)
        top_seq[:, :, cur_len] = top_tok
        top_bidx = running_bidx[ar, top_beam]
        top_bidx[:, :, cur_len - plen] = top_beam + (np.arange(A) * G)[:, None]
        if nospeech is not None:
            top_tlp = running_tlp[ar, top_beam]
            top_tlp[:, :, cur_len - plen] = top_scores - running_scores[ar, top_beam]
        hits = (top_tok == opts.eos_token) | (cur_len + 1 >= max_length)
        # running beams of the next iteration
        run_lp = top_scores + hits.astype(np.float32) * NEG
        nxt = _topk_desc(run_lp, G)
        running_seq = top_seq[ar, nxt]
        running_scores = np.take_along_axis(run_lp, nxt, 1)
        running_bidx = top_bidx[ar, nxt]
        if nospeech is not None:
            running_tlp = top_tlp[ar, nxt]
        parents = np.take_along_axis(top_beam, nxt, 1)
        next_tok = np.take_along_axis(top_tok, nxt, 1)
        # finished beams
        did_finish = hits & top_mask[None, :]
        lp = top_scores / np.float32((cur_len + 1 - plen) ** length_penalty)
        lp = lp + (~unsat).astype(np.float32) * NEG
        lp = lp + (~did_finish).astype(np.float32) * NEG
        m_scores = np.concatenate([beam_scores, lp], 1)
        m_seq = np.concatenate([sequences, top_seq], 1)
        m_fin = np.concatenate([finished, did_finish], 1)
        m_bidx = np.concatenate([bidx, top_bidx], 1)
        sel = _topk_desc(m_scores, G)
        sequences = m_seq[ar, sel]
        bidx = m_bidx[ar, sel]
        if nospeech is not None:
            tlp = np.concatenate([tlp, top_tlp], 1)[ar, sel]
        beam_scores = np.take_along_axis(m_scores, sel, 1)
        finished = np.take_along_axis(m_fin, sel, 1)
        cur_len += 1
        # early-stop heuristic (early_stopping=False): can the best running beam still beat the worst finished one?
        best_possible = running_scores[:, :1] / np.float32((cur_len - plen) ** length_penalty)
        worst_finished = np.where(finished, beam_scores.min(axis=1, keepdims=True), NEG)
        unsat = unsat & np.any(best_possible > worst_finished, axis=1, keepdims=True)
        if not (unsat.any() and not hits.all()):
            break
        glob_parent = (parents + (np.arange(A) * G)[:, None]).reshape(-1)
        eng.decode_reorder(glob_parent, next_tok.reshape(-1))
    gen: List[np.ndarray] = []
    eos_seen = []
    for a in range(A):
        row = sequences[a, 0, plen:cur_len].astype(np.int64)
        cut = np.where(row == opts.eos_token)[0]
        eos_seen.append(len(cut) > 0)
        gen.append(row[: cut[0]] if len(cut) else row)
    out = (gen, steps, eos_seen)
    if return_beam_indices:
        out += (bidx[:, 0, :].astype(np.int64),)
    if nospeech is not None:
        out += (tlp[:, 0, :],)
    return out
