"""Float64 restatement of the decoder's prompt forward (what bw_decode_prefill computes): all n teacher-forced positions of Q
sequences at once, full-sequence form, engine weight naming.  Returns every layer's K / V rows.  The keyword arguments restate
the bug classes the GPU tests must be able to see:
  leak          each row also attends to the next `leak` positions (a missing / shifted causal mask);
  cross_keep    bool [S]: encoder keys kept (a dropped cross-attention key tile);
  stale         (t0, value): rows at positions >= t0 read the K / V row t0 - 1 of the previous pass as `value` (read before it
                was written across a pass boundary).
Checked against oracle/step_ref.decoder_step (itself checked against transformers) in tests/test_prefill_ref_cpu.py."""
from __future__ import annotations

import torch


def _ln(x, g, b):
    m = x.mean(-1, keepdim=True)
    v = (x - m).pow(2).mean(-1, keepdim=True)
    return (x - m) / torch.sqrt(v + 1e-5) * g + b


def _attend(q, k, v, mask):
    """q [Q, H, n, 64], k / v [Q, H, m, 64], mask bool [Q or 1, 1 or H, n, m] (True = visible)"""
    s = q @ k.transpose(-1, -2)
    s = s.masked_fill(~mask, float("-inf"))
    return torch.softmax(s, -1) @ v


def prefill_kv(w, n_layers: int, tokens, cross_k, cross_v, G: int = 1, leak: int = 0, cross_keep=None, stale=None):
    """w: engine-named decoder weights (int8 kinds already dequantised to s * q); tokens [Q, >= n] with n = tokens.shape[1];
    cross_k / cross_v [L][A'][H][S][64] (A' >= Q / G).  -> (K, V) float64 [L][Q][n][D]."""
    dev = w["dec.embed"].device
    W = lambda name: w[name].to(device=dev, dtype=torch.float64)
    tok = torch.as_tensor(tokens).to(device=dev, dtype=torch.long)
    Q, n = tok.shape
    D = w["dec.embed"].shape[1]
    H = D // 64
    heads = lambda t: t.view(Q, -1, H, 64).transpose(1, 2)  # [Q, rows, D] -> [Q, H, rows, 64]
    merge = lambda t: t.transpose(1, 2).reshape(Q, -1, D)
    x = W("dec.embed")[tok] + W("dec.pos")[:n][None]
    t = torch.arange(n, device=dev)
    self_mask = (t[None, :] <= t[:, None] + leak)[None, None]
    Ks, Vs = [], []
    for l in range(n_layers):
        p = f"dec.{l}."
        qkv = _ln(x, W(p + "ln1.g"), W(p + "ln1.b")) @ W(p + "wqkv").T + W(p + "bqkv")
        q, k, v = qkv[..., :D] * 0.125, qkv[..., D:2 * D], qkv[..., 2 * D:]
        Ks.append(k)
        Vs.append(v)
        kh, vh = heads(k), heads(v)
        if stale is None:
            ao = _attend(heads(q), kh, vh, self_mask)
        else:  # rows >= t0 see row t0 - 1 as the planted value, rows < t0 see it as it is
            t0, val = stale
            ks, vs = kh.clone(), vh.clone()
            ks[:, :, t0 - 1] = val
            vs[:, :, t0 - 1] = val
            early = (t >= t0)[None, None, :, None]
            ao = torch.where(early, _attend(heads(q), ks, vs, self_mask), _attend(heads(q), kh, vh, self_mask))
        x = x + merge(ao) @ W(p + "wo").T + W(p + "bo")
        xq = (_ln(x, W(p + "ln2.g"), W(p + "ln2.b")) @ W(p + "xwq").T + W(p + "xbq")) * 0.125
        ck = cross_k[l][: Q // G].to(device=dev, dtype=torch.float64).repeat_interleave(G, 0)  # [Q, H, S, 64]
        cv = cross_v[l][: Q // G].to(device=dev, dtype=torch.float64).repeat_interleave(G, 0)
        S = ck.shape[2]
        keep = torch.ones(S, dtype=torch.bool, device=dev) if cross_keep is None else torch.as_tensor(cross_keep, device=dev)
        xo = _attend(heads(xq), ck, cv, keep[None, None, None, :].expand(1, 1, n, S))
        x = x + merge(xo) @ W(p + "xwo").T + W(p + "xbo")
        h = torch.nn.functional.gelu(_ln(x, W(p + "ln3.g"), W(p + "ln3.b")) @ W(p + "w1").T + W(p + "b1"))
        x = x + h @ W(p + "w2").T + W(p + "b2")
    return torch.stack(Ks), torch.stack(Vs)
