"""ORACLE (test infrastructure, never the product path).

One Whisper decoder step restated in torch float64 from explicit state, the way TF/models/whisper/modeling_whisper.py's
decoder layer computes it: pre-LN layers (eps 1e-5), q scaled by 1/8 after its bias, k without bias, cross-attention v with
its bias (already inside the cross V cache), exact GELU, tied LM head.  The newest self K/V row is rounded to the cache's
element type before attention, as every engine path does.

Weights are named as `engine.pack_weights` names them.  Tensors may live on any device; pass them in float64 to avoid a
conversion per call.
"""
from __future__ import annotations

from typing import Callable, Dict, Optional, Sequence

import torch
import torch.nn.functional as F


def _ln(x, g, b):
    return F.layer_norm(x, x.shape[-1:], g, b, eps=1e-5)


def _attend(q, k, v, keep):
    """q [Q, H, 64]; k, v [Q, H, n, 64]; keep None or bool [n].  -> (out [Q, H, 64], raw scores [Q, H, n]).
    A query whose keys are all dropped gets a zero output."""
    s = torch.einsum("qhd,qhnd->qhn", q, k)
    z = s if keep is None else s.masked_fill(~keep, float("-inf"))
    p = torch.softmax(z, dim=-1).nan_to_num(0.0)
    return torch.einsum("qhn,qhnd->qhd", p, v), s


@torch.no_grad()
def decoder_step(w: Dict[str, torch.Tensor], n_layers: int, self_k, self_v, cross_k, cross_v, tokens, pos: int, G: int = 1,
                 anc=None, align_heads: Sequence[Sequence[int]] = (), round_operands: bool = False,
                 self_keep=None, cross_keep=None, hook: Optional[Callable] = None) -> dict:
    """One step of Q = tokens.shape[0] sequences (A = Q / G audios, beams of an audio adjacent) at position `pos`.

    self_k / self_v: [L][slots >= Q][Tmax][D] in the element type (the cache); rows < pos are read, through anc [Q][Tmax]
                     (sequence q reads position s from slot anc[q][s]) when it is given, else from slot q.
    cross_k / cross_v: [L][A'][H][S][64] (A' >= A).   tokens: [Q][>= pos + 1].
    round_operands: round the GEMM operands to the element type where the batched engine step does (LayerNorm outputs,
                    attention outputs, GELU output).
    self_keep: bool [pos + 1] / cross_keep: bool [S]: keys kept (None: all).
    hook(l, kind, q, k_new): called before layer l's self ("self") / cross ("cross") attention reads its keys, with the
                    scaled query [Q][H][64] and (self only) the newest key row [Q][H][64]; it may edit the caches in place.
    Returns k_new / v_new [L][Q][D] (element type), dx [Q][D] (final residual), xattn [Q][D] (last layer's cross-attention
    output), logits [Q][V], align [Q][len(align_heads)][S] (raw scaled scores) and q_self [L][Q][H][64]."""
    et = self_k.dtype
    dev = w["dec.embed"].device
    f64 = lambda t: t.to(device=dev, dtype=torch.float64)
    op = (lambda t: t.to(et).double()) if round_operands else (lambda t: t)
    W = lambda name: f64(w[name])
    Q = tokens.shape[0]
    A = Q // G
    D = w["dec.embed"].shape[1]
    H = D // 64
    S = cross_k.shape[3]
    tok = torch.as_tensor(tokens)[:, pos].to(device=dev, dtype=torch.long)
    x = W("dec.embed")[tok] + W("dec.pos")[pos][None]
    if anc is not None:
        slot = torch.as_tensor(anc)[:, :pos].to(device=dev, dtype=torch.long)             # [Q, pos]
    else:
        slot = torch.arange(Q, device=dev)[:, None].expand(Q, pos)
    sidx = torch.arange(pos, device=dev)[None].expand(Q, pos)
    beam_audio = torch.arange(Q, device=dev) // G
    slots = {tuple(p): i for i, p in enumerate(align_heads)}
    out = {"k_new": [], "v_new": [], "q_self": [], "align": torch.zeros(Q, len(align_heads), S, dtype=torch.float64, device=dev)}
    for l in range(n_layers):
        p = f"dec.{l}."
        h = op(_ln(x, W(p + "ln1.g"), W(p + "ln1.b")))
        qkv = h @ W(p + "wqkv").T + W(p + "bqkv")
        q = (qkv[:, :D] / 8).view(Q, H, 64)
        k_new, v_new = qkv[:, D:2 * D].to(et), qkv[:, 2 * D:].to(et)
        out["k_new"].append(k_new)
        out["v_new"].append(v_new)
        out["q_self"].append(q)
        if hook:
            hook(l, "self", q, k_new.double().view(Q, H, 64))
        kp = f64(self_k[l][slot, sidx])                                                   # [Q, pos, D]
        vp = f64(self_v[l][slot, sidx])
        k = torch.cat([kp, f64(k_new)[:, None]], 1).view(Q, pos + 1, H, 64).transpose(1, 2)
        v = torch.cat([vp, f64(v_new)[:, None]], 1).view(Q, pos + 1, H, 64).transpose(1, 2)
        o, _ = _attend(q, k, v, None if self_keep is None else torch.as_tensor(self_keep, device=dev))
        x = x + op(o.reshape(Q, D)) @ W(p + "wo").T + W(p + "bo")
        h = op(_ln(x, W(p + "ln2.g"), W(p + "ln2.b")))
        cq = ((h @ W(p + "xwq").T + W(p + "xbq")) / 8).view(Q, H, 64)
        if hook:
            hook(l, "cross", cq, None)
        ck, cv = f64(cross_k[l][:A])[beam_audio], f64(cross_v[l][:A])[beam_audio]        # [Q, H, S, 64]
        co, sc = _attend(cq, ck, cv, None if cross_keep is None else torch.as_tensor(cross_keep, device=dev))
        for hh in range(H):
            if (l, hh) in slots:
                out["align"][:, slots[(l, hh)]] = sc[:, hh]
        out["xattn"] = co.reshape(Q, D)
        x = x + op(co.reshape(Q, D)) @ W(p + "xwo").T + W(p + "xbo")
        h = op(_ln(x, W(p + "ln3.g"), W(p + "ln3.b")))
        f = op(F.gelu(h @ W(p + "w1").T + W(p + "b1")))
        x = x + f @ W(p + "w2").T + W(p + "b2")
    out["dx"] = x
    h = op(_ln(x, W("dec.lnf.g"), W("dec.lnf.b")))
    out["logits"] = h @ W("dec.embed").T
    for key in ("k_new", "v_new", "q_self"):
        out[key] = torch.stack(out[key])
    return out
