"""ORACLE (test infrastructure, never the product path).

Log-mel and the Whisper encoder restated in float64, the way TF/models/whisper/feature_extraction_whisper.py:135-164 and
TF/models/whisper/modeling_whisper.py's encoder compute them:

  log-mel   reflect-padded 400-sample frames every 160 samples (the last frame dropped), periodic Hann(400), rfft, power,
            the engine's slaney bank (thewhisper_b200.features.mel_filter_bank), log10(max(., 1e-10)), a per-item floor at
            max - 8, then (x + 4) / 4.
  encoder   conv1 (k3, p1) -> GELU -> conv2 (k3, s2, p1) -> GELU -> + pos; pre-LN layers (eps 1e-5) with q scaled by 1/8,
            k without bias, exact GELU; the final LayerNorm; then every decoder layer's cross K (no bias) and cross V (+ xbv),
            head-major [L][B][H][S][64].

Weights are named as `engine.pack_weights` names them (conv kernels [co][tap][ci], fused wqkv / bqkv).  Every stage is a
function of explicit upstream tensors in the engine's layouts, so a test can feed the engine's own inputs to one stage; `encode`
chains them and, given an element type `et`, rounds to it wherever the engine stores a 16-bit value (mel_tm, h1, xn, qkv, ao,
hbuf, enc_out, cross K/V).

Ablations (each restates one plausible bug, so a test can show that its inputs would reveal it): `symmetric_window`,
`reflect_off_by_one`, `batch_max` (log-mel); `pos_shift` (rows of the positional table used one row late); `drop_keys_from`
(keys >= that index masked); `leak_next` (the keys of the last 128-key tile beyond S admitted unmasked: they are the next item's
rows, or zeros after the last item, as the attention kernel reads them); `v_bias_to_k` (xbv added to K instead of V);
`tanh_gelu` (the tanh approximation instead of the exact GELU).
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np
import torch
import torch.nn.functional as F

from thewhisper_b200.features import HOP, N_FFT, mel_filter_bank


# ------------------------------------------------------------------------------------------------------------------
# log-mel
# ------------------------------------------------------------------------------------------------------------------
def logmel(pcm: np.ndarray, n_mels: int = 128, *, symmetric_window: bool = False, reflect_off_by_one: bool = False,
           batch_max: bool = False) -> np.ndarray:
    """pcm [B, n_samples] (any float type, n_samples a multiple of 160) -> [B, n_mels, n_samples / 160] float64."""
    x = np.atleast_2d(np.asarray(pcm, dtype=np.float32)).astype(np.float64)
    frames = x.shape[1] // HOP
    xp = np.pad(x, ((0, 0), (N_FFT // 2, N_FFT // 2)), mode="symmetric" if reflect_off_by_one else "reflect")
    n = np.arange(N_FFT)
    win = 0.5 - 0.5 * np.cos(2 * np.pi * n / (N_FFT - 1 if symmetric_window else N_FFT))
    idx = n[None, :] + HOP * np.arange(frames)[:, None]                                   # [frames, 400]
    power = np.abs(np.fft.rfft(xp[:, idx] * win, axis=-1)) ** 2                           # [B, frames, 201]
    mel = np.einsum("bfk,km->bmf", power, mel_filter_bank(n_mels).astype(np.float64))
    lg = np.log10(np.maximum(mel, 1e-10))
    top = lg.max() if batch_max else lg.max(axis=(1, 2), keepdims=True)
    return (np.maximum(lg, top - 8.0) + 4.0) / 4.0


# ------------------------------------------------------------------------------------------------------------------
# encoder stages (torch float64; any device)
# ------------------------------------------------------------------------------------------------------------------
def _f64(t):
    return t.double() if torch.is_tensor(t) else torch.as_tensor(t, dtype=torch.float64)


def _rnd(t, et):
    return t if et is None else t.to(et).double()


def gelu(x, tanh_gelu: bool = False):
    return F.gelu(x, approximate="tanh" if tanh_gelu else "none")


def layer_norm(x, g, b):
    return F.layer_norm(x, x.shape[-1:], _f64(g), _f64(b), eps=1e-5)


def mel_tm(mel):
    """[B, n_mels, F] -> the conv stem's input [B, F + 2, n_mels]: time-major with a zero row either side."""
    return F.pad(_f64(mel).transpose(1, 2), (0, 0, 1, 1))


def conv1(w, m_tm, tanh_gelu: bool = False):
    """m_tm [B, F + 2, n_mels] (padded) -> GELU(conv1) [B, F, D] (rows 1..F of the engine's padded h1)."""
    D = w["enc.conv1.b"].shape[0]
    m = _f64(m_tm)
    W = _f64(w["enc.conv1.w"]).view(D, 3, m.shape[2])
    Fr = m.shape[1] - 2
    acc = sum(m[:, tap:tap + Fr] @ W[:, tap].T for tap in range(3))
    return gelu(acc + _f64(w["enc.conv1.b"]), tanh_gelu)


def conv2_pos(w, h1p, pos_shift: int = 0, tanh_gelu: bool = False):
    """h1p [B, F + 2, D] (padded) -> GELU(conv2, stride 2) + pos [B, S, D]."""
    D = w["enc.conv2.b"].shape[0]
    h = _f64(h1p)
    W = _f64(w["enc.conv2.w"]).view(D, 3, D)
    S = (h.shape[1] - 2) // 2
    acc = sum(h[:, tap:tap + 2 * S:2] @ W[:, tap].T for tap in range(3))
    pos = _f64(w["enc.pos"])[:S]
    if pos_shift:
        pos = pos.roll(pos_shift, 0)
    return gelu(acc + _f64(w["enc.conv2.b"]), tanh_gelu) + pos


def ln1_qkv(w, l, x, et=None):
    """Layer l's LayerNorm 1 and fused q/k/v projection (q unscaled, k bias zero): x [B, S, D] -> qkv [B, S, 3D]."""
    p = f"enc.{l}."
    xn = _rnd(layer_norm(_f64(x), w[p + "ln1.g"], w[p + "ln1.b"]), et)
    return xn @ _f64(w[p + "wqkv"]).T + _f64(w[p + "bqkv"])


def attention(qkv, H: int, drop_keys_from: Optional[int] = None, leak_next: bool = False):
    """Non-causal self-attention of each item: qkv [B, S, 3D] -> [B, S, D], scores q k^T / 8."""
    qkv = _f64(qkv)
    B, S, D3 = qkv.shape
    D = D3 // 3
    q = qkv[..., :D].reshape(B, S, H, 64).transpose(1, 2)
    if leak_next:  # item b reads rows [b S, b S + ceil(S / 128) 128) of the flat [B S] qkv rows, zeros past the last item
        T = (S + 127) // 128 * 128
        flat = torch.cat([qkv.reshape(B * S, D3), qkv.new_zeros(T, D3)])
        kv = torch.stack([flat[b * S:b * S + T] for b in range(B)])
    else:
        kv = qkv
    k = kv[..., D:2 * D].reshape(B, -1, H, 64).transpose(1, 2)
    v = kv[..., 2 * D:].reshape(B, -1, H, 64).transpose(1, 2)
    s = q @ k.transpose(-1, -2) / 8.0
    if drop_keys_from is not None:
        s[..., drop_keys_from:] = float("-inf")
    return (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(B, S, D)


def out_ln2(w, l, x, ao, et=None):
    """Out-projection + residual, then LayerNorm 2: -> (x_mid [B, S, D], xn [B, S, D])."""
    p = f"enc.{l}."
    x_mid = _f64(x) + _f64(ao) @ _f64(w[p + "wo"]).T + _f64(w[p + "bo"])
    return x_mid, _rnd(layer_norm(x_mid, w[p + "ln2.g"], w[p + "ln2.b"]), et)


def fc1(w, l, xn, tanh_gelu: bool = False):
    p = f"enc.{l}."
    return gelu(_f64(xn) @ _f64(w[p + "w1"]).T + _f64(w[p + "b1"]), tanh_gelu)


def fc2(w, l, h, x_mid):
    p = f"enc.{l}."
    return _f64(x_mid) + _f64(h) @ _f64(w[p + "w2"]).T + _f64(w[p + "b2"])


def final_ln(w, x):
    return layer_norm(_f64(x), w["enc.lnf.g"], w["enc.lnf.b"])


def cross_kv(w, n_dec: int, enc_out, H: int, v_bias_to_k: bool = False):
    """enc_out [B, S, D] -> (K, V) [L][B][H][S][64]: K without bias, V with xbv."""
    e = _f64(enc_out)
    B, S, D = e.shape
    hm = lambda t: t.view(B, S, H, 64).transpose(1, 2)
    ks, vs = [], []
    for l in range(n_dec):
        p = f"dec.{l}."
        k = e @ _f64(w[p + "xwk"]).T
        v = e @ _f64(w[p + "xwv"]).T
        bias = _f64(w[p + "xbv"])
        ks.append(hm(k + bias if v_bias_to_k else k))
        vs.append(hm(v if v_bias_to_k else v + bias))
    return torch.stack(ks), torch.stack(vs)


@torch.no_grad()
def encode(w: Dict[str, torch.Tensor], mel, n_layers: int, n_dec: int, H: int, et=None, pos_shift: int = 0,
           drop_keys_from: Optional[int] = None, leak_next: bool = False, v_bias_to_k: bool = False,
           tanh_gelu: bool = False) -> dict:
    """The whole pass from mel [B, n_mels, F]: -> dict of h1 [B, F, D], x [n_layers + 1][B, S, D] (the residual stream at
    the input of each layer and after the last), enc_out [B, S, D], cross_k / cross_v [L][B][H][S][64].  With `et`, every
    value the engine stores in 16 bits is rounded to it."""
    m = _rnd(mel_tm(mel), et)
    h1 = _rnd(conv1(w, m, tanh_gelu), et)
    x = conv2_pos(w, F.pad(h1, (0, 0, 1, 1)), pos_shift, tanh_gelu)
    xs = [x]
    for l in range(n_layers):
        qkv = _rnd(ln1_qkv(w, l, x, et), et)
        ao = _rnd(attention(qkv, H, drop_keys_from, leak_next), et)
        x_mid, xn = out_ln2(w, l, x, ao, et)
        x = fc2(w, l, _rnd(fc1(w, l, xn, tanh_gelu), et), x_mid)
        xs.append(x)
    enc_out = _rnd(final_ln(w, x), et)
    ck, cv = cross_kv(w, n_dec, enc_out, H, v_bias_to_k)
    return dict(h1=h1, x=xs, enc_out=enc_out, cross_k=_rnd(ck, et), cross_v=_rnd(cv, et))
