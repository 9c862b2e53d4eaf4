"""tests/prefill_ref.prefill_kv (the float64 prompt forward the prefill GPU tests compare with) against n steps of
oracle/step_ref.decoder_step, which is itself checked against transformers (tests/test_step_ref_cpu.py); and its ablation
switches change what they claim to change."""
import torch

from oracle.step_ref import decoder_step
from tests.prefill_ref import prefill_kv


def _weights(D=128, ffn=256, L=2, V=300, T=16, seed=0):
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    w = {"dec.embed": rn(V, D) * 0.5, "dec.pos": rn(T, D), "dec.lnf.g": 1 + 0.1 * rn(D), "dec.lnf.b": 0.1 * rn(D)}
    for l in range(L):
        p = f"dec.{l}."
        for k in ("ln1", "ln2", "ln3"):
            w[p + k + ".g"], w[p + k + ".b"] = 1 + 0.1 * rn(D), 0.1 * rn(D)
        w[p + "wqkv"], w[p + "bqkv"] = rn(3 * D, D) / D ** 0.5, 0.1 * rn(3 * D)
        for k, b in (("wo", "bo"), ("xwq", "xbq"), ("xwo", "xbo")):
            w[p + k], w[p + b] = rn(D, D) / D ** 0.5, 0.1 * rn(D)
        w[p + "w1"], w[p + "b1"] = rn(ffn, D) / D ** 0.5, 0.1 * rn(ffn)
        w[p + "w2"], w[p + "b2"] = rn(D, ffn) / ffn ** 0.5, 0.1 * rn(D)
    return w


def test_prefill_ref_matches_step_oracle():
    D, L, H, S, T, n, A, G = 128, 2, 2, 20, 16, 9, 2, 2
    Q = A * G
    w = _weights(D=D, L=L, T=T)
    g = torch.Generator().manual_seed(1)
    ck = torch.randn(L, A, H, S, 64, generator=g, dtype=torch.float64)
    cv = torch.randn(L, A, H, S, 64, generator=g, dtype=torch.float64)
    tokens = torch.randint(0, 300, (A, n), generator=g).repeat_interleave(G, 0)
    tokens[1, 3] = 7  # beams of one audio need not share their rows
    K, V = prefill_kv(w, L, tokens, ck, cv, G=G)
    sk = torch.zeros(L, Q, T, D, dtype=torch.float64)
    sv = torch.zeros_like(sk)
    for pos in range(n):
        out = decoder_step(w, L, sk, sv, ck, cv, tokens.numpy(), pos, G=G)
        sk[:, :, pos], sv[:, :, pos] = out["k_new"], out["v_new"]
    assert (K - sk[:, :, :n]).abs().max().item() < 1e-9
    assert (V - sv[:, :, :n]).abs().max().item() < 1e-9
    # the ablation switches: a leak changes rows < n - 1 of layers >= 1 only, the last row cannot see further
    Kl, _ = prefill_kv(w, L, tokens, ck, cv, G=G, leak=1)
    assert torch.equal(Kl[0], K[0]) and (Kl[1, :, : n - 1] - K[1, :, : n - 1]).abs().max() > 1e-3
    assert (Kl[1, :, n - 1] - K[1, :, n - 1]).abs().max() < 1e-12
    keep = torch.ones(S, dtype=torch.bool)
    keep[16:] = False
    Kc, _ = prefill_kv(w, L, tokens, ck, cv, G=G, cross_keep=keep)
    assert torch.equal(Kc[0], K[0]) and (Kc[1] - K[1]).abs().max() > 1e-3
    Ks, _ = prefill_kv(w, L, tokens, ck, cv, G=G, stale=(5, 3.0))
    assert torch.equal(Ks[0], K[0]) and (Ks[1, :, :5] - K[1, :, :5]).abs().max() < 1e-12 and (Ks[1, :, 5:] - K[1, :, 5:]).abs().max() > 1e-3
