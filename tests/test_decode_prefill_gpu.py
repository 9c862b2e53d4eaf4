"""bw_decode_prefill: after decode_begin, decode_prefill(n) must leave the engine in the state n decode_run steps leave -- every
layer's self K/V rows 0..n-1 of every sequence slot, pos = n -- so that the next step computes the same logits, token and K/V
row n.

Per cell (random decoder weights, random cross K/V) the same prompt is decoded both ways on one engine, in one pass and in >= 3
passes whose boundaries are not multiples of the attention kernels' 64-row tiles, and:
  * every layer's K/V rows 0..n-1 of the prefill AND of the teacher-forced steps are compared with the float64 prompt forward
    (tests/prefill_ref.py, fed s * q for int8 weights) under the same bounds, and with each other;
  * the step after (persistent, per-op or batched by Q): logits relative to their standard deviation, the selected token where
    the top-2 margin is clear of the bound, K/V row n;
  * cache rows >= n and slots >= Q keep a planted sentinel.
test_prefill_ablations_are_caught restates four bug classes in float64 on planted inputs and shows each lands outside these
bounds: a row that sees position t + 1, a row written one position late, the last cross-attention key tile dropped (its keys
planted to carry the attention), and a K/V row of the previous pass read before it was written (the cache holds a sentinel).
"""
import numpy as np
import pytest
import torch

from tests.prefill_ref import prefill_kv
from tests.test_decode_step_gpu import DTYPES, V, make_weights

pytestmark = pytest.mark.gpu

TMAX = 448
DIMS = {"tiny500": (128, 2, 512, 2, 500), "small1500": (256, 4, 1024, 3, 1500)}
NS = (1, 7, 63, 64, 65, 200, 443)
# (1, 2): per-op step after the prefill; (1, 1), (3, 1): persistent; (1, 5), (3, 5): batched with beams; 64 x 5 = 320 slots,
# 12 positions per 4096-row pass
AGS = ((1, 1), (1, 2), (3, 1), (1, 5), (3, 5))
BIG = {(64, 1): (64, 443), (64, 5): (12, 65)}
PF_ROWS = 4096  # api.cu PREFILL_ROWS
# Bounds, per element type: (K/V relative rms, K/V max |diff| / rms) against the float64 prompt forward, the same for the prefill
# and for the teacher-forced steps; (K/V relative rms, max / rms, logits max |diff| / std) between the prefill and the steps.
# Measured maxima over all cells on an NVIDIA H100 80GB HBM3 at 700 W (printed per run), prefill / steps vs float64:
#   bf16 rel rms 3.4e-3 / 3.2e-3, max/rms 2.5e-2 / 2.3e-2; fp16 rel rms 4.0e-4 / 3.9e-4, max/rms 2.8e-3 / 2.9e-3;
#   prefill vs steps: bf16 3.9e-3, 3.1e-2, logits 1.95e-2 sigma; fp16 4.4e-4, 3.9e-3, logits 2.6e-3 sigma.
# The bounds are 2.5-4x those; the smallest ablation effect (a row that sees t + 1) is 20x the max/rms bound.
TOL64 = {"bf16": (1.2e-2, 8e-2), "fp16": (1.5e-3, 1e-2)}
TOL = {"bf16": (1e-2, 8e-2, 4.5e-2), "fp16": (1.2e-3, 1e-2, 6e-3)}
SENTINEL = 3.0


def _engine(dname, tname, w8):
    from thewhisper_b200.engine import INT8_LAYER_KINDS, ModelDims, WhisperEngine, quantize_rows

    D, H, ffn, L, S = DIMS[dname]
    w = make_weights(DIMS[dname], DTYPES[tname])
    if w8:
        names = ["dec.embed"] + [f"dec.{l}.{k}" for l in range(L) for k in INT8_LAYER_KINDS]
        for n in names:
            w[n], w[n + ".scale"] = quantize_rows(w[n].float())
    w64 = {k: v.double() for k, v in w.items() if k.startswith("dec.") and not k.endswith(".scale")}
    if w8:
        for n in names:
            w64[n] = w[n].double() * w[n + ".scale"].double()[:, None]
    dims = ModelDims(D, H, ffn, 0, L, 128, V, S, TMAX)
    eng = WhisperEngine(None, dims, chunk_length_s=S * 30 / 1500, max_audios=64, max_beams=5, weights=w)
    g = torch.Generator(device="cuda").manual_seed(7)
    for name in ("cross_k", "cross_v"):
        n = L * 64 * H * S * 64
        eng.write_buffer(name, torch.randn(n, generator=g, device="cuda").to(DTYPES[tname]))
    return eng, w64


def _opts():
    from thewhisper_b200 import synthetic as S
    from thewhisper_b200.engine import DecodeOptions

    return DecodeOptions(eos_token=S.EOS, pad_token=S.EOS, suppress_tokens=S.default_suppress_tokens(),
                         begin_suppress_tokens=list(S.BEGIN_SUPPRESS))


def _caches(eng, tname):
    D, L = eng.dims.d_model, eng.dims.dec_layers
    shape = (L, 64 * 5, TMAX, D)
    return eng.buffer("self_k", DTYPES[tname], shape).clone(), eng.buffer("self_v", DTYPES[tname], shape).clone()


def _plant(eng, tname):
    D, L = eng.dims.d_model, eng.dims.dec_layers
    n = L * 64 * 5 * TMAX * D
    for name in ("self_k", "self_v"):
        eng.write_buffer(name, torch.full((n,), SENTINEL, dtype=DTYPES[tname], device="cuda"))


def _run(eng, tname, prompts, A, G, n, how):
    """-> (K, V caches after the forced positions, logits / tokens / K, V after one more step, pos after the prefill)"""
    _plant(eng, tname)
    eng.decode_begin(prompts, A, G, _opts())
    if how == "steps":
        eng.decode_run(n)
    else:
        eng.decode_prefill(n, how)
    pos = eng.decode_read()[2]
    k0, v0 = _caches(eng, tname)
    eng.decode_run(1)
    lg = eng.logits().clone()
    toks = eng.decode_read()[0]
    k1, v1 = _caches(eng, tname)
    return k0, v0, lg, toks, k1, v1, pos


def _rel(a, b):
    a, b = a.double(), b.double()
    rms = b.pow(2).mean().sqrt().item()
    return (a - b).pow(2).mean().sqrt().item() / rms, (a - b).abs().max().item() / rms


def _cross(eng, tname):
    D, H, L, S = eng.dims.d_model, eng.dims.n_heads, eng.dims.dec_layers, eng.S
    return (eng.buffer("cross_k", DTYPES[tname], (L, 64, H, S, 64)).double(),
            eng.buffer("cross_v", DTYPES[tname], (L, 64, H, S, 64)).double())


def _vs64(a, k64, Q, n, stats, key):
    rel, mx = _rel(a[:, :Q, :n], k64)
    stats[key + "_rel"] = max(stats.get(key + "_rel", 0.0), rel)
    stats[key + "_max"] = max(stats.get(key + "_max", 0.0), mx)
    return rel, mx


def _check(tname, ref, got, Q, n, label, stats, kv64, fails):
    kr, vr, lr, tr, k1r, v1r, _ = ref
    kg, vg, lgot, tg, k1g, v1g, pos = got
    if pos != n:
        fails.append((label, "pos", pos))
    tol, t64 = TOL[tname], TOL64[tname]
    for name, a, b, r64 in (("K", kg, kr, kv64[0]), ("V", vg, vr, kv64[1])):
        rel, mx = _rel(a[:, :Q, :n], b[:, :Q, :n])
        stats["diff_rel"] = max(stats.get("diff_rel", 0.0), rel)
        stats["diff_max"] = max(stats.get("diff_max", 0.0), mx)
        if rel > tol[0] or mx > tol[1]:
            fails.append((label, name, "prefill vs steps", rel, mx))
        rel, mx = _vs64(a, r64, Q, n, stats, "pf64")
        if rel > t64[0] or mx > t64[1]:
            fails.append((label, name, "prefill vs float64", rel, mx))
        # nothing outside rows 0..n-1 of slots < Q was written by the forced positions
        if not bool((a[:, Q:] == SENTINEL).all()) or not bool((a[:, :Q, n:] == SENTINEL).all()):
            fails.append((label, name, "row >= n or slot >= Q written"))
    std = lr.double().std().item()
    dl = (lgot.double() - lr.double()).abs().max().item() / std
    stats["logits"] = max(stats.get("logits", 0.0), dl)
    if dl > tol[2]:
        fails.append((label, "logits", dl))
    top2 = torch.topk(lr.double(), 2, dim=-1).values
    clear = (top2[:, 0] - top2[:, 1]) / std > 2 * tol[2]
    for q in range(Q):
        if clear[q] and tg[q, n + 1] != tr[q, n + 1]:
            fails.append((label, "token", q))
    for a, b in ((k1g, k1r), (v1g, v1r)):
        rel, mx = _rel(a[:, :Q, n], b[:, :Q, n])
        if rel > tol[0] or mx > tol[1]:
            fails.append((label, "row n", rel, mx))


def _passes_rows(Q, n):
    """max_rows_per_pass giving >= 3 passes whose boundaries are not multiples of 64 (None when n < 3)"""
    if n < 3:
        return None
    per = min(max(1, n // 3), PF_ROWS // Q)
    if per % 64 == 0:
        per -= 1
    return Q * per


CELLS = [(d, t, w8) for d in DIMS for t in ("bf16", "fp16") for w8 in (False, True)]


@pytest.mark.parametrize("dname,tname,w8", CELLS, ids=[f"{d}-{t}-{'int8' if w else '16bit'}" for d, t, w in CELLS])
def test_prefill_matches_forced_steps(cuda, dname, tname, w8):
    eng, w64 = _engine(dname, tname, w8)
    L = DIMS[dname][3]
    ck, cv = _cross(eng, tname)
    rng = np.random.default_rng(11)
    stats, fails = {}, []
    cells = [(ag, n) for ag in AGS for n in NS] + [(ag, n) for ag, ns in BIG.items() for n in ns]
    try:
        for (A, G), n in cells:
            Q = A * G
            prompt = rng.integers(0, 50257, size=(A, n + 1)).astype(np.int32)
            prompts = np.repeat(prompt, G, axis=0)
            kv64 = prefill_kv(w64, L, prompts[:, :n], ck, cv, G=G)
            ref = _run(eng, tname, prompts, A, G, n, "steps")
            for name, a, r64 in (("K", ref[0], kv64[0]), ("V", ref[1], kv64[1])):
                rel, mx = _vs64(a, r64, Q, n, stats, "steps64")
                if rel > TOL64[tname][0] or mx > TOL64[tname][1]:
                    fails.append(((A, G, n), name, "steps vs float64", rel, mx))
            _check(tname, ref, _run(eng, tname, prompts, A, G, n, 0), Q, n, (A, G, n, "one pass"), stats, kv64, fails)
            mr = _passes_rows(Q, n)
            if mr is not None:
                _check(tname, ref, _run(eng, tname, prompts, A, G, n, mr), Q, n, (A, G, n, f"rows {mr}"), stats, kv64, fails)
            del kv64
        print(f"\n[{dname} {tname} {'int8' if w8 else '16-bit'}] measured max: "
              + ", ".join(f"{k} {v:.2e}" for k, v in sorted(stats.items())) + f"; bounds float64 {TOL64[tname]}, prefill vs steps {TOL[tname]}")
        assert not fails, fails[:10]
    finally:
        eng.close()


def test_prefill_ablations_are_caught(cuda):
    """On planted inputs, the float64 restatement of each bug class lands outside the bounds the cells above apply, while the
    prefill itself (in passes with boundaries at 43, 86, 129) lands inside them."""
    eng, w64 = _engine("tiny500", "bf16", False)
    D, H, ffn, L, S = DIMS["tiny500"]
    try:
        A, G, n = 1, 1, 130
        # plant: the keys of the last (partial) 64-key tile of every head scaled so that they carry the cross attention
        ck = eng.buffer("cross_k", torch.bfloat16, (L, 64, H, S, 64)).clone()
        last = (S - 1) // 64 * 64
        ck[:, :, :, last:] *= 4
        eng.write_buffer("cross_k", ck)
        ck64, cv64 = _cross(eng, "bf16")
        rng = np.random.default_rng(3)
        prompts = rng.integers(0, 50257, size=(1, n + 1)).astype(np.int32)
        k64, _ = prefill_kv(w64, L, prompts[:, :n], ck64, cv64)
        kp = _run(eng, "bf16", prompts, A, G, n, 43)[0][:, :1, :n]
        t64 = TOL64["bf16"]
        rel, mx = _rel(kp, k64)
        print(f"\n[ablation] prefill vs float64: K rel rms {rel:.2e}, max/rms {mx:.2e} (bounds {t64})")
        assert rel <= t64[0] and mx <= t64[1]
        keep = torch.ones(S, dtype=torch.bool)
        keep[last:] = False
        bugs = {
            "sees t + 1": prefill_kv(w64, L, prompts[:, :n], ck64, cv64, leak=1)[0],
            "row one position late": torch.cat([k64[:, :, :1], k64[:, :, :-1]], dim=2),
            "last cross key tile dropped": prefill_kv(w64, L, prompts[:, :n], ck64, cv64, cross_keep=keep)[0],
            "previous pass row read before written": prefill_kv(w64, L, prompts[:, :n], ck64, cv64, stale=(86, SENTINEL))[0],
        }
        for label, bad in bugs.items():
            rel, mx = _rel(bad, k64)
            print(f"[ablation {label}] K rel rms {rel:.2e} ({rel / t64[0]:.1f}x bound), max/rms {mx:.2e} ({mx / t64[1]:.1f}x bound)")
            assert max(rel / t64[0], mx / t64[1]) >= 10, label  # every bound at or below 1/10 of the effect it must catch
    finally:
        eng.close()


def test_prefill_argument_checks(cuda):
    from thewhisper_b200 import _lib

    eng, _ = _engine("tiny500", "bf16", False)
    try:
        prompts = np.zeros((2, 5), dtype=np.int32)
        eng.decode_begin(prompts, 2, 1, _opts())
        for bad in ((0, 0), (5, 0), (2, 1)):  # n = 0, n > begin_index - 1, max_rows_per_pass < Q
            with pytest.raises(_lib.BwError):
                eng.decode_prefill(*bad)
        eng.decode_run(1)
        with pytest.raises(_lib.BwError, match="must come first"):
            eng.decode_prefill(2)
        eng.decode_begin(prompts, 2, 1, _opts())
        eng.decode_prefill(4, 2)  # one position per pass
        assert eng.decode_read()[2] == 4
    finally:
        eng.close()
