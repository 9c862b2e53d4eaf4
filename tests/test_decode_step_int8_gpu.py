"""One decoder step with int8 decoder weights, on every step path, against the float64 restatement (oracle/step_ref.py) fed
the dequantised weights s[n] * q[n, k].

The machinery (weights, state injection, planted attention scores, the per-position checks and their bounds) is that of
tests/test_decode_step_gpu.py, imported.  The dequantisation is exact (|q| <= 128 converts exactly and the scale multiplies
the fp32 dot product once per row), so the arithmetic class of each path is that of its 16-bit version and the same bounds
(TOL, KV_ULPS per class) apply.  On the batched step the int8 weight tiles are converted to the 16-bit wgmma operand in shared
memory and the scale multiplies each split-K partial sum, so its cells are held to the batched-class bounds.

Each quantised kind gets one planted row whose codes run through all 256 values (-128 included), written past the quantiser.
"""
import numpy as np
import pytest
import torch

from tests import test_decode_step_gpu as T

pytestmark = pytest.mark.gpu

KINDS = ("wqkv", "wo", "xwq", "xwo", "w1", "w2")
# Measured maxima over all cells on an NVIDIA H100 80GB HBM3 at a 700 W power limit (logits, dx, attention, alignment; tiny /
# small, large-v3 in brackets), all within the 16-bit file's bounds for the same class, which apply unchanged:
#   fp32 bf16:    6.2e-4 (1.5e-3), 3.8e-4 (1.2e-3), 2.6e-4 (1.5e-3), 1.9e-4 (3.0e-4); K/V rows within 1 ulp at every layer
#   fp32 fp16:    7.3e-5 (1.7e-4), 5.3e-5 (2.0e-4), 8.4e-5 (1.7e-4), 1.6e-5 (4.3e-5)
#   batched bf16: 1.6e-2 (2.7e-2), 8.6e-3 (3.7e-2), 2.1e-2 (6.6e-2), 4.1e-3 (7.9e-3); K/V 2.5 (6) ulps
#   batched fp16: 2.3e-3 (3.5e-3), 1.4e-3 (3.2e-3), 4.1e-3 (5.6e-3), 5.2e-4 (9.4e-4); K/V 3 (6) ulps
CELLS = [(d, t, p, ag) for d in ("tiny500", "tiny750", "small1500") for t in ("bf16", "fp16") for p in T.PATHS for ag in T.SMALL_AG[p]
         if not (p.startswith("mega") and ag[1] > 1)]
CELLS += [("large1500",) + c for c in T.LARGE_CELLS]


def quantized_weights(dname, tname, plant=True, seed=0):
    """(engine weights with int8 decoder matrices, their float64 restatement for the oracle).  The fp32 weights of
    T.make_weights are the checkpoint: the quantiser reads them, the other tensors take the engine's 16-bit type."""
    from thewhisper_b200.engine import quantize_rows

    w32 = T.make_weights(T.DIMS[dname], torch.float32, seed=seed)
    dtype = T.DTYPES[tname]
    L = T.DIMS[dname][3]
    w, w64 = {}, {}
    quant = ["dec.embed"] + [f"dec.{l}.{k}" for l in range(L) for k in KINDS]
    for n, t in w32.items():
        if n in quant:
            q, s = quantize_rows(t)
            if plant:  # row 1: codes -128 .. 127 (repeated), the row's scale kept
                K = q.shape[1]
                q[1] = (torch.arange(K, device=q.device) % 256 - 128).to(torch.int8)
            w[n], w[n + ".scale"] = q, s
            w64[n] = s.double()[:, None] * q.double()
        elif t.dtype == torch.float32 and t.dim() == 2 and not n.startswith("enc.pos") and n != "dec.pos":
            w[n] = t.to(dtype)
            w64[n] = w[n].double()
        else:
            w[n] = t
            w64[n] = t.double()
    return w, {k: v for k, v in w64.items() if k.startswith("dec.")}


class Rig8(T.Rig):
    def weights(self, dname, tname):
        if self.key_w != (dname, tname):
            self.close()
            self.w = self.w64 = None
            torch.cuda.empty_cache()
            self.w, self.w64 = quantized_weights(dname, tname)
            self.key_w = (dname, tname)
        return self.w, self.w64


@pytest.fixture(scope="module")
def rig8():
    r = Rig8()
    yield r
    r.close()


@pytest.mark.parametrize("dname,tname,path,ag", CELLS, ids=[f"{d}-{t}-{p}-A{a}G{g}" for d, t, p, (a, g) in CELLS])
def test_decode_step_int8_matches_reference(cuda, rig8, dname, tname, path, ag):
    A, G = ag
    print(f"\n[int8 {dname} {tname} {path} A={A} G={G}]")
    T.run_cell(rig8, dname, tname, path, A, G, T.LARGE_POSITIONS if dname == "large1500" else T.POSITIONS)
    assert rig8.eng.decoder_weights == "int8"


def test_int8_ablations_are_visible(cuda):
    """The inputs above separate these bugs from correct code: the unquantised weights, one kind's scales shifted by one row,
    the embedding scale dropped from the lookup must each move the logits by >= 10x the bound."""
    from oracle.step_ref import decoder_step

    dname, tname, pos = "tiny500", "bf16", 145
    w, w64 = quantized_weights(dname, tname)
    c = T.make_case(w64, dname, tname, "perop", 1, 1, 1, 1, pos)
    D, H, ffn, L, Sx = T.DIMS[dname]
    args = (L, c["self_k"], c["self_v"], c["cross_k"], c["cross_v"], c["tokens"][:1], pos)
    lg = decoder_step(w64, *args)["logits"]
    scale = float(lg.std())
    tol = T.TOL[("fp32", tname)][0]
    w32 = T.make_weights(T.DIMS[dname], torch.float32)
    variants = {"unquantised": {k: (w32[k].double() if k in w64 and w32[k].dim() == 2 and "ln" not in k else v) for k, v in w64.items()}}
    for kind in KINDS:
        n = f"dec.0.{kind}"
        sh = dict(w64)
        s = w[n + ".scale"].double()
        sh[n] = torch.roll(s, 1)[:, None] * w[n].double()
        variants[f"{kind} scales shifted"] = sh
    emb = dict(w64)
    tok = int(c["tokens"][0, pos])
    emb["dec.embed"] = w64["dec.embed"].clone()
    emb["dec.embed"][tok] = w["dec.embed"][tok].double()  # the looked-up row without its scale
    variants["embed scale dropped"] = emb
    for k, v in variants.items():
        e = float((decoder_step(v, *args)["logits"] - lg).abs().max()) / scale
        print(f"  ablation {k}: {e:.3f} (bound {tol:.0e})")
        assert e >= 10 * tol, (k, e)


def test_int8_encoder_output_and_cross_kv_are_bit_identical(cuda):
    """xwk / xwv stay 16-bit: the encoder output and cross K/V of an int8 engine equal those of a 16-bit engine bit for bit."""
    import json
    import os

    from tests.conftest import GOLD
    from thewhisper_b200 import synthetic as S
    from thewhisper_b200.engine import ModelDims, WhisperEngine

    meta = json.load(open(os.path.join(GOLD, "model_tiny10.json")))
    model = S.make_hf_model(meta["preset"], seed=meta["seed"], layer_gain=meta.get("layer_gain", 1.0))
    pcm = np.stack([S.synth_audio(10, seed=1000 + i) for i in range(2)])
    out = {}
    for fmt in (None, "int8"):
        eng = WhisperEngine(model.state_dict(), ModelDims.from_hf_config(model.config), chunk_length_s=10, max_audios=2,
                            decoder_weights=fmt)
        try:
            eng.logmel(pcm)
            eng.encode(2)
            L, H = eng.dims.dec_layers, eng.dims.n_heads
            out[fmt] = [eng.buffer("enc_out", eng.dtype, (2, eng.S, eng.dims.d_model))] + [
                eng.buffer(n, eng.dtype, (L, 2, H, eng.S, 64)) for n in ("cross_k", "cross_v")]
        finally:
            eng.close()
    for a, b in zip(out[None], out["int8"]):
        assert torch.equal(a, b)


def test_finalize_rejects_mixed_or_missing_scales(cuda):
    from thewhisper_b200 import _lib
    from thewhisper_b200.engine import ModelDims, WhisperEngine

    dname, tname = "tiny500", "bf16"
    D, H, ffn, L, S = T.DIMS[dname]
    dims = ModelDims(D, H, ffn, 0, L, 128, T.V, S, T.TMAX)
    w8, _ = quantized_weights(dname, tname, plant=False)

    def build(w, **kw):
        eng = WhisperEngine(None, dims, chunk_length_s=S * 30 / 1500, weights=w, **kw)
        eng.close()

    build(w8)  # complete: accepted
    missing = {k: v for k, v in w8.items() if k != "dec.1.w2.scale"}
    with pytest.raises(_lib.BwError, match=r"dec\.1\.w2\.scale"):
        build(missing)
    w16 = {k: (v.to(torch.bfloat16) if v.dtype == torch.int8 else v) for k, v in w8.items() if not k.endswith(".scale")}
    build(w16)
    with pytest.raises(_lib.BwError, match=r"dec\.0\.wo\.scale"):  # a scale without dec.embed.scale
        build(dict(w16, **{"dec.0.wo.scale": w8["dec.0.wo.scale"]}))
    with pytest.raises(_lib.BwError, match=r"dec\.0\.xwk\.scale"):  # xwk is never quantised
        build(dict(w8, **{"dec.0.xwk.scale": w8["dec.0.wo.scale"]}))
    with pytest.raises(_lib.BwError, match="int8"):  # the requested format must be the preloaded one
        build(w16, decoder_weights="int8")
