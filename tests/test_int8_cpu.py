"""CPU checks of the int8 decoder-weight format: the quantiser, what pack_weights emits, the weight broadcast's flat layout,
and the persistent step's shared-memory plan for 1-byte weight rows."""
import ctypes as C

import pytest
import torch

from thewhisper_b200.engine import INT8_LAYER_KINDS, ModelDims, decoder_weights_of, pack_weights, quantize_rows


def test_quantize_rows_rounds_half_to_even_and_clamps():
    # row 0: amax 127 -> s = 1, so w / s is w itself: .5 cases round to even
    w = torch.tensor([[0.5, 1.5, 2.5, -0.5, -1.5, -2.5, 127.0, 3.49],
                      [0.0] * 8,
                      [1e-3, -2e-3, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0]], dtype=torch.float32)
    q, s = quantize_rows(w)
    assert q.dtype == torch.int8 and s.dtype == torch.float32 and q.shape == w.shape and s.shape == (3,)
    assert q[0].tolist() == [0, 2, 2, 0, -2, -2, 127, 3]
    assert s[1].item() == 1.0 and q[1].abs().sum().item() == 0  # an all-zero row: s = 1, codes 0
    assert q[2, 1].item() == -127 and q[2, 0].item() == round(1e-3 / (2e-3 / 127))  # the row's amax maps to +-127
    # the clamp: a value just past 127 s cannot leave [-127, 127]
    q2, _ = quantize_rows(torch.tensor([[1.0, -1.0, 0.999]]))
    assert q2.min().item() >= -127 and q2.max().item() <= 127


def test_quantize_rows_round_trip_is_exact_s_times_q():
    g = torch.Generator().manual_seed(0)
    w = torch.randn(64, 96, generator=g) * torch.linspace(1e-3, 10, 64)[:, None]
    q, s = quantize_rows(w)
    deq = s.double()[:, None] * q.double()
    # per element the error is at most half a step (the rounding), and s * q is what the kernels compute with
    assert ((deq - w.double()).abs() <= s.double()[:, None] / 2 * (1 + 1e-6)).all()
    assert torch.equal(q.abs().amax(dim=1), torch.full((64,), 127, dtype=torch.int8))
    # a bf16 cast first would change the codes: the quantiser reads the checkpoint's own values
    q16, _ = quantize_rows(w.to(torch.bfloat16).float())
    assert not torch.equal(q16, q)


def _tiny_sd():
    from thewhisper_b200 import synthetic as S

    model = S.make_hf_model("tiny-test", seed=0)
    return model, model.state_dict()


def test_pack_weights_int8_names_and_dtypes():
    model, sd = _tiny_sd()
    dims = ModelDims.from_hf_config(model.config)
    pos = sd["model.encoder.embed_positions.weight"].float()
    w16 = pack_weights(sd, dims, pos, torch.device("cpu"), torch.bfloat16)
    w8 = pack_weights(sd, dims, pos, torch.device("cpu"), torch.bfloat16, "int8")
    assert decoder_weights_of(w16) is None and decoder_weights_of(w8) == "int8"
    quant = ["dec.embed"] + [f"dec.{i}.{k}" for i in range(dims.dec_layers) for k in INT8_LAYER_KINDS]
    assert set(w8) == set(w16) | {n + ".scale" for n in quant}  # no 16-bit duplicate, nothing else added
    for n in quant:
        assert w8[n].dtype == torch.int8 and w8[n].shape == w16[n].shape, n
        assert w8[n + ".scale"].dtype == torch.float32 and w8[n + ".scale"].shape == (w16[n].shape[0],), n
        assert w8[n].is_contiguous() and w8[n + ".scale"].is_contiguous()
    for n, t in w16.items():
        if n not in quant:  # encoder, cross K/V projections (xwk / xwv), vectors: the 16-bit engine's tensors
            assert w8[n].dtype == t.dtype and torch.equal(w8[n], t), n
    for i in range(dims.dec_layers):
        assert w8[f"dec.{i}.xwk"].dtype == torch.bfloat16 and w8[f"dec.{i}.xwv"].dtype == torch.bfloat16
    # the codes are those of the checkpoint's fp32 values (fused q/k/v rows in the engine's order)
    p = "model.decoder.layers.0."
    wqkv = torch.cat([sd[p + "self_attn.q_proj.weight"], sd[p + "self_attn.k_proj.weight"], sd[p + "self_attn.v_proj.weight"]], 0)
    q, s = quantize_rows(wqkv)
    assert torch.equal(w8["dec.0.wqkv"], q) and torch.equal(w8["dec.0.wqkv.scale"], s)
    with pytest.raises(ValueError):
        pack_weights(sd, dims, pos, torch.device("cpu"), torch.bfloat16, "int4")


def test_flatten_round_trip_with_int8_and_scales():
    from thewhisper_b200.parallel import flatten_weights, views_of

    model, sd = _tiny_sd()
    dims = ModelDims.from_hf_config(model.config)
    w8 = pack_weights(sd, dims, sd["model.encoder.embed_positions.weight"].float(), torch.device("cpu"), torch.bfloat16, "int8")
    flat, meta, views = flatten_weights(w8, torch.device("cpu"))
    again = views_of(flat.clone(), meta)
    assert set(again) == set(w8)
    for n, t in w8.items():
        assert again[n].dtype == t.dtype and again[n].shape == t.shape and torch.equal(again[n], t), n
        assert (views[n].data_ptr() - flat.data_ptr()) % 256 == 0  # 256-byte aligned offsets (TMA / vector loads)
    assert decoder_weights_of(again) == "int8"


OPTIN = 227 * 1024  # opt-in shared memory per block of an H100 (sm_90)


@pytest.mark.parametrize("sms", [114, 132, 148])
@pytest.mark.parametrize("Q", [1, 2])
def test_mega_plan_w8_is_double_buffered(sms, Q):
    """With 1-byte rows at large-v3 dims the slab regions are about half their 16-bit size and the pool is bound by the
    attention scratch (~147 KB), so every case keeps double-buffered slabs, at <= 188 KB of dynamic smem."""
    from tests.test_mega_plan_cpu import _static_smem

    from thewhisper_b200 import _lib, build

    build.build()
    lib = _lib.load()
    static = _static_smem(_lib.LIB_PATH)
    out = (C.c_int64 * 2)()
    rc = lib.bw_op_mega_plan_w8(Q, 1280, 5120, sms, OPTIN, static, out)
    smem, p0_off = int(out[0]), int(out[1])
    assert rc == 0 and p0_off > 0 and smem + static <= OPTIN, (sms, Q, rc, smem, p0_off, static)
    assert smem <= 188 * 1024, smem
    # the attention scratch (ATT_OFF + 448 keys x 256 B + the 12-warp fold) is the pool, not the two slab regions
    att = 32 * 1024 + 448 * 256 + 12 * 72 * 4
    fixed = 64 * 4 + Q * 5120 * 4 + 128
    assert smem == fixed + att, (smem, fixed + att)
    out16 = (C.c_int64 * 2)()
    assert lib.bw_op_mega_plan(Q, 1280, 5120, sms, OPTIN, static, out16) == 0
    assert smem <= int(out16[0])
