"""The float64 log-mel and encoder restatement (oracle/enc_ref.py) agrees with transformers.  The GPU stage tests
(tests/test_encode_stage_gpu.py) compare the engine's kernels against this restatement with tight bounds, so it is proven
here first: a failure there then points at a kernel, not at the reference.

Measured maxima (this file prints them):
  log-mel vs WhisperFeatureExtractor (float32 arithmetic): 2.1e-5 absolute; vs tests/golden/logmel.npz: 2.9e-6
  encoder vs WhisperEncoder in float64, relative to the output rms: 6.9e-15 (S = 500), 7.2e-15 (S = 600), 6.9e-15 (S = 1500)
"""
import os

import numpy as np
import pytest
import torch


def _cases():
    from thewhisper_b200 import synthetic as S

    rng = np.random.RandomState(3)
    n = 160000
    imp = np.zeros(n, dtype=np.float32)
    imp[0], imp[-1] = 1.0, -0.7
    sq = np.clip(2.0 * np.sign(np.sin(2 * np.pi * 330 * np.arange(n) / 16000)), -1, 1).astype(np.float32)
    return {"noise": (0.1 * rng.randn(n)).astype(np.float32), "impulses": imp, "square": sq,
            "speech": S.synth_audio(10, seed=5), "two_tone": S.two_tone(10)}


def test_logmel_ref_matches_feature_extractor():
    from oracle.enc_ref import logmel
    from tests.conftest import GOLD
    from thewhisper_b200 import synthetic as S

    fe = S.make_feature_extractor(10)
    worst = 0.0
    for name, x in _cases().items():
        want = fe(x, sampling_rate=16000, return_tensors="np")["input_features"][0].astype(np.float64)
        got = logmel(x[None])[0]
        err = float(np.abs(got - want).max())
        worst = max(worst, err)
        assert err < 5e-5, (name, err)
    gold = np.load(os.path.join(GOLD, "logmel.npz"))
    gerr = float(np.abs(logmel(S.two_tone(10)[None])[0][:, ::25] - gold["two_tone_10s_sub"]).max())
    x = (np.random.RandomState(0).randn(160000) * 0.1).astype(np.float32)
    gerr = max(gerr, float(np.abs(logmel(x[None])[0][:, ::10] - gold["noise_10s_sub"]).max()))
    assert gerr < 5e-5, gerr
    # a batch is per-item: a quiet item next to a loud one keeps its own floor
    quiet, loud = 1e-3 * _cases()["noise"], _cases()["square"]
    both = logmel(np.stack([loud, quiet]))
    assert np.array_equal(both[1], logmel(quiet[None])[0])
    assert np.abs(logmel(np.stack([loud, quiet]), batch_max=True)[1] - both[1]).max() > 0.1
    print(f"\nlog-mel restatement: max |d| {worst:.1e} vs WhisperFeatureExtractor, {gerr:.1e} vs the golden fixture")


@pytest.mark.parametrize("S_", [500, 600, 1500])
def test_encoder_ref_matches_transformers(S_):
    from oracle import enc_ref, hf_ref
    from thewhisper_b200 import synthetic as S
    from thewhisper_b200.engine import ModelDims, pack_weights

    model = S.make_hf_model("tiny-test", layer_gain=8)
    if S_ != 1500:
        hf_ref.interpolate_positions(model, S_ * 30 / 1500)
    enc = model.model.encoder.double().eval()
    dims = ModelDims.from_hf_config(model.config)
    sd = model.state_dict()
    w = pack_weights(sd, dims, sd["model.encoder.embed_positions.weight"], device="cpu", dtype=torch.float64)
    mel = torch.from_numpy(np.stack([hf_ref.logmel(S.make_feature_extractor(S_ * 30 // 1500), S.synth_audio(S_ / 50, seed=s))
                                     for s in (1, 2)])).double()
    with torch.no_grad():
        want = enc(mel).last_hidden_state
    ref = enc_ref.encode(w, mel, dims.enc_layers, dims.dec_layers, dims.n_heads)
    assert ref["enc_out"].shape == (2, S_, dims.d_model)
    err = float((ref["enc_out"] - want).abs().max() / want.pow(2).mean().sqrt())
    assert err < 1e-12, err
    # cross K/V restated from their definition: [L][B][H][S][64]
    l = dims.dec_layers - 1
    k = want @ w[f"dec.{l}.xwk"].T
    v = want @ w[f"dec.{l}.xwv"].T + w[f"dec.{l}.xbv"]
    H = dims.n_heads
    assert torch.allclose(ref["cross_k"][l], k.view(2, S_, H, 64).transpose(1, 2), atol=1e-12)
    assert torch.allclose(ref["cross_v"][l], v.view(2, S_, H, 64).transpose(1, 2), atol=1e-12)
    print(f"\nencoder restatement S={S_}: max |d| {err:.1e} of the output rms vs transformers WhisperEncoder (float64)")
