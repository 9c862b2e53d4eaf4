"""The float64 decoder-step restatement (oracle/step_ref.py) agrees with transformers at every position of a 448-token
sequence.  The GPU step tests (tests/test_decode_step_gpu.py) compare the engine's kernels against this restatement with
tight bounds, so it is proven here first: a failure there then points at a kernel, not at the reference."""
import numpy as np
import torch


def test_step_ref_matches_transformers_all_positions():
    from oracle import hf_ref
    from oracle.step_ref import decoder_step
    from thewhisper_b200 import synthetic as S
    from thewhisper_b200.engine import ModelDims, pack_weights

    model = S.make_hf_model("tiny-test", layer_gain=8)
    dims = ModelDims.from_hf_config(model.config)
    sd = model.state_dict()
    w = pack_weights(sd, dims, sd["model.encoder.embed_positions.weight"], device="cpu", dtype=torch.float32)
    w = {k: v.double() for k, v in w.items() if k.startswith("dec.")}
    L, D, H, T = dims.dec_layers, dims.d_model, dims.n_heads, dims.max_target_positions
    fe = S.make_feature_extractor(30)
    mel = hf_ref.logmel(fe, S.synth_audio(30, seed=1000))
    with torch.no_grad():
        enc = model.model.encoder(torch.from_numpy(mel)[None]).last_hidden_state  # [1, S, D] fp32
    Sx = enc.shape[1]
    e64 = enc[0].double()
    ck = torch.stack([(e64 @ w[f"dec.{l}.xwk"].T).view(Sx, H, 64).transpose(0, 1) for l in range(L)])[:, None]
    cv = torch.stack([(e64 @ w[f"dec.{l}.xwv"].T + w[f"dec.{l}.xbv"]).view(Sx, H, 64).transpose(0, 1) for l in range(L)])[:, None]
    rng = np.random.RandomState(7)
    ids = [S.SOT, S.LANG_EN, S.TRANSCRIBE, S.NOTIMESTAMPS] + rng.randint(0, S.EOS, size=T - 4).tolist()
    with torch.no_grad():
        ref = model(encoder_outputs=(enc,), decoder_input_ids=torch.tensor([ids])).logits[0].double()  # [T, V] fp32
    # the restatement grows its own fp32 cache (the element type of an fp32 checkpoint) one step at a time
    self_k = torch.zeros(L, 1, T, D, dtype=torch.float32)
    self_v = torch.zeros_like(self_k)
    toks = torch.tensor([ids])
    scale = float(ref.std())
    worst = 0.0
    for pos in range(T):
        out = decoder_step(w, L, self_k, self_v, ck, cv, toks, pos)
        self_k[:, 0, pos] = out["k_new"][:, 0]
        self_v[:, 0, pos] = out["v_new"][:, 0]
        err = float((out["logits"][0] - ref[pos]).abs().max()) / scale
        worst = max(worst, err)
        assert err < 1e-4, (pos, err)
    print(f"\nstep_ref vs transformers fp32 over {T} positions: max |dlogit| = {worst:.2e} of the logit std ({scale:.3f})")
