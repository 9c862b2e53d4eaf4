"""Sequential long-form transcription on the GPU:
  * bw_logmel_long against the float64 restatement (oracle/enc_ref.py) at the bound of the chunk log-mel test, for sample counts
    just past the window, not a multiple of 160, 10 minutes, and a batch of three unequal lengths with their zero tails; and
    bit-identical to bw_logmel at one window;
  * the per-sequence key start of decoder self-attention (left-padded decoder inputs) on the per-op step, the batched step and
    the prefill: one step against the float64 step restatement with the keys below the start dropped (logits, appended K/V rows,
    the last layer's cross-attention output), NaN planted in the K/V rows below the start, the K/V rows of a pad query (no key:
    a zero self-attention output), an off-by-one ablation, and the path a key start selects at Q = 2;
  * the step-graph cache: bounded, least recently used evicted;
  * long-form through ASRPipeline on tiny10 and small30: every greedy decode call replayed through transformers (tie-aware, with
    the decoder attention mask of a conditioned window), plain / word / conditioned / int8; beam 5 on fp16 against the live
    transformers transcript; one large-v3-shape call on 10 minutes of audio."""
import json
import os

import numpy as np
import pytest
import torch

from tests.conftest import GOLD
from tests.test_encode_stage_gpu import LOGMEL_ABS

pytestmark = pytest.mark.gpu


def _engine(preset="tiny-test", chunk=10, max_audios=3, max_beams=1, dtype=torch.bfloat16, layer_gain=8.0):
    from thewhisper_b200 import synthetic as S
    from thewhisper_b200.engine import ModelDims, WhisperEngine

    model = S.make_hf_model(preset, seed=0, layer_gain=layer_gain)
    return WhisperEngine(model.state_dict(), ModelDims.from_hf_config(model.config), chunk_length_s=chunk, max_audios=max_audios,
                         max_beams=max_beams, dtype=dtype), model


# ------------------------------------------------------------------------------------------------------------------
# long log-mel
# ------------------------------------------------------------------------------------------------------------------
def test_logmel_long_matches_reference(cuda):
    from oracle import enc_ref as R

    eng, _ = _engine()
    n = eng.n_samples
    rng = np.random.RandomState(11)
    t = lambda k: np.arange(k) / 16000
    one = (0.1 * rng.randn(n)).astype(np.float32)
    # at one window: bit-identical to the chunk entry point
    assert torch.equal(eng.logmel_long(one[None]), eng.logmel(one[None], return_f32=True))
    worst = 0.0
    for L in (n + 1, n + 1234, 10 * 60 * 16000):
        pcm = (0.3 * np.sin(2 * np.pi * 440 * t(L)) + 0.05 * rng.randn(L)).astype(np.float32)[None]
        got = eng.logmel_long(pcm)
        assert got.shape == (1, 128, L // 160)
        ref = _ref_any(R, pcm)
        err = float(np.abs(got.double().cpu().numpy() - ref).max())
        print(f"\n[log-mel long] L={L}: max |d| {err:.2e}")
        worst = max(worst, err)
    lens = (n + 777, 3 * n + 160 * 7 + 33, n // 2)
    Lmax = max(lens)
    pcm = np.zeros((3, Lmax), dtype=np.float32)
    for i, L in enumerate(lens):
        pcm[i, :L] = (0.2 * rng.randn(L) * (1 + i)).astype(np.float32)
    got = eng.logmel_long(pcm).double().cpu().numpy()
    ref = _ref_any(R, pcm)
    err = float(np.abs(got - ref).max())
    print(f"[log-mel long] batch of {lens} padded to {Lmax}: max |d| {err:.2e} (bound {LOGMEL_ABS:.0e})")
    worst = max(worst, err)
    for i, L in enumerate(lens):  # the zero tail of a shorter row sits at its row's clamp floor
        tail = got[i, :, (L + 400) // 160:]
        assert tail.size == 0 or np.allclose(tail, tail.min()), i
    assert worst < LOGMEL_ABS


def _ref_any(R, pcm):
    """enc_ref.logmel for a sample count that is not a multiple of 160: the same frames, the reflect pad taken at the true end."""
    from thewhisper_b200.features import HOP, N_FFT, mel_filter_bank

    x = np.asarray(pcm, dtype=np.float64)
    frames = x.shape[1] // HOP
    xp = np.pad(x, ((0, 0), (N_FFT // 2, N_FFT // 2)), mode="reflect")
    nn = np.arange(N_FFT)
    win = 0.5 - 0.5 * np.cos(2 * np.pi * nn / N_FFT)
    out = np.empty((x.shape[0], 128, frames))
    bank = mel_filter_bank(128).astype(np.float64)
    for f0 in range(0, frames, 4096):  # (bounded memory at 10 minutes)
        idx = nn[None, :] + HOP * np.arange(f0, min(frames, f0 + 4096))[:, None]
        power = np.abs(np.fft.rfft(xp[:, idx] * win, axis=-1)) ** 2
        out[:, :, f0: f0 + idx.shape[0]] = np.log10(np.maximum(np.einsum("bfk,km->bmf", power, bank), 1e-10))
    top = out.max(axis=(1, 2), keepdims=True)
    return (np.maximum(out, top - 8.0) + 4.0) / 4.0


# ------------------------------------------------------------------------------------------------------------------
# key start
# ------------------------------------------------------------------------------------------------------------------
PLEN = 48


def _key_start_step(eng, k0, prefill):
    """Left-padded prompts of PLEN tokens with key starts k0, the forced positions by steps or by one prefill, NaN planted in the
    K/V rows below each start, then one step at position PLEN - 1.  -> dict of the engine's and the float64 restatement's values:
    logits (also with the start one lower: the ablation), the K/V rows the step appends, the last layer's cross-attention output,
    and the K/V rows of the last pad position k0 - 1 (a query with no key: written with a zero self-attention output)."""
    from oracle.step_ref import decoder_step
    from thewhisper_b200.engine import DecodeOptions

    Q = len(k0)
    d = eng.dims
    rng = np.random.RandomState(5)
    prompts = rng.randint(0, 50000, size=(Q, PLEN)).astype(np.int32)
    for q, k in enumerate(k0):
        prompts[q, :k] = 50257
    opts = DecodeOptions(eos_token=50257, pad_token=50257)
    eng.encode(Q)
    eng.decode_begin(prompts, Q, 1, opts, key_start=list(k0))
    if prefill:
        eng.decode_prefill(PLEN - 1)
    else:
        eng.decode_run(PLEN - 1)
    et, L, D, Qm, T = eng.dtype, d.dec_layers, d.d_model, eng.max_audios * eng.max_beams, d.max_target_positions
    sk = eng.buffer("self_k", et, (L, Qm, T, D)).clone()
    sv = eng.buffer("self_v", et, (L, Qm, T, D)).clone()
    ck = eng.buffer("cross_k", et, (L, eng.max_audios, d.n_heads, eng.S, 64))
    cv = eng.buffer("cross_v", et, (L, eng.max_audios, d.n_heads, eng.S, 64))
    nk, nv = sk.clone(), sv.clone()
    for q, k in enumerate(k0):
        nk[:, q, :k] = float("nan")
        nv[:, q, :k] = float("nan")
    eng.write_buffer("self_k", nk)
    eng.write_buffer("self_v", nv)
    eng.decode_run(1)
    pos = PLEN - 1
    batched = Q >= 3  # the batched step (BW_BATCH_MIN's default); below it the per-op step (a key start declines the persistent one)
    out = {"logits": eng.logits()[:Q].double(), "k_new": eng.buffer("self_k", et, (L, Qm, T, D))[:, :Q, pos],
           "v_new": eng.buffer("self_v", et, (L, Qm, T, D))[:, :Q, pos],
           "xattn": (eng.buffer("dba", et, (Qm, D)) if batched else eng.buffer("dattn", torch.float32, (Qm, D)))[:Q].double()}
    w64 = {k: v.double() for k, v in eng.weights.items()}
    ref = {"logits": [], "off": [], "k_new": [], "v_new": [], "xattn": [], "pad_k": [], "pad_v": [], "pad_k_ref": [], "pad_v_ref": []}
    step = lambda q, p, keep, rnd: decoder_step(w64, L, sk[:, q:q + 1], sv[:, q:q + 1], ck[:, q:q + 1], cv[:, q:q + 1], prompts[q:q + 1],
                                               p, self_keep=keep, round_operands=rnd)
    for q, k in enumerate(k0):
        r = step(q, pos, torch.arange(pos + 1) >= k, batched)
        ref["logits"].append(r["logits"][0])
        ref["k_new"].append(r["k_new"][:, 0])
        ref["v_new"].append(r["v_new"][:, 0])
        ref["xattn"].append(r["xattn"][0])
        ref["off"].append(step(q, pos, torch.arange(pos + 1) >= max(k - 1, 0), batched)["logits"][0])
        if k > 0:  # the pad query at k0 - 1 sees no key at all
            r = step(q, k - 1, torch.zeros(k, dtype=torch.bool), batched or prefill)
            ref["pad_k_ref"].append(r["k_new"][:, 0])
            ref["pad_v_ref"].append(r["v_new"][:, 0])
            ref["pad_k"].append(sk[:, q, k - 1])
            ref["pad_v"].append(sv[:, q, k - 1])
    return out, ref


@pytest.mark.parametrize("path,k0", [("perop", (1, 37)), ("perop", (0, PLEN - 1)), ("batched", (0, 1, 37)), ("batched", (PLEN - 1, 37, 1)),
                                     ("prefill", (1, 37)), ("prefill", (0, 1, PLEN - 1))])
def test_key_start_step_matches_reference(cuda, path, k0):
    from tests.test_decode_step_gpu import KV_ULPS, _ulps

    eng, _ = _engine(max_audios=3)
    got, ref = _key_start_step(eng, k0, prefill=(path == "prefill"))
    want, off = torch.stack(ref["logits"]), torch.stack(ref["off"])
    assert torch.isfinite(got["logits"]).all()
    scale = want.std(dim=-1, keepdim=True)
    err = float(((got["logits"] - want).abs() / scale).max())
    # fp32-activation bf16 bound of tests/test_decode_step_gpu.py; at Q = 3 (batched step) 2x the largest deviation measured here on an
    # NVIDIA H100 80GB HBM3 at 700 W (6.8e-3 of the logit std), below that file's batched bound so the off-by-one ablation lands outside
    batched = len(k0) >= 3
    tol = 1.5e-2 if batched else 4e-3
    print(f"\n[key start {path} {k0}] logits max |d| / std {err:.2e} (bound {tol:.0e})")
    assert err < tol
    moved = [float(((off[q] - want[q]).abs() / scale[q]).max()) for q in range(len(k0)) if k0[q] > 0]
    print(f"[key start {path} {k0}] start - 1 ablation moves the logits by {min(moved):.2e}")
    assert min(moved) > tol
    # the K/V rows this step appends, within the step tests' ulp bounds
    kv_bound = KV_ULPS["batched" if batched else "fp32"]
    for name in ("k_new", "v_new"):
        u = max(_ulps(got[name][:, q], ref[name][q], eng.dtype) for q in range(len(k0)))
        print(f"[key start {path} {k0}] appended {name} rows: {u:.2f} ulps (bound {kv_bound})")
        assert u <= kv_bound
    # the last layer's cross-attention output (downstream of every layer's masked self-attention)
    xw = torch.stack(ref["xattn"])
    xerr = float(((got["xattn"] - xw).abs() / xw.pow(2).mean(-1, keepdim=True).sqrt()).max())
    xtol = 5e-2 if batched else 5e-3  # (tests/test_decode_step_gpu.py's attention-output bounds, batched / fp32 bf16)
    print(f"[key start {path} {k0}] cross-attention output max |d| / rms {xerr:.2e} (bound {xtol:.0e})")
    assert xerr < xtol
    # a pad query (no key): its K/V rows in every layer are those of a zero self-attention output -- finite, and as restated
    pad_bound = KV_ULPS["batched" if (batched or path == "prefill") else "fp32"]
    for name in ("k", "v"):
        for g, w in zip(ref[f"pad_{name}"], ref[f"pad_{name}_ref"]):
            assert torch.isfinite(g).all()
            u = _ulps(g, w, eng.dtype)
            print(f"[key start {path} {k0}] pad-query {name} rows: {u:.2f} ulps (bound {pad_bound})")
            assert u <= pad_bound


def test_key_start_declines_persistent_step(cuda):
    from thewhisper_b200.engine import DecodeOptions

    eng, _ = _engine(max_audios=2)
    opts = DecodeOptions(eos_token=50257, pad_token=50257)
    prompts = np.full((2, 8), 220, dtype=np.int32)
    prompts[0, :3] = 50257
    eng.encode(2)
    for ks, most in ((None, 2), ([3, 0], None)):
        eng.decode_begin(prompts, 2, 1, opts, key_start=ks)
        before = eng.decode_kernel_launches()
        eng.decode_run(4)
        per_step = (eng.decode_kernel_launches() - before) / 4
        print(f"\n[key start {ks}] {per_step:.0f} kernels per step at Q = 2")
        if most is not None:
            assert per_step <= most
        else:
            assert per_step > 2
    eng.decode_begin(prompts, 2, 1, opts, key_start=[0, 0])  # every start 0: the unmasked path
    before = eng.decode_kernel_launches()
    eng.decode_run(1)
    assert eng.decode_kernel_launches() - before <= 2


def test_step_graph_cache_is_bounded(cuda, monkeypatch):
    """Every new begin_index captures a step graph; past BW_STEP_GRAPHS the least recently used one is evicted and recaptured when
    it is needed again, with the same results."""
    from thewhisper_b200.engine import DecodeOptions

    monkeypatch.setenv("BW_STEP_GRAPHS", "4")
    eng, _ = _engine(max_audios=1)
    opts = DecodeOptions(eos_token=50257, pad_token=50257)
    eng.encode(1)
    first = None
    for plen in (3, 4, 5, 6, 7, 8, 3):
        eng.greedy(np.full((1, plen), 220, dtype=np.int32), 1, opts, 4)
        if plen == 3:
            toks = eng.decode_read()[0][0, :7].tolist()
            assert first is None or toks == first
            first = toks
    g = eng.graph_stats()
    print(f"\n[step graphs] {g}")
    assert g["cached"] == 4 and g["captured"] == 7 and g["evicted"] == 3


# ------------------------------------------------------------------------------------------------------------------
# pipeline
# ------------------------------------------------------------------------------------------------------------------
class _Recorder:
    def __init__(self, pipe):
        self.records = []
        gen, eng = pipe.generator, pipe.engine
        os_, od = eng.set_mel, gen._decode
        self._mel = None

        def set_mel(m):
            self._mel = m.float().cpu().numpy()
            return os_(m)

        def _decode(prompts, A, opts, max_new, num_beams, **kw):
            out = od(prompts, A, opts, max_new, num_beams, **kw)
            self.records.append({"mel": self._mel[:A].copy(), "prompts": np.array(prompts), "gen": [np.asarray(g) for g in out[0]],
                                 "eos_seen": list(out[2]), "opts": opts, "max_new": max_new})
            return out

        eng.set_mel, gen._decode = set_mel, _decode


def _masked_teacher_forced(pad):
    """hf_ref.teacher_forced_logits with transformers' decoder_attention_mask of a left-padded decoder input."""

    @torch.no_grad()
    def tf(model, mel, ids):
        ids = list(ids)
        k0 = next((i for i, t in enumerate(ids) if t != pad), 0)
        mask = torch.ones(1, len(ids), dtype=torch.long)
        mask[0, :k0] = 0
        x = torch.from_numpy(mel)[None].to(model.dtype)
        return model(input_features=x, decoder_input_ids=torch.tensor([ids]), decoder_attention_mask=mask).logits[0].float().numpy()

    return tf


@pytest.mark.parametrize("name,mode", [("tiny10", "plain"), ("tiny10", "word"), ("tiny10", "cond"), ("tiny10", "int8"),
                                       ("small30", "plain"), ("small30", "cond")])
def test_longform_pipeline_replays_through_transformers(cuda, monkeypatch, name, mode):
    from oracle import hf_ref
    from tests.parity_utils import assert_oracle_greedy
    from thewhisper_b200 import synthetic as S
    from thewhisper_b200.nvidia import ASRPipeline

    meta = json.load(open(os.path.join(GOLD, f"model_{name}.json")))
    chunk = meta["chunk_s"]
    model = S.make_hf_model(meta["preset"], seed=0, layer_gain=meta["layer_gain"])
    pipe = ASRPipeline(model, feature_extractor=S.make_feature_extractor(chunk), tokenizer=S.make_tokenizer(), chunk_length_s=chunk,
                       device="cuda", batch_size=3, **({"decoder_weights": "int8"} if mode == "int8" else {}))
    rec = _Recorder(pipe)
    gk = {"num_beams": 1, "do_sample": False, "language": "en", "task": "transcribe", "max_new_tokens": 48,
          "condition_on_prev_tokens": mode == "cond"}
    audios = [S.synth_audio(sec * chunk / 10, seed=6000 + k) for k, sec in enumerate((31.0, 7.5, 22.2))]
    out = pipe(audios, chunk_length_s=0, batch_size=3, return_timestamps="word" if mode == "word" else True, generate_kwargs=gk)
    assert len(out) == 3 and all(isinstance(o["text"], str) for o in out)
    assert len(rec.records) >= 2
    om = S.make_hf_model(meta["preset"], seed=0, layer_gain=meta["layer_gain"])
    if mode == "int8":
        from tests.test_pipeline_int8_gpu import _dequantised

        om = _dequantised(om)
    if chunk < 30:
        hf_ref.interpolate_positions(om, chunk)
    if mode == "cond":  # conditioned windows start with <|startofprev|> or, left-padded, with pad (small30 reaches both)
        assert any(np.isin(r["prompts"][:, 0], (50257, 50362)).any() for r in rec.records), "no conditioned window"
        if name == "small30":
            assert any((r["prompts"][:, 0] == 50257).any() for r in rec.records), "no left-padded window"
    monkeypatch.setattr(hf_ref, "teacher_forced_logits", _masked_teacher_forced(50257))
    n_tok = sum(len(g) for r in rec.records for g in r["gen"])
    near = assert_oracle_greedy(rec.records, om, max_near_ties=max(6, n_tok // 20))  # (every other token is the oracle's arg-max)
    print(f"\n[long form {name} {mode}] {len(rec.records)} decode calls, {n_tok} tokens, {near} near ties")


def test_longform_beam5_fp16_matches_transformers(cuda):
    from oracle import hf_ref
    from tests.test_pipeline_gpu import _check_text
    from thewhisper_b200 import synthetic as S
    from thewhisper_b200.nvidia import ASRPipeline

    meta = json.load(open(os.path.join(GOLD, "model_tiny10.json")))
    chunk = meta["chunk_s"]
    model = S.make_hf_model(meta["preset"], seed=0, layer_gain=meta["layer_gain"])
    pipe = ASRPipeline(model, feature_extractor=S.make_feature_extractor(chunk), tokenizer=S.make_tokenizer(), chunk_length_s=chunk,
                       device="cuda", torch_dtype=torch.float16, batch_size=1)
    ref = hf_ref.make_ref_pipeline(S.make_hf_model(meta["preset"], seed=0, layer_gain=meta["layer_gain"]), S.make_feature_extractor(chunk),
                                   S.make_tokenizer(), chunk_length_s=chunk)
    gk = {"num_beams": 5, "do_sample": False, "language": "en", "task": "transcribe", "max_new_tokens": 32}
    audio = S.synth_audio(33.0, seed=6100)
    got = pipe(audio.copy(), chunk_length_s=0, return_timestamps=True, generate_kwargs=dict(gk))
    want = ref(audio.copy(), chunk_length_s=0, return_timestamps=True, generate_kwargs=dict(gk))
    print(f"\n[long form beam5 fp16] ours {got['text'][:80]!r}\n                      ref  {want['text'][:80]!r}")
    _check_text(got["text"], want["text"])


def test_longform_large_v3_ten_minutes(cuda):
    """Large-v3 shapes, random weights, one 10-minute input: the per-call feature buffer and the seek loop hold."""
    from thewhisper_b200 import synthetic as S
    from thewhisper_b200.nvidia import ASRPipeline

    model = S.make_hf_model("large-v3", seed=0)
    pipe = ASRPipeline(model, feature_extractor=S.make_feature_extractor(30), tokenizer=S.make_tokenizer(), chunk_length_s=30,
                       device="cuda", torch_dtype=torch.float16, batch_size=1)
    audio = S.synth_audio(600.0, seed=6200)
    out = pipe(audio, chunk_length_s=0, return_timestamps=True,
               generate_kwargs={"num_beams": 1, "language": "en", "task": "transcribe", "max_new_tokens": 24})
    st = pipe.engine.stats
    print(f"\n[long form large-v3 10 min] {st['chunks_encoded']} windows encoded, {st['decode_steps']} decoder steps, "
          f"peak {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")
    assert isinstance(out["text"], str) and st["chunks_encoded"] >= 20
