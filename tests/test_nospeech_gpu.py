"""No-speech skipping on the GPU:
  * step level: the scores select_kernel writes -- lp (processed log-prob of the selected token), lmass (allowed mass) and nsp (the
    no-speech probability) -- against float64 on the planted exact logits of tests/test_select_gpu.py, on the persistent step (which
    then runs select_kernel after it), the per-op and the batched step, bf16 / fp16, 16-bit / int8 weights, and beam search at
    (A, G) = (3, 2), (2, 5), (1, 8).  nsp is checked at a forced position and at begin_index - 1.  Three bugs, restated in float64,
    must land outside the bound: the lse over the raw instead of the allowed logits, nsp read one position late, and the text mass
    kept when a timestamp is forced;
  * path and invariance: the persistent step declines its fused select only with scores on; tokens and logits are byte-identical with
    scores on and off; the no-speech position is not part of the step graph (a conditioned window captures what it captured before);
  * pipeline: long-form calls with the thresholds on tiny10, greedy / word / int8 / conditioned, every window's skip decision and
    statistics replayed through transformers (tie-aware), and beam 5 in fp16 against the live transformers pipeline;
  * large-v3 shape: a 10-minute input with silent stretches finishes and skips windows."""
import json
import os

import numpy as np
import pytest
import torch

from tests import test_decode_step_gpu as T
from tests import test_select_cases_cpu as C
from tests import test_select_gpu as SG
from tests.conftest import GOLD
from tests.test_nospeech_cpu import NS_FACTOR, _audio, _lse, _scale_nospeech

pytestmark = pytest.mark.gpu

NSTOK = 50363  # <|nospeech|> of the synthetic vocabulary
# |device - float64| of lp and lmass (fp32, __expf sums over 51866 logits) and the relative error of nsp.  The bounds are about
# 2.5x the maxima measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit, the same in every cell (printed by each cell).
LP_TOL = 8.5e-6   # measured 3.3e-6 (lmass), 2.5e-6 (lp)
NSP_RTOL = 6.5e-6  # measured 2.5e-6


def _proc(case, row, r0):
    o = case.opts()
    from oracle import whisper_ref as R

    return R.process_logits(row, case.seq(r0), case.begin, suppress=o.suppress_tokens, begin_suppress=o.begin_suppress_tokens,
                            ts_rules=o.timestamp_rules, ts_begin=o.timestamp_begin, no_ts=o.no_timestamps_token, eos=o.eos_token,
                            max_initial_ts=o.max_initial_timestamp_index if o.max_initial_timestamp_index >= 0 else None, details=True)


def _step(eng, w, env, case, A, G, st):
    """One step of the case with scores on; compares lp / lmass with float64, and nsp when the step is the first generated one
    (the no-speech position at begin_index - 1, as with a single init token); otherwise nsp must stay unwritten."""
    D = w["dec.lnf.g"].shape[0]
    i = (SG.GREEDY + SG.BEAM).index(case)
    w["dec.lnf.b"].copy_(torch.from_numpy(SG.PLANTED[D][1][i]).float().cuda())
    row = SG.PLANTED[D][2][i]
    Q = A * G
    Qm = eng.max_audios * eng.max_beams
    spec = case.row_spec(Q)
    with T._env(env):
        eng.decode_begin(np.array([case.prompt()] * Q, dtype=np.int32), A, G, case.opts(), begin_index=case.begin)
        first = case.cur_len == case.begin
        eng.decode_scores_enable(case.cur_len - 1 if first else -1, NSTOK)
    tok = np.full((Qm, T.TMAX), case.pad, dtype=np.int32)
    for q in range(Q):
        s = case.seq(q % len(case.rows))
        tok[q, :len(s)] = s
    fin = np.zeros(Qm, dtype=np.int32)
    if not case.beam:
        fin[:Q] = [int(f) for _, f in spec]
    for name, t in (("tokens", tok), ("finished", fin), ("pos", np.array([case.cur_len - 1], dtype=np.int32))):
        eng.write_buffer(name, torch.from_numpy(t).cuda())
    torch.cuda.synchronize()
    k0 = eng.decode_kernel_launches()
    if case.beam:
        eng.decode_beam_step(np.array([r for _, r in spec], dtype=np.float32))
    else:
        eng.decode_run(1)
    torch.cuda.synchronize()
    kernels = eng.decode_kernel_launches() - k0
    assert torch.equal(eng.logits().double(), torch.from_numpy(row)[None].cuda().expand(Q, C.V)), case.name
    lp, lmass, nsp = eng.decode_scores()
    ref = SG._reference(case, Q, G)
    raw_lse = _lse(row)
    ns_ref = float(np.exp(row[NSTOK] - raw_lse))
    for q in range(Q):
        r0 = q % len(case.rows)
        s, pre, _ = _proc(case, row, r0)
        allowed = np.isfinite(s)
        if not allowed.any():
            continue
        a_lse = _lse(row[allowed])
        lm_ref = a_lse - raw_lse
        st["lmass"] = max(st["lmass"], abs(float(lmass[q, case.cur_len]) - lm_ref))
        pre_ok = np.isfinite(pre)
        st["abl_textmass"] = max(st["abl_textmass"], abs((_lse(row[pre_ok]) - raw_lse) - lm_ref))
        if not case.beam:
            t, _, _ = ref[q]
            lp_ref = 0.0 if spec[q][1] else float(row[t]) - a_lse
            st["lp"] = max(st["lp"], abs(float(lp[q, case.cur_len]) - lp_ref))
            if not spec[q][1]:
                st["abl_rawlse"] = max(st["abl_rawlse"], abs((float(row[t]) - raw_lse) - lp_ref))
        if first:
            st["nsp"] = max(st["nsp"], abs(float(nsp[q]) - ns_ref) / ns_ref)
        else:
            assert nsp[q] == 0.0, (case.name, q, nsp[q])
        st["rows"] += 1
    st["first_step"] += int(first)
    return kernels


def _forced_nsp(eng, w, env, st):
    """nsp at a forced position (the input before begin_index, as with a prompt or history): the step consuming position 1 writes it
    from its logits; the next step, over other logits, leaves it (and the tokens) alone.  The ablation reads the next position's."""
    D = w["dec.lnf.g"].shape[0]
    case = next(c for c in SG.GREEDY if c.begin == 4)
    x, y = 0, len(SG.GREEDY) - 1
    with T._env(env):
        eng.decode_begin(np.array([case.prompt()], dtype=np.int32), 1, 1, case.opts(), begin_index=4)
        eng.decode_scores_enable(1, NSTOK)
    eng.write_buffer("pos", torch.tensor([1], dtype=torch.int32, device="cuda"))
    toks0, _, _ = eng.decode_read()
    for i in (x, y):
        w["dec.lnf.b"].copy_(torch.from_numpy(SG.PLANTED[D][1][i]).float().cuda())
        eng.decode_run(1)
    torch.cuda.synchronize()
    _, _, nsp = eng.decode_scores()
    toks1, _, pos = eng.decode_read()
    assert pos == 3 and np.array_equal(toks0, toks1)
    want = float(np.exp(SG.PLANTED[D][2][x][NSTOK] - _lse(SG.PLANTED[D][2][x])))
    late = float(np.exp(SG.PLANTED[D][2][y][NSTOK] - _lse(SG.PLANTED[D][2][y])))
    st["nsp"] = max(st["nsp"], abs(float(nsp[0]) - want) / want)
    st["abl_late"] = max(st["abl_late"], abs(late - want) / want)
    st["forced"] += 1


def _stats():
    return dict(rows=0, lp=0.0, lmass=0.0, nsp=0.0, abl_rawlse=0.0, abl_textmass=0.0, abl_late=0.0, first_step=0, forced=0)


def _report(label, st):
    print(f"\n[{label}] {st['rows']} rows ({st['first_step']} first steps, {st['forced']} forced): max |lp err| {st['lp']:.2e}, "
          f"|lmass err| {st['lmass']:.2e} (bound {LP_TOL:.1e}), nsp rel err {st['nsp']:.2e} (bound {NSP_RTOL:.1e}); ablations "
          f"raw lse {st['abl_rawlse']:.2e}, text mass under forcing {st['abl_textmass']:.2e}, nsp one late {st['abl_late']:.2e}")
    assert st["lp"] <= LP_TOL and st["lmass"] <= LP_TOL and st["nsp"] <= NSP_RTOL, st


GREEDY_CELLS = [(t, w8, p) for t in ("bf16", "fp16") for w8 in (False, True) for p in ("mega", "perop", "batched")]


@pytest.mark.parametrize("tname,int8,path", GREEDY_CELLS, ids=[f"{t}-{'int8' if w8 else '16bit'}-{p}" for t, w8, p in GREEDY_CELLS])
def test_step_scores_greedy(cuda, tname, int8, path):
    A = SG._greedy_A(path)
    env = SG.PATHS[path]
    eng, w = SG.make_engine(SG.DIMS["tiny"], tname, int8, env, A, 1)
    try:
        st = _stats()
        for case in SG.GREEDY:
            k = _step(eng, w, env, case, A, 1, st)
            if path == "mega":  # with scores on, the persistent step leaves selection to select_kernel, timestamp rules or not
                assert k == 2, (case.name, k)
            else:
                assert k > 2, (path, case.name, k)
        _forced_nsp(eng, w, env, st)
    finally:
        eng.close()
    _report(f"scores greedy {tname} {'int8' if int8 else '16-bit'} {path} A={A}", st)
    assert st["first_step"] > 0 and st["forced"] > 0
    # the three bugs, restated in float64, land outside the bound
    assert st["abl_rawlse"] > LP_TOL and st["abl_textmass"] > LP_TOL and st["abl_late"] > NSP_RTOL, st


BEAM_CELLS = [(t, p) for t in ("bf16", "fp16") for p in ("perop", "batched")]


@pytest.mark.parametrize("tname,path", BEAM_CELLS, ids=[f"{t}-{p}" for t, p in BEAM_CELLS])
def test_step_scores_beam(cuda, tname, path):
    env = SG.PATHS[path]
    eng, w = SG.make_engine(SG.DIMS["tiny"], tname, False, env, 3, 8)
    try:
        for A, G in SG.BEAM_AG:
            st = _stats()
            for case in SG.BEAM:
                assert _step(eng, w, env, case, A, G, st) > 2
            _report(f"scores beam {tname} {path} A={A} G={G}", st)
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------------------------
# path and invariance
# ------------------------------------------------------------------------------------------------------------------
def _tiny_engine(A=3, G=1, dtype=torch.bfloat16, decoder_weights=None):
    from thewhisper_b200 import synthetic as S
    from thewhisper_b200.engine import ModelDims, WhisperEngine

    model = S.make_hf_model("tiny-test", seed=0, layer_gain=8.0)
    eng = WhisperEngine(model.state_dict(), ModelDims.from_hf_config(model.config), chunk_length_s=10, max_audios=A, max_beams=G,
                        dtype=dtype, decoder_weights=decoder_weights)
    pcm = np.stack([_audio(10.0, 900 + a) for a in range(A)])
    eng.logmel(pcm)
    eng.encode(A)
    return eng, model


def _steps(eng, A, opts, scores, n=24):
    from thewhisper_b200 import synthetic as S

    prompts = np.array([[S.SOT, S.LANG_EN, S.TRANSCRIBE] + ([] if opts.timestamp_rules else [S.NOTIMESTAMPS])] * A, dtype=np.int32)
    eng.decode_begin(prompts, A, 1, opts)
    if scores:
        eng.decode_scores_enable(0, NSTOK)
    eng.decode_run(prompts.shape[1] - 1)
    lgs = []
    k0 = eng.decode_kernel_launches()
    for _ in range(n):
        eng.decode_run(1)
        lgs.append(eng.logits().cpu().numpy().copy())
    per_step = (eng.decode_kernel_launches() - k0) / n
    toks, fin, _ = eng.decode_read()
    return toks, np.stack(lgs), per_step


@pytest.mark.parametrize("path", ["mega", "perop", "batched"])
def test_tokens_and_logits_identical_with_scores(cuda, path):
    from thewhisper_b200 import synthetic as S
    from thewhisper_b200.engine import DecodeOptions

    env = SG.PATHS[path]
    A = SG._greedy_A(path)
    with T._env(env):
        eng, model = _tiny_engine(A)
    g = model.generation_config
    try:
        for ts in (False, True):
            opts = DecodeOptions(eos_token=S.EOS, pad_token=S.EOS, suppress_tokens=list(g.suppress_tokens),
                                 begin_suppress_tokens=list(g.begin_suppress_tokens), timestamp_rules=ts,
                                 max_initial_timestamp_index=50 if ts else -1)
            with T._env(env):
                t0, l0, k_off = _steps(eng, A, opts, False)
                t1, l1, k_on = _steps(eng, A, opts, True)
            assert np.array_equal(t0, t1) and l0.tobytes() == l1.tobytes(), (path, ts)
            if path == "mega":
                assert (k_off, k_on) == ((2, 2) if ts else (1, 2)), (ts, k_off, k_on)
            print(f"\n[invariance {path} ts={ts}] kernels per step {k_off:g} -> {k_on:g}, tokens and logits identical")
    finally:
        eng.close()


def test_nospeech_position_is_not_in_the_graph_key(cuda):
    """Conditioned windows: one capture per begin_index, whatever the no-speech position, with scores as without."""
    from thewhisper_b200 import synthetic as S
    from thewhisper_b200.engine import DecodeOptions

    eng, model = _tiny_engine(2)
    g = model.generation_config
    opts = DecodeOptions(eos_token=S.EOS, pad_token=S.EOS, suppress_tokens=list(g.suppress_tokens),
                         begin_suppress_tokens=list(g.begin_suppress_tokens), timestamp_rules=True, max_initial_timestamp_index=50)
    init = [S.SOT, S.LANG_EN, S.TRANSCRIBE]
    try:
        counts = {}
        for scores in (False, True):
            c0 = eng.graph_stats()["captured"]
            for hist in (4, 5, 6):
                prompts = np.array([[S.STARTOFPREV] + [300 + i for i in range(hist)] + init] * 2, dtype=np.int32)
                for ns in ((1 + hist, 2 + hist) if scores else (None,)):
                    eng.decode_begin(prompts, 2, 1, opts, key_start=[0, 2])
                    if ns is not None:
                        eng.decode_scores_enable(ns, NSTOK)
                    eng.teacher_force(prompts.shape[1], True, ns)
                    eng.decode_run(3)
            counts[scores] = eng.graph_stats()["captured"] - c0
        print(f"\n[graph key] captures for 3 conditioned begin indices: {counts[False]} without scores, {counts[True]} with "
              f"scores at 2 no-speech positions each")
        assert counts == {False: 3, True: 3}, counts
        with pytest.raises(Exception, match="before it"):  # enabling after a step is refused
            eng.decode_scores_enable(0, NSTOK)
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------------------------
# pipeline
# ------------------------------------------------------------------------------------------------------------------
TH = {"no_speech_threshold": 0.5, "logprob_threshold": -8.3, "temperature": 0.0}  # (see tests/test_nospeech_cpu.py)
# a window whose avg_logprob lies within LP_MARGIN of logprob_threshold, or whose no_speech_prob within NS_MARGIN of
# no_speech_threshold, is counted and printed, not compared: 16-bit decoder arithmetic moves both statistics
LP_MARGIN, NS_MARGIN = 0.1, 0.05


class _Windows:
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
            self.records.append({"mel": self._mel[:A].copy(), "prompts": np.array(prompts), "gen": [np.asarray(x) for x in out[0]],
                                 "eos_seen": list(out[2]), "opts": opts, "max_new": max_new, "n_init": kw.get("n_init"),
                                 "scores": gen._window_scores})
            return out

        eng.set_mel, gen._decode = set_mel, _decode


@torch.no_grad()
def _replay(rec, om, pad, eos):
    """transformers' avg_logprob and no_speech_prob of every row of a recorded greedy window: its decoder over the window's input
    and tokens (decoder attention mask for the left pads), the processors restated by oracle/whisper_ref.process_logits."""
    from oracle import whisper_ref as R

    o = rec["opts"]
    out = []
    for a, gen in enumerate(rec["gen"]):
        prompt = rec["prompts"][a].tolist()
        toks = list(gen) + ([eos] if rec["eos_seen"][a] else [])
        ids = prompt + toks
        k0 = next((i for i, t in enumerate(ids) if t != pad), 0)
        mask = torch.ones(1, len(ids), dtype=torch.long)
        mask[0, :k0] = 0
        x = torch.from_numpy(rec["mel"][a])[None].to(om.dtype)
        lg = om(input_features=x, decoder_input_ids=torch.tensor([ids]), decoder_attention_mask=mask).logits[0].double().numpy()
        plen = len(prompt)
        tot = 0.0
        for i, t in enumerate(toks):
            raw = lg[plen - 1 + i]
            s = R.process_logits(raw.astype(np.float32), ids[:plen + i], plen, suppress=o.suppress_tokens,
                                 begin_suppress=o.begin_suppress_tokens, ts_rules=o.timestamp_rules, ts_begin=o.timestamp_begin,
                                 no_ts=o.no_timestamps_token, eos=o.eos_token,
                                 max_initial_ts=o.max_initial_timestamp_index if o.max_initial_timestamp_index >= 0 else None)
            tot += float(raw[t]) - _lse(raw[np.isfinite(s)])
        row = lg[plen - rec["n_init"]]
        out.append((tot / len(toks), float(np.exp(row[NSTOK] - _lse(row)))))
    return out


@pytest.mark.parametrize("mode", ["plain", "word", "int8", "cond"])
def test_pipeline_skip_decisions_replay_through_transformers(cuda, monkeypatch, mode):
    from oracle import hf_ref
    from tests.parity_utils import assert_oracle_greedy
    from tests.test_longform_gpu import _masked_teacher_forced
    from thewhisper_b200 import synthetic as S
    from thewhisper_b200.nvidia import ASRPipeline

    meta = json.load(open(os.path.join(GOLD, "model_tiny10.json")))
    chunk = meta["chunk_s"]
    edit = _scale_nospeech(NS_FACTOR)
    model = S.make_hf_model(meta["preset"], seed=0, layer_gain=meta["layer_gain"])
    edit(model)
    pipe = ASRPipeline(model, feature_extractor=S.make_feature_extractor(chunk), tokenizer=S.make_tokenizer(), chunk_length_s=chunk,
                       device="cuda", batch_size=3, **({"decoder_weights": "int8"} if mode == "int8" else {}))
    rec = _Windows(pipe)
    gk = dict({"num_beams": 1, "language": "en", "task": "transcribe", "max_new_tokens": 24, "condition_on_prev_tokens": mode == "cond"}, **TH)
    audios = [_audio(sec, 3000 + k) for k, sec in enumerate((37.3, 25.0, 58.6))]
    out = pipe(audios, chunk_length_s=0, batch_size=3, return_timestamps="word" if mode == "word" else True, generate_kwargs=gk)
    assert len(out) == 3
    om = S.make_hf_model(meta["preset"], seed=0, layer_gain=meta["layer_gain"])
    edit(om)
    if mode == "int8":
        from tests.test_pipeline_int8_gpu import _dequantised

        om = _dequantised(om)
    hf_ref.interpolate_positions(om, chunk)
    g = om.generation_config
    decided = {"skip": 0, "keep": 0, "near": 0}
    for r in rec.records:
        avg, ns = r["scores"]
        for a, (ra, rn) in enumerate(_replay(r, om, g.pad_token_id, g.eos_token_id)):
            ours = bool(avg[a] < TH["logprob_threshold"] and ns[a] > TH["no_speech_threshold"])
            if abs(ra - TH["logprob_threshold"]) < LP_MARGIN or abs(rn - TH["no_speech_threshold"]) < NS_MARGIN:
                decided["near"] += 1
                print(f"  near a threshold: avg_logprob {avg[a]:.4f} (transformers {ra:.4f}), no_speech_prob {ns[a]:.4f} ({rn:.4f})")
                continue
            want = bool(ra < TH["logprob_threshold"] and rn > TH["no_speech_threshold"])
            assert ours == want, (a, avg[a], ra, ns[a], rn)
            decided["skip" if want else "keep"] += 1
    monkeypatch.setattr(hf_ref, "teacher_forced_logits", _masked_teacher_forced(g.pad_token_id))
    n_tok = sum(len(x) for r in rec.records for x in r["gen"])
    near = assert_oracle_greedy(rec.records, om, max_near_ties=max(6, n_tok // 20))
    st = pipe.generator.window_stats
    print(f"\n[no-speech {mode}] {len(rec.records)} windows decoded, decisions {decided}, {near} near token ties, window stats {st}, "
          f"forced steps added by the <|startoftranscript|> split: {pipe.engine.stats['sot_split_steps']}")
    assert decided["skip"] > 0 and decided["keep"] > 0, decided


def test_beam5_fp16_matches_transformers(cuda):
    from oracle import hf_ref
    from tests.test_pipeline_gpu import _check_text
    from thewhisper_b200 import synthetic as S
    from thewhisper_b200.nvidia import ASRPipeline

    meta = json.load(open(os.path.join(GOLD, "model_tiny10.json")))
    chunk = meta["chunk_s"]
    edit = _scale_nospeech(NS_FACTOR)
    model = S.make_hf_model(meta["preset"], seed=0, layer_gain=meta["layer_gain"])
    edit(model)
    pipe = ASRPipeline(model, feature_extractor=S.make_feature_extractor(chunk), tokenizer=S.make_tokenizer(), chunk_length_s=chunk,
                       device="cuda", torch_dtype=torch.float16, batch_size=1)
    rm = S.make_hf_model(meta["preset"], seed=0, layer_gain=meta["layer_gain"])
    edit(rm)
    ref = hf_ref.make_ref_pipeline(rm, S.make_feature_extractor(chunk), S.make_tokenizer(), chunk_length_s=chunk)
    gk = dict({"num_beams": 5, "language": "en", "task": "transcribe", "max_new_tokens": 24}, **TH)
    audio = _audio(37.3, 3001)
    got = pipe(audio.copy(), chunk_length_s=0, return_timestamps=True, generate_kwargs=dict(gk))
    want = ref(audio.copy(), chunk_length_s=0, return_timestamps=True, generate_kwargs=dict(gk))
    print(f"\n[no-speech beam5 fp16] skipped {pipe.generator.window_stats['skipped']} of {pipe.generator.window_stats['windows']} "
          f"windows\n  ours {got['text'][:80]!r}\n  ref  {want['text'][:80]!r}")
    _check_text(got["text"], want["text"])


def test_large_v3_ten_minutes_skips_silence(cuda):
    """Large-v3 shapes, random weights, 10 minutes with zeroed stretches: the call finishes and skips windows.  Random weights
    model no speech, so the thresholds here (avg_logprob below 0, no_speech_prob above 0) skip every window."""
    from thewhisper_b200 import synthetic as S
    from thewhisper_b200.nvidia import ASRPipeline

    model = S.make_hf_model("large-v3", seed=0)
    pipe = ASRPipeline(model, feature_extractor=S.make_feature_extractor(30), tokenizer=S.make_tokenizer(), chunk_length_s=30,
                       device="cuda", torch_dtype=torch.float16, batch_size=1)
    audio = S.synth_audio(600.0, seed=6200)
    for k in range(0, 600, 120):
        audio[(k + 30) * 16000:(k + 90) * 16000] = 0.0
    out = pipe(audio, chunk_length_s=0, return_timestamps=True,
               generate_kwargs={"num_beams": 1, "language": "en", "task": "transcribe", "max_new_tokens": 24, "temperature": 0.0,
                                "no_speech_threshold": 0.0, "logprob_threshold": 0.0})
    st, ws = pipe.engine.stats, pipe.generator.window_stats
    print(f"\n[no-speech large-v3 10 min] {ws['windows']} windows, {ws['skipped']} skipped, {st['decode_steps']} decoder steps")
    assert isinstance(out["text"], str) and ws["skipped"] > 0 and ws["windows"] >= 20
