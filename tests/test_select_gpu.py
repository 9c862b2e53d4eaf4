"""Token selection of the real decoder step, on every step path, against the float64 references of
tests/test_select_cases_cpu.py: greedy argmax with suppression, begin suppression, the Whisper timestamp rules, ties,
pad / finished, and the beam candidate lists.

The cases plant exact logits through the final LayerNorm (g = 0, b = beta) and the tied embedding (see
tests/test_select_cases_cpu.py); the engine binds dec.lnf.b by pointer, so a case switches its logit row by writing beta
into that tensor in place.  Each case then writes the token history, `finished` and `pos` (as tests/test_decode_step_gpu.py
does), runs one step, checks that the logits are the planted values bit for bit, and compares the selection exactly.
The decoder layers are random; they cannot reach the logits.
"""
import numpy as np
import pytest
import torch

from tests import test_decode_step_gpu as T
from tests import test_select_cases_cpu as C

pytestmark = pytest.mark.gpu

TMAX, V = T.TMAX, C.V
DIMS = {"tiny": (128, 2, 512, 2, 500), "large": (1280, 20, 5120, 2, 1500)}  # (D, H, ffn, decoder layers, S); large-v3 width
PATHS = {
    "mega": {},                                           # fused greedy select in the persistent kernel (no timestamp rules)
    "mega-nofuse": {"BW_NO_FUSED_SELECT": "1"},           # persistent step + select_kernel
    "perop": {"BW_NO_MEGA": "1", "BW_BATCH_MIN": "1000"},
    "batched": {"BW_NO_MEGA": "1", "BW_BATCH_MIN": "1"},
}
DTYPES = T.DTYPES
GREEDY = C.greedy_cases()
BEAM = C.beam_cases()
PLANTED = {D: C.plant(GREEDY + BEAM, D) for D in (128, 1280)}
BEAM_AG = [(3, 2), (2, 5), (1, 8)]
# Beam scores: |device - float64 reference| over every finite candidate.  The device computes logit - lse + run in fp32 with
# an __expf sum over the 51866 raw logits.  Measured maximum 2.37e-6 on an NVIDIA H100 80GB HBM3 at a 700 W power limit (the
# same in every beam cell); the bound is about 2.5x that.
SCORE_TOL = 6e-6


def _greedy_A(path):
    return 2 if path.startswith("mega") else 3  # the persistent step runs at most two sequences


def make_engine(dims, tname, int8, env, A, G):
    """An engine whose tied embedding holds the planted columns, final LayerNorm g = 0, b = 0 (set per case)."""
    from thewhisper_b200.engine import ModelDims, WhisperEngine, quantize_rows

    D, H, ffn, L, S = dims
    E = torch.from_numpy(PLANTED[D][0]).float().cuda()
    if int8:
        w = T.make_weights(dims, torch.float32)
        for n in list(w):
            if n.startswith("dec.") and n.split(".")[-1] in ("wqkv", "wo", "xwq", "xwo", "w1", "w2"):
                w[n], w[n + ".scale"] = quantize_rows(w[n])
            elif w[n].dim() == 2 and n not in ("enc.pos", "dec.pos"):
                w[n] = w[n].to(DTYPES[tname])
        w["dec.embed"] = torch.round(E * 16).to(torch.int8)
        w["dec.embed.scale"] = torch.full((V,), 1 / 16, device="cuda")  # codes * 2^-4 is E exactly
    else:
        w = T.make_weights(dims, DTYPES[tname])
        w["dec.embed"] = E.to(DTYPES[tname])
    w["dec.lnf.g"] = torch.zeros(D, device="cuda")
    w["dec.lnf.b"] = torch.zeros(D, device="cuda")
    with T._env(env):
        eng = WhisperEngine(None, ModelDims(D, H, ffn, 0, L, 128, V, S, TMAX), chunk_length_s=S * 30 / 1500, max_audios=A,
                            max_beams=G, weights=w)
    dt = DTYPES[tname]
    Qm = A * G
    for name, shape in (("self_k", (L, Qm, TMAX, D)), ("self_v", (L, Qm, TMAX, D)), ("cross_k", (L, A, H, S, 64)),
                        ("cross_v", (L, A, H, S, 64))):
        eng.write_buffer(name, torch.zeros(shape, dtype=dt, device="cuda"))  # finite state: the LayerNorm input stays finite
    return eng, w


_REF = {}


def _reference(case, Q, G):
    key = (case.name, Q, G)
    if key not in _REF:
        _REF[key] = C.reference(case, C.plant_row(case), Q, G)
    return _REF[key]


def run_case(eng, w, env, case, A, G, stats):
    """One step of `case` with A audios x G beams; checks logits, then tokens / finished / pos or the candidate lists."""
    D = w["dec.lnf.g"].shape[0]
    i = (GREEDY + BEAM).index(case)
    beta = torch.from_numpy(PLANTED[D][1][i]).float().cuda()
    row = torch.from_numpy(PLANTED[D][2][i]).cuda()
    w["dec.lnf.b"].copy_(beta)
    Q = A * G
    Qm = eng.max_audios * eng.max_beams
    spec = case.row_spec(Q)
    with T._env(env):
        eng.decode_begin(np.array([case.prompt()] * Q, dtype=np.int32), A, G, case.opts(), begin_index=case.begin)
    tok = np.full((Qm, TMAX), case.pad, dtype=np.int32)
    for q in range(Q):
        s = case.seq(q % len(case.rows))
        tok[q, :len(s)] = s
    fin = np.zeros(Qm, dtype=np.int32)
    if not case.beam:
        fin[:Q] = [int(f) for _, f in spec]
    pos = case.cur_len - 1
    for name, t in (("tokens", tok), ("finished", fin), ("pos", np.array([pos], dtype=np.int32))):
        eng.write_buffer(name, torch.from_numpy(t).cuda())
    torch.cuda.synchronize()
    k0 = eng.decode_kernel_launches()
    if case.beam:
        cs, ct = eng.decode_beam_step(np.array([r for _, r in spec], dtype=np.float32))
    else:
        eng.decode_run(1)
    torch.cuda.synchronize()
    kernels = eng.decode_kernel_launches() - k0
    lg = eng.logits().double()
    assert torch.equal(lg, row[None].expand(Q, V)), (case.name, "logits are not the planted values")
    ref = _reference(case, Q, G)
    margins = [abs(m) for *_, m in ref if np.isfinite(m) and m != 0]  # (margin 0: the exact tie, counted apart)
    if margins:
        stats["margin"] = min(stats["margin"], min(margins))
    stats["ties"] += sum(m == 0 for *_, m in ref)
    stats["cases"] += 1
    if case.beam:
        for q in range(Q):
            scores, ids, _ = ref[q]
            assert np.array_equal(ct[q], ids), (case.name, q, ct[q].tolist(), ids.tolist())
            f = ids >= 0
            assert np.all(np.isneginf(cs[q][~f])), (case.name, q, cs[q])
            err = float(np.abs(cs[q][f].astype(np.float64) - scores[f]).max()) if f.any() else 0.0
            stats["score"] = max(stats["score"], err)
            assert err <= SCORE_TOL, (case.name, q, err)
        return kernels
    toks, fin_after, pos_after = eng.decode_read()
    want = tok[:Q].copy()
    for q, (t, f, _) in enumerate(ref):
        want[q, case.cur_len] = t
    assert pos_after == case.cur_len, (case.name, pos_after)
    assert np.array_equal(toks[:, case.cur_len], want[:, case.cur_len]), (case.name, toks[:, case.cur_len], want[:, case.cur_len])
    assert np.array_equal(toks, want), (case.name, "a token other than the step's changed")
    assert np.array_equal(fin_after, [int(f) for _, f, _ in ref]), (case.name, fin_after, [f for _, f, _ in ref])
    return kernels


def _stats():
    return dict(cases=0, margin=float("inf"), ties=0, score=0.0)


def _report(label, st):
    line = f"[{label}] {st['cases']} cases, smallest rule margin decided {st['margin']:.3g} (+ {st['ties']} rows at an exact tie)"
    if st["score"] or "beam" in label:
        line += f", worst beam score error {st['score']:.2e} (bound {SCORE_TOL:.0e})"
    print("\n" + line)


def run_greedy(eng, w, env, path, A, stats):
    for case in GREEDY:
        k = run_case(eng, w, env, case, A, 1, stats)
        if path == "mega":  # one kernel per step: the fused select; two: the persistent step + select_kernel
            assert k == (2 if case.ts else 1), (case.name, k)
        elif path == "mega-nofuse":
            assert k == 2, (case.name, k)
        else:
            assert k > 2, (path, case.name, k)


GREEDY_CELLS = [(t, w8, p) for t in ("bf16", "fp16") for w8 in (False, True) for p in PATHS]


@pytest.mark.parametrize("tname,int8,path", GREEDY_CELLS, ids=[f"{t}-{'int8' if w8 else '16bit'}-{p}" for t, w8, p in GREEDY_CELLS])
def test_greedy_select(cuda, tname, int8, path):
    A = _greedy_A(path)
    eng, w = make_engine(DIMS["tiny"], tname, int8, PATHS[path], A, 1)
    try:
        st = _stats()
        run_greedy(eng, w, PATHS[path], path, A, st)
    finally:
        eng.close()
    _report(f"greedy {tname} {'int8' if int8 else '16-bit'} {path} A={A}", st)


BEAM_CELLS = [(t, p) for t in ("bf16", "fp16") for p in ("perop", "batched")]


@pytest.mark.parametrize("tname,path", BEAM_CELLS, ids=[f"{t}-{p}" for t, p in BEAM_CELLS])
def test_beam_candidates(cuda, tname, path):
    eng, w = make_engine(DIMS["tiny"], tname, False, PATHS[path], 3, 8)
    try:
        for A, G in BEAM_AG:
            st = _stats()
            for case in BEAM:
                k = run_case(eng, w, PATHS[path], case, A, G, st)
                assert k > 2, (path, case.name, k)
            _report(f"beam {tname} {path} A={A} G={G}", st)
    finally:
        eng.close()


@pytest.mark.parametrize("path", ["mega", "batched"])
def test_greedy_select_large_width(cuda, path):
    """D = 1280: the LM-head loops at K = 1280."""
    A = _greedy_A(path)
    eng, w = make_engine(DIMS["large"], "bf16", False, PATHS[path], A, 1)
    try:
        st = _stats()
        run_greedy(eng, w, PATHS[path], path, A, st)
    finally:
        eng.close()
    _report(f"greedy large-width bf16 {path} A={A}", st)


def test_graph_cache_reuse(cuda):
    """One engine, the greedy and beam cases run twice with the option sets revisited in reverse order (timestamp rules,
    max_initial_timestamp_index, begin_index 3 / 4, G, pad all change between neighbours): every replayed step graph must
    still select what the reference selects, as must an engine that captures no graphs.  An option that changes the select
    arguments but is missing from the graph key would replay a graph of another option set."""
    runs = [(c, 2, 1) for c in GREEDY] + [(c, a, g) for a, g in ((2, 2), (1, 5), (2, 8)) for c in BEAM]
    for env, passes in (({}, (runs, runs[::-1])), ({"BW_NO_GRAPH": "1"}, (runs,))):
        eng, w = make_engine(DIMS["tiny"], "bf16", False, env, 2, 8)
        try:
            st = _stats()
            for p in passes:
                for case, A, G in p:
                    run_case(eng, w, env, case, A, G, st)
        finally:
            eng.close()
        _report(f"graph cache {'no graphs' if env else 'two passes'}", st)
