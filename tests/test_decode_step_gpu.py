"""One decoder step from injected state, on every step path, at every cache length, against the float64 restatement
(oracle/step_ref.py, itself checked against transformers by tests/test_step_ref_cpu.py).

The step graph reads `pos` from device memory, so a test can write any decoder state (tokens, pos, the self K/V caches of all
layers, the cross K/V, the beam block table `anc`) through `WhisperEngine.write_buffer`, run exactly one step and compare
everything the step wrote against the reference computed from the same state.  Encoder error is out of the picture and the
bounds are tight.

The inputs are made to tell bugs apart: before each layer's attention the reference's own query plants the scores of chosen
keys (the key before `pos`, keys on both sides of 128 and 144, the first keys of the last 128-key chunk, keys on both sides of
every cross-attention split boundary, key S - 1), so that the softmax maximum sits in a late chunk while the early chunks keep
mass.  Each test then checks its own inputs: dropping keys >= 128, the row at `pos`, the last cross-attention split, or the
block table must move the logits by at least 10x the bound, else the test could not see that bug.
"""
import contextlib
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

POSITIONS = (0, 1, 127, 128, 129, 143, 144, 145, 255, 256, 383, 446, 447)
LARGE_POSITIONS = (129, 144, 145, 447)
BEGIN = 4   # begin_index of the decode (prompt of 4 tokens)
TMAX = 448
V = 51866

DIMS = {  # name: (d_model, heads, ffn, decoder layers, S)
    "tiny500": (128, 2, 512, 2, 500),
    "tiny750": (128, 2, 512, 2, 750),
    "small1500": (256, 4, 1024, 3, 1500),
    "large1500": (1280, 20, 5120, 32, 1500),
}
PATHS = {  # environment switches (read at engine creation / step-graph capture)
    "mega": {},
    "mega-single": {"BW_MEGA_FLAGS": "66"},  # default bit 6 + bit 1: single-buffered weight slabs
    "perop": {"BW_NO_MEGA": "1"},
    "batched": {"BW_NO_MEGA": "1", "BW_BATCH_MIN": "1"},
    "xstream": {"BW_NO_MEGA": "1", "BW_BATCH_MIN": "1", "BW_XATTN_STREAM_MIN": "1"},
}
SMALL_AG = {"mega": [(1, 1), (2, 1)], "mega-single": [(1, 1)], "perop": [(1, 1), (1, 2)], "batched": [(3, 1), (2, 5)],
            "xstream": [(2, 1), (1, 3), (1, 5), (1, 6)]}
LARGE_CELLS = [("bf16", "mega", (1, 1)), ("bf16", "mega", (2, 1)), ("bf16", "perop", (1, 1)), ("bf16", "batched", (8, 1)),
               ("bf16", "batched", (2, 5)), ("fp16", "mega", (1, 1)), ("fp16", "batched", (8, 1))]
DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}

CELLS = [(d, t, p, ag) for d in ("tiny500", "tiny750", "small1500") for t in ("bf16", "fp16") for p in PATHS for ag in SMALL_AG[p]]
CELLS += [("tiny500", "bf16", "mega", (1, 2))]  # does not apply: kept as a reported skip
CELLS += [("large1500",) + c for c in LARGE_CELLS]

# Bounds, relative to the reference's scale (logits: their standard deviation; dx / attention output / alignment scores: their
# rms), per arithmetic class and element type.  The persistent and per-op paths keep fp32 activations (compared with
# round_operands=False); the batched path rounds its GEMM operands (compared with round_operands=True), where a rounding that
# falls the other way than in float64 moves an operand by one ulp and the next layers with it.  Measured maxima on an
# NVIDIA H100 80GB HBM3 at a 700 W power limit, over all cells (tiny / small; large-v3 where it differs):
#   fp32 bf16:    logits 4.1e-4 (1.09e-3 at 32 layers), dx 3.2e-4 (1.07e-3), attention 2.2e-4 (1.46e-3), alignment 9.1e-5 (2.2e-4)
#   fp32 fp16:    logits 1.1e-4 (1.6e-4), dx 7.1e-5 (1.3e-4), attention 1.1e-4 (1.6e-4), alignment 2.3e-5 (3.4e-5)
#   batched bf16: logits 1.4e-2, dx 7.5e-3, attention 2.5e-2 (a bf16 operand: half an ulp is 2e-3 of its rms), alignment 3.1e-3
#   batched fp16: logits 1.5e-3, dx 7.6e-4, attention 1.9e-3, alignment 3.5e-4
#   at large-v3 (32 layers) the batched path drifts further: bf16 logits 2.6e-2, dx 2.0e-2, attention 6.6e-2, alignment 8.4e-3;
#   fp16 logits 3.4e-3, dx 2.5e-3, attention 5.0e-3, alignment 7.8e-4
# The bounds are about 2-3x those; every logit bound stays at or below 1/10 of the smallest ablation effect (0.45 of the logit
# std on tiny / small, 1.10 at large-v3).
TOL = {  # (class, dtype[, dims]): (logits, dx, attention output, alignment scores)
    ("fp32", "bf16"): (4e-3, 4e-3, 5e-3, 1e-3),
    ("fp32", "fp16"): (5e-4, 4e-4, 5e-4, 1e-4),
    ("batched", "bf16"): (4e-2, 2.5e-2, 5e-2, 1e-2),
    ("batched", "fp16"): (5e-3, 3e-3, 6e-3, 1.2e-3),
    ("batched", "bf16", "large1500"): (8e-2, 5e-2, 1.5e-1, 2e-2),
    ("batched", "fp16", "large1500"): (1e-2, 7e-3, 1.5e-2, 2.5e-3),
}
# The appended K/V row of layer 0 is within 1 ulp on every path, and on the fp32-activation paths at every layer.  On the batched
# path the operand roundings that fall the other way reach the later layers' rows and grow with depth: measured up to 2.25 ulps
# on tiny / small, 6 ulps at layer 13 of large-v3.
KV_ULPS = {"fp32": 1.0, "batched": 16.0}


def _cls(path):
    return "batched" if path in ("batched", "xstream") else "fp32"


def _pos_class(pos):
    return "<128" if pos < 128 else ("128-144" if pos <= 144 else ">144")


@contextlib.contextmanager
def _env(env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def make_weights(dims, dtype, seed=0, dev="cuda"):
    """Decoder weights in the engine's naming, generated on the device: matrices N(0, 1/K) (so activations stay O(1)), the
    tied embedding scaled so that logits have a standard deviation of about 2.  The encoder is never run here (0 layers);
    its stem / table / final LayerNorm are bound to zeros."""
    D, H, ffn, L, S = dims
    g = torch.Generator(device=dev).manual_seed(seed)
    rn = lambda *shape: torch.randn(*shape, generator=g, device=dev)
    mat = lambda n, k: (rn(n, k) / k ** 0.5).to(dtype)
    vec = lambda n, s=0.1, c=0.0: (c + s * rn(n)).float()
    w = {"enc.conv1.w": torch.zeros(D, 3 * 128, dtype=dtype, device=dev), "enc.conv2.w": torch.zeros(D, 3 * D, dtype=dtype, device=dev)}
    for n in ("enc.conv1.b", "enc.conv2.b", "enc.lnf.g", "enc.lnf.b"):
        w[n] = torch.zeros(D, device=dev)
    w["enc.pos"] = torch.zeros(S, D, device=dev)
    w["dec.embed"] = (rn(V, D) * (2.0 / D ** 0.5)).to(dtype)
    w["dec.pos"] = rn(TMAX, D)
    w["dec.lnf.g"], w["dec.lnf.b"] = vec(D, 0.1, 1.0), vec(D)
    for l in range(L):
        p = f"dec.{l}."
        for n in ("ln1", "ln2", "ln3"):
            w[p + n + ".g"], w[p + n + ".b"] = vec(D, 0.1, 1.0), vec(D)
        w[p + "wqkv"] = mat(3 * D, D)
        w[p + "bqkv"] = torch.cat([vec(D), torch.zeros(D, device=dev), vec(D)])
        w[p + "wo"], w[p + "bo"] = mat(D, D), vec(D)
        w[p + "xwq"], w[p + "xbq"] = mat(D, D), vec(D)
        w[p + "xwk"], w[p + "xwv"], w[p + "xbv"] = mat(D, D), mat(D, D), vec(D)
        w[p + "xwo"], w[p + "xbo"] = mat(D, D), vec(D)
        w[p + "w1"], w[p + "b1"] = mat(ffn, D), vec(ffn)
        w[p + "w2"], w[p + "b2"] = mat(D, ffn), vec(D)
    return w


class Rig:
    """Weights (+ their float64 copy for the reference) and engines, one configuration alive at a time (large-v3 caches at
    40 sequence slots are 3 GB)."""

    def __init__(self):
        self.key_w = self.key_e = None
        self.w = self.w64 = self.eng = None

    def weights(self, dname, tname):
        if self.key_w != (dname, tname):
            self.close()
            self.w = self.w64 = None
            torch.cuda.empty_cache()
            self.w = make_weights(DIMS[dname], DTYPES[tname])
            self.w64 = {k: v.double() for k, v in self.w.items() if k.startswith("dec.")}
            self.key_w = (dname, tname)
        return self.w, self.w64

    def engine(self, dname, tname, path, ags):
        from thewhisper_b200.engine import ModelDims, WhisperEngine

        w, _ = self.weights(dname, tname)
        key = (dname, tname, path)
        if self.key_e != key:
            self.close()
            D, H, ffn, L, S = DIMS[dname]
            dims = ModelDims(D, H, ffn, 0, L, 128, V, S, TMAX)
            with _env(PATHS[path]):
                self.eng = WhisperEngine(None, dims, chunk_length_s=S * 30 / 1500, max_audios=max(a for a, _ in ags),
                                         max_beams=max(g for _, g in ags), alignment_heads=[[0, 0], [L - 1, H - 1]], weights=w)
            self.key_e = key
        return self.eng

    def close(self):
        if self.eng is not None:
            self.eng.close()
        self.eng, self.key_e = None, None


@pytest.fixture(scope="module")
def rig():
    r = Rig()
    yield r
    r.close()


def _opts():
    from thewhisper_b200 import synthetic as S
    from thewhisper_b200.engine import DecodeOptions

    return DecodeOptions(eos_token=S.EOS, pad_token=S.EOS, suppress_tokens=S.default_suppress_tokens(),
                         begin_suppress_tokens=list(S.BEGIN_SUPPRESS), record_alignment=True)


def _cross_split(path, S, Q, H, num_sms=None):
    """Keys per cross-attention split (or tile) of the path: the persistent step's nsplit rule (api.cu), 12 splits on the
    per-op / batched split kernel, 128-key tiles on the streaming kernel."""
    if path.startswith("mega"):
        ns = (num_sms or torch.cuda.get_device_properties(0).multi_processor_count) // (Q * H)
        ns = min(max(ns, (S + 255) // 256), 12)
        return (S + ns - 1) // ns
    return 128 if path == "xstream" else (S + 11) // 12


def _ulps(got, want, dtype):
    """max |got - want| in units of the element type's spacing at the larger of |want| and the rms of `want` (an element that
    cancels to near zero is not held to the spacing of its own tiny magnitude)."""
    mant, emin = (7, -126) if dtype == torch.bfloat16 else (10, -14)
    w = want.double()
    mag = torch.maximum(w.abs(), w.pow(2).mean().sqrt()).clamp_min(2.0 ** emin)
    e = torch.floor(torch.log2(mag))
    return ((got.double() - w).abs() / torch.exp2(e - mant)).max().item()


def _masked_argmax(row, sup, at_begin, bsup):
    r = row.clone()
    r[sup] = -float("inf")
    if at_begin:
        r[bsup] = -float("inf")
    return int(torch.argmax(r)), r  # first maximum: ties go to the smaller id


def make_case(w64, dname, tname, path, A, G, Am, Qm, pos, dev="cuda"):
    """Decoder state at `pos` with planted attention scores, the float64 reference step from it, and the effect of each
    ablation on the logits (relative to their standard deviation)."""
    from oracle.step_ref import decoder_step
    from thewhisper_b200 import synthetic as S

    D, H, ffn, L, Sx = DIMS[dname]
    dtype = DTYPES[tname]
    Q = A * G
    ks = _cross_split(path, Sx, Q, H)
    last_split = ((Sx + ks - 1) // ks - 1) * ks
    gen = torch.Generator(device=dev).manual_seed(1000 * pos + 10 * Q + G)
    rn = lambda *shape: torch.randn(*shape, generator=gen, device=dev)
    ri = lambda lo, hi, shape: torch.randint(lo, hi, shape, generator=gen, device=dev)
    self_k = rn(L, Qm, TMAX, D).to(dtype)
    self_v = rn(L, Qm, TMAX, D).to(dtype)
    cross_k = rn(L, Am, H, Sx, 64).to(dtype)
    cross_v = rn(L, Am, H, Sx, 64).to(dtype)
    tokens = ri(0, S.EOS, (Qm, TMAX)).int()
    tokens[:, :BEGIN] = torch.tensor([S.SOT, S.LANG_EN, S.TRANSCRIBE, S.NOTIMESTAMPS], device=dev, dtype=torch.int32)
    anc = torch.arange(Qm, device=dev, dtype=torch.int32)[:, None].repeat(1, TMAX)
    if G > 1 and pos > 0:  # a block table a beam search could leave: past rows from any beam of the same audio, the last
        aud = torch.arange(Q, device=dev)[:, None] // G    # one from another beam (as after a reorder that switched beams)
        anc[:Q, :pos] = (aud * G + ri(0, G, (Q, pos))).int()
        own = torch.arange(Q, device=dev) - aud[:, 0] * G
        anc[:Q, pos - 1] = (aud[:, 0] * G + (own + 1 + ri(0, G - 1, (Q,))) % G).int()
    finished = torch.zeros(Qm, dtype=torch.int32, device=dev)
    if Q > 1:
        finished[Q - 1] = 1  # a finished sequence gets the pad token
    # ---- planted scores (self: relative to the score of the row at pos; cross: absolute)
    planted = sorted({pos - 1, 127, 128, 143, 144, 255, 256, (pos // 128) * 128, (pos // 128) * 128 + 1} & set(range(pos)))
    late = [s for s in planted if s >= 128]
    top = late[-1] if late else pos - 1
    base_self = -5.0 + 0.5 * rn(Q, pos, H)
    base_self[:, planted] = -1.0
    if pos > 0:
        base_self[:, top] = 1.0
    xplant = sorted({b + d for b in range(ks, Sx, ks) for d in (-1, 0)})
    base_cross = -4.0 + 0.5 * rn(L, Am, H, Sx)
    base_cross[..., xplant] = 0.0
    base_cross[..., Sx - 1] = 3.0
    anc_ref = anc[:Q] if G > 1 else None

    def hook(l, kind, q, k_new):
        if kind == "self":
            if pos == 0:
                return
            s_pos = (q * k_new).sum(-1)                                     # [Q, H]
            for qi in range(Q):
                slots = anc_ref[qi, :pos].long() if G > 1 else torch.full((pos,), qi, device=dev)
                idx = torch.arange(pos, device=dev)
                rows = self_k[l][slots, idx].double().view(pos, H, 64)
                qq = q[qi]
                cur = (rows * qq).sum(-1)
                tgt = s_pos[qi][None] + base_self[qi]
                rows += ((tgt - cur) / (qq * qq).sum(-1))[..., None] * qq
                self_k[l][slots, idx] = rows.view(pos, D).to(dtype)
        else:
            for a in range(A):
                qq = q[a * G]                                                # beam 0 of the audio
                K = cross_k[l][a].double()                                   # [H, S, 64]
                cur = torch.einsum("hsd,hd->hs", K, qq)
                K += ((base_cross[l, a] - cur) / (qq * qq).sum(-1)[:, None])[..., None] * qq[:, None]
                cross_k[l][a] = K.to(dtype)

    ro = _cls(path) == "batched"
    args = (w64, L, self_k, self_v, cross_k, cross_v, tokens[:Q], pos)
    kw = dict(G=G, anc=anc_ref, align_heads=[[0, 0], [L - 1, H - 1]], round_operands=ro)
    ref = decoder_step(*args, hook=hook, **kw)
    lg_ref = ref["logits"]
    scale = float(lg_ref.std())
    # ---- the inputs must separate these bugs from correct code (checked by the caller against its bound)
    abl = {}
    if pos > 128:
        keep = torch.arange(pos + 1, device=dev)
        abl["keys>=128"] = decoder_step(*args, self_keep=(keep < 128) | (keep == pos), **kw)
    abl["row pos"] = decoder_step(*args, self_keep=torch.arange(pos + 1, device=dev) < pos, **kw)
    abl["last split"] = decoder_step(*args, cross_keep=torch.arange(Sx, device=dev) < last_split, **kw)
    if G > 1 and pos > 0:
        abl["anc"] = decoder_step(*args, **dict(kw, anc=None))
    effects = {k: float((v["logits"] - lg_ref).abs().max()) / scale for k, v in abl.items()}
    return dict(self_k=self_k, self_v=self_v, cross_k=cross_k, cross_v=cross_v, tokens=tokens, anc=anc, finished=finished,
                ref=ref, effects=effects)


def run_cell(rig, dname, tname, path, A, G, positions):
    from thewhisper_b200 import synthetic as S

    D, H, ffn, L, Sx = DIMS[dname]
    dtype = DTYPES[tname]
    ags = [ag for _, p, ag in LARGE_CELLS if p == path] if dname == "large1500" else SMALL_AG[path]
    eng = rig.engine(dname, tname, path, ags)
    w64 = rig.w64
    Am, Qm = eng.max_audios, eng.max_audios * eng.max_beams
    Q = A * G
    cls = _cls(path)
    tol_lg, tol_dx, tol_xa, tol_al = TOL.get((cls, tname, dname), TOL[(cls, tname)])
    opts = _opts()
    sup = torch.tensor(opts.suppress_tokens, device="cuda")
    bsup = torch.tensor(opts.begin_suppress_tokens, device="cuda")
    Ha, Tcap = 2, eng.max_align_steps
    dev = "cuda"
    stats = {}
    for pos in positions:
        c = make_case(w64, dname, tname, path, A, G, Am, Qm, pos)
        self_k, self_v, cross_k, cross_v = c["self_k"], c["self_v"], c["cross_k"], c["cross_v"]
        tokens, anc, finished, ref, effects = c["tokens"], c["anc"], c["finished"], c["ref"], c["effects"]
        lg_ref = ref["logits"]
        scale = float(lg_ref.std())
        for k, e in effects.items():
            assert e >= 10 * tol_lg, (pos, k, e, tol_lg)  # else this input could not reveal that bug
        # ---- the engine: begin a decode, overwrite its state, one step
        with _env(PATHS[path]):
            eng.decode_begin(np.array([[S.SOT, S.LANG_EN, S.TRANSCRIBE, S.NOTIMESTAMPS]] * Q, dtype=np.int32), A, G, opts,
                             begin_index=BEGIN)
        for name, t in (("self_k", self_k), ("self_v", self_v), ("cross_k", cross_k), ("cross_v", cross_v), ("tokens", tokens),
                        ("anc", anc), ("finished", finished), ("pos", torch.tensor([pos], dtype=torch.int32, device=dev))):
            eng.write_buffer(name, t)
        align0 = eng.buffer("align", torch.float32, (Qm, Ha, Tcap, Sx)).clone()
        k0 = eng.decode_kernel_launches()
        eng.decode_run(1)
        torch.cuda.synchronize()
        per_step = eng.decode_kernel_launches() - k0
        assert (per_step <= 2) == path.startswith("mega"), (path, per_step)
        # ---- appended K/V rows of every layer (1 ulp), every other row untouched
        sk = eng.buffer("self_k", dtype, (L, Qm, TMAX, D))
        sv = eng.buffer("self_v", dtype, (L, Qm, TMAX, D))
        kv_ulp = 0.0
        for l in range(L):
            u = max(_ulps(sk[l, :Q, pos], ref["k_new"][l], dtype), _ulps(sv[l, :Q, pos], ref["v_new"][l], dtype))
            assert u <= (1.0 if l == 0 else KV_ULPS[cls]), (pos, "first diverging layer", l, u)
            kv_ulp = max(kv_ulp, u)
        sk[:, :Q, pos] = self_k[:, :Q, pos]
        sv[:, :Q, pos] = self_v[:, :Q, pos]
        assert torch.equal(sk, self_k) and torch.equal(sv, self_v), (pos, "a cache row other than (q < Q, pos) changed")
        assert torch.equal(eng.buffer("cross_k", dtype, cross_k.shape), cross_k)
        assert torch.equal(eng.buffer("cross_v", dtype, cross_v.shape), cross_v)
        # ---- residual, last cross-attention output, logits, alignment scores
        dx = eng.buffer("dx", torch.float32, (Qm, D))[:Q].double()
        e_dx = float((dx - ref["dx"]).abs().max() / ref["dx"].pow(2).mean().sqrt())
        xa = (eng.buffer("dba", dtype, (Qm, D)) if cls == "batched" else eng.buffer("dattn", torch.float32, (Qm, D)))[:Q].double()
        e_xa = float((xa - ref["xattn"]).abs().max() / ref["xattn"].pow(2).mean().sqrt())
        lg = eng.logits().double()
        e_lg = float((lg - lg_ref).abs().max()) / scale
        al = eng.buffer("align", torch.float32, (Qm, Ha, Tcap, Sx))
        step = pos - BEGIN
        e_al = 0.0
        if 0 <= step < Tcap:
            e_al = float((al[:Q, :, step].double() - ref["align"]).abs().max() / ref["align"].pow(2).mean().sqrt())
            al[:Q, :, step] = align0[:Q, :, step]
        assert torch.equal(al, align0), (pos, "alignment rows other than the step's changed")
        # ---- token selection, finished, pos
        toks, fin, pos_after = eng.decode_read()
        assert pos_after == pos + 1
        want_tok = tokens.cpu().numpy()[:Q].copy()
        want_fin = finished.cpu().numpy()[:Q].copy()
        cur_len = pos + 1
        if BEGIN <= cur_len < TMAX:
            for q in range(Q):
                mine, _ = _masked_argmax(lg[q], sup, cur_len == BEGIN, bsup)
                theirs, rrow = _masked_argmax(lg_ref[q], sup, cur_len == BEGIN, bsup)
                if want_fin[q]:
                    want_tok[q, cur_len] = S.EOS
                    continue
                want_tok[q, cur_len] = mine
                assert mine == theirs or float(rrow[theirs] - rrow[mine]) < tol_lg * scale, (pos, q, mine, theirs)
                want_fin[q] = int(mine == S.EOS)
        assert np.array_equal(toks, want_tok), (pos, "tokens")  # at pos = 447 nothing is written: row q + 1 is intact
        assert np.array_equal(fin, want_fin), (pos, fin, want_fin)
        c = stats.setdefault(_pos_class(pos), dict(logits=0.0, dx=0.0, xattn=0.0, align=0.0, kv_ulp=0.0, ablation=float("inf")))
        for k, v in (("logits", e_lg), ("dx", e_dx), ("xattn", e_xa), ("align", e_al), ("kv_ulp", kv_ulp)):
            c[k] = max(c[k], v)
        c["ablation"] = min([c["ablation"]] + list(effects.values()))
        print(f"  pos {pos:3d}: logits {e_lg:.2e} dx {e_dx:.2e} xattn {e_xa:.2e} align {e_al:.2e} kv {kv_ulp:.2f} ulp | "
              + " ".join(f"{k} {v:.3f}" for k, v in effects.items()))
        assert e_lg < tol_lg and e_dx < tol_dx and e_xa < tol_xa and e_al < tol_al, (pos, e_lg, e_dx, e_xa, e_al)
    for k, c in stats.items():
        print(f"[{dname} {tname} {path} A={A} G={G}] pos {k:>7}: worst logits {c['logits']:.2e} dx {c['dx']:.2e} "
              f"xattn {c['xattn']:.2e} align {c['align']:.2e} kv {c['kv_ulp']:.2f} ulp; smallest ablation {c['ablation']:.3f} "
              f"(bound {tol_lg:.0e})")


@pytest.mark.parametrize("dname,tname,path,ag", CELLS, ids=[f"{d}-{t}-{p}-A{a}G{g}" for d, t, p, (a, g) in CELLS])
def test_decode_step_matches_reference(cuda, rig, dname, tname, path, ag):
    A, G = ag
    if path.startswith("mega") and G > 1:
        pytest.skip("the persistent step runs one sequence per audio (G = 1); beams take the per-op or batched step")
    print(f"\n[{dname} {tname} {path} A={A} G={G}]")
    run_cell(rig, dname, tname, path, A, G, LARGE_POSITIONS if dname == "large1500" else POSITIONS)


# ------------------------------------------------------------------------------------------------------------------
# the C-ABI stops at the last position
# ------------------------------------------------------------------------------------------------------------------
def test_decode_run_stops_at_last_position(cuda, rig):
    """bw_decode_run refuses steps past position Tmax - 1 before launching anything.  A build without that check would run
    the step at pos = Tmax out of bounds, so the test first makes sure the check is there: a negative step count is refused
    only by a build that has it."""
    from thewhisper_b200 import _lib
    from thewhisper_b200 import synthetic as S

    eng = rig.engine("tiny500", "bf16", "mega", SMALL_AG["mega"])
    prompt = np.array([[S.SOT, S.LANG_EN, S.TRANSCRIBE, S.NOTIMESTAMPS]], dtype=np.int32)
    eng.decode_begin(prompt, 1, 1, _opts())
    try:
        eng.decode_run(-1)
    except _lib.BwError:
        pass
    else:
        pytest.fail("bw_decode_run accepts a negative step count: the last-position check is missing, not testing further")
    with pytest.raises(_lib.BwError, match="past the last position"):
        eng.decode_run(TMAX + 1)
    assert eng.decode_read()[2] == 0  # nothing was launched
    eng.decode_run(TMAX - 1)
    eng.decode_run(1)  # the step at pos = Tmax - 1 is allowed (and writes no token)
    toks, _, pos = eng.decode_read()
    assert pos == TMAX
    with pytest.raises(_lib.BwError, match="past the last position"):
        eng.decode_run(1)
    assert eng.decode_read()[2] == TMAX
    eng.decode_begin(prompt, 1, 1, _opts())  # a new decode starts counting again
    eng.decode_run(1)
    assert eng.decode_read()[2] == 1


# ------------------------------------------------------------------------------------------------------------------
# greedy to the last position: the cache written step by step is the cache read later
# ------------------------------------------------------------------------------------------------------------------
_TINY = {}


@pytest.mark.parametrize("path", ["mega", "perop", "batched"])
def test_greedy_to_last_position(cuda, path):
    """tiny10 with EOS suppressed, greedy until the host loop stops at Tmax (444 new tokens), against the live fp32 oracle
    with the near-tie protocol of tests/test_large_gpu.py: the engine's logits are first teacher-forced over its own 448-token
    sequence to measure the logit error at the oracle's top-8 tokens; every generated token must then be the oracle's processed
    arg-max given the same prefix, unless the oracle rates it within twice that error of its own arg-max."""
    import json

    from oracle import hf_ref
    from tests.conftest import GOLD
    from thewhisper_b200 import synthetic as S
    from thewhisper_b200.engine import DecodeOptions, ModelDims, WhisperEngine

    if not _TINY:
        meta = json.load(open(os.path.join(GOLD, "model_tiny10.json")))
        model = S.make_hf_model(meta["preset"], seed=meta["seed"], layer_gain=meta.get("layer_gain", 1.0))
        model.generation_config = S.make_generation_config(meta["preset"], eos_suppressed=True)
        hf_ref.interpolate_positions(model, 10)
        mel = hf_ref.logmel(S.make_feature_extractor(10), S.synth_audio(10, seed=1000))
        with torch.no_grad():
            enc = model.model.encoder(torch.from_numpy(mel)[None]).last_hidden_state
        _TINY.update(model=model, mel=mel, enc=enc, ref={})
    model, mel = _TINY["model"], _TINY["mel"]
    env = {"mega": {}, "perop": {"BW_NO_MEGA": "1", "BW_BATCH_MIN": "1000"}, "batched": {"BW_NO_MEGA": "1", "BW_BATCH_MIN": "1"}}[path]
    with _env(env):
        eng = WhisperEngine(model.state_dict(), ModelDims.from_hf_config(model.config), chunk_length_s=10, max_audios=1)
        try:
            g = model.generation_config
            opts = DecodeOptions(eos_token=S.EOS, pad_token=S.EOS, suppress_tokens=list(g.suppress_tokens),
                                 begin_suppress_tokens=list(g.begin_suppress_tokens))
            eng.set_mel(torch.from_numpy(mel[None]))
            eng.encode(1)
            prompt = np.array([[S.SOT, S.LANG_EN, S.TRANSCRIBE, S.NOTIMESTAMPS]], dtype=np.int32)
            k0 = eng.decode_kernel_launches()
            gen, toks, n = eng.greedy(prompt, 1, opts, max_new_tokens=10 ** 6)
            per_step = (eng.decode_kernel_launches() - k0) / (TMAX - 1)
            assert (per_step <= 2) == (path == "mega"), (path, per_step)
            gen = gen[0]
            assert n == TMAX - 4 and len(gen) == TMAX - 4, (n, len(gen))
            assert eng.decode_read()[2] == TMAX - 1  # the last token came from the step at Tmax - 2: the loop stopped there
            full = prompt[0].tolist() + gen.tolist()
            key = tuple(full)
            if key not in _TINY["ref"]:
                with torch.no_grad():
                    out = model(encoder_outputs=(_TINY["enc"],), decoder_input_ids=torch.tensor([full]))
                _TINY["ref"][key] = out.logits[0].float().numpy()
            ref = _TINY["ref"][key]
            # the engine teacher-forced over its own sequence: the measured error at the oracle's top-8 tokens
            eng.decode_begin(np.array([full], dtype=np.int32), 1, 1, opts)
            worst_top = 0.0
            for t in range(TMAX):
                eng.decode_run(1)
                lg = eng.logits()[0].cpu().numpy()
                top = np.argsort(-ref[t])[:8]
                worst_top = max(worst_top, float(np.abs(lg[top] - ref[t][top]).max()))
        finally:
            eng.close()
    tol = 2.0 * worst_top
    near = 0
    for i, tok in enumerate(gen):
        row = ref[3 + i].copy()
        row[list(g.suppress_tokens)] = -np.inf
        if i == 0:
            row[list(g.begin_suppress_tokens)] = -np.inf
        best = int(np.argmax(row))
        if tok != best:
            gap = float(row[best] - row[tok])
            assert gap < tol, (i, int(tok), best, gap, tol)
            near += 1
    print(f"\n[tiny10 {path}] greedy to Tmax: {len(gen)} tokens, {near} admissible near ties (oracle margin < {tol:.4f}; "
          f"max |dlogit| at the oracle's top-8 over 448 teacher-forced positions {worst_top:.4f})")
    assert near <= len(gen) // 40, near  # measured on the H100: 4 (persistent), 4 (per-op), 5 (batched) of 444
