"""Log-mel and every encoder stage, on every encoder path, in bf16 and fp16, against the float64 restatement
(oracle/enc_ref.py, itself checked against transformers by tests/test_enc_ref_cpu.py).

Engines are built with enc_layers = 0, 1, ..., L over one weight dict, so layer l's intermediates are the last-layer buffers
of the depth-(l + 1) engine (`qkv`, `ao`, `xn` = LayerNorm 2, `hbuf`, `x_enc`) and its input is `x_enc` of the depth-l
engine.  Every stage is computed from the engine's own upstream tensor, so errors do not drift and the 16-bit stages are held
to 1-3 ulps and to the fraction of elements that differ from the correctly rounded value.  The whole pass from the mel is
compared once more against the rounding reference, with a drift bound.

The inputs are made to tell bugs apart:
  - mel frames 0, 1, F-2 and F-1 carry large values, so the conv stem's zero padding and last rows matter;
  - one column of the positional table is large only at rows 0, 127, 128 and S-1, every layer passes that column through
    unchanged, and head 0's k weights and q bias are aligned with it: that head's largest scores sit on the first key, on both
    sides of the 128-key tile boundary and on the ragged last tile, while the other heads keep diffuse scores;
  - neighbouring items have different mels, and the first key of every item is a planted one, so a last tile that reads the
    next item's rows unmasked is visible.
Each cell checks its own inputs: the restatement with a plausible bug (positional rows one late, key S-1 masked, the next
item's keys admitted, tanh GELU, the V bias on K; for the log-mel a symmetric window, reflect padding off by one, a batch-wide
maximum) must move the compared output by at least 10x its bound.
"""
import contextlib
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

V = 51866
TMAX = 448
DIMS = {  # name: (d_model, heads, ffn, encoder layers, decoder layers)
    "tiny": (128, 2, 512, 2, 2),
    "small": (256, 4, 1024, 3, 2),
    "large-v3": (1280, 20, 5120, 32, 2),
    "turbo": (1280, 20, 5120, 32, 4),
}
PATHS = {  # environment switches, read at engine creation
    "default": {},
    "gemm2=0": {"BW_GEMM2": "0"},
    "vdirect=0": {"BW_ATTN_VDIRECT": "0"},
    "simt": {"BW_GEMM_IMPL": "simt"},
    "pdl": {"BW_ENC_PDL": "1"},
}
S_VALUES = (100, 365, 500, 600, 750, 1500)
DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}

CELLS = [(d, t, p, S, (1, 3)) for d in ("tiny", "small") for t in DTYPES for p in PATHS for S in S_VALUES]
CELLS += [("large-v3", t, "default", 1500, (1, 2)) for t in DTYPES] + [("large-v3", "bf16", "gemm2=0", 1500, (1, 2))]
CELLS += [("turbo", t, "default", 500, (1, 2)) for t in DTYPES]

# Bounds.  Measured maxima on an NVIDIA H100 80GB HBM3 at a 400 W power limit, over all cells (tiny / small; large-v3 and
# turbo where it differs):
#   16-bit stages from the engine's own inputs, in ulps: qkv 1.11 (an xn element rounded the other way than in float64 moves
#     the planted k dimension), xn 1.0, h1 / hbuf / enc_out / cross K/V 0.51
#   elements that differ from the correctly rounded float64 value: bf16 h1 2.3e-3, qkv 2.2e-3, others 8.1e-4;
#     fp16 h1 3.8e-3, qkv 1.1e-2, others 6.9e-3
#   conv2 + GELU + pos (fp32): 9.3e-6 (4.7e-5) of the rms; fc2 + residual (fp32): 3.5e-6 (5.5e-6)
#   attention output: bf16 2.7e-2 (3.6e-2), fp16 3.4e-3 (4.8e-3) of the rms (P is rounded to the element type in the kernel)
#   the whole pass from the mel (enc_out, cross V): bf16 3.1e-2, fp16 3.9e-3 of the rms
#   log-mel: 1.4e-5 absolute
# The bounds are 2-3x those and at most 1/10 of the smallest ablation effect, except two:
#   - bf16 attention: the smallest ablation moves the output by 0.47 of its rms, so its bound is 1.7x the measured error
#     at tiny / small and 1.25x at large-v3;
#   - bf16 h1: tanh GELU changes 2.5% of the elements, and no bound above the measured 0.23% is 10x below that.  That
#     ablation is asserted in fp16 (17%), where the conv1 epilogue runs the same code.
# Smallest ablation effects: pos shift 6.2 of the rms; key S-1 masked 0.47, next item's keys 0.49; tanh GELU in fc1 7.5%
# (bf16) / 31% (fp16) of the elements; V bias on K 38 (bf16) / 299 (fp16) ulps; log-mel 0.45 absolute.
ULPS = {"qkv": 3.0, "xn": 2.0, "other": 1.0}
MISMATCH = {"bf16": {"conv1": 5e-3, "qkv": 5e-3, "other": 2e-3}, "fp16": {"conv1": 1e-2, "qkv": 3e-2, "other": 1.5e-2}}
REL = {"stem": 1e-4, "fc2": 1.5e-5, ("attn", "bf16"): 4.5e-2, ("attn", "fp16"): 1e-2}
DRIFT = {"bf16": 8e-2, "fp16": 1e-2}
LOGMEL_ABS = 4e-5


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


def _rms(t):
    return float(t.double().pow(2).mean().sqrt())


def _rel(got, want):
    return float((got.double() - want.double()).abs().max()) / _rms(want)


def _ulps(got, want, dtype):
    """max |got - want| in units of the element type's spacing at the larger of |want| and the rms of `want`."""
    mant, emin = (7, -126) if dtype == torch.bfloat16 else (10, -14)
    w = want.double()
    mag = torch.maximum(w.abs(), w.pow(2).mean().sqrt()).clamp_min(2.0 ** emin)
    return float(((got.double() - w).abs() / torch.exp2(torch.floor(torch.log2(mag)) - mant)).max())


def _mismatch(got, want, dtype):
    """Fraction of elements that differ from the correctly rounded value."""
    return float((got.to(dtype) != want.to(dtype)).double().mean())


def plant(dims, S):
    """The planted column, the rows that carry it, and its value: large enough that LayerNorm leaves about 6 there."""
    D = dims[0]
    return D - 1, sorted({0, 127, 128, S - 1} & set(range(S))), 6.0 / (1.0 - 36.0 / D) ** 0.5


def make_weights(dims, dtype, seed=0, dev="cuda"):
    """Encoder + decoder weights in the engine's naming, generated on the device: matrices N(0, 1/K) (the encoder's out-proj
    and fc2 scaled by 1/sqrt(L), so that the residual stream stays O(1) to the last layer), LayerNorm gains 1 +- 0.1.
    Column c of the residual stream only ever holds the positional table (conv2, out-proj and fc2 write zeros there,
    LayerNorm 1's bias is 0 there); head 0's first q / k dimensions read it: q = 3 (bias only), k = 3 x[c], so a planted
    key scores about 7 above the others in that head."""
    D, H, ffn, Le, Ld = dims
    c = D - 1
    g = torch.Generator(device=dev).manual_seed(seed)
    rn = lambda *shape: torch.randn(*shape, generator=g, device=dev)
    mat = lambda n, k: rn(n, k) / k ** 0.5
    vec = lambda n, s=0.1, m=0.0: (m + s * rn(n)).float()
    w = {"enc.conv1.w": mat(D, 3 * 128), "enc.conv1.b": vec(D), "enc.conv2.w": mat(D, 3 * D), "enc.conv2.b": vec(D),
         "enc.lnf.g": vec(D, 0.1, 1.0), "enc.lnf.b": vec(D)}
    w["enc.conv2.w"][c] = 0
    w["enc.conv2.b"][c] = 0
    for l in range(Le):
        p = f"enc.{l}."
        for n in ("ln1", "ln2"):
            w[p + n + ".g"], w[p + n + ".b"] = vec(D, 0.1, 1.0), vec(D)
        w[p + "ln1.b"][c] = 0
        w[p + "wqkv"] = mat(3 * D, D)
        w[p + "bqkv"] = torch.cat([vec(D), torch.zeros(D, device=dev), vec(D)])
        w[p + "wqkv"][0] = 0
        w[p + "bqkv"][0] = 3.0
        w[p + "wqkv"][D] = 0
        w[p + "wqkv"][D, c] = 3.0
        w[p + "wo"], w[p + "bo"] = mat(D, D) / Le ** 0.5, vec(D)
        w[p + "w1"], w[p + "b1"] = mat(ffn, D), vec(ffn)
        w[p + "w2"], w[p + "b2"] = mat(D, ffn) / Le ** 0.5, vec(D)
        for n in ("wo", "bo", "w2", "b2"):
            w[p + n][c] = 0
    w["dec.embed"] = rn(V, D) / D ** 0.5
    w["dec.pos"] = rn(TMAX, D)
    w["dec.lnf.g"], w["dec.lnf.b"] = vec(D, 0.1, 1.0), vec(D)
    for l in range(Ld):
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
    return {k: (v.to(dtype) if v.dim() == 2 and k != "dec.pos" else v.float()).contiguous() for k, v in w.items()}


def make_pos(dims, S, seed=1, dev="cuda"):
    """A random positional table with distinct rows; the planted column is zero except at its rows."""
    c, rows, val = plant(dims, S)
    pos = torch.randn(S, dims[0], generator=torch.Generator(device=dev).manual_seed(seed), device=dev)
    pos[:, c] = 0
    pos[rows, c] = val
    return pos.contiguous()


def make_mel(n, S, seed=2, dev="cuda"):
    """n different log-mel-like items [n, 128, 2S]; frames 0, 1, F-2 and F-1 carry large values."""
    g = torch.Generator(device=dev).manual_seed(seed)
    F_ = 2 * S
    mel = 0.5 * torch.randn(n, 128, F_, generator=g, device=dev) + 0.3 * torch.randn(n, 128, 1, generator=g, device=dev)
    edge = [0, 1, F_ - 2, F_ - 1]
    mel[:, :, edge] = 4.0 * torch.sign(torch.randn(n, 128, 4, generator=g, device=dev))
    return mel


class Rig:
    """One weight dict per (dims, type); engines of every depth of one cell."""

    def __init__(self):
        self.key_w, self.w, self.engines = None, None, {}

    def weights(self, dname, tname):
        if self.key_w != (dname, tname):
            self.close()
            self.w = None
            torch.cuda.empty_cache()
            self.w = make_weights(DIMS[dname], DTYPES[tname])
            self.key_w = (dname, tname)
        return self.w

    def build(self, dname, tname, path, S, depths, A):
        from thewhisper_b200.engine import ModelDims, WhisperEngine

        self.close()
        w = self.weights(dname, tname)
        w["enc.pos"] = make_pos(DIMS[dname], S)
        D, H, ffn, Le, Ld = DIMS[dname]
        with _env(PATHS[path]):
            for d in depths:
                eng = WhisperEngine(None, ModelDims(D, H, ffn, d, Ld, 128, V, S, TMAX), chunk_length_s=S * 30 / 1500,
                                    max_audios=A, weights=w)
                assert eng.S == S, (eng.S, S)
                self.engines[d] = eng
        return self.engines

    def close(self):
        for e in self.engines.values():
            e.close()
        self.engines = {}


@pytest.fixture(scope="module")
def rig():
    r = Rig()
    yield r
    r.close()


SENTINEL = 4096.0  # exactly representable in float32, bf16 and fp16
_DEFAULT_OUT = {}  # (dims, type, S, B) -> the default path's outputs, for the bit-identity of BW_ENC_PDL=1


def _run(eng, mel, B):
    """set_mel + encode(B) twice (stream, then the captured graph); returns the buffers of the first call.  Slots >= B of
    x_enc, enc_out and cross K/V hold a sentinel beforehand and must still hold it."""
    A, S, D, F_, H = eng.max_audios, eng.S, eng.dims.d_model, eng.frames, eng.dims.n_heads
    Ld, ffn, et = eng.dims.dec_layers, eng.dims.ffn, eng.dtype
    shapes = {"mel_tm": (et, (A, F_ + 2, 128)), "h1": (et, (A, F_ + 2, D)), "x_enc": (torch.float32, (A, S, D)),
              "qkv": (et, (A, S, 3 * D)), "ao": (et, (A, S, D)), "xn": (et, (A, S, D)), "hbuf": (et, (A, S, ffn)),
              "enc_out": (et, (A, S, D)), "cross_k": (et, (Ld, A, H, S, 64)), "cross_v": (et, (Ld, A, H, S, 64))}
    for name in ("x_enc", "enc_out", "cross_k", "cross_v"):
        t, shp = shapes[name]
        eng.write_buffer(name, torch.full(shp, SENTINEL, dtype=t, device="cuda"))
    eng.set_mel(mel[:B])
    outs = []
    for _ in range(2):
        eng.encode(B)
        torch.cuda.synchronize()
        outs.append({n: eng.buffer(n, t, shp).clone() for n, (t, shp) in shapes.items()})
    for n in outs[0]:
        assert torch.equal(outs[0][n], outs[1][n]), (n, "the graph replay differs from the stream call")
    o = outs[0]
    for name in ("x_enc", "enc_out"):
        assert bool((o[name][B:] == SENTINEL).all()), (name, "a slot >= B was written")
    for name in ("cross_k", "cross_v"):
        assert bool((o[name][:, B:] == SENTINEL).all()), (name, "a slot >= B was written")
    return o


def _same_gemm_path(path, S, B0, B1):
    if path in ("gemm2=0", "simt"):
        return True
    return (B0 * S >= 1024) == (B1 * S >= 1024)  # gemm2_min_rows: the flat-row kernel from 1024 rows on


@pytest.mark.parametrize("dname,tname,path,S,Bs", CELLS, ids=[f"{d}-{t}-{p}-S{S}" for d, t, p, S, _ in CELLS])
def test_encode_stages_match_reference(cuda, rig, dname, tname, path, S, Bs):
    from oracle import enc_ref as R
    from thewhisper_b200 import _lib

    D, H, ffn, Le, Ld = DIMS[dname]
    et = DTYPES[tname]
    large = dname in ("large-v3", "turbo")
    depths = sorted({0, 1, 2, Le - 1, Le}) if large else list(range(Le + 1))
    try:
        engines = rig.build(dname, tname, path, S, depths, max(Bs))
    except _lib.BwError as ex:  # a shape the engine does not take must be refused at creation, with a message
        assert str(ex), ex
        pytest.skip(f"engine refuses S={S}: {ex}")
    w = rig.w
    mel = make_mel(max(Bs), S)
    c, rows, _ = plant(DIMS[dname], S)
    mm, tol_attn, tol_drift = MISMATCH[tname], REL[("attn", tname)], DRIFT[tname]
    worst, abl, bad = {}, {}, []

    def note(stage, err, bound, effects=None):
        worst[stage] = max(worst.get(stage, 0.0), err)
        if not err <= bound:
            bad.append((stage, err, bound))
        for k, e in (effects or {}).items():
            abl[(stage, k)] = min(abl.get((stage, k), float("inf")), e)
            if not e >= 10 * bound:
                bad.append((stage, "ablation " + k, e, bound))

    per_b = {}
    for B in Bs:
        out = {d: _run(engines[d], mel, B) for d in depths}
        per_b[B] = out
        # ---- set_mel: bit-exact rounding, zero pad rows
        mt = out[depths[0]]["mel_tm"][:B]
        assert torch.equal(mt[:, 1:-1], mel[:B].transpose(1, 2).to(et)), "mel_tm"
        assert not mt[:, 0].any() and not mt[:, -1].any(), "mel_tm pad rows"
        # ---- conv1 + GELU: engine mel_tm -> h1 (pad rows zero)
        h1 = out[0]["h1"][:B]
        assert not h1[:, 0].any() and not h1[:, -1].any(), "h1 pad rows"
        ref = R.conv1(w, mt)
        note("conv1 ulp", _ulps(h1[:, 1:-1], ref, et), ULPS["other"])
        # in bf16 the tanh approximation moves GELU by about 3% of an ulp, too little for this count to see; fp16 shows it
        note("conv1 mismatch", _mismatch(h1[:, 1:-1], ref, et), mm["conv1"],
             {"tanh gelu": _mismatch(R.conv1(w, mt, tanh_gelu=True), ref, et)} if tname == "fp16" else None)
        # ---- conv2 + GELU + pos: engine h1 -> x_enc at depth 0
        ref = R.conv2_pos(w, h1)
        note("conv2+pos", _rel(out[0]["x_enc"][:B], ref), REL["stem"], {"pos shift": _rel(R.conv2_pos(w, h1, pos_shift=1), ref)})
        # ---- encoder layers: layer l = the last layer of the depth-(l + 1) engine
        for d in depths[1:]:
            if d - 1 not in out:
                continue
            l, o, x_in = d - 1, out[d], out[d - 1]["x_enc"][:B]
            ref = R.ln1_qkv(w, l, x_in, et)
            note("ln1+qkv ulp", _ulps(o["qkv"][:B], ref, et), ULPS["qkv"])
            note("ln1+qkv mismatch", _mismatch(o["qkv"][:B], ref, et), mm["qkv"])
            qkv = o["qkv"][:B]
            ref = R.attention(qkv, H)
            eff = {"key S-1 masked": _rel(R.attention(qkv, H, drop_keys_from=S - 1), ref)}
            if B > 1:
                eff["next item's keys"] = _rel(R.attention(qkv, H, leak_next=True), ref)
            note("attention", _rel(o["ao"][:B], ref), tol_attn, eff)
            x_mid, ref = R.out_ln2(w, l, x_in, o["ao"][:B], et)
            note("out-proj+ln2 ulp", _ulps(o["xn"][:B], ref, et), ULPS["xn"])
            note("out-proj+ln2 mismatch", _mismatch(o["xn"][:B], ref, et), mm["other"])
            ref = R.fc1(w, l, o["xn"][:B])
            note("fc1 ulp", _ulps(o["hbuf"][:B], ref, et), ULPS["other"])
            note("fc1 mismatch", _mismatch(o["hbuf"][:B], ref, et), mm["other"],
                 {"tanh gelu": _mismatch(R.fc1(w, l, o["xn"][:B], tanh_gelu=True), ref, et)})
            note("fc2", _rel(o["x_enc"][:B], R.fc2(w, l, o["hbuf"][:B], x_mid)), REL["fc2"])
        # ---- final LayerNorm and cross K/V of every decoder layer, every item
        for d in depths:
            o = out[d]
            ref = R.final_ln(w, o["x_enc"][:B])
            note("final ln ulp", _ulps(o["enc_out"][:B], ref, et), ULPS["other"])
            note("final ln mismatch", _mismatch(o["enc_out"][:B], ref, et), mm["other"])
        o = out[Le]
        ck, cv = R.cross_kv(w, Ld, o["enc_out"][:B], H)
        ak, av = R.cross_kv(w, Ld, o["enc_out"][:B], H, v_bias_to_k=True)
        note("cross K ulp", _ulps(o["cross_k"][:, :B], ck, et), ULPS["other"], {"V bias on K": _ulps(ak.to(et), ck, et)})
        note("cross V ulp", _ulps(o["cross_v"][:, :B], cv, et), ULPS["other"], {"V bias on K": _ulps(av.to(et), cv, et)})
        note("cross K/V mismatch", max(_mismatch(o["cross_k"][:, :B], ck, et), _mismatch(o["cross_v"][:, :B], cv, et)),
             mm["other"])
        # ---- drift: the whole pass from the mel against the rounding reference
        full = R.encode(w, mel[:B], Le, Ld, H, et=et)
        note("drift enc-out", _rel(o["enc_out"][:B], full["enc_out"]), tol_drift)
        note("drift cross V", _rel(o["cross_v"][:, :B], full["cross_v"]), tol_drift)
        key = (dname, tname, S, B)
        if path == "default":
            _DEFAULT_OUT[key] = {n: o[n].clone() for n in ("x_enc", "enc_out", "cross_k", "cross_v")}
        elif path == "pdl" and key in _DEFAULT_OUT:
            for n, t in _DEFAULT_OUT[key].items():
                assert torch.equal(o[n], t), (n, "BW_ENC_PDL=1 differs from the default")
    # ---- an item's outputs at the two batch sizes: bit-identical on the same GEMM path, else both within the bounds above
    B0, B1 = Bs
    if _same_gemm_path(path, S, B0, B1):
        for d in depths:
            for n in ("x_enc", "qkv", "ao", "hbuf", "enc_out"):
                assert torch.equal(per_b[B0][d][n][:B0], per_b[B1][d][n][:B0]), (d, n, f"B={B0} and B={B1} differ")
            for n in ("cross_k", "cross_v"):
                assert torch.equal(per_b[B0][d][n][:, :B0], per_b[B1][d][n][:, :B0]), (d, n, f"B={B0} and B={B1} differ")
    print(f"\n[{dname} {tname} {path} S={S}] " + "  ".join(f"{k} {v:.2e}" for k, v in worst.items()))
    print("    smallest ablation effects: " + "  ".join(f"{s}/{k} {v:.2e}" for (s, k), v in abl.items()))
    assert not bad, bad


# ------------------------------------------------------------------------------------------------------------------
# the encoder graph replays read the current input
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tname", list(DTYPES))
def test_encode_graph_replay_reads_new_input(cuda, rig, tname):
    """encode(3) twice (the second call captures and replays the graph), encode(1) on other mels, then new mels and a
    replayed encode(3): the outputs are those of a stream call on the new mels, not those of the old ones."""
    S = 500
    engines = rig.build("tiny", tname, "default", S, [DIMS["tiny"][3]], 3)
    eng = next(iter(engines.values()))
    old, new = make_mel(3, S, seed=5), make_mel(3, S, seed=6)
    names = ("enc_out", "cross_k", "cross_v")
    shp = lambda n: (3, S, 128) if n == "enc_out" else (2, 3, 2, S, 64)
    eng.set_mel(new)
    eng.encode(3)
    want = {n: eng.buffer(n, eng.dtype, shp(n)).clone() for n in names}  # the stream call on the new mels
    eng.set_mel(old)
    eng.encode(3)  # captured and replayed
    stale = {n: eng.buffer(n, eng.dtype, shp(n)).clone() for n in names}
    eng.set_mel(new[:1])
    eng.encode(1)
    eng.set_mel(new)
    eng.encode(3)  # replayed
    for n in names:
        got = eng.buffer(n, eng.dtype, shp(n))
        assert torch.equal(got, want[n]), n
        assert not torch.equal(got, stale[n]), n


# ------------------------------------------------------------------------------------------------------------------
# log-mel
# ------------------------------------------------------------------------------------------------------------------
def _pcm_cases(n):
    rng = np.random.RandomState(4)
    t = np.arange(n) / 16000
    imp = np.zeros(n, dtype=np.float32)
    imp[0], imp[-1] = 1.0, -0.8
    return {
        "white noise": (0.1 * rng.randn(n)).astype(np.float32),
        "silence": np.zeros(n, dtype=np.float32),
        "impulses at 0 and n-1": imp,
        "clipped square": np.clip(1.5 * np.sign(np.sin(2 * np.pi * 220 * t)), -1, 1).astype(np.float32),
        "loud": (0.9 * np.sin(2 * np.pi * 1000 * t) + 0.05 * rng.randn(n)).astype(np.float32),
        "quiet": (1e-4 * rng.randn(n)).astype(np.float32),
    }


@pytest.mark.parametrize("tname", list(DTYPES))
def test_logmel_matches_reference(cuda, rig, tname):
    """bw_logmel on batches of three (white noise, silence, reflect-edge impulses; a clipped square, a loud item next to a
    quiet one; then the quiet item again with louder neighbours gone, which needs the per-item maximum reset): the fp32
    mel against the float64 restatement, and mel_tm bit-exactly the rounded fp32 mel with zero pad rows."""
    from oracle import enc_ref as R

    S = 500
    eng = next(iter(rig.build("tiny", tname, "default", S, [0], 3).values()))
    et, F_ = eng.dtype, eng.frames
    cases = _pcm_cases(eng.n_samples)
    batches = [["white noise", "silence", "impulses at 0 and n-1"], ["clipped square", "loud", "quiet"],
               ["quiet", "silence", "white noise"]]
    worst, effects = 0.0, {"symmetric window": 0.0, "reflect off by one": 0.0, "batch-wide max": 0.0}
    for names in batches:
        pcm = np.stack([cases[n] for n in names])
        got = eng.logmel(pcm, return_f32=True).double().cpu().numpy()
        ref = R.logmel(pcm)
        err = float(np.abs(got - ref).max())
        print(f"\n[log-mel {tname}] {', '.join(names)}: max |d| {err:.2e}")
        worst = max(worst, err)
        mt = eng.buffer("mel_tm", et, (3, F_ + 2, 128))
        f32 = torch.from_numpy(got).cuda().float()
        assert torch.equal(mt[:, 1:-1], f32.transpose(1, 2).to(et)), "mel_tm is not the rounded fp32 mel"
        assert not mt[:, 0].any() and not mt[:, -1].any(), "mel_tm pad rows"
        for k, kw in (("symmetric window", dict(symmetric_window=True)), ("reflect off by one", dict(reflect_off_by_one=True)),
                      ("batch-wide max", dict(batch_max=True))):
            effects[k] = max(effects[k], float(np.abs(R.logmel(pcm, **kw) - ref).max()))
    print(f"[log-mel {tname}] worst {worst:.2e} (bound {LOGMEL_ABS:.0e}); ablation effects "
          + "  ".join(f"{k} {v:.2e}" for k, v in effects.items()))
    assert worst < LOGMEL_ABS
    for k, e in effects.items():
        assert e >= 10 * LOGMEL_ABS, (k, e)
