"""Token selection cases with planted, exactly known logits, and their float64 references (oracle/whisper_ref.select_greedy,
beam_candidates).  tests/test_select_gpu.py runs every case through the real decoder step on every step path.

How the logits are planted: with the final decoder LayerNorm at g = 0, b = beta, every row of the LM-head input is beta
whatever the layers computed, so logits[v] = sum_j beta_j * E[v, j] (E = the tied embedding).  Every beta_j is a power of
two or zero, so beta survives the 16-bit rounding of the batched step.  E holds k * 2^-4 with integer |k| <= 127 and a last
column of 127 * 2^-4 in every row that no case selects, so every row lies on the per-row int8 grid of engine.quantize_rows
(scale 2^-4) and the values are exact in bf16 and fp16.  A case owns one column (its background -127/16 everywhere, its
planted values on its ids) or, when it needs margins finer than 2^-4, three columns weighted 1, 2^-7, 2^-14; every logit
then is a sum of at most three terms within 24 significant bits, so the fp32 dot products of every path (split-K included)
are exact and the kernels see exactly the values the references see.

Each case names the rules it exercises as ablations: the reference with that rule removed or changed (ties to the larger
id, no begin suppression, `>=` for the last allowed initial timestamp, eos in place of pad, no forcing rule, the monotonic
bound off by one, ...) must give a different answer, else the case could not catch that bug.
"""
from __future__ import annotations

import dataclasses
import itertools
from typing import Dict, List, Tuple

import numpy as np
import pytest

from oracle import whisper_ref as R
from thewhisper_b200 import synthetic as S

V = S.VOCAB
EOS, TB, NOTS = S.EOS, S.TIMESTAMP_BEGIN, S.NOTIMESTAMPS
PAD = 50256                                 # a pad id other than eos: a path that writes eos for a finished row is seen
SUPPRESS = sorted(set(S.default_suppress_tokens()) | {4096, 4127})   # + bit 0 and bit 31 of mask word 128
BEGIN_SUPPRESS = list(S.BEGIN_SUPPRESS)      # [220, EOS]
PROMPT = [S.SOT, S.LANG_EN, S.TRANSCRIBE, S.NOTIMESTAMPS]
BG = -127                                    # background code of a case's main column (value -127/16 at beta 1)
FINE = (1.0, 2.0 ** -7, 2.0 ** -14)          # column weights of a fine-margin case (relative to its scale)
MARGINS = (2.0 ** -10, 2.0 ** -13, -2.0 ** -10, -2.0 ** -13)
BEAM_G = (2, 5, 8)


@dataclasses.dataclass
class Case:
    name: str
    group: str
    values: Dict[int, float]                 # planted logits (all other ids: BG / 16 * scale)
    rows: List[Tuple[list, float]]           # per sequence: (generated history, finished flag (greedy) or running score (beam))
    ablations: Tuple[str, ...]
    beam: bool = False
    ts: bool = False
    mit: int = -1
    begin: int = 4
    pad: int = EOS
    scale: float = 1.0                       # beta of the case's main column (a power of two)
    margin: float = float("nan")             # planted probability-rule margin (probability-rule cases)

    def opts(self, **over):
        from thewhisper_b200.engine import DecodeOptions

        kw = dict(eos_token=EOS, pad_token=self.pad, suppress_tokens=SUPPRESS, begin_suppress_tokens=BEGIN_SUPPRESS,
                  timestamp_rules=self.ts, max_initial_timestamp_index=self.mit)
        kw.update(over)
        return DecodeOptions(**kw)

    def prompt(self):
        return PROMPT[:self.begin]

    def seq(self, r):
        return self.prompt() + list(self.rows[r][0])

    @property
    def cur_len(self):
        return self.begin + len(self.rows[0][0])

    def row_spec(self, n):
        """n sequences: the case's rows, cycled."""
        return [self.rows[i % len(self.rows)] for i in range(n)]


def _greedy(name, group, values, abl, hist=(440, 1000), rows=None, **kw):
    rows = rows or [(list(hist), 0), (list(hist), 1), (list(hist), 0)]  # a finished row among the first two (A = 2 cells)
    return Case(name, group, values, rows, tuple(abl), **kw)


def _prob_case(margin):
    """Eight timestamps at 1.0 (each below the best text token) whose log-sum-exp exceeds text id 700 by `margin`."""
    hist = [TB + 2, 500]
    c = _greedy(f"prob{'+' if margin > 0 else '-'}2^{int(np.log2(abs(margin)))}", "probability rule",
                {**{TB + 10 + i: 1.0 for i in range(8)}, 700: 0.0}, ["rule-shift"], hist=hist, ts=True, begin=3, margin=margin)
    row = plant_row(c)
    mask = R.rule_masks(V, c.seq(0), c.begin, c.opts())
    lse = R._logsumexp(np.where(mask, -np.inf, row)[TB:])
    c.values[700] = round((lse - margin) * 2 ** 18) / 2 ** 18
    return c


def greedy_cases() -> List[Case]:
    g = _greedy
    ts = dict(ts=True, begin=3)
    cs = [
        # ties: same row pair of the fused select's LM-head warp, far apart, the same select_kernel thread, three-way
        g("tie-pair", "ties", {6: 5, 7: 5, 9: 4}, ["ties-larger"]),
        g("tie-far", "ties", {7: 5, 51000: 5}, ["ties-larger"]),
        g("tie-thread", "ties", {7: 5, 1031: 5}, ["ties-larger"]),
        g("tie-cta", "ties", {130: 5, 26000: 5}, ["ties-larger"]),
        g("tie-3way", "ties", {300: 5, 25000: 5, 50001: 5}, ["ties-larger"]),
        # best text == best timestamp and every other timestamp ~227 below: logsumexp(ts) equals the max in fp32 and float64,
        # the rule does not fire (a timestamp strictly above the best text always fires it: logsumexp >= max)
        g("tie-text-ts", "ties", {700: 100, TB + 10: 100}, ["ties-larger"], hist=[TB + 2, 500], scale=16.0, **ts),
        # ends of the vocabulary
        g("id-0", "vocab ends", {0: 5, 1: 4}, ["drop-ends"]),
        g("id-last", "vocab ends", {V - 1: 5, V - 2: 4}, ["drop-ends"]),
        g("id-last-ts", "vocab ends", {V - 1: 5, 700: 3}, ["drop-ends"], hist=[TB + 2, 500], **ts),
        g("eos-1-masked", "vocab ends", {EOS - 1: 6, EOS: 5, TB + 5: 2}, ["eos-masked", "no-text-after-ts"], hist=[500, TB + 5], **ts),
        g("eos", "vocab ends", {EOS: 5, 10: 4}, ["no-finish"]),
        # suppression: bit 0 and bit 31 of one mask word, the runner-up in the same word
        g("sup-bit0", "suppression", {4096: 6, 4097: 5}, ["no-suppress"]),
        g("sup-bit31", "suppression", {4127: 6, 4126: 5}, ["no-suppress"]),
        # the first generated step: begin suppression, and one step later
        g("begin-220", "begin step", {220: 6, 221: 5}, ["no-begin-suppress"], hist=[]),
        g("begin-eos", "begin step", {EOS: 6, 1000: 5}, ["no-begin-suppress"], hist=[]),
        g("after-begin-eos", "begin step", {EOS: 6, 1000: 5}, ["begin-always", "no-finish"], hist=[1000]),
        # pad != eos
        g("pad-eos", "finished / pad", {EOS: 6, 10: 5}, ["eos-for-pad"], pad=PAD),
        g("pad-text", "finished / pad", {10: 6}, ["eos-for-pad"], pad=PAD,
          rows=[([440, 1000], 1), ([440, 1000], 0), ([440, 1000], 1)]),
        # timestamp rules
        g("first-step", "timestamp rules", {500: 6, NOTS: 5.5, TB + 1: 2}, ["no-first-text-mask"], hist=[], mit=50, **ts),
        g("first-mit-1", "timestamp rules", {V - 1: 6, TB + 60: 5}, ["mit-50"], hist=[], mit=-1, **ts),
    ]
    for k in (0, 3, 50):
        cs.append(g(f"first-mit{k}-at", "timestamp rules", {TB + k: 6, TB + k + 1: 5}, ["ge-last-allowed"], hist=[], mit=k, **ts))
        cs.append(g(f"first-mit{k}-over", "timestamp rules", {TB + k: 5, TB + k + 1: 6}, ["ge-last-allowed", "no-mit"], hist=[], mit=k,
                    **ts))
    cs += [
        g("text-ts", "timestamp rules", {600: 7, TB + 4: 6, TB + 5: 5, EOS: 4}, ["no-text-after-ts", "mono-excl"], hist=[500, TB + 5], **ts),
        g("ts-ts", "timestamp rules", {TB + 9: 7, 600: 5}, ["no-ts-pair-block"], hist=[500, TB + 5, TB + 7], **ts),
        g("single-ts", "timestamp rules", {TB + 9: 7, 600: 5}, ["penult-short"], hist=[TB + 5], **ts),
        g("ts-text", "timestamp rules", {TB + 5: 7, TB + 6: 6, 600: 1}, ["mono-incl"], hist=[TB + 5, 500], **ts),
        g("nots-masked", "timestamp rules", {NOTS: 7, 600: 6}, ["no-nots-mask"], hist=[TB + 5, 500], **ts),
    ]
    cs += [_prob_case(m) for m in MARGINS]
    return cs


def beam_cases() -> List[Case]:
    runs = [0.0, -1.5, -3.25, -0.5]
    hist, tsh = [440, 1000], [TB + 2, 500]
    b = lambda name, values, abl, h, **kw: Case(name, "beam", values, [(list(h), r) for r in runs], tuple(abl), beam=True, **kw)
    # 18 planted ids, ties straddling positions 2G = 4, 10 and 16; the higher-id member of each tie planted first
    ranked = [(900, 7.0), (800, 6.5), (30, 6.0), (2000, 5.5), (60, 5.5), (3000, 5.0), (3100, 4.75), (51000, 4.5), (12, 4.25),
              (40000, 4.0), (41, 4.0), (5000, 3.75), (5001, 3.5), (6000, 3.25), (7, 3.0), (45000, 2.75), (44999, 2.75),
              (100, 2.5)]
    return [
        b("beam-ties", {**dict(ranked), 4096: 7.5, 4127: 7.25}, ["ties-larger", "no-suppress"], hist),
        b("beam-force", {**{TB + 10 + i: 4.0 - (i // 2) / 16 for i in range(20)}, 700: 4.5, TB + 2: 7.5}, ["no-force"], tsh, ts=True,
          begin=3),
        b("beam-noforce", {700: 7.0, 701: 6.5, 702: 6.5, TB + 3: 5.0, TB + 4: 5.5, TB + 2: 7.5, NOTS: 7.25},
          ["mono-incl", "no-nots-mask"], tsh, ts=True, begin=3),
        b("beam-first-mit3", {TB: 2.0, TB + 1: 3.0, TB + 2: 3.0, TB + 3: 1.0, TB + 4: 5.0, 500: 6.0}, ["no-mit"], [], ts=True, begin=3,
          mit=3),
        b("beam-first-mit0", {TB: 2.0, TB + 1: 5.0, 500: 6.0}, ["no-mit"], [], ts=True, begin=3, mit=0),
    ]


# ------------------------------------------------------------------------------------------------------------------
# planting
# ------------------------------------------------------------------------------------------------------------------
def _codes(x):
    """x = k1/16 + k2/2048 + k3/262144 with |k| <= 127 (x on the 2^-18 grid, |x| < 8)."""
    k1 = int(round(x * 16))
    k2 = int(round((x - k1 / 16) * 2048))
    k3 = int(round((x - k1 / 16 - k2 / 2048) * 2 ** 18))
    assert max(abs(k1), abs(k2), abs(k3)) <= 127 and k1 / 16 + k2 / 2048 + k3 / 2 ** 18 == x, x
    return k1, k2, k3


def _needs_fine(c):
    return any(v / c.scale * 16 != round(v / c.scale * 16) for v in c.values.values())


def plant_row(c):
    """The case's exact logit row (float64 [V])."""
    row = np.full(V, BG / 16 * c.scale)
    for t, v in c.values.items():
        row[t] = v
    return row


def plant(cases, D):
    """-> (E float64 [V, D] of codes / 16, per case its beta float64 [D], its exact logit row float64 [V])."""
    E = np.zeros((V, D))
    E[:, D - 1] = 127 / 16
    col = 0
    betas, rows = [], []
    for c in cases:
        fine = _needs_fine(c)
        cols = [col, col + 1, col + 2] if fine else [col]
        col += len(cols)
        assert col <= D - 1, "more case columns than the embedding has"
        E[:, cols[0]] = BG / 16
        beta = np.zeros(D)
        for j, w in zip(cols, FINE):
            beta[j] = c.scale * w
        for t, v in c.values.items():
            ks = _codes(v / c.scale) if fine else (int(round(v / c.scale * 16)),)
            assert all(abs(k) <= 127 for k in ks), (c.name, t, v)
            for j, k in zip(cols, ks):
                E[t, j] = k / 16
        betas.append(beta)
        rows.append(E @ beta)
    return E, betas, rows


# ------------------------------------------------------------------------------------------------------------------
# ablations: the reference with one rule removed or changed
# ------------------------------------------------------------------------------------------------------------------
def _last_ts(hist):
    return [t for t in hist if t >= TB][-1]


def ablated_kwargs(c, r, abl):
    """-> (opts, reference keyword arguments, finish rule on) for sequence r of case c with ablation `abl`."""
    opts = c.opts()
    seq = c.seq(r)
    hist = c.rows[r][0]
    kw = {}
    mask = lambda o=opts, s=seq: R.rule_masks(V, s, c.begin, o)
    plain = R.rule_masks(V, seq, c.begin, c.opts(timestamp_rules=False))  # suppression only
    finish = True
    if abl == "ties-larger":
        kw["larger_id_ties"] = True
    elif abl == "no-suppress":
        opts = c.opts(suppress_tokens=[])
    elif abl == "no-begin-suppress":
        opts = c.opts(begin_suppress_tokens=[])
    elif abl == "begin-always":
        opts = c.opts(suppress_tokens=sorted(set(SUPPRESS) | set(BEGIN_SUPPRESS)))
    elif abl == "eos-for-pad":
        opts = c.opts(pad_token=EOS)
    elif abl == "no-finish":
        finish = False
    elif abl == "no-force":
        kw["rule_shift"] = -np.inf
    elif abl == "rule-shift":  # a timestamp log-sum-exp off by twice the planted margin, against the planted side
        kw["rule_shift"] = -2 * c.margin
    elif abl == "no-mit":
        opts = c.opts(max_initial_timestamp_index=-1)
    elif abl == "mit-50":
        opts = c.opts(max_initial_timestamp_index=50)
    elif abl == "penult-short":  # a lone generated timestamp read as text -> timestamp
        kw["mask"] = mask(s=c.prompt() + [500] + list(hist))
    else:
        m = mask()
        if abl == "drop-ends":
            m[[0, V - 1]] = True
        elif abl == "eos-masked":  # `v <= eos` for the text below eos
            m[EOS] = True
        elif abl == "no-text-after-ts":
            m[:EOS] = plain[:EOS]
        elif abl == "no-first-text-mask":
            m[:TB] = plain[:TB]
            m[NOTS] = True
        elif abl == "ge-last-allowed":
            m[TB + c.mit] = True
        elif abl == "no-ts-pair-block":
            m[TB:] = plain[TB:]
            m[TB:_last_ts(hist) + 1] = True
        elif abl == "mono-incl":  # the last timestamp allowed again after text
            m[_last_ts(hist)] = False
        elif abl == "mono-excl":  # the last timestamp masked right after it (text -> timestamp)
            m[_last_ts(hist)] = True
        elif abl == "no-nots-mask":
            m[NOTS] = plain[NOTS]
        else:
            raise KeyError(abl)
        kw["mask"] = m
    return opts, kw, finish


def reference(c, row, n_seq, G=1, abl=None):
    """Per sequence of the case's first n_seq rows: greedy (token, finished, margin) or beam (scores, ids, margin)."""
    out = []
    for r, (hist, flag) in enumerate(c.row_spec(n_seq)):
        r0 = r % len(c.rows)
        opts, kw, finish = ablated_kwargs(c, r0, abl) if abl else (c.opts(), {}, True)
        if c.beam:
            out.append(R.beam_candidates(row, c.seq(r0), c.begin, flag, 2 * G, opts, **kw))
        else:
            tok, fin, m = R.select_greedy(row, c.seq(r0), c.begin, bool(flag), opts, **kw)
            out.append((tok, fin if finish else bool(flag), m))
    return out


def _same(a, b):
    if isinstance(a[0], np.ndarray):
        return np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    return a[:2] == b[:2]


ALL = greedy_cases() + beam_cases()


# ------------------------------------------------------------------------------------------------------------------
# tests
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [128, 1280])
def test_planted_values_are_exact(D):
    import torch

    from thewhisper_b200.engine import quantize_rows

    E, betas, rows = plant(ALL, D)
    for dt in (torch.bfloat16, torch.float16):
        assert torch.equal(torch.from_numpy(E).to(dt).double(), torch.from_numpy(E)), dt
    q, s = quantize_rows(torch.from_numpy(E).float())
    assert torch.equal(s, torch.full_like(s, 1 / 16)) and torch.equal(q.double() * s.double()[:, None], torch.from_numpy(E))
    for c, beta, row in zip(ALL, betas, rows):
        nz = np.nonzero(beta)[0]
        for b in beta[nz]:
            assert b == 2.0 ** np.round(np.log2(b)) and torch.tensor(b).half().double() == b, (c.name, b)
        assert np.array_equal(row, plant_row(c)), c.name
        for t in list(c.values) + [V // 2]:  # every partial sum of the (at most three) terms is exact in fp32
            terms = E[t, nz] * beta[nz]
            for k in range(1, len(terms) + 1):
                for sub in itertools.permutations(terms, k):
                    acc = np.float32(0)
                    for x in sub:
                        acc = np.float32(acc + np.float32(x))
                    assert float(acc) == sum(sub), (c.name, t, sub)


def _hf(c, row, r):
    """transformers' processors (+ argmax / topk) on the case's row for sequence r."""
    import torch
    from transformers.generation.logits_process import (SuppressTokensAtBeginLogitsProcessor, SuppressTokensLogitsProcessor,
                                                        WhisperTimeStampLogitsProcessor)

    g = S.make_generation_config("tiny-test")
    g.max_initial_timestamp_index = c.mit if c.mit >= 0 else None
    procs = [SuppressTokensAtBeginLogitsProcessor(BEGIN_SUPPRESS, begin_index=c.begin), SuppressTokensLogitsProcessor(SUPPRESS)]
    if c.ts:
        procs.append(WhisperTimeStampLogitsProcessor(g, begin_index=c.begin))
    x = torch.from_numpy(row.astype(np.float32))[None]
    if c.beam:  # (in float64: torch's fp32 log_softmax over 51866 entries is off by ~1e-4 here)
        x = torch.log_softmax(x.double(), dim=-1)
    ids = torch.tensor([c.seq(r)])
    for p in procs:
        x = p(ids, x)
    if not c.beam:
        return int(x[0].argmax())
    return x[0].double() + c.rows[r][1]


@pytest.mark.parametrize("case", ALL, ids=[c.name for c in ALL])
def test_reference_matches_transformers(case):
    import torch

    row = plant_row(case)
    for r in range(len(case.rows)):
        if not case.beam:
            tok, _, _ = R.select_greedy(row, case.seq(r), case.begin, False, case.opts())
            assert tok == _hf(case, row, r), (case.name, r)
            continue
        hf = _hf(case, row, r)
        for G in BEAM_G:
            n = 2 * G
            scores, ids, _ = R.beam_candidates(row, case.seq(r), case.begin, case.rows[r][1], n, case.opts())
            v, i = torch.topk(hf, n)
            fin = torch.isfinite(v)
            assert int(fin.sum()) == int((ids >= 0).sum()), (case.name, r, G)
            np.testing.assert_allclose(v[fin].numpy(), scores[ids >= 0], rtol=0, atol=1e-9)
            full = np.sort(hf.numpy())[::-1]
            if n < len(full) and full[n - 1] == full[n]:
                continue  # a tie at the boundary: topk may keep either member
            assert set(i[fin].tolist()) == set(ids[ids >= 0].tolist()), (case.name, r, G)


@pytest.mark.parametrize("case", ALL, ids=[c.name for c in ALL])
def test_each_ablation_changes_the_answer(case):
    row = plant_row(case)
    assert case.ablations
    for G in (BEAM_G if case.beam else (1,)):
        n = len(case.rows)
        want = reference(case, row, n, G)
        for abl in case.ablations:
            got = reference(case, row, n, G, abl)
            assert any(not _same(a, b) for a, b in zip(want, got)), (case.name, abl, G)


def test_planted_rule_margins():
    """Margins of the probability-rule cases as planted (within 2^-17 of the target), and one cur_len per case (the step's
    pos is shared by its sequences)."""
    for c in ALL:
        assert len({len(h) for h, _ in c.rows}) == 1, c.name
        if np.isfinite(c.margin):
            _, _, m = R.select_greedy(plant_row(c), c.seq(0), c.begin, False, c.opts())
            assert abs(m - c.margin) < 2 ** -17 and np.sign(m) == np.sign(c.margin), (c.name, m, c.margin)
