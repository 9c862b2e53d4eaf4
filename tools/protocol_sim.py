"""Happens-before simulator for the hand-over protocol of the persistent decoder-step kernels (no GPU needed).

Every CTA is a sequential program of abstract operations -- plain writes / reads of buffer elements with a symbolic version,
commutative adds into an accumulator, release-signal / acquire-wait on counters, grid barriers.  A random scheduler runs the
CTAs; vector clocks decide whether a write happens-before a read (and whether a later write is ordered after every earlier
access of the same element).  The simulator reports deadlocks, reads of the wrong version and unordered (racy) accesses.
It models WHAT synchronises with WHAT in csrc/decode_mega3.cu (and in decode_mega.cu with the V_P2P / V_PROD variants), not
the arithmetic.   python tools/protocol_sim.py [--schedules N]"""
from __future__ import annotations

import argparse
import random
from collections import defaultdict


class Sim:
    def __init__(self, n_cta: int, seed: int):
        self.G = n_cta
        self.rng = random.Random(seed)
        self.vc = [[0] * n_cta for _ in range(n_cta)]
        self.counters = defaultdict(lambda: {"val": 0, "vc": [0] * n_cta})
        self.cells = {}  # (buf, idx) -> {"w": (version, vc), "reads": [vc...], "adds": [vc...]}
        self.errors = []

    @staticmethod
    def hb(a, b):  # vector clock a <= b
        return all(x <= y for x, y in zip(a, b))

    def join(self, b, other):
        self.vc[b] = [max(x, y) for x, y in zip(self.vc[b], other)]

    def tick(self, b):
        self.vc[b][b] += 1

    # ---- memory ----
    def write(self, b, buf, idxs, version):
        self.tick(b)
        now = list(self.vc[b])
        for i in idxs:
            c = self.cells.get((buf, i))
            if c:
                if c["w"] and not self.hb(c["w"][1], now):
                    self.errors.append(f"CTA {b}: write {buf}[{i}]={version} not ordered after write {c['w'][0]}")
                for r in c["reads"]:
                    if not self.hb(r, now):
                        self.errors.append(f"CTA {b}: write {buf}[{i}]={version} races with an earlier read")
                        break
                for r in c["adds"]:
                    if not self.hb(r, now):
                        self.errors.append(f"CTA {b}: write {buf}[{i}]={version} races with an add")
                        break
            self.cells[(buf, i)] = {"w": (version, now), "reads": [], "adds": []}

    def add(self, b, buf, idxs):
        self.tick(b)
        now = list(self.vc[b])
        for i in idxs:
            c = self.cells.get((buf, i))
            if not c or not c["w"]:
                self.errors.append(f"CTA {b}: add into {buf}[{i}] before it was ever cleared")
                continue
            if not self.hb(c["w"][1], now):
                self.errors.append(f"CTA {b}: add into {buf}[{i}] not ordered after the clear")
            if c["reads"]:
                self.errors.append(f"CTA {b}: add into {buf}[{i}] after somebody already read this round")
            c["adds"].append(now)

    def read(self, b, buf, idxs, version=None, n_adds=None):
        self.tick(b)
        now = list(self.vc[b])
        for i in idxs:
            c = self.cells.get((buf, i))
            if not c or not c["w"]:
                self.errors.append(f"CTA {b}: read of unwritten {buf}[{i}]")
                continue
            if not self.hb(c["w"][1], now):
                self.errors.append(f"CTA {b}: read {buf}[{i}] (want {version}) races with write {c['w'][0]}")
            elif version is not None and c["w"][0] != version:
                self.errors.append(f"CTA {b}: read {buf}[{i}] sees {c['w'][0]}, wants {version}")
            if n_adds is not None:
                if len(c["adds"]) != n_adds:
                    self.errors.append(f"CTA {b}: read {buf}[{i}] sees {len(c['adds'])} adds, wants {n_adds}")
                for r in c["adds"]:
                    if not self.hb(r, now):
                        self.errors.append(f"CTA {b}: read {buf}[{i}] races with an add")
                        break
            c["reads"].append(now)

    # ---- run ----
    def run(self, programs):
        pc = [0] * self.G
        arrived = set()
        bar_vc = [0] * self.G
        steps = 0
        while True:
            runnable = []
            for b in range(self.G):
                if pc[b] >= len(programs[b]):
                    continue
                op = programs[b][pc[b]]
                if op[0] == "wait":
                    if self.counters[op[1]]["val"] >= op[2]:
                        runnable.append(b)
                elif op[0] == "barrier":
                    if b not in arrived:
                        runnable.append(b)
                else:
                    runnable.append(b)
            if not runnable:
                if all(pc[b] >= len(programs[b]) for b in range(self.G)):
                    return
                stuck = [(b, programs[b][pc[b]]) for b in range(self.G) if pc[b] < len(programs[b])][:4]
                self.errors.append(f"DEADLOCK: {stuck}")
                return
            b = self.rng.choice(runnable)
            op = programs[b][pc[b]]
            steps += 1
            if op[0] == "w":
                self.write(b, op[1], op[2], op[3])
            elif op[0] == "r":
                self.read(b, op[1], op[2], op[3], op[4] if len(op) > 4 else None)
            elif op[0] == "add":
                self.add(b, op[1], op[2])
            elif op[0] == "signal":  # red.release
                self.tick(b)
                c = self.counters[op[1]]
                c["val"] += 1
                c["vc"] = [max(x, y) for x, y in zip(c["vc"], self.vc[b])]
            elif op[0] == "wait":    # ld.acquire poll
                self.join(b, self.counters[op[1]]["vc"])
            elif op[0] == "merge":   # atom.acq_rel on a per-head counter; the last arriver runs the ops in op[3]
                self.tick(b)
                c = self.counters[op[1]]
                self.join(b, c["vc"])
                c["vc"] = [max(x, y) for x, y in zip(c["vc"], self.vc[b])]
                c["val"] += 1
                if c["val"] == op[2]:
                    programs[b][pc[b] + 1:pc[b] + 1] = list(op[3])
            elif op[0] == "barrier":
                self.tick(b)
                arrived.add(b)
                bar_vc = [max(x, y) for x, y in zip(bar_vc, self.vc[b])]
                if len(arrived) == self.G:
                    for c in range(self.G):
                        self.join(c, bar_vc)
                        pc[c] += 1
                    arrived = set()
                    bar_vc = [0] * self.G
                continue
            pc[b] += 1
            if len(self.errors) > 20:
                return


def rows_of(b, N, G):
    rc = (N + G - 1) // G
    n0 = min(N, b * rc)
    return range(n0, min(N, n0 + rc))


def heads_of(rows, D):
    if len(rows) == 0:
        return []
    h0, h1 = (rows[0] % D) // 64, (rows[-1] % D) // 64
    return [h0] if h0 == h1 else [h0, h1]


def expected(h, D, nblk, rc):
    return sum((b * D + h * 64 + 63) // rc - (b * D + h * 64) // rc + 1 for b in range(nblk))


def mega3_programs(G, D, H, ffn, nsplit, L):
    """One decoder step of csrc/decode_mega3.cu."""
    allD, allF = range(D), range(ffn)
    rs = (D + nsplit - 1) // nsplit
    P = [[] for _ in range(G)]
    for b in range(G):
        p = P[b]
        item = b < H * nsplit
        ih, ij = (b // nsplit, b % nsplit) if item else (0, 0)
        sl = range(min(D, ij * rs), min(D, ij * rs + rs)) if item else range(0)
        if b == 0:
            p.append(("w", "dx", allD, "x0@0"))
        p.append(("barrier",))
        for l in range(L):
            # ---- LN1 + QKV
            p.append(("r", "dx", allD, f"x0@{l}"))
            if b == 0 and l > 0:
                p.append(("w", "accB", allD, f"zeroB@{l}"))
            rq = rows_of(b, 3 * D, G)
            p.append(("w", "dqkv", rq, f"qkv@{l}"))
            p.append(("w", "kv", [(l, r) for r in rq if r >= D], f"kv@{l}"))
            for h in heads_of(rq, D):
                p.append(("signal", ("qkv", h)))
            # ---- self-attention + out-projection slice
            if item:
                p.append(("wait", ("qkv", ih), (l + 1) * expected(ih, D, 3, (3 * D + G - 1) // G)))
                need = [blk * D + ih * 64 + d for blk in range(3) for d in range(64)]
                p.append(("r", "dqkv", need, f"qkv@{l}"))
                p.append(("r", "kv", [(l, r) for r in need if r >= D], f"kv@{l}"))
                p.append(("add", "accA", sl))
            p.append(("barrier",))
            # ---- LN2 + cross-q: x1 = dx + bo + accA -> dx2
            p.append(("r", "dx", allD, f"x0@{l}"))
            p.append(("r", "accA", allD, None, H))
            if b == 0:
                p.append(("w", "dx2", allD, f"x1@{l}"))
            rx = rows_of(b, D, G)
            p.append(("w", "dq", rx, f"xq@{l}"))
            for h in heads_of(rx, D):
                p.append(("signal", ("xq", h)))
            # ---- cross-attention + exchange + out-projection slice
            if item:
                p.append(("wait", ("xq", ih), (l + 1) * expected(ih, D, 1, (D + G - 1) // G)))
                p.append(("r", "dq", [ih * 64 + d for d in range(64)], f"xq@{l}"))
                p.append(("w", "part", [(ih, ij)], f"part@{l}"))
                p.append(("signal", ("xhead", ih)))
                p.append(("wait", ("xhead", ih), (l + 1) * nsplit))
                p.append(("r", "part", [(ih, j) for j in range(nsplit)], f"part@{l}"))
                p.append(("add", "accB", sl))
            p.append(("barrier",))
            # ---- LN3 + fc1: x2 = dx2 + xbo + accB -> dx; accA cleared
            p.append(("r", "dx2", allD, f"x1@{l}"))
            p.append(("r", "accB", allD, None, H))
            if b == 0:
                p.append(("w", "dx", allD, f"x2@{l}"))
                p.append(("w", "accA", allD, f"zeroA@{l}"))
            p.append(("w", "dh", rows_of(b, ffn, G), f"h@{l}"))
            p.append(("barrier",))
            # ---- fc2: x3 = x2 + W2 h, in place
            p.append(("r", "dh", allF, f"h@{l}"))
            p.append(("r", "dx", rows_of(b, D, G), f"x2@{l}"))
            p.append(("w", "dx", rows_of(b, D, G), f"x0@{l + 1}"))
            p.append(("barrier",))
        p.append(("r", "dx", allD, f"x0@{L}"))
        if b == 0:
            p.append(("w", "accB", allD, "zeroB@end"))
    return P


def mega1_programs(G, D, H, ffn, nsplit, L, p2p=False, prod=False):
    """One decoder step of csrc/decode_mega.cu (8 phases per layer); p2p / prod = the V_P2P / V_PROD variants."""
    allD, allF = range(D), range(ffn)
    P = [[] for _ in range(G)]
    for b in range(G):
        p = P[b]
        if b == 0:
            p.append(("w", "dx", allD, "x@0"))
        p.append(("barrier",))
        for l in range(L):
            rq, rd = rows_of(b, 3 * D, G), rows_of(b, D, G)
            # A: LN1 + QKV
            p.append(("r", "dx", allD, f"x@{l}"))
            p.append(("w", "dqkv", rq, f"qkv@{l}"))
            p.append(("w", "kv", [(l, r) for r in rq if r >= D], f"kv@{l}"))
            if p2p:
                for h in heads_of(rq, D):
                    p.append(("signal", ("qkv", h)))
            else:
                p.append(("barrier",))
            # B: self-attention, CTA = head
            if b < H:
                if p2p:
                    p.append(("wait", ("qkv", b), (l + 1) * expected(b, D, 3, (3 * D + G - 1) // G)))
                need = [blk * D + b * 64 + d for blk in range(3) for d in range(64)]
                p.append(("r", "dqkv", need, f"qkv@{l}"))
                p.append(("r", "kv", [(l, r) for r in need if r >= D], f"kv@{l}"))
                p.append(("w", "dattn", range(b * 64, b * 64 + 64), f"a@{l}"))
                if prod:
                    p.append(("signal", ("prodB",)))
            if prod:
                p.append(("wait", ("prodB",), (l + 1) * H))
            else:
                p.append(("barrier",))
            # C: out-proj + residual
            p.append(("r", "dattn", allD, f"a@{l}"))
            p.append(("r", "dx", rd, f"x@{l}"))
            p.append(("w", "dx", rd, f"x1@{l}"))
            p.append(("barrier",))
            # D: LN2 + cross-q
            p.append(("r", "dx", allD, f"x1@{l}"))
            p.append(("w", "dq", rd, f"xq@{l}"))
            if p2p:
                for h in heads_of(rd, D):
                    p.append(("signal", ("xq", h)))
            else:
                p.append(("barrier",))
            # E: cross-attention, (head, split) items.  Shipped: every split only writes its partials, and every CTA merges all
            # of them while staging F (writing its own rows of dattn); V_PROD: the last-arriving split of a head merges
            if b < H * nsplit:
                h, j = b // nsplit, b % nsplit
                if p2p:
                    p.append(("wait", ("xq", h), (l + 1) * expected(h, D, 1, (D + G - 1) // G)))
                p.append(("r", "dq", [h * 64 + d for d in range(64)], f"xq@{l}"))
                p.append(("w", "part", [(h, j)], f"part@{l}"))
                if prod:
                    tail = [("r", "part", [(h, jj) for jj in range(nsplit)], f"part@{l}"),
                            ("w", "dattn", range(h * 64, h * 64 + 64), f"a2@{l}"), ("signal", ("prodE",))]
                    p.append(("merge", ("xc", h), (l + 1) * nsplit, tail))
            if prod:
                p.append(("wait", ("prodE",), (l + 1) * H))
            else:
                p.append(("barrier",))
            # F: cross out-proj + residual
            if prod:
                p.append(("r", "dattn", allD, f"a2@{l}"))
            else:
                p.append(("r", "part", [(h, jj) for h in range(H) for jj in range(nsplit)], f"part@{l}"))
                p.append(("w", "dattn", rd, f"a2@{l}"))
            p.append(("r", "dx", rd, f"x1@{l}"))
            p.append(("w", "dx", rd, f"x2@{l}"))
            p.append(("barrier",))
            # G: LN3 + fc1
            p.append(("r", "dx", allD, f"x2@{l}"))
            p.append(("w", "dh", rows_of(b, ffn, G), f"h@{l}"))
            p.append(("barrier",))
            # H: fc2 + residual
            p.append(("r", "dh", allF, f"h@{l}"))
            p.append(("r", "dx", rd, f"x2@{l}"))
            p.append(("w", "dx", rd, f"x@{l + 1}"))
            p.append(("barrier",))
        p.append(("r", "dx", allD, f"x@{L}"))
    return P


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--schedules", type=int, default=20)
    args = ap.parse_args()
    G, D, H, ffn, nsplit, L = 24, 256, 4, 384, 5, 3
    bad = 0
    for seed in range(args.schedules):
        sim = Sim(G, seed)
        # state at kernel start: both accumulators are clear (bw_decode_begin / the previous step)
        sim.write(0, "accA", range(D), "zeroA@start")
        sim.write(0, "accB", range(D), "zeroB@start")
        sim.vc = [list(sim.vc[0]) for _ in range(G)]  # (the launch boundary orders everything before the kernel)
        sim.run(mega3_programs(G, D, H, ffn, nsplit, L))
        if sim.errors:
            bad += 1
            print(f"schedule {seed}: {len(sim.errors)} problems, first: {sim.errors[0]}")
    print(f"decode_mega3 protocol: {args.schedules - bad}/{args.schedules} random schedules clean "
          f"(G={G} CTAs, D={D}, H={H}, nsplit={nsplit}, L={L})")
    total_bad = bad
    for p2p, prod in ((False, False), (True, False), (False, True), (True, True)):
        bad = 0
        for seed in range(args.schedules):
            sim = Sim(G, 1000 + seed)
            sim.run(mega1_programs(G, D, H, ffn, nsplit, L, p2p, prod))
            if sim.errors:
                bad += 1
                print(f"  decode_mega p2p={p2p} prod={prod} schedule {seed}: first problem: {sim.errors[0]}")
        print(f"decode_mega protocol (V_P2P={p2p}, V_PROD={prod}): {args.schedules - bad}/{args.schedules} random schedules clean")
        total_bad += bad
    return 1 if total_bad else 0


if __name__ == "__main__":
    raise SystemExit(main())
