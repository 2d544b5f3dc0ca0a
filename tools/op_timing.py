#!/usr/bin/env python
"""Device time of the rigid solve with per-case operating points (raftk_cases.op) against the same solve without them.

Two shapes, each solved through DeviceSession (tables resident, CUDA events around solve()), the variants alternated round by
round in one process so that they see the same card state:
  cfg2   VolturnUS-S, 1 design x 64 cases x 1024 bins (bench.py's cfg2 shape)
  sweep  1250 copies of that design x 16 cases x 256 bins (one GPU's shard of a design sweep)
Variants: no tables; a design-level A_w / B_w; 8 operating points shared by every design (op_shared = 1); one operating point
per case (64 for cfg2, 16 for the sweep).  Prints the card's name and power limit, then one line per shape and variant:
the median and min of the per-solve device time over the rounds.
Usage: python tools/op_timing.py [--rounds R] [--out FILE]"""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return "unknown card"


def shape(nD, nC, nw):
    from raft_b200 import grid, solver
    z = np.load(os.path.join(ROOT, "tests", "golden", "cfg2_VolturnUS-S_nw64.npz"))
    P = grid.regrid({k[2:]: z[k] for k in z.files if k.startswith("P_")}, nw, 0.512)
    rng = np.random.default_rng(1)
    cases = dict(Hs=rng.uniform(1, 9, nC), Tp=rng.uniform(6, 17, nC), gamma=np.zeros(nC), beta_deg=rng.uniform(-180, 180, nC),
                 spec=np.zeros(nC, dtype=np.int32))
    M = np.abs(np.asarray(P["M0"])).max()

    def tables(lead):
        A = rng.normal(size=lead + (6, 6, nw)) * 0.01 * M / 36
        B = np.abs(rng.normal(size=lead + (6, 6, nw))) * 2e4
        return A, B
    A1, B1 = tables(())
    Pw = dict(P, A_w=A1, B_w=B1)
    A8, B8 = tables((8,))
    An, Bn = tables((nC,))
    variants = [("none", [P] * nD, solver.CaseTable(cases)),
                ("design A_w", [Pw] * nD, solver.CaseTable(cases)),
                ("8 shared ops", [P] * nD, solver.CaseTable(cases, ops=dict(op=np.arange(nC, dtype=np.int32) % 8, A_w=A8, B_w=B8))),
                ("%d ops" % nC, [P] * nD, solver.CaseTable(cases, ops=dict(op=np.arange(nC, dtype=np.int32), A_w=An, B_w=Bn)))]
    return [(name, solver.DeviceSession(solver.DesignBatch(packs), ct)) for name, packs, ct in variants]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from raft_b200 import solver
    lines = ["card: %s" % card()]
    for label, dims in (("cfg2", (1, 64, 1024)), ("sweep", (1250, 16, 256))):
        sess = shape(*dims)
        ms, kern = {n: [] for n, _ in sess}, {}
        for n, s in sess:                                   # warm-up: module load, plan blobs
            s.solve()
        torch.cuda.synchronize()
        for _ in range(a.rounds):
            for n, s in sess:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                s.solve()
                e1.record()
                e1.synchronize()
                ms[n].append(e0.elapsed_time(e1))
                kern[n] = solver.last_dispatch()["kernel"]
        for n, _ in sess:
            lines.append("%-5s %d designs x %d cases x %d bins  %-14s median %8.3f ms  min %8.3f ms  (%d rounds, kernel %s)"
                         % ((label,) + dims + (n, np.median(ms[n]), np.min(ms[n]), a.rounds, kern[n])))
        del sess
        torch.cuda.empty_cache()
    text = "\n".join(lines)
    print(text)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(text + "\n")


if __name__ == "__main__":
    main()
