#!/usr/bin/env python
"""Device time of the generalised-DOF solve with per-case operating points (raftk_cases.op on raftk_general_*) against the
same solve without them.

The 150-DOF VolturnUS-S-flexible design of the flexops_bem fixture (marin_semi BEM and the rotor node: n_fd = 11), 64 cases
(seeded sea states, one train each), on the fixture's 40 bins and on a 256-bin grid, solved through GeneralSession (tables
resident, CUDA events around solve()).  Variants, alternated round by round in one process so that they see the same card
state: no operating points; n_op = 1 (one point for every case); one point per case (64).  The points are the fixture's
packed points, cycled, regridded by linear interpolation on the 256-bin grid.  Prints the card's name and power limit, then
one line per grid and variant: the median and min of the per-solve device time over the rounds.
Usage: python tools/general_op_timing.py [--rounds R] [--out FILE]"""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return "unknown card"


def regrid(P, fd, ops, nw):
    """The design, fd and operating points on nw bins over the same frequency range (linear interpolation of every w-indexed
    table; wave numbers from the deep-water relation where the grid is new)."""
    w0 = np.asarray(P["w"])
    w = np.linspace(w0[0], w0[-1], nw)
    if nw == len(w0):
        return P, fd, ops
    interp = lambda a: np.apply_along_axis(lambda v: np.interp(w, w0, v.real) + (1j * np.interp(w, w0, v.imag) if np.iscomplexobj(v) else 0), -1, a)  # noqa: E731
    Q = dict(P, w=w, k=np.interp(w, w0, np.asarray(P["k"])), dw=np.float64(w[1] - w[0]))
    if P.get("node_Imat_w") is not None:
        Q["node_Imat_w"] = interp(np.asarray(P["node_Imat_w"]))
    f = dict(fd, A_w=np.ascontiguousarray(interp(fd["A_w"])), B_w=np.ascontiguousarray(interp(fd["B_w"])))
    if fd.get("X_BEM") is not None:
        f["X_BEM"] = np.ascontiguousarray(interp(fd["X_BEM"]))
    o = dict(ops, A_w=np.ascontiguousarray(interp(ops["A_w"])), B_w=np.ascontiguousarray(interp(ops["B_w"])))
    return Q, f, o


def sessions(nC, nw):
    from test_general_operating_points import load_flexops
    from raft_b200 import solver
    P, M, B, Cm, fd, ops, z = load_flexops("bem")
    P, fd, ops = regrid(P, fd, ops, nw)
    rng = np.random.default_rng(1)
    cases = dict(Hs=rng.uniform(1, 9, nC), Tp=rng.uniform(6, 17, nC), gamma=np.zeros(nC), beta_deg=rng.uniform(-180, 180, nC),
                 spec=np.zeros(nC, dtype=np.int32))
    A, Bt = ops["A_w"][0], ops["B_w"][0]                       # [n_op, n_fd, n_fd, nw], cycled to one point per case
    per = np.arange(nC) % len(A)
    variants = [("none", solver.CaseTable(cases)),
                ("n_op = 1", solver.CaseTable(cases, ops=dict(op=np.zeros(nC, np.int32), A_w=A[:1], B_w=Bt[:1]))),
                ("%d ops" % nC, solver.CaseTable(cases, ops=dict(op=np.arange(nC, dtype=np.int32), A_w=A[per], B_w=Bt[per])))]
    return [(name, solver.GeneralSession(P, M, B, Cm, ct, fd=fd)) for name, ct in variants], int(z["n_iter"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from raft_b200 import solver
    lines = ["card: %s" % card()]
    nC = 64
    for nw in (40, 256):
        sess, n_iter = sessions(nC, nw)
        ms, kern = {n: [] for n, _ in sess}, {}
        for n, s in sess:                                   # warm-up: module load, smem opt-in
            s.solve(n_iter=n_iter)
        torch.cuda.synchronize()
        for _ in range(a.rounds):
            for n, s in sess:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                s.solve(n_iter=n_iter)
                e1.record()
                e1.synchronize()
                ms[n].append(e0.elapsed_time(e1))
                kern[n] = solver.last_dispatch()["kernel"]
        for n, _ in sess:
            lines.append("150 DOFs x %d cases x %3d bins  %-9s median %8.3f ms  min %8.3f ms  (%d rounds, kernel %s)"
                         % (nC, nw, n, np.median(ms[n]), np.min(ms[n]), a.rounds, kern[n]))
        del sess
        torch.cuda.empty_cache()
    text = "\n".join(lines)
    print(text)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(text + "\n")


if __name__ == "__main__":
    main()
