#!/usr/bin/env python
"""Cost of the frequency-dependent terms on the generalised-DOF solve: the bench's flex workload (bench_extra.flex_design:
150 DOFs, 200 bins, 64 cases) solved through GeneralSession with fd = None and with fd = BEM coefficients of marin_semi
(bem.read_hydro on tests/golden/wamit_marin_semi.npz at that grid) plus a 12-DOF synthetic rotor block (DOFs 0-5 and
144-149, as tests/golden/make_golden_flexfd.py builds them).  The two are alternated within one run, CUDA events around each
solve, and the card name and power limit are printed with the numbers.

Usage:  python tools/general_fd_timing.py [--reps 7] [--nw 200] [--cases 64]
"""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def fd_tables(P):
    from raft_b200 import bem
    n, w = int(P["gen_nDOF"]), np.asarray(P["w"], dtype=float)
    z = np.load(os.path.join(ROOT, "tests", "golden", "wamit_marin_semi.npz"))
    h = bem.read_hydro(z["A"], z["B"], z["w1"], z["Re"], z["Im"], z["w3"], z["heads"], w)
    idx = np.r_[0:6, n - 6:n].astype(np.int32)
    rng = np.random.default_rng(11)
    A_w, B_w = np.zeros([12, 12, len(w)]), np.zeros([12, 12, len(w)])
    A_w[:6, :6], B_w[:6, :6] = h["A_BEM"], h["B_BEM"]
    s = np.sqrt(np.array([1e5, 1e5, 1e5, 1e7, 1e7, 1e7]))
    for tab, base in ((A_w, 0.2), (B_w, 0.6)):
        G = rng.standard_normal([6, 6])
        S = (G @ G.T / 6.0 + np.eye(6)) * np.outer(s, s) * base
        tab[6:, 6:] = S[:, :, None] * (1.0 + 0.5 * np.sin(w))[None, None, :] / (1.0 + 0.3 * w ** 2)[None, None, :]
    T0 = np.zeros([6, n])
    T0[:, :6] = np.eye(6)
    return dict(fd_idx=idx, A_w=A_w, B_w=B_w, X_BEM=np.ascontiguousarray(h["X_BEM"][:, :6]), bem_headings=h["BEM_headings"],
                heading_adjust=0.0, T0=T0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--nw", type=int, default=200)
    ap.add_argument("--cases", type=int, default=64)
    args = ap.parse_args()
    import torch
    import bench_extra
    from raft_b200 import solver
    dev = torch.device("cuda", 0)
    P, M, B, Cm = bench_extra.flex_design(args.nw)
    nC = args.cases
    rng = np.random.default_rng(6)
    cs = solver.CaseTable(dict(Hs=rng.uniform(1, 10, nC), Tp=rng.uniform(5, 18, nC), gamma=np.zeros(nC), beta_deg=rng.uniform(-180, 180, nC),
                               spec=np.zeros(nC, dtype=np.int32)))
    sess = {"fd=None": solver.GeneralSession(P, M, B, Cm, cs, device=dev),
            "fd": solver.GeneralSession(P, M, B, Cm, cs, device=dev, fd=fd_tables(P))}
    for s in sess.values():
        s.solve(n_iter=10)
    torch.cuda.synchronize()
    times = {k: [] for k in sess}
    for _ in range(args.reps):
        for k, s in sess.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            s.solve(n_iter=10)
            b.record()
            b.synchronize()
            times[k].append(a.elapsed_time(b))
    passes = {k: s.status[:, 0].cpu().numpy() for k, s in sess.items()}
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                            # pragma: no cover
        smi = "nvidia-smi unavailable (%s)" % e
    print("device: %s | %s" % (torch.cuda.get_device_name(0), smi))
    print("shape: %d DOFs, %d bins, %d cases, n_iter 10" % (int(P["gen_nDOF"]), args.nw, nC))
    for k, t in times.items():
        t = np.array(t)
        print("%-8s median %.2f ms  min %.2f  max %.2f  (%d reps)  passes: mean %.2f" % (k, np.median(t), t.min(), t.max(), len(t), passes[k].mean()))
    r = np.array(times["fd"]) / np.array(times["fd=None"])
    print("fd / fd=None per alternation: median %.4f  min %.4f  max %.4f" % (np.median(r), r.min(), r.max()))


if __name__ == "__main__":
    main()
