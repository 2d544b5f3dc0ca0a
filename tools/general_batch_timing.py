#!/usr/bin/env python
"""Design batches of flexible FOWTs (raftk_general_batch_solve_dynamics_dev through GeneralBatchSession) against one
GeneralSession solve per design, on one GPU.

1. The VolturnUS-S-flexible fixture (150 DOFs, 40 bins), 6 seeded sea states, 64 seeded variants (M / C entries scaled by up to
   1 %, drag coefficients by 0.9-1.1): one batched device-resident solve against a loop of 64 GeneralSession solves on the
   same tables.
2. The bench's flex shape (bench_extra.flex_design: 150 DOFs, 200 bins, 64 cases) for a few variants, where one design's
   call already fills the GPU.

The two arms alternate within one run; each ends in a device synchronise and is timed with CUDA events.  Reported: ms per
design for each arm and whether the outputs (Xi, status) are bit-identical.  The card name and power limit are printed with
the numbers.

Usage:  python tools/general_batch_timing.py [--reps 5] [--variants 64] [--flex-variants 3]
"""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def sea_states(nC, seed):
    from raft_b200 import solver
    rng = np.random.default_rng(seed)
    return solver.CaseTable(dict(Hs=rng.uniform(1, 10, nC), Tp=rng.uniform(5, 18, nC), gamma=np.zeros(nC),
                                 beta_deg=rng.uniform(-180, 180, nC), spec=np.zeros(nC, dtype=np.int32)))


def variants(P, M, B, Cm, count, seed):
    """Design 0 as given, then seeded variants: M / C entries scaled (symmetrically) by up to 1 %, drag coefficients by 0.9-1.1."""
    rng = np.random.default_rng(seed)
    out = [(P, M, B, Cm)]
    for _ in range(count - 1):
        M1 = M * (1.0 + 0.01 * rng.uniform(-1, 1, M.shape))
        C1 = Cm * (1.0 + 0.01 * rng.uniform(-1, 1, Cm.shape))
        P1 = dict(P)
        for k in ("node_Cd_q", "node_Cd_p1", "node_Cd_p2", "node_Cd_End"):
            P1[k] = np.asarray(P[k]) * rng.uniform(0.9, 1.1, np.shape(P[k]))
        out.append((P1, 0.5 * (M1 + M1.T), B, 0.5 * (C1 + C1.T)))
    return out


def compare(torch, solver, designs, cs, reps, label):
    dev = torch.device("cuda", 0)
    batch = solver.GeneralBatchSession(designs, cs, device=dev)
    loop = [solver.GeneralSession(P, M, B, Cm, cs, device=dev) for P, M, B, Cm in designs]

    def run_batch():
        batch.solve(n_iter=10)
        torch.cuda.synchronize()

    def run_loop():
        for s in loop:
            s.solve(n_iter=10)
        torch.cuda.synchronize()
    run_batch()
    run_loop()
    same = all(np.array_equal(batch.Xi[d].cpu().numpy(), s.Xi.cpu().numpy()) and np.array_equal(batch.status[d].cpu().numpy(), s.status.cpu().numpy())
               for d, s in enumerate(loop))
    tb, tl = [], []
    for _ in range(reps):                              # alternated
        for fn, acc in ((run_batch, tb), (run_loop, tl)):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            acc.append(a.elapsed_time(b))
    nD = len(designs)
    st = batch.status.cpu().numpy()
    tb, tl = np.array(tb), np.array(tl)
    print("%s: %d designs x %d cases, %d DOFs, %d bins, n_iter 10; passes: mean %.2f; batch workspace %.2f GB"
          % (label, nD, cs.n_cases, batch.n, batch.nw, st[..., 0].mean(), batch.workspace_bytes / 1e9))
    print("  batched solve     median %9.2f ms (min %9.2f, max %9.2f)  = %7.3f ms per design" % (np.median(tb), tb.min(), tb.max(), np.median(tb) / nD))
    print("  loop of sessions  median %9.2f ms (min %9.2f, max %9.2f)  = %7.3f ms per design" % (np.median(tl), tl.min(), tl.max(), np.median(tl) / nD))
    print("  loop / batch %.3fx over %d alternated reps; outputs bit-identical: %s" % (np.median(tl) / np.median(tb), reps, same))
    del batch, loop
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--variants", type=int, default=64)
    ap.add_argument("--flex-variants", type=int, default=3)
    args = ap.parse_args()
    import torch
    import bench_extra
    from raft_b200 import solver
    from test_general_stream import _flexout
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                            # pragma: no cover
        smi = "nvidia-smi unavailable (%s)" % e
    print("device: %s | %s" % (torch.cuda.get_device_name(0), smi))
    P, M, B, Cm, _, _, _ = _flexout()
    compare(torch, solver, variants(P, M, B, Cm, args.variants, 1), sea_states(6, 6), args.reps, "VolturnUS-S-flexible")
    P, M, B, Cm = bench_extra.flex_design(200)
    compare(torch, solver, variants(P, M, B, Cm, args.flex_variants, 2), sea_states(64, 6), args.reps, "bench flex shape")


if __name__ == "__main__":
    main()
