#!/usr/bin/env python
"""Streamed generalised-DOF solve (raftk_general_solve_dynamics_stream_dev through GeneralSession(max_chunk_cases=K)) on one GPU.

1. The bench's flex workload (bench_extra.flex_design: 150 DOFs, 200 bins, 64 cases): the single-table entry and the streamed
   one at chunks of 64, 16 and 4 cases, alternated within one run, CUDA events around each solve: the cost of the chunking.
2. A table the single-table entry cannot allocate on an 80 GB card: 150 DOFs x 1024 bins x 256 cases (about 98 GB of
   workspace in one piece), streamed under a 16 GiB budget (solver.general_chunk_for_budget): cases and (case, bin) systems
   solved per second.

Every streamed result is compared with the single-table one where both fit (bit for bit).  The card name and power limit are
printed with the numbers.

Usage:  python tools/general_stream_timing.py [--reps 5] [--big-reps 2] [--budget-gb 16]
"""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def sea_states(nC, seed):
    from raft_b200 import solver
    rng = np.random.default_rng(seed)
    return solver.CaseTable(dict(Hs=rng.uniform(1, 10, nC), Tp=rng.uniform(5, 18, nC), gamma=np.zeros(nC),
                                 beta_deg=rng.uniform(-180, 180, nC), spec=np.zeros(nC, dtype=np.int32)))


def timed(torch, fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--big-reps", type=int, default=2)
    ap.add_argument("--budget-gb", type=float, default=16.0)       # GiB
    ap.add_argument("--big-nw", type=int, default=1024)
    ap.add_argument("--big-cases", type=int, default=256)
    args = ap.parse_args()
    import torch
    import bench_extra
    from raft_b200 import solver
    dev = torch.device("cuda", 0)
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                            # pragma: no cover
        smi = "nvidia-smi unavailable (%s)" % e
    print("device: %s | %s" % (torch.cuda.get_device_name(0), smi))

    # 1. the bench flex shape, single table against chunks
    P, M, B, Cm = bench_extra.flex_design(200)
    n, nC = int(P["gen_nDOF"]), 64
    cs = sea_states(nC, 6)
    sess = {"single": solver.GeneralSession(P, M, B, Cm, cs, device=dev)}
    for K in (64, 16, 4):
        sess["chunk %d" % K] = solver.GeneralSession(P, M, B, Cm, cs, device=dev, max_chunk_cases=K)
    for s in sess.values():
        s.solve(n_iter=10)
    torch.cuda.synchronize()
    ref = sess["single"].Xi.cpu().numpy(), sess["single"].status.cpu().numpy()
    same = {k: np.array_equal(s.Xi.cpu().numpy(), ref[0]) and np.array_equal(s.status.cpu().numpy(), ref[1]) for k, s in sess.items()}
    times = {k: [] for k in sess}
    for _ in range(args.reps):
        for k, s in sess.items():
            times[k].append(timed(torch, lambda: s.solve(n_iter=10)))
    print("flex shape: %d DOFs, 200 bins, %d cases, n_iter 10; passes: mean %.2f" % (n, nC, ref[1][:, 0].mean()))
    t0 = np.median(times["single"])
    for k, t in times.items():
        t = np.array(t)
        print("  %-9s workspace %7.2f GB  median %8.2f ms  min %8.2f  max %8.2f  (%d reps)  vs single %.3fx  bit-identical: %s"
              % (k, sess[k].workspace_bytes / 1e9, np.median(t), t.min(), t.max(), len(t), np.median(t) / t0, same[k]))
    del sess
    torch.cuda.empty_cache()

    # 2. a table the single-table entry cannot allocate
    nw, nC = args.big_nw, args.big_cases
    P, M, B, Cm = bench_extra.flex_design(nw)
    cs = sea_states(nC, 7)
    budget = int(args.budget_gb * (1 << 30))
    single = solver.general_stream_workspace_bytes(P, None, None, nC, 0)
    K = solver.general_chunk_for_budget(P, None, None, nC, budget)
    s = solver.GeneralSession(P, M, B, Cm, cs, device=dev, max_chunk_cases=K)
    s.solve(n_iter=10)
    torch.cuda.synchronize()
    t = np.array([timed(torch, lambda: s.solve(n_iter=10)) for _ in range(args.big_reps)])
    st = s.status.cpu().numpy()
    ms = np.median(t)
    print("big table: %d DOFs, %d bins, %d cases, n_iter 10: single-table workspace %.1f GB; streamed in chunks of %d cases "
          "(%d chunks) in %.2f GB (budget %.1f GB)" % (n, nw, nC, single / 1e9, K, -(-nC // K), s.workspace_bytes / 1e9, budget / 1e9))
    print("  median %.1f ms  min %.1f  max %.1f  (%d reps): %.1f cases/s, %.0f (case, bin) systems/s per pass-set; passes: mean %.2f, "
          "converged %d/%d, flags %d" % (ms, t.min(), t.max(), len(t), nC / (ms / 1e3), nC * nw / (ms / 1e3), st[:, 0].mean(),
                                        int(st[:, 1].sum()), nC, int((st[:, 2] != 0).sum())))


if __name__ == "__main__":
    main()
