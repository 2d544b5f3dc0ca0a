#!/usr/bin/env python
"""Batches of farms (DeviceSession.farm_response(n_fowt=N): raftk_farm_batch_response_ws_dev) against one DeviceSession
solve + farm_response per farm, on one GPU.

Shapes: the shipped farm (N = 2 FOWTs, 100 bins, 1 case) and N = 8, each for F = 64 and F = 512 candidate layouts.  Farm f is
bench_extra.farm_designs' array with every FOWT moved by a seeded offset of up to 400 m and a seeded SPD array stiffness of
its own.  Both arms work on device-resident tables and run the per-FOWT drag linearisation and the system response:

  loop   F sessions of N designs: solve() + farm_response() on each, one device synchronise at the end
  batch  one session of F * N designs: solve() + farm_response(n_fowt=N), one device synchronise

The arms alternate within one process; a sample is a host-clock window around `inner` repetitions ending in the synchronise,
with `inner` chosen so that a window lasts at least --window seconds.  Reported: ms per sweep of F farms for each arm, the
ratio, and whether Xi_sys / info of the two arms are bit-identical.  The card's name, power limit and clocks are read
(nothing is set) and printed with the numbers.

Usage:  python tools/farm_batch_timing.py [--reps 7] [--window 0.25] [--farms 64 512] [--fowts 2 8]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def layouts(N, F, nw):
    """-> (packs [F][N], C_arr [F,6N,6N]): farm 0 on the 1600 m grid, the others with every FOWT moved (member ends and
    reference point together) and their own array stiffness."""
    import bench_extra
    base, C0, _ = bench_extra.farm_designs(N, nw=nw, max_freq=0.002 * nw)
    rng = np.random.default_rng(100 * N + F)
    packs, C_arr = [base], [C0]
    for f in range(1, F):
        row = []
        for P in base:
            r = np.append(rng.uniform(-400.0, 400.0, size=2), 0.0)
            Q = dict(P)
            for k in ("mem_rA", "node_r", "prp"):
                Q[k] = np.asarray(P[k], dtype=float) + r
            Q["x_ref"], Q["y_ref"] = float(P["x_ref"]) + r[0], float(P["y_ref"]) + r[1]
            row.append(Q)
        packs.append(row)
        A = rng.normal(size=(6 * N, 6 * N)) * 2e4
        C_arr.append(A @ A.T / (6 * N) + np.diag([5e4] * (6 * N)))
    return packs, np.array(C_arr)


def compare(torch, solver, N, F, nw, reps, window):
    dev = torch.device("cuda", 0)
    packs, C_arr = layouts(N, F, nw)
    cs = solver.CaseTable(dict(Hs=np.array([6.0]), Tp=np.array([12.0]), gamma=np.zeros(1), beta_deg=np.zeros(1), spec=np.zeros(1, dtype=np.int32)))
    want = ("Xi", "status", "B_drag", "F_drag", "F_iner")
    batch = solver.DeviceSession(solver.DesignBatch([P for row in packs for P in row]), cs, device=dev, want=want)
    loop = [solver.DeviceSession(solver.DesignBatch(row), cs, device=dev, want=want) for row in packs]

    def run_batch():
        batch.solve(n_iter=10)
        return batch.farm_response(C_arr=C_arr, n_fowt=N)

    def run_loop():
        return [(s.solve(n_iter=10), s.farm_response(C_arr=C_arr[f]))[1] for f, s in enumerate(loop)]

    xb, ib = run_batch()
    kernel = solver.last_dispatch()["kernel"]
    single = run_loop()
    torch.cuda.synchronize()
    same = all(np.array_equal(xb[f].cpu().numpy(), x.cpu().numpy()) and np.array_equal(ib[f].cpu().numpy(), i.cpu().numpy())
               for f, (x, i) in enumerate(single))

    def sample(fn, inner):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(inner):
            fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / inner * 1e3

    inner = {}
    for name, fn in (("batch", run_batch), ("loop", run_loop)):       # warm-up doubles as the choice of `inner`
        sample(fn, 2)
        inner[name] = max(1, int(np.ceil(window * 1e3 / sample(fn, 3))))
    tb, tl = [], []
    for _ in range(reps):                                              # alternated
        tb.append(sample(run_batch, inner["batch"]))
        tl.append(sample(run_loop, inner["loop"]))
    tb, tl = np.array(tb), np.array(tl)
    passes = batch.out["status"][..., 0].float().mean().item()
    print("N = %d FOWTs x F = %d farms, %d bins, 1 case, n_iter 10 (passes: mean %.2f); system kernel %s" % (N, F, nw, passes, kernel))
    print("  batch  median %9.3f ms per sweep (min %9.3f, max %9.3f; %d sweeps per sample) = %8.2f us per farm"
          % (np.median(tb), tb.min(), tb.max(), inner["batch"], np.median(tb) / F * 1e3))
    print("  loop   median %9.3f ms per sweep (min %9.3f, max %9.3f; %d sweeps per sample) = %8.2f us per farm"
          % (np.median(tl), tl.min(), tl.max(), inner["loop"], np.median(tl) / F * 1e3))
    print("  loop / batch %.2fx over %d alternated samples; Xi_sys and info bit-identical: %s" % (np.median(tl) / np.median(tb), reps, same))
    del batch, loop
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--window", type=float, default=0.25)
    ap.add_argument("--farms", type=int, nargs="+", default=[64, 512])
    ap.add_argument("--fowts", type=int, nargs="+", default=[2, 8])
    ap.add_argument("--nw", type=int, default=100)
    args = ap.parse_args()
    import torch
    from raft_b200 import solver
    if not torch.cuda.is_available():
        raise SystemExit("farm_batch_timing.py measures on a CUDA device; none is available")
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm,clocks.mem", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                            # pragma: no cover
        smi = "nvidia-smi unavailable (%s)" % e
    print("device: %s | name, power limit, max SM clock, SM clock, memory clock: %s" % (torch.cuda.get_device_name(0), smi))
    for N in args.fowts:
        for F in args.farms:
            compare(torch, solver, N, F, args.nw, args.reps, args.window)


if __name__ == "__main__":
    main()
