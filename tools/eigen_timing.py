#!/usr/bin/env python
"""Natural frequencies and mode shapes on the GPU (solver.solve_eigen, DeviceSession.eigen: raftk_eigen_*) against the host
loop a sweep user writes today, np.linalg.eig(np.linalg.solve(M, C)) on the stacked systems, on one GPU.

Shapes:
  sweep   the 1250 VolturnUS-S geometry variants of bench.py's sweep workload (sweep.build_variants_batched), 6 DOFs:
          DeviceSession.eigen on the resident M0 / C0 (DOF order) against numpy on the same matrices
  flex    256 seeded perturbations (diagonal congruences) of the 150-DOF VolturnUS-S-flexible system of the eigen fixture:
          solve_eigen (host arrays in and out, ascending order) against numpy
  farm24  64 seeded perturbations of the 144-DOF farm of the eigen fixture (DOF order)
  n300    16 seeded systems of 300 DOFs: H in the workspace slab
The arms alternate; a sample is a host-clock window around one call that ends in a device synchronise (GPU arm) or around
the numpy loop (host arm).  Reported: the median ms of each arm, the ratio, the kernel that ran, and the worst eigenvalue
difference against numpy, |lam - lam_np| / max|lam_np| per system after sorting both ascending.  The card's name and power
limit are read (nothing is set) and printed with the numbers.

Usage:  python tools/eigen_timing.py [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def congruences(M, K, nS, seed, amp=0.05):
    rng = np.random.default_rng(seed)
    n = len(M)
    D = 1.0 + amp * rng.uniform(-1, 1, size=(nS, n))
    E = 1.0 + amp * rng.uniform(-1, 1, size=(nS, n))
    return D[:, :, None] * M[None] * D[:, None, :], E[:, :, None] * K[None] * E[:, None, :]


def seeded(n, nS, seed):
    rng = np.random.default_rng(seed)
    A = rng.normal(size=(nS, n, n))
    M = A @ np.swapaxes(A, 1, 2) / n + np.eye(n) * 2.0
    B = rng.normal(size=(nS, n, n))
    return M, (B @ np.swapaxes(B, 1, 2) / n + np.eye(n)) * 100.0


def parity(lam, M, K):
    """worst |lam - lam_np| / max|lam_np| over the systems, both sorted ascending"""
    w = np.linalg.eigvals(np.linalg.solve(M, K))
    a, b = np.sort_complex(np.asarray(lam, dtype=complex)), np.sort_complex(w)
    return float((np.abs(a - b).max(axis=1) / np.abs(b).max(axis=1)).max())


def host_arm(M, K):
    return [np.linalg.eig(np.linalg.solve(M[s], K[s])) for s in range(len(M))]


def timed(fn, sync):
    t0 = time.perf_counter()
    r = fn()
    sync()
    return (time.perf_counter() - t0) * 1e3, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch
    from raft_b200 import solver, sweep
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("card: %s (nvidia-smi; nothing set)   host CPUs: %d   numpy %s" % (q.stdout.strip(), os.cpu_count(), np.__version__))
    dev = torch.device("cuda", 0)
    sync = torch.cuda.synchronize
    nothing = lambda: None  # noqa: E731

    # sweep: bench.py's sweep shard, 6 DOFs per design
    base = json.load(open(os.path.join(ROOT, "tests", "golden", "designs.json")))["cfg2_VolturnUS-S_nw64"]
    z = np.load(os.path.join(ROOT, "tests", "golden", "cfg2_VolturnUS-S_nw64.npz"))
    mats = dict(M_struc=z["P_M0"] - z["A_hydro_morison"], C_struc=z["P_C0"] - z["C_moor"], C_moor=z["C_moor"])
    fac = sweep.sample_factors(1250, seed=40)
    batch = sweep.build_variants_batched(base, mats, fac, nw=64, max_freq=0.40, depth=float(z["P_depth"]))
    cs = solver.CaseTable(dict(Hs=[6.0], Tp=[12.0], gamma=[0.0], beta_deg=[0.0], spec=np.zeros(1, dtype=np.int32)))
    sess = solver.DeviceSession(batch, cs, device=dev)
    Ms = np.array(batch.arrays["M0"]).reshape(-1, 6, 6)
    Ks = np.array(batch.arrays["C0"]).reshape(-1, 6, 6)

    fx = np.load(os.path.join(ROOT, "tests", "golden", "eigen_VolturnUS-S-flexible.npz"))
    f24 = np.load(os.path.join(ROOT, "tests", "golden", "eigen_farm24.npz"))
    shapes = [
        ("sweep 1250 x 6 DOF (DeviceSession.eigen)", Ms, Ks, "dof", lambda: sess.eigen()),
        ("flex 256 x 150 DOF (solve_eigen)", *congruences(fx["M_tot"], fx["C_tot"], 256, 1), "ascending", None),
        ("farm24 64 x 144 DOF (solve_eigen)", *congruences(f24["M_tot"], f24["C_tot"], 64, 2), "dof", None),
        ("n300 16 x 300 DOF (solve_eigen)", *seeded(300, 16, 3), "dof", None),
    ]
    for name, M, K, sort, dev_call in shapes:
        gpu_call = dev_call or (lambda M=M, K=K, sort=sort: solver.solve_eigen(M, K, sort=sort))
        timed(gpu_call, sync)                                         # warm-up: module load, shared-memory opt-in, arena
        kern = solver.last_dispatch()["kernel"]
        tg, th = [], []
        for _ in range(args.reps):
            t, r = timed(gpu_call, sync)
            tg.append(t)
            t, _ = timed(lambda M=M, K=K: host_arm(M, K), nothing)
            th.append(t)
        lam = r["lam"].cpu().numpy() if dev_call else r["lam"]
        info = r["info"].cpu().numpy() if dev_call else r["info"]
        bad = int(np.count_nonzero(info & ~solver.EIG_COMPLEX))
        g, h = float(np.median(tg)), float(np.median(th))
        print("%-44s GPU %9.2f ms   numpy %10.2f ms   x%7.1f   kernel %-13s flagged %d   worst |dlam|/max|lam| %.1e"
              % (name, g, h, h / g, kern, bad, parity(lam, M, K)))


if __name__ == "__main__":
    main()
