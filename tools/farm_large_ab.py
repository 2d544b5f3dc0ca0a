"""k_farm_response_global against torch.linalg.solve on the same assembled complex128 systems, one GPU.

For each N: the bench farm (bench_extra.farm_designs, 1024 bins, seeded SPD array stiffness) with --cases sea states; the
per-FOWT solve runs once, then
  kernel: DeviceSession.farm_response (assembly of every (case, bin) system + LU + back substitution), CUDA events;
  torch : the same Z_sys [nC*nw, 6N, 6N] and right-hand sides assembled once on the device with torch from the session's
          outputs, then torch.linalg.solve alone is timed (assembly outside the timing).
Both results are compared (max difference over a case's bins relative to its largest amplitude).  Prints one JSON line per N.

Usage: python tools/farm_large_ab.py --turbines 21 32 64 --cases 8 --reps 5
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _events(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def run(N, nC, reps):
    import torch
    import bench_extra
    from raft_b200 import solver
    packs, C_arr, _ = bench_extra.farm_designs(N)
    rng = np.random.default_rng(5)
    cs = dict(Hs=rng.uniform(1, 10, nC), Tp=rng.uniform(5, 18, nC), gamma=np.zeros(nC), beta_deg=rng.uniform(-180, 180, nC),
              spec=np.zeros(nC, dtype=np.int32))
    batch, cases = solver.DesignBatch(packs), solver.CaseTable(cs)
    dev = torch.device("cuda", 0)
    sess = solver.DeviceSession(batch, cases, device=dev, want=("Xi", "status", "B_drag", "F_drag", "F_iner"))
    sess.solve(n_iter=10)
    n, nw = 6 * N, batch.nw
    ms_kernel = _events(lambda: sess.farm_response(C_arr=C_arr), reps)
    kernel = solver.last_dispatch()["kernel"]
    xi = sess._farm[2].clone()                                                        # [nC, n, nw]
    # the same systems assembled with torch: blockdiag(-w^2 M0 + i w (B0 + B_drag) + C0) + C_arr, F = F_drag + F_iner
    w = torch.tensor(packs[0]["w"], dtype=torch.float64, device=dev)
    M0 = torch.tensor(np.stack([P["M0"] for P in packs]), device=dev)
    B0 = torch.tensor(np.stack([P["B0"] for P in packs]), device=dev)
    C0 = torch.tensor(np.stack([P["C0"] for P in packs]), device=dev)
    Bd = sess.out["B_drag"]                                                           # [N, nC, 6, 6]
    Z = torch.zeros([nC, nw, n, n], dtype=torch.complex128, device=dev)
    Z += torch.tensor(C_arr, dtype=torch.complex128, device=dev)
    for i in range(N):
        blk = (-w[None, :, None, None] ** 2 * M0[i] + C0[i]) + 1j * w[None, :, None, None] * (B0[i] + Bd[i])[:, None]
        Z[:, :, 6 * i:6 * i + 6, 6 * i:6 * i + 6] += blk
    F = (sess.out["F_drag"] + sess.out["F_iner"]).permute(1, 0, 2, 3).reshape(nC, n, nw).permute(0, 2, 1).contiguous()
    Zf, Ff = Z.reshape(nC * nw, n, n), F.reshape(nC * nw, n, 1)
    ms_torch = _events(lambda: torch.linalg.solve(Zf, Ff), reps)
    X = torch.linalg.solve(Zf, Ff).reshape(nC, nw, n).permute(0, 2, 1)
    diff = float(((X - xi).abs().amax(dim=(1, 2)) / xi.abs().amax(dim=(1, 2))).max())          # per case, over all bins
    flops = ((8.0 / 3.0) * n ** 3 + 8.0 * n * n) * nC * nw
    res = dict(n_fowt=N, n_dof=n, cases=nC, nw=nw, systems=nC * nw, kernel=kernel, kernel_ms=ms_kernel, torch_solve_ms=ms_torch,
               kernel_gflops=flops / (ms_kernel * 1e-3) / 1e9, torch_gflops=flops / (ms_torch * 1e-3) / 1e9,
               speedup_vs_torch=ms_torch / ms_kernel, max_rel_diff=diff, reps=reps,
               note="kernel time includes the assembly of every system; torch time is torch.linalg.solve alone",
               gpu=torch.cuda.get_device_name(0))
    del sess, Z, F, Zf, Ff, X
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--turbines", type=int, nargs="+", default=[21, 32, 64])
    ap.add_argument("--cases", type=int, default=8)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    for N in args.turbines:
        print(json.dumps(run(N, args.cases, args.reps)), flush=True)


if __name__ == "__main__":
    main()
