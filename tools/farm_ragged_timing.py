#!/usr/bin/env python
"""A ragged farm batch (DeviceSession.farm_response(farm_sizes=...): raftk_farm_ragged_response_ws_dev) against the two ways
a mixed-size study ran before it, on one GPU (profiles/h100_farm_ragged.txt).

Workload: --farms farms whose sizes cycle through --sizes (default 32 farms of N in {2, 4, 8, 16, 32, 64}), one case, --nw
bins.  The farms of size N are tools/farm_batch_timing.layouts(N, F_N): bench_extra.farm_designs' array with every FOWT
moved by a seeded offset and a seeded SPD array stiffness of its own.  Every arm works on device-resident tables and runs the
per-FOWT drag linearisation and the coupled system response:

  ragged   one session of every farm's FOWTs: solve() + farm_response(farm_sizes=sizes)
  per-N    (a) one session per distinct N: solve() + farm_response(n_fowt=N) on each
  per-farm (b) one session per farm: solve() + farm_response() on each

The arms alternate within one process.  A sample is CUDA events recorded on the current stream around `inner` repetitions
of an arm, `inner` chosen so that a window lasts at least --window seconds.  Reported: ms per sweep of the whole study for
each arm (median and range over --reps samples), the speed-ups of the ragged call over (a) and (b), and whether every farm's
Xi_sys / info are bit-identical across the three arms.  The card's name, power limit and clocks are read (nothing is set)
and printed with the numbers.

Usage:  python tools/farm_ragged_timing.py [--reps 7] [--window 0.5] [--farms 32] [--sizes 2 4 8 16 32 64] [--nw 50]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--window", type=float, default=0.5)
    ap.add_argument("--farms", type=int, default=32)
    ap.add_argument("--sizes", type=int, nargs="+", default=[2, 4, 8, 16, 32, 64])
    ap.add_argument("--nw", type=int, default=50)
    args = ap.parse_args()
    import torch
    from farm_batch_timing import layouts
    from raft_b200 import solver
    assert torch.cuda.is_available(), "this measurement needs a CUDA device"
    dev = torch.device("cuda", 0)
    sizes = [args.sizes[f % len(args.sizes)] for f in range(args.farms)]
    distinct = sorted(set(sizes))
    by_n = {N: layouts(N, sizes.count(N), args.nw) for N in distinct}
    packs, C_arr, seen = [], [], {N: 0 for N in distinct}
    for N in sizes:                                      # farm order of the ragged batch: the sizes interleaved
        packs.append(by_n[N][0][seen[N]])
        C_arr.append(by_n[N][1][seen[N]])
        seen[N] += 1
    cs = solver.CaseTable(dict(Hs=np.array([6.0]), Tp=np.array([12.0]), gamma=np.zeros(1), beta_deg=np.zeros(1), spec=np.zeros(1, dtype=np.int32)))
    want = ("Xi", "status", "B_drag", "F_drag", "F_iner")
    rag = solver.DeviceSession(solver.DesignBatch([P for row in packs for P in row]), cs, device=dev, want=want)
    per_n = {N: solver.DeviceSession(solver.DesignBatch([P for row in by_n[N][0] for P in row]), cs, device=dev, want=want) for N in distinct}
    per_farm = [solver.DeviceSession(solver.DesignBatch(row), cs, device=dev, want=want) for row in packs]

    def run_ragged():
        rag.solve(n_iter=10)
        return rag.farm_response(C_arr=C_arr, farm_sizes=sizes)

    def run_per_n():
        return {N: (s.solve(n_iter=10), s.farm_response(C_arr=by_n[N][1], n_fowt=N))[1] for N, s in per_n.items()}

    def run_per_farm():
        return [(s.solve(n_iter=10), s.farm_response(C_arr=C_arr[f]))[1] for f, s in enumerate(per_farm)]

    xr, ir = run_ragged()
    classes = solver.last_dispatch()["farm_classes"]
    xn, xf = run_per_n(), run_per_farm()
    torch.cuda.synchronize()
    same, seen = True, {N: 0 for N in distinct}
    for f, N in enumerate(sizes):
        k = seen[N]
        seen[N] += 1
        a, ia = xr[f].cpu().numpy(), ir[f].cpu().numpy()
        same &= np.array_equal(a, xn[N][0][k].cpu().numpy()) and np.array_equal(ia, xn[N][1][k].cpu().numpy())
        same &= np.array_equal(a, xf[f][0].cpu().numpy()) and np.array_equal(ia, xf[f][1].cpu().numpy())

    def sample(fn, inner):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(inner):
            fn()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) / inner

    arms = (("ragged", run_ragged), ("per-N", run_per_n), ("per-farm", run_per_farm))
    inner = {}
    for name, fn in arms:                                # warm-up, then the repetitions that fill one window
        fn()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        inner[name] = max(1, int(args.window / max(time.perf_counter() - t0, 1e-6)))
    ms = {name: [] for name, _ in arms}
    for _ in range(args.reps):
        for name, fn in arms:
            ms[name].append(sample(fn, inner[name]))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    med = {k: float(np.median(v)) for k, v in ms.items()}
    print("card: %s" % q)
    print("study: %d farms, sizes %s (%d FOWTs), 1 case, %d bins; ragged call launched %s" % (len(sizes), sizes, sum(sizes), args.nw,
                                                                                           ", ".join(classes)))
    for name, _ in arms:
        print("%-9s %9.3f ms per study (median of %d, range %.3f - %.3f; %d calls per window)" % (
            name, med[name], args.reps, min(ms[name]), max(ms[name]), inner[name]))
    print("speed-up of the ragged call: %.2fx over one call per distinct N (a), %.2fx over one call per farm (b)" % (
        med["per-N"] / med["ragged"], med["per-farm"] / med["ragged"]))
    print("Xi_sys and info bit-identical across the three arms: %s" % same)
    return 0 if same else 1


if __name__ == "__main__":
    sys.exit(main())
