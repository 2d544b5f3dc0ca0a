#!/usr/bin/env python
"""When do k_rao_fused2's CTAs start?  Runs bench.py's cfg2 step (1024 bins x 64 sea states) through a diagnostic build of
the library compiled with -DRAFTK_F2_WAVE_TRACE, which stores %smid and %globaltimer at entry and exit of every CTA, and
prints the occupancy queries of the launch and a histogram of the CTA start times.

  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -shared -Xcompiler -fPIC -DRAFTK_F2_WAVE_TRACE \\
       -o build/libraftk_wavetrace.so raft_b200/csrc/raftk.cu
  python tools/fused2_waves.py build/libraftk_wavetrace.so [--steps 3] [--xchg cluster|grid]
"""
import argparse
import ctypes as C
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("lib")
    ap.add_argument("--steps", type=int, default=3, help="traced steps, each reported")
    ap.add_argument("--xchg", default="", help="RAFTK_FUSED2_XCHG for the traced steps (default: the planner's choice)")
    a = ap.parse_args()
    os.environ["RAFTK_LIB"] = os.path.abspath(a.lib)
    if a.xchg:
        os.environ["RAFTK_FUSED2_XCHG"] = a.xchg
    import torch
    import bench
    from raft_b200 import solver
    from raft_b200._lib import check, lib
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print("GPU:", gpu)
    designs, cs, cfg = bench.build_workload(argparse.Namespace(workload="cfg2", nw=0, cases=0, designs=0), 0, 1)
    dev = torch.device("cuda", 0)
    sess = solver.DeviceSession(solver.DesignBatch(designs), solver.CaseTable(cs), device=dev)
    occ = (C.c_int * 5)()
    check(lib.raftk_f2_occupancy(C.byref(sess.d_struct), sess.cases.n_cases, 0, occ))
    clusters, resident, grid, CS, smem = list(occ)
    units = sess.batch.n_designs * sess.cases.n_cases
    n = units * CS
    print("workload: %s" % cfg["workload"])
    print("launch: %d units x %d CTAs = %d CTAs of 128 threads, %d B dynamic shared memory" % (units, CS, n, smem))
    print("cudaOccupancyMaxActiveClusters = %d (of %d clusters); cudaOccupancyMaxActiveBlocksPerMultiprocessor x SMs = %d CTAs"
          % (clusters, units, resident))
    print("exchange: %s" % ("grid (cooperative launch, rows in L2)" if grid else "cluster (distributed shared memory)"))
    for _ in range(5):
        sess.solve(n_iter=10, tol=0.01, xi_start=0.0)
    torch.cuda.synchronize()
    buf = (C.c_ulonglong * (3 * n))()
    for s in range(a.steps):
        sess.solve(n_iter=10, tol=0.01, xi_start=0.0)
        torch.cuda.synchronize()
        check(lib.raftk_f2_trace_read(buf, n))
        t = np.frombuffer(buf, dtype=np.uint64).reshape(n, 3).astype(np.int64)
        sm, t0, t1 = t[:, 0], t[:, 1], t[:, 2]
        base = t0.min()
        start, end = (t0 - base) / 1e3, (t1 - base) / 1e3        # us
        first_exit = end.min()
        late = start > first_exit
        print("\nstep %d: kernel span %.1f us (first CTA start to last CTA exit); first CTA exit at %.1f us"
              % (s, end.max(), first_exit))
        print("  CTAs starting after the first CTA exit: %d of %d (%d clusters); distinct SMs used %d"
              % (int(late.sum()), n, int(late.reshape(units, CS).any(1).sum()), len(np.unique(sm))))
        print("  CTAs per SM at the start (<= 5 us): max %d" % np.bincount(sm[start <= 5.0].astype(np.int64)).max())
        edges = [0, 1, 2, 5, 10, 20, 50, 100, 150, 200, 250, 300, 350, 400, 500, 1e9]
        h, _ = np.histogram(start, bins=edges)
        print("  start-time histogram (us from the first start):")
        for lo, hi, c in zip(edges[:-1], edges[1:], h):
            if c:
                print("    [%5g, %5s) %4d CTAs" % (lo, ("%g" % hi) if hi < 1e9 else "inf", c))
        if late.any():
            print("  late CTAs start %.1f..%.1f us; they start after %d..%d CTAs have exited"
                  % (start[late].min(), start[late].max(), int((end < start[late].min()).sum()), int((end < start[late].max()).sum())))
        dur = end - start
        print("  CTA duration (us): min %.1f median %.1f max %.1f" % (dur.min(), np.median(dur), dur.max()))
        st = sess.out["status"].cpu().numpy()[0]
        print("  passes per unit: %s" % dict(zip(*[x.tolist() for x in np.unique(st[:, 0], return_counts=True)])))
    # device time of the solve kernel and of the counter reset the grid variant enqueues before it (torch.profiler)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(20):
            sess.solve(n_iter=10, tol=0.01, xi_start=0.0)
        torch.cuda.synchronize()
    for ev in prof.key_averages():
        if "k_rao_fused2" in ev.key or "emset" in ev.key:
            t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
            print("profiler: %-60s count %3d  mean %.2f us" % (ev.key[:60], ev.count, t / max(ev.count, 1)))


if __name__ == "__main__":
    main()
