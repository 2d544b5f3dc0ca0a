"""Measure the margins of the fused solvers' step-class tolerance (DESIGN.md section 6).  CPU only.

For the golden designs, the synthetic designs the suite solves and a sample of the VolturnUS-S sweep family, every node's
phase key (q_x,q_y)*step and depth key q_z*step is classed by the kernels' rule (greedy, raftk_fused.cuh step_classes_warp)
at a candidate tolerance and at 1e-11, the tolerance before it was tightened.  Prints the largest relative difference that
is merged into a class, the smallest relative difference between two class keys, whether every design keeps the class
counts it had at 1e-11, and k_max * L_max * tol for the grids the suite and the benchmark use (the phase a node walked
along a member at worst accumulates from merged keys).

    python tools/step_class_tolerance.py [--tol 5e-14] [--family 1250]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def design_keys(a, d):
    """Keys per node of design ``d`` of raftk_designs columns ``a`` (as the kernels form them) -> (wkeys, hkeys, spans)."""
    m0, m1 = int(a["member_offset"][d]), int(a["member_offset"][d + 1])
    wk, hk, spans = [], [], []
    for m in range(m0, m1):
        q = a["mem_frame"][m][:3]
        ls = a["node_ls"][a["mem_node_start"][m]:a["mem_node_start"][m + 1]]
        spans.append(float(ls[-1] - ls[0]) if len(ls) else 0.0)
        for step in np.diff(ls):
            kx, ky, kz = q[0] * step, q[1] * step, q[2] * step
            if abs(kx) > 1e-14 or abs(ky) > 1e-14:
                wk.append((kx, ky))
            if abs(kz) > 1e-14:
                hk.append((kz,))
    return wk, hk, spans


def greedy(keys, rtol):
    """-> (class keys, largest merged relative difference)."""
    reps, worst = [], 0.0
    for k in keys:
        mag = sum(abs(x) for x in k)
        for r in reps:
            if all(abs(a - b) <= rtol * mag for a, b in zip(r, k)):
                worst = max(worst, max(abs(a - b) for a, b in zip(r, k)) / mag)
                break
        else:
            reps.append(k)
    return reps, worst


def closest(reps):
    best = np.inf
    for i in range(len(reps)):
        for j in range(i):
            mag = sum(abs(x) for x in reps[i])
            best = min(best, max(abs(a - b) for a, b in zip(reps[i], reps[j])) / mag)
    return best


def designs():
    from conftest import load_golden
    from test_dispatch_solve import _random_packed
    from raft_b200 import solver
    out = []
    for f in sorted(os.listdir(os.path.join(ROOT, "tests", "golden"))):
        if f.endswith(".npz"):
            _, P = load_golden(f[:-4])
            if "node_ls" in P and "mem_q" in P and not any(k.startswith("gen_") for k in P):
                out.append(("golden " + f[:-4], solver.DesignBatch([{k: v for k, v in P.items() if not k.startswith("qs_")}]).arrays, 1))
    for seed in (1, 2, 3, 4, 24):
        out.append(("random seed %d" % seed, solver.DesignBatch(_random_packed(seed)).arrays, 1))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tol", type=float, default=5e-14)
    ap.add_argument("--family", type=int, default=1250)
    args = ap.parse_args()
    from conftest import load_golden
    from raft_b200 import grid, sweep
    sets = designs()
    base = json.load(open(os.path.join(ROOT, "tests", "golden", "designs.json")))["cfg2_VolturnUS-S_nw64"]
    _, P = load_golden("cfg2_VolturnUS-S_nw64")
    mats = dict(M_struc=P["M0"], C_struc=P["C0"])
    fam = sweep.build_variants_batched(base, mats, sweep.sample_factors(args.family, seed=40), nw=64, max_freq=0.40,
                                       depth=float(P["depth"]), native=False)
    sets.append(("sweep family (%d designs)" % args.family, fam.arrays, fam.n_designs))
    worst_merge, min_gap, l_max, same = 0.0, np.inf, 0.0, True
    for name, a, nD in sets:
        wm, gap = 0.0, np.inf
        for d in range(nD):
            wk, hk, spans = design_keys(a, d)
            l_max = max(l_max, max(spans, default=0.0))
            for keys in (wk, hk):
                r_old, _ = greedy(keys, 1e-11)
                r_new, m = greedy(keys, args.tol)
                same &= len(r_old) == len(r_new)
                wm = max(wm, m)
                gap = min(gap, closest(r_new))
        print("%-40s largest merged %.2e   closest distinct %.2e" % (name, wm, gap))
        worst_merge, min_gap = max(worst_merge, wm), min(min_gap, gap)
    k_max = float(grid.wave_number(np.array([2 * np.pi * 0.512]), 1e4)[0])       # the benchmark's top bin, deep water
    print("tol %.1e: largest merged %.2e, closest distinct %.2e, class counts as at 1e-11: %s" % (args.tol, worst_merge, min_gap, same))
    print("k_max %.3f rad/m (0.512 Hz), L_max %.1f m (longest member walk): k_max L_max tol = %.2e"
          % (k_max, l_max, k_max * l_max * args.tol))


if __name__ == "__main__":
    main()
