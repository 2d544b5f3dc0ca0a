"""Cost of a submerged rotor's inertial wave excitation at cfg2's shape on one GPU: VolturnUS-S on 1024 bins (max_freq
0.512 Hz) x 64 JONSWAP sea states, the same design solved without and with one synthetic submerged rotor, alternating, through
a DeviceSession (k_rao_fused2 in its rotor-free and rotor instantiations).  Prints the card, its power limit and the step
times (CUDA-synchronised wall clock, median of --steps after --warmup) as JSON lines.

    python tools/mhk_timing.py [--steps 20] [--warmup 3] [--rounds 3]
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


def synthetic_rotor_table():
    """One submerged rotor as packer.pack_rotor_excitation packs it: a hub 16 m below the waterline, off the axis, with a
    seeded symmetric I_hydro, a small rotation R_q and a hub node rigidly tied to the PRP."""
    import types
    from raft_b200 import packer
    rng = np.random.default_rng(0)
    A = rng.normal(size=(6, 6))
    I6 = A @ A.T * 4e4 + np.diag([3e5, 8e4, 8e4, 2e6, 1e6, 1e6])
    c, s_ = np.cos(0.2), np.sin(0.2)
    R = np.array([[c, -s_, 0.0], [s_, c, 0.0], [0.0, 0.0, 1.0]])
    r3 = np.array([-6.0, 3.5, -16.0])
    T = np.vstack([np.eye(6), np.eye(6)])
    T[6:9, 3:] = np.array([[0, r3[2], -r3[1]], [-r3[2], 0, r3[0]], [r3[1], -r3[0], 0]])
    rot = types.SimpleNamespace(r3=r3, I_hydro=I6, R_q=R, nodeList=[types.SimpleNamespace(id=1)])
    return packer.pack_rotor_excitation(types.SimpleNamespace(rotorList=[rot], T=T, r6=np.zeros(6)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import torch
    from raft_b200 import grid, solver
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(json.dumps(dict(card=card)))
    z = np.load(os.path.join(ROOT, "tests", "golden", "cfg2_VolturnUS-S_nw64.npz"))
    P0 = grid.regrid({k[2:]: z[k] for k in z.files if k.startswith("P_")}, 1024, 0.512)
    P1 = dict(P0, **synthetic_rotor_table())
    rng = np.random.default_rng(2)
    n = 64
    ct = solver.CaseTable(dict(Hs=rng.uniform(1, 10, n), Tp=rng.uniform(5, 18, n), gamma=np.zeros(n), beta_deg=np.zeros(n),
                               spec=np.zeros(n, dtype=np.int32)))
    sessions = {name: solver.DeviceSession(solver.DesignBatch(P), ct) for name, P in (("no_rotor", P0), ("rotor", P1))}
    for s in sessions.values():
        for _ in range(args.warmup):
            s.solve(n_iter=10)
    torch.cuda.synchronize()
    times = {k: [] for k in sessions}
    for _ in range(args.rounds):
        for name, s in sessions.items():
            for _ in range(args.steps):
                t0 = time.perf_counter()
                out = s.solve(n_iter=10)
                torch.cuda.synchronize()
                times[name].append((time.perf_counter() - t0) * 1e3)
            print(json.dumps(dict(variant=name, kernel=solver.last_dispatch()["kernel"],
                                  passes_max=int(out["status"][..., 0].max()), ms_median=float(np.median(times[name][-args.steps:])))))
    med = {k: float(np.median(v)) for k, v in times.items()}
    print(json.dumps(dict(summary=med, spread_ms={k: [float(np.min(v)), float(np.max(v))] for k, v in times.items()},
                          rotor_over_no_rotor=med["rotor"] / med["no_rotor"])))


if __name__ == "__main__":
    main()
