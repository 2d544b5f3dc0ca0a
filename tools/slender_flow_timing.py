"""potSecOrder 1: the host flow (solver.solve_dynamics_slender) against the device flow (solver.SlenderSession, one call, no
host synchronisation) on VolturnUS-S, 64 sea states, at the reference's second-order grid and at the fine grid of
tools/slender_timing.py, and on a 256-design build_variants sample.  CUDA events around the device flow, a host clock around
the host flow (it ends in a synchronise).  Prints one JSON line per row, with the QTF chunk size and the workspace bytes.

    python tools/slender_flow_timing.py [--reps 3] [--chunk 0]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def cases(n, seed=0):
    rng = np.random.default_rng(seed)
    return dict(Hs=rng.uniform(1.5, 9.0, n), Tp=rng.uniform(6.0, 17.0, n), gamma=np.zeros(n), beta_deg=rng.uniform(-180, 180, n),
                spec=np.zeros(n, dtype=np.int32))


def fine_grid(P, nw2):
    """The second-order grid of tools/slender_timing.py: nw2 frequencies up to the fixture's last one."""
    from raft_b200 import grid
    qw = np.linspace(P["qs_w"][0], P["qs_w"][-1], nw2)
    return dict(P, qs_w=qw, qs_k=grid.wave_number(qw, float(P["qs_depth"])))


def time_row(name, packed, ct, reps, chunk, host=True):
    import torch
    from raft_b200 import solver
    s = solver.SlenderSession(packed, ct, want=("Xi", "status", "F_2nd"), qtf_chunk=chunk)
    s.solve()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dev = []
    for _ in range(reps):
        a.record()
        s.solve()
        b.record()
        b.synchronize()
        dev.append(a.elapsed_time(b))
    hst = []
    if host:
        solver.solve_dynamics_slender(packed, ct)
        for _ in range(reps):
            t0 = time.perf_counter()
            solver.solve_dynamics_slender(packed, ct)
            hst.append((time.perf_counter() - t0) * 1e3)
    units = len(packed) * ct.n_cases
    print(json.dumps(dict(row=name, designs=len(packed), cases=ct.n_cases, nw=int(s.batch.nw), nw2=int(s.slender.nw2),
                          qtf_chunk=chunk or units, workspace_bytes=s.workspace_bytes, device_ms=min(dev),
                          host_flow_ms=min(hst) if hst else None)), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--chunk", type=int, default=0)
    ap.add_argument("--designs", type=int, default=256)
    args = ap.parse_args()
    import torch
    from raft_b200 import solver, sweep
    name = torch.cuda.get_device_name()
    props = os.popen("nvidia-smi --query-gpu=power.limit --format=csv,noheader").read().strip()
    print(json.dumps(dict(gpu=name, power_limit=props)), flush=True)
    z = np.load(os.path.join(ROOT, "tests", "golden", "slender_VolturnUS-S.npz"))
    P = {k[2:]: z[k] for k in z.files if k.startswith("P_")}
    ct = solver.CaseTable(cases(64))
    time_row("VolturnUS-S reference grid", [P], ct, args.reps, args.chunk)
    time_row("VolturnUS-S fine grid", [fine_grid(P, 120)], ct, args.reps, args.chunk)
    D = json.load(open(os.path.join(ROOT, "tests", "golden", "designs.json")))["test_VolturnUS-S"]
    base = dict(D, platform=dict(D["platform"], potSecOrder=1), site=dict(D["site"], water_depth=float(P["depth"])))
    mats = dict(M_struc=P["M0"] - z["A_hydro_morison"], C_struc=P["C0"] - z["C_moor"], C_moor=z["C_moor"])
    packed = sweep.build_variants(base, mats, sweep.sample_factors(args.designs, seed=40), len(P["w"]), float(P["w"][-1]) / (2 * np.pi),
                                  float(P["depth"]))
    time_row("build_variants x %d" % args.designs, packed, solver.CaseTable(cases(16)), args.reps, args.chunk or 1024)


if __name__ == "__main__":
    main()
