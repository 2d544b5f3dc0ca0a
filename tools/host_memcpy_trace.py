"""The host<->device copies of one cfg2 raftk_solve_dynamics_host call (1024 bins x 64 sea states, page-locked Xi and status,
so the solve kernel stores those straight into host memory), as torch.profiler records them: kind and bytes, in order.
Run it against two builds (RAFTK_LIB=...) to compare their copy patterns.

    python tools/host_memcpy_trace.py"""
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    from torch.profiler import ProfilerActivity, profile
    from raft_b200 import grid, solver
    z = np.load(os.path.join(ROOT, "tests", "golden", "cfg2_VolturnUS-S_nw64.npz"))
    P = grid.regrid({k[2:]: z[k] for k in z.files if k.startswith("P_")}, 1024, 0.512)
    rng = np.random.default_rng(2)
    nC = 64
    ct = solver.CaseTable(dict(Hs=rng.uniform(2, 8, nC), Tp=rng.uniform(6, 14, nC), gamma=np.zeros(nC), beta_deg=rng.uniform(-90, 90, nC),
                               spec=np.zeros(nC, dtype=np.int32)))
    batch = solver.DesignBatch(P)
    out = dict(Xi=solver.pinned_empty([1, nC, 6, 1024], np.complex128), status=solver.pinned_empty([1, nC, 4], np.int32))
    solver.solve_dynamics(batch, ct, out=out)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        solver.solve_dynamics(batch, ct, out=out)
        torch.cuda.synchronize()
    assert solver.last_dispatch()["direct_d2h"]
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        ev = json.load(open(path))["traceEvents"]
    copies = sorted((e for e in ev if e.get("cat") == "gpu_memcpy"), key=lambda e: e["ts"])
    for e in copies:
        print("%s %d" % (e["name"], e["args"].get("bytes", -1)))


if __name__ == "__main__":
    main()
