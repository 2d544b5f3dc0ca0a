#!/usr/bin/env python
"""Device timing of the slender-body QTF kernels (k_slender_tables + k_slender_pairs + k_slender_fill) through
raftk_qtf_slender_dev: the reference's own test grid (23 frequencies, VolturnUS-S, 53 nodes) for 1 and 64 (heading, RAO)
pairs, and a finer second-order grid (92 frequencies).  CUDA events on torch's current stream."""
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from raft_b200 import grid, solver  # noqa: E402
from raft_b200._lib import check, lib  # noqa: E402

z = np.load(os.path.join(ROOT, "tests", "golden", "slender_VolturnUS-S.npz"))
P = {k[2:]: z[k] for k in z.files if k.startswith("P_")}
dev = torch.device("cuda", 0)


def run(P, n, label, reps=5):
    nw2 = len(P["qs_w"])
    keep = {}

    def to_dev(name, a):
        keep[name] = torch.from_numpy(a).to(dev)
        return keep[name].data_ptr()
    s = solver._slender_struct(P, to_dev)
    rng = np.random.default_rng(7)
    beta = torch.from_numpy(rng.uniform(-np.pi, np.pi, n)).to(dev)
    Xi = (rng.normal(size=(n, 6, nw2)) + 1j * rng.normal(size=(n, 6, nw2))) * np.array([1, 1, 1, 0.03, 0.03, 0.03])[None, :, None]
    Xi = torch.from_numpy(np.ascontiguousarray(Xi).view(np.float64)).to(dev)
    q = torch.zeros(n * nw2 * nw2 * 6 * 2, dtype=torch.float64, device=dev)
    wb = lib.raftk_qtf_slender_workspace_bytes(C.byref(s), n)
    ws = torch.empty(wb, dtype=torch.uint8, device=dev)
    st = torch.cuda.current_stream(dev).cuda_stream

    def go():
        check(lib.raftk_qtf_slender_dev(C.byref(s), n, beta.data_ptr(), Xi.data_ptr(), q.data_ptr(), ws.data_ptr(), wb, st))
    for _ in range(2):
        go()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        go()
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / reps
    pairs = n * nw2 * (nw2 + 1) // 2
    return {label: dict(ms=ms, qtf_per_s=n / (ms * 1e-3), node_pairs_per_s=pairs * s.n_nodes / (ms * 1e-3), nw2=nw2, n=n)}


res = {}
res.update(run(P, 1, "test_grid_1case"))
res.update(run(P, 64, "test_grid_64cases"))
w2 = np.arange(0.040, 0.200 + 0.5 * 0.002, 0.002) * 2 * np.pi
Pf = dict(P, qs_w=w2, qs_k=np.array([grid.wave_number(np.array([x]), float(P["qs_depth"]))[0] for x in w2]))
res.update(run(Pf, 16, "fine_grid_16cases"))
print(json.dumps(dict(workload="raftk_qtf_slender_dev, VolturnUS-S (53 strip nodes, 2 MCF columns)", **res)))
