#!/usr/bin/env python
"""Rotor speed, generator torque and blade pitch statistics on one GPU: raftk_rotor_stats_dev against numpy on the host.

Two shapes, seeded and resident on the device:
  sweep  1250 rigid designs x 8 cases (one train each) x 1024 bins, one rotor per design, per-design C / V_w / gains;
  farms  16 farms x 64 FOWTs (6N = 384 DOFs, one rotor per FOWT at col0 = 6 i) x 8 cases x 256 bins, shared tables.
Device arm: the raftk_rotor_stats_dev struct and outputs prepared once, then CUDA events around 20 back-to-back launches
(kernel_ms: their mean, median over --reps after a warm-up; the host-side set-up of a session call is not in it); numpy arm: the vectorised restatement of
raft_fowt.py:2643-2675 from host arrays.  Reported per shape: the medians, the bytes the kernel must move (each rotor's
hub columns of Xi, C, V_w, the std and PSD writes) over its time, as a share of the H100 SXM data-sheet 3.35 TB/s, and
the largest relative std difference against numpy.  The card's name and power limit are read (nothing is set) and printed
with the numbers.

Usage:  python tools/rotor_timing.py [--reps 7]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
RPM, DEG = 1 / 0.1047, 57.29577951308232
LAUNCHES = 20


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip()
    except Exception:                                              # noqa: BLE001
        return "unknown"


def numpy_stats(R, C_, V_w, g, w, Xi, dw, col0):
    """Xi [nU, nC, n, nw] with one row per case; R [nrot, 6]; tables [nU or 1, nC, nrot, ...]."""
    hub = np.stack([np.einsum("b,ucbw->ucw", R[k], Xi[:, :, c0:c0 + 6]) for k, c0 in enumerate(col0)], axis=2)   # [nU, nC, nrot, nw]
    a = np.abs(C_) ** 2 * (np.abs(hub) ** 2 + np.abs(V_w) ** 2 / w ** 2)
    w2 = w ** 2
    ch = np.stack([w2 * a, (g[..., 1:2] ** 2 + w2 * g[..., 0:1] ** 2) * a, (g[..., 3:4] ** 2 + w2 * g[..., 2:3] ** 2) * a], axis=3)
    s = np.array([RPM, 1.0, DEG])
    return np.sqrt(0.5 * ch.sum(axis=-1)) * s, s[:, None] ** 2 * 0.5 * ch / dw


def run(shape, nU, nC, n, nw, nrot, per_unit, reps, torch, solver):
    rng = np.random.default_rng(7)
    dev = torch.device("cuda", 0)
    w = np.linspace(2.0 / nw, 2.0, nw)
    dw = w[1] - w[0]
    Xi = rng.normal(size=(nU, nC, n, nw)) + 1j * rng.normal(size=(nU, nC, n, nw))
    lead = (nU,) if per_unit else ()
    R = rng.normal(size=(nrot, 6))
    C_ = (rng.normal(size=lead + (nC, nrot, nw)) + 1j * rng.normal(size=lead + (nC, nrot, nw))) * 0.1
    V_w = rng.normal(size=lead + (nC, nrot, nw)) + 0j
    g = rng.normal(size=lead + (nC, nrot, 4))
    col0 = 6 * np.arange(nrot, dtype=np.int32)
    dXi, dW = torch.from_numpy(Xi).to(dev), torch.from_numpy(w).to(dev)
    dR, dC, dV, dG = (torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in (R, C_, V_w, g))
    stream = torch.cuda.current_stream(dev).cuda_stream

    # the struct and outputs are prepared once (what DeviceSession.rotor_stats does per call on the host), so the event
    # window holds only back-to-back kernel launches
    ro, rows, cols = solver._rotor_struct(dR, dC, dV, dG, nU, nw, dw, None, col0)
    sd = torch.empty([nU, nC, nrot, 3], dtype=torch.float64, device=dev)
    P = torch.empty([nU, nC, nrot, 3, nw], dtype=torch.float64, device=dev)
    ro.R, ro.C, ro.V_w, ro.gains = dR.data_ptr(), dC.data_ptr(), dV.data_ptr(), dG.data_ptr()
    ro.std, ro.psd = sd.data_ptr(), P.data_ptr()

    def launch():
        solver.check(solver.lib.raftk_rotor_stats_dev(nU, nC, n, nw, dW.data_ptr(), dXi.data_ptr(), C.byref(ro), stream))

    launch()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    td, th = [], []
    for rep in range(reps):
        e0.record()
        for _ in range(LAUNCHES):
            launch()
        e1.record()
        torch.cuda.synchronize()
        td.append(e0.elapsed_time(e1) / LAUNCHES)
        if rep < 2:
            t0 = time.perf_counter()
            sn, pn = numpy_stats(R, C_ if per_unit else C_[None], V_w if per_unit else V_w[None], g if per_unit else g[None], w, Xi, dw, col0)
            th.append((time.perf_counter() - t0) * 1e3)
    tab = (nU if per_unit else 1) * nC * nrot
    need = nU * nC * nrot * 6 * nw * 16 + tab * nw * 32 + tab * 32 + nU * nC * nrot * 3 * (nw + 1) * 8
    ms = float(np.median(td))
    err = float(np.abs(sd.cpu().numpy() - sn).max() / np.abs(sn).max())
    return dict(shape=shape, units=nU, cases=nC, dof=n, nw=nw, rotors=nrot, kernel_ms=ms, numpy_ms=float(np.median(th)),
                numpy_over_kernel=float(np.median(th)) / ms, bytes=int(need), GBps=need / ms / 1e6,
                share_of_3350GBps=need / ms / 1e6 / 3350.0, std_rel_vs_numpy=err)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    a = ap.parse_args()
    import torch
    from raft_b200 import solver
    res = [run("sweep", 1250, 8, 6, 1024, 1, True, a.reps, torch, solver),
           run("farms", 16, 8, 384, 256, 64, False, a.reps, torch, solver)]
    print(json.dumps(dict(card=card(), reps=a.reps, results=res)))


if __name__ == "__main__":
    main()
