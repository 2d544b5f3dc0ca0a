#!/usr/bin/env python
"""Mooring tension statistics of a farm batch on one GPU: raftk_farm_channel_stats_dev (one pass over Xi_sys per bin tile
for every channel) against what a farm-batch user could run before it -- a loop over the farms of
raftk_general_channel_stats_dev (one CTA per (unit, channel), each re-reading the unit's whole Xi) -- and numpy on the host.

Shape: F = 16 farms of N = 64 FOWTs (6N = 384 DOFs), nC = 8 cases, nw = 256 bins, 12N = 768 channels (a per-farm R, wpow 0),
seeded Xi_sys resident on the device.  Device arms: a host-clock window around the call(s) ending in a device synchronise;
the numpy arm: R_f @ Xi_sys[f, r] per (farm, row) plus the PSD / std reductions, from host arrays.  The arms alternate;
reported: the median ms of each arm over --reps, and whether std and PSD of the two device arms are bit-identical.  The
card's name and power limit are read (nothing is set) and printed with the numbers.

Usage:  python tools/tension_timing.py [--reps 5] [--farms 16] [--fowts 64] [--cases 8] [--nw 256]
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


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip()
    except Exception:                                              # noqa: BLE001
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--farms", type=int, default=16)
    ap.add_argument("--fowts", type=int, default=64)
    ap.add_argument("--cases", type=int, default=8)
    ap.add_argument("--nw", type=int, default=256)
    a = ap.parse_args()
    import torch
    from raft_b200 import _lib, solver
    lib = _lib.lib
    F, N, nC, nw = a.farms, a.fowts, a.cases, a.nw
    n, nch = 6 * N, 12 * N
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(1)
    Xi = (rng.normal(size=(F, nC, n, nw)) + 1j * rng.normal(size=(F, nC, n, nw))).astype(np.complex128)
    R = rng.normal(size=(F, nch, n))
    wpow = np.zeros(nch, dtype=np.int32)
    w = np.linspace(0.01, 2.56, nw)
    dw = float(w[0])
    dXi, dR, dW = torch.from_numpy(Xi).to(dev), torch.from_numpy(R).to(dev), torch.from_numpy(w).to(dev)
    dP = torch.from_numpy(wpow).to(dev)
    sdA = torch.zeros([F, nC, nch], dtype=torch.float64, device=dev)
    psA = torch.zeros([F, nC, nch, nw], dtype=torch.float64, device=dev)
    sdB, psB = torch.zeros_like(sdA), torch.zeros_like(psA)
    ch = _lib.RaftkFarmChannels()
    ch.n_ch, ch.R_shared, ch.R, ch.wpow, ch.dw = nch, 0, dR.data_ptr(), wpow.ctypes.data, dw
    ch.std, ch.psd, ch.amp = sdA.data_ptr(), psA.data_ptr(), None
    stream = torch.cuda.current_stream(dev).cuda_stream

    def batched():
        _lib.check(lib.raftk_farm_channel_stats_dev(F, nC, n, nw, dW.data_ptr(), dXi.data_ptr(), C.byref(ch), None, 0, stream))

    def loop():
        for f in range(F):
            _lib.check(lib.raftk_general_channel_stats_dev(nC, n, nch, nw, dw, dW.data_ptr(), dR[f].data_ptr(), dP.data_ptr(), dXi[f].data_ptr(),
                                                           sdB[f].data_ptr(), psB[f].data_ptr(), None, stream))

    def host():
        sd, ps = np.zeros([F, nC, nch]), np.zeros([F, nC, nch, nw])
        for f in range(F):
            Y = np.matmul(R[f], Xi[f])                            # [nC, nch, nw]
            a2 = Y.real ** 2 + Y.imag ** 2
            ps[f] = 0.5 * a2 / dw
            sd[f] = np.sqrt(0.5 * a2.sum(axis=-1))
        return sd, ps

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, r

    timed(batched), timed(loop)                                    # warm-up: module load, shared-memory opt-in
    tA, tB, tH = [], [], []
    sd_np = ps_np = None
    for rep in range(a.reps):
        tA.append(timed(batched)[0])
        tB.append(timed(loop)[0])
        if rep < 2:
            t, (sd_np, ps_np) = timed(host)
            tH.append(t)
    same = bool(torch.equal(sdA, sdB) and torch.equal(psA, psB))
    err_np = float(np.abs(sdA.cpu().numpy() - sd_np).max() / np.abs(sd_np).max())
    res = dict(shape=dict(farms=F, fowts=N, dof=n, cases=nC, nw=nw, channels=nch), card=card(),
               batched_ms=float(np.median(tA)), loop_general_ms=float(np.median(tB)), numpy_ms=float(np.median(tH)),
               loop_over_batched=float(np.median(tB) / np.median(tA)), numpy_over_batched=float(np.median(tH) / np.median(tA)),
               bit_identical_std_psd=same, std_rel_vs_numpy=err_np, reps=a.reps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
