"""Device time of raftk_fatigue_dev on resident responses against the bytes it must read, and against numpy.

Shapes: (a) a rigid design sweep, 1250 designs x 8 cases x 1024 bins, 4 complex-coefficient channels shared by every design
(AxRNA / AyRNA / AzRNA / Mbase, the DeviceSession.fatigue path); (b) 16 farms of 64 FOWTs (384 DOFs) x 8 cases x 256 bins, 768
tension rows per farm (DeviceSession.fatigue(farm=True)); (c) a flexible batch, 64 designs x 8 cases of 2 trains x 150 DOFs x
200 bins, 15 rows per design (GeneralBatchSession.fatigue).  Xi is seeded random data of those shapes: the kernels' work does
not depend on the values.  Device time: CUDA events around one call (moments, finish and lifetime kernels), median of 7
repetitions of 10 calls after a warm-up.  Bytes: Xi plus the coefficients or rows, read once; share of the 3.35 TB/s HBM3
data-sheet bandwidth.  numpy: the same moments and closed form in float64 on the host (for (b) one farm, scaled by 16).
Usage: python tools/fatigue_timing.py [out.txt]"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from raft_b200 import solver  # noqa: E402
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import test_fatigue as ref  # noqa: E402

HBM = 3.35e12


def device_time(fn, reps=7, inner=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(inner):
            fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) / inner * 1e-3)
    return float(np.median(ts)), float(min(ts)), float(max(ts))


def numpy_fatigue(Xi, w, row0, m, **ch):
    t0 = time.perf_counter()
    lam = ref.np_moments(ref.np_amplitudes(Xi, w, **ch), w, row0)
    out = ref.np_fatigue(lam, m)
    return time.perf_counter() - t0, lam, out


def run(name, U, nR, n, nw, nch, form, row0, numpy_units):
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(1)
    Xi = torch.complex(torch.randn(U, nR, n, nw, device=dev, dtype=torch.float64, generator=g),
                       torch.randn(U, nR, n, nw, device=dev, dtype=torch.float64, generator=g))
    w = torch.arange(1, nw + 1, device=dev, dtype=torch.float64) * (3.0 / nw)
    rng = np.random.default_rng(2)
    if form == "coef":
        ch = dict(coef=rng.normal(size=(nch, n, nw)) + 1j * rng.normal(size=(nch, n, nw)))
        ch_bytes = nch * n * nw * 16
    else:
        ch = dict(R=rng.normal(size=(U, nch, n)), wpow=np.zeros(nch, dtype=np.int32))
        ch_bytes = U * nch * n * 8
    dch = {k: (torch.from_numpy(v).to(dev) if k != "wpow" else v) for k, v in ch.items()}
    keep = []

    def call():
        be = solver._Device(dev)
        out = solver._fatigue(be, Xi, w, 4.0, dch.get("R"), dch.get("wpow"), dch.get("coef"), row0, 1.0, "dirlik", None, True, True, 0)
        keep[:] = [out, be]
        return out
    t_med, t_min, t_max = device_time(call)
    out = call()
    torch.cuda.synchronize()
    xi_bytes = U * nR * n * nw * 16
    by = xi_bytes + ch_bytes
    # numpy on the first numpy_units units; agreement with the device on them
    Xh = Xi[:numpy_units].cpu().numpy()
    chh = dict(ch)
    if "R" in chh:
        chh["R"] = chh["R"][:numpy_units]
    t_np, lam, o_np = numpy_fatigue(Xh, w.cpu().numpy(), row0, 4.0, **chh)
    err_m = float(np.max(np.abs(out["moments"][:numpy_units].cpu().numpy() - lam) / np.abs(lam)))
    err_d = float(np.max(np.abs(out["DEL"][:numpy_units].cpu().numpy() - o_np["DEL"]) / np.abs(o_np["DEL"])))
    t_np_full = t_np * U / numpy_units
    return dict(shape=name, units=U, rows=nR, n_dof=n, nw=nw, nch=nch, form=form, device_s_median=t_med, device_s_min=t_min,
                device_s_max=t_max, bytes_read=by, xi_bytes=xi_bytes, GBps=by / t_med / 1e9, share_of_3p35TBps=by / t_med / HBM,
                numpy_s=t_np_full, numpy_units_timed=numpy_units, speedup_vs_numpy=t_np_full / t_med,
                max_rel_err_moments_vs_numpy=err_m, max_rel_err_DEL_vs_numpy=err_d)


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else None
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    lines = ["device: " + smi]
    res = [run("sweep 1250 x 8 cases x 1024 bins x 4 coef channels", 1250, 8, 6, 1024, 4, "coef", np.arange(9, dtype=np.int32), 1250),
           run("16 farms x 64 FOWTs x 8 cases x 256 bins x 768 tension rows", 16, 8, 384, 256, 768, "R", np.arange(9, dtype=np.int32), 1),
           run("flexible batch 64 designs x 8 cases x 2 trains x 150 DOFs x 200 bins x 15 rows", 64, 16, 150, 200, 15, "R",
               np.arange(0, 17, 2, dtype=np.int32), 64)]
    for r in res:
        lines.append(json.dumps(r))
    txt = "\n".join(lines)
    print(txt)
    if out:
        with open(out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
