"""Device time of raftk_stress_ring_dev on resident responses, against the per-angle solver.fatigue loop it replaces and
against numpy.

Shapes: (a) a rigid design sweep, 1250 designs x 8 cases x 1024 bins x 50 angles, the fore-aft moment as complex per-bin
coefficients shared by every design (a rigid tower's Mbase, the DeviceSession.stress_ring path); (b) a flexible batch,
256 FOWTs of 150 DOFs x 8 cases x 256 bins x 50 angles, fore-aft and side-side rows per design (GeneralBatchSession.
stress_ring).  Xi is seeded random data of those shapes: the kernels' work does not depend on the values.  Every call gives
std / avg / max / min, DEL (m = 4, Dirlik) and the hot spot.
Device time: CUDA events around one call, median of 7 repetitions of 5 calls after a warm-up.  Per-angle loop: what a user
could do without stress_ring, 50 solver.fatigue calls on the device, one per angle with the explicit row R_theta = c (cos R_FA -
sin R_SS) (or c cos theta coef_FA); also one fatigue call with the 50 rows as 50 channels.  numpy: the three cross sums and
the closed form over the angles in float64 on the host for the first units, scaled to all.
Usage: python tools/stress_timing.py [out.txt]"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from raft_b200 import solver  # noqa: E402

HBM = 3.35e12


def device_time(fn, reps=7, inner=5):
    for _ in range(2):
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


def numpy_stress(Xi, w, fa, ss, angles, c):
    """std [U, nC, nA] of one ring, one row per case, from the three cross sums (fa / ss: real rows [U, n] or complex
    coefficients [n, nw]; ss may be None)."""
    t0 = time.perf_counter()
    if np.iscomplexobj(fa):
        a = np.einsum("bw,ucbw->ucw", fa, Xi)
        b = np.zeros_like(a) if ss is None else np.einsum("bw,ucbw->ucw", ss, Xi)
    else:
        a, b = np.einsum("ub,ucbw->ucw", fa, Xi), np.einsum("ub,ucbw->ucw", ss, Xi)
    S = np.stack([np.stack([np.sum(w ** k * q, axis=-1) for k in (0, 1, 2, 4)], -1)
                  for q in (0.5 * np.abs(a) ** 2, 0.5 * np.abs(b) ** 2, 0.5 * (a * np.conj(b)).real)], 2)      # [U, nC, 3, 4]
    cs, sn = np.cos(angles), np.sin(angles)
    lam = c * c * (cs[:, None] ** 2 * S[:, :, None, 0] - 2 * (sn * cs)[:, None] * S[:, :, None, 2] + sn[:, None] ** 2 * S[:, :, None, 1])
    return time.perf_counter() - t0, np.sqrt(np.maximum(lam[..., 0], 0))


def run(name, U, nC, n, nw, form, numpy_units):
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(1)
    Xi = torch.complex(torch.randn(U, nC, n, nw, device=dev, dtype=torch.float64, generator=g),
                       torch.randn(U, nC, n, nw, device=dev, dtype=torch.float64, generator=g))
    w = torch.arange(1, nw + 1, device=dev, dtype=torch.float64) * (3.0 / nw)
    dw = 3.0 / nw
    rng = np.random.default_rng(2)
    angles = np.linspace(0, 2 * np.pi, 50)
    d, t = 10.0, 0.083
    c = (d / 2) / (np.pi / 8 * t * d ** 3) / 1e6
    if form == "coef":
        fa_h, ss_h = rng.normal(size=(n, nw)) + 1j * rng.normal(size=(n, nw)), None
        fa, ss = torch.from_numpy(fa_h).to(dev), None
        rows = [dict(coef=torch.from_numpy((c * np.cos(th) * fa_h)[None]).to(dev)) for th in angles]
        all_rows = dict(coef=torch.from_numpy(c * np.cos(angles)[:, None, None] * fa_h[None]).to(dev))
        ch_bytes = n * nw * 16
    else:
        fa_h, ss_h = rng.normal(size=(U, n)), rng.normal(size=(U, n))
        fa, ss = torch.from_numpy(fa_h[:, None]).to(dev), torch.from_numpy(ss_h[:, None]).to(dev)
        Rt = c * (np.cos(angles)[None, :, None] * fa_h[:, None] - np.sin(angles)[None, :, None] * ss_h[:, None])    # [U, nA, n]
        rows = [dict(R=torch.from_numpy(np.ascontiguousarray(Rt[:, j:j + 1])).to(dev)) for j in range(len(angles))]
        all_rows = dict(R=torch.from_numpy(Rt).to(dev))
        ch_bytes = U * 2 * n * 8
    keep = []

    def stress():
        be = solver._Device(dev)
        out = solver._stress_ring(be, Xi, w, fa, ss, angles, d, t, 4.0, 1.0, "dirlik", None, None, None, False, None, None, dw, 0)
        keep[:] = [out, be]
        return out

    def fat(ch):
        be = solver._Device(dev)
        out = solver._fatigue(be, Xi, w, 4.0, ch.get("R"), None, ch.get("coef"), None, 1.0, "dirlik", None, False, False, 0)
        keep.append((out, be))
        return out

    def loop():
        keep.clear()
        return [fat(ch) for ch in rows]

    def one():
        keep.clear()
        return fat(all_rows)
    t_s = device_time(stress)
    t_loop = device_time(loop, reps=5, inner=1)
    t_one = device_time(one)
    out = stress()
    ref = loop()
    torch.cuda.synchronize()
    DEL = out["DEL"][:, :, 0].cpu().numpy()                                # [U, nC, nA]
    DEL_loop = np.stack([r["DEL"][:, :, 0].cpu().numpy() for r in ref], -1)
    err_del = float(np.max(np.abs(DEL - DEL_loop) / np.abs(DEL_loop)))
    Xh = Xi[:numpy_units].cpu().numpy()
    t_np, sd_np = numpy_stress(Xh, w.cpu().numpy(), fa_h if form == "coef" else fa_h[:numpy_units], None if ss_h is None else ss_h[:numpy_units],
                               angles, c)
    sd = out["std"][:numpy_units, :, 0].cpu().numpy()
    err_sd = float(np.max(np.abs(sd - sd_np) / np.max(sd_np)))
    t_np_full = t_np * U / numpy_units
    by = U * nC * n * nw * 16 + ch_bytes
    return dict(shape=name, units=U, cases=nC, n_dof=n, nw=nw, angles=len(angles), form=form,
                stress_ring_s_median=t_s[0], stress_ring_s_min=t_s[1], stress_ring_s_max=t_s[2],
                fatigue_loop_50_calls_s_median=t_loop[0], fatigue_one_call_50_rows_s_median=t_one[0],
                speedup_vs_fatigue_loop=t_loop[0] / t_s[0], speedup_vs_fatigue_one_call=t_one[0] / t_s[0],
                bytes_read=by, GBps=by / t_s[0] / 1e9, share_of_3p35TBps=by / t_s[0] / HBM,
                numpy_s=t_np_full, numpy_units_timed=numpy_units, speedup_vs_numpy=t_np_full / t_s[0],
                max_rel_err_DEL_vs_fatigue_loop=err_del, max_err_std_vs_numpy_rel_to_max=err_sd)


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else None
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    lines = ["device: " + smi]
    res = [run("rigid sweep 1250 designs x 8 cases x 1024 bins x 50 angles, Mbase coefficients (fore-aft only)", 1250, 8, 6, 1024, "coef", 125),
           run("flexible batch 256 FOWTs x 150 DOFs x 8 cases x 256 bins x 50 angles, MbaseY / MbaseX rows", 256, 8, 150, 256, "R", 32)]
    for r in res:
        lines.append(json.dumps(r))
    txt = "\n".join(lines)
    print(txt)
    if out:
        with open(out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
