#!/usr/bin/env python
"""Generate tests/golden/stress_VolturnUS-S-flexible.npz (run in the BUILD CONTAINER only, like make_golden.py, whose
harness and helpers it uses): tower-base axial stress around the circumference of a flexible FOWT, from the unmodified
reference's helpers.getSigmaXPSD on its own tower-base loads.

The run is that of make_golden_flexout.py (VolturnUS-S-flexible, 150 DOFs, the same three cases, one of them with two
wave trains), case by case: Model.solveDynamics, then the tower-base internal loads Fi_base = -Kf[base] Xi_internal that
FOWT.saveTurbineOutputs forms (raft_fowt.py:2541-2560), and getSigmaXPSD(Fi_base[:, 4], Fi_base[:, 3], w, angles, d, t)
(helpers.py:1164), the fore-aft moment MbaseY and the side-side moment MbaseX, at the helper's defaults (50 angles over
[0, 2 pi], d = 10, t = 0.083) and at a second set of angles, d and t.

A quirk of the helper: its sigmaX is [nw, nA] (or [rows * nw, nA] for a case with several rows, which np.meshgrid
flattens) and getPSD sums over axis 0, so what it returns per angle is sum over the case's rows and bins of
1/2 |sigma_x|^2 / dw, i.e. std(theta)^2 / dw -- not a per-bin PSD.  The fixture stores exactly that (ref_run_case<i>_
sigPSD_<set>), and the tests compare std^2 / dw with it.

Stored per case i: Fi_base fore-aft / side-side amplitudes of all rows of Model.Xi (trains + the zero row) [nRows, nw],
the reference's MbaseY_avg / MbaseX_avg (saveTurbineOutputs), and per set s the helper's output [nA]; per set its
angles, d and t.

Usage:  python tests/golden/make_golden_stress.py
"""
import contextlib
import copy
import io
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import OUT, rh  # noqa: E402

SETS = dict(default=(np.linspace(0, 2 * np.pi, 50), 10.0, 0.083),
            other=(np.linspace(-0.3, 3.5, 23), 8.5, 0.05))


def fixture_stress(name, yaml_path):
    t0 = time.time()
    raft = rh.load_reference()
    from raft import helpers
    design = rh.load_design(yaml_path, strip=False)
    design.pop("mooring", None)
    design["platform"]["potSecOrder"] = 0
    with contextlib.redirect_stdout(io.StringIO()):
        model = raft.Model(copy.deepcopy(design))
        fowt = model.fowtList[0]
        fowt.setPosition(np.zeros(fowt.nDOF))
        fowt.calcStatics()
        fowt.calcTurbineConstants(rh.make_case(), ptfm_pitch=0)
        fowt.calcHydroConstants()
    n = fowt.nDOF
    Cmoor = np.zeros([n, n])
    Cmoor[:6, :6] = rh.C_MOOR_DEFAULT
    fowt.C_moor = Cmoor
    tow = fowt.memberList[fowt.nplatmems]
    i0, i1 = tow.nodeList[0].id, tow.nodeList[-1].id
    first = tow.nodeList[0].r0[2] <= tow.nodeList[-1].r0[2]
    cases = [rh.make_case(6.0, 12.0, 30.0), rh.make_case(2.0, 8.0, -60.0)]
    c3 = rh.make_case()
    c3.update(wave_heading=[0.0, 60.0], wave_period=[10.0, 14.0], wave_height=[4.0, 2.0], wave_spectrum=["JONSWAP"] * 2, wave_gamma=[0.0, 0.0])
    cases.append(c3)
    w = np.asarray(fowt.w, dtype=float)
    out = dict(w=w, n_cases=np.int32(len(cases)))
    for s, (angles, d, t) in SETS.items():
        out["%s_angles" % s], out["%s_d" % s], out["%s_t" % s] = angles, np.float64(d), np.float64(t)
    for ic, case in enumerate(cases):
        rh.solve_dynamics(model, case)
        res = {}
        with contextlib.redirect_stdout(io.StringIO()):
            fowt.saveTurbineOutputs(res, case)
        Xi_int = fowt.Xi_fullDOF[:, i0 * 6:(i1 + 1) * 6, :]
        Fi = np.stack([-tow.Kf @ Xi_int[h] for h in range(Xi_int.shape[0])])
        Fi_base = Fi[:, 0:6, :] if first else Fi[:, -6:, :]
        out["ref_run_case%d_FA" % ic] = np.array(Fi_base[:, 4, :])
        out["ref_run_case%d_SS" % ic] = np.array(Fi_base[:, 3, :])
        out["ref_run_case%d_MbaseY_avg" % ic] = np.array(res["MbaseY_avg"])
        out["ref_run_case%d_MbaseX_avg" % ic] = np.array(res["MbaseX_avg"])
        out["ref_run_case%d_MbaseY_std" % ic] = np.array(res["MbaseY_std"])
        for s, (angles, d, t) in SETS.items():
            psd = helpers.getSigmaXPSD(Fi_base[:, 4], Fi_base[:, 3], w, angles, d, t)[0]
            out["ref_run_case%d_sigPSD_%s" % (ic, s)] = np.asarray(psd, dtype=float)
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **out)
    print("%-28s nDOF=%3d nw=%3d cases=%d  %.1f s  %.0f KB" % (name, n, len(w), len(cases), time.time() - t0, os.path.getsize(path) / 1024))


if __name__ == "__main__":
    fixture_stress("stress_VolturnUS-S-flexible", os.path.join(rh.REF_ROOT, "tests", "test_data", "VolturnUS-S-flexible.yaml"))
