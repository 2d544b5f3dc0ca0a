#!/usr/bin/env python
"""Generate tests/golden/flexout_VolturnUS-S-flexible.npz (run in the BUILD CONTAINER only, like make_golden.py, whose
harness and helpers it uses): a flexible FOWT through the unmodified reference's Model.solveDynamics with several wave
trains and FOWT.saveTurbineOutputs.

Usage:  python tests/golden/make_golden_flexout.py
"""
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import OUT, count_passes, packer, rh  # noqa: E402


def fixture_flexout(name, yaml_path):
    """Flexible FOWT (nDOF = 150) through Model.solveDynamics and FOWT.saveTurbineOutputs of the unmodified reference:
    two single-train cases and one case with two wave trains (raft_model.py:1200-1236 with nDOF > 6), the packed output
    channels (packer.pack_general_channels) and the statistics saveTurbineOutputs stores for them (raft_fowt.py:2299-2604).
    Same set-up as fixture_flexible: turbine kept (flexible tower), CCBlade stubbed, mooring stripped, synthetic C_moor on
    the rigid-body DOFs, the design's own frequency grid."""
    import contextlib
    import copy
    import io
    t0 = time.time()
    raft = rh.load_reference()
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
    P = packer.pack_general_dofs(fowt)
    ch = packer.pack_general_channels(fowt)
    out = {"P_" + k: np.asarray(v) for k, v in P.items()}
    out["gen_M"] = np.sum(fowt.A_aero, axis=3)[:, :, 0] + fowt.M_struc + fowt.A_hydro_morison
    out["gen_B"] = np.sum(fowt.B_aero, axis=3)[:, :, 0] + fowt.B_struc + np.sum(fowt.B_gyro, axis=2)
    out["gen_C"] = fowt.C_struc + fowt.C_hydro + Cmoor + fowt.C_elast
    out["n_iter"], out["xi_start"] = np.int32(int(model.nIter)), np.float64(model.XiStart)
    out["ch_names"] = np.array(["%s:%s" % (nm, "" if ir is None else ir) for nm, ir in ch["names"]])
    out["ch_R"], out["ch_wpow"], out["ch_avg"] = ch["R"], ch["wpow"], ch["avg"]
    cases = [rh.make_case(6.0, 12.0, 30.0), rh.make_case(2.0, 8.0, -60.0)]
    c3 = rh.make_case()
    c3.update(wave_heading=[0.0, 60.0], wave_period=[10.0, 14.0], wave_height=[4.0, 2.0], wave_spectrum=["JONSWAP"] * 2, wave_gamma=[0.0, 0.0])
    cases.append(c3)
    chans = ["surge", "sway", "heave", "roll", "pitch", "yaw", "AxRNA", "AyRNA", "AzRNA",
             "FbaseX", "FbaseY", "FbaseZ", "MbaseX", "MbaseY", "MbaseZ", "Mbase"]
    keys = [c + s for c in chans for s in ("_avg", "_std", "_max", "_min", "_PSD")] + [c + "_RA" for c in chans[:6]]
    cnt, orig = count_passes(fowt)
    for ic, case in enumerate(cases):
        cnt[0] = 0
        x = rh.solve_dynamics(model, case)
        out["ref_run_case%d_passes" % ic] = np.int32(cnt[0])
        res = {}
        with contextlib.redirect_stdout(io.StringIO()):
            fowt.saveTurbineOutputs(res, case)
        out["ref_run_case%d_Xi" % ic] = np.array(x)                      # Model.Xi [nWaves+1, nDOF, nw]
        out["ref_run_case%d_trains" % ic] = np.array([np.atleast_1d(case[k]) for k in ("wave_height", "wave_period", "wave_heading")], dtype=float).T
        for k in keys:
            out["ref_run_case%d_%s" % (ic, k)] = np.array(res[k])
    fowt.calcHydroLinearization = orig
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **out)
    print("%-28s nDOF=%3d nw=%3d cases=%d  %.1f s  %.0f KB" % (name, n, len(P["w"]), len(cases), time.time() - t0, os.path.getsize(path) / 1024))


if __name__ == "__main__":
    fixture_flexout("flexout_VolturnUS-S-flexible", os.path.join(rh.REF_ROOT, "tests", "test_data", "VolturnUS-S-flexible.yaml"))
