#!/usr/bin/env python
"""Generate tests/golden/ops_<name>.npz: every load case solved at its own turbine operating point by the UNMODIFIED
reference, run under oracle/ref_harness.py as make_golden_rotor.py runs it.

Model.solveStatics is patched to the case-by-case hook where the reference calls calcTurbineConstants(case)
(raft_model.py:602, 730, 957).  Inside it the reference's own FOWT.calcTurbineConstants(case) runs, with Rotor.calcAero
replaced by a seeded stand-in that returns calcAero's structure (f_aero0, f_aero, a_aero, b_aero): only the [0, 0] entries
set, then rotateMatrix6 by R_q (raft_rotor.py:879-896), seeded by the wind speed so that equal speeds give equal arrays, with
a positive damping of a realistic size.  The reference then does its own T^T a T, its gating (wind_speed 0,
turbine_status) and its gyroscopic term, for which I_drivetrain is set nonzero.  The rotor outputs' calcAero results
(control transfer function, wind amplitudes, gains, operating point) are make_golden_rotor.py's stand-ins, set in the same
hook, so that rotors= is checked on the same run.  Statics, mooring and lines2ss are as in make_golden_tmoor.py.

Each file stores what make_golden_rotor.py stores (design_json, cases_json, w, mat<i>_*, hubT<i>, in<i>_*, Xi_c<c>, C_array,
the rotor keys fowt<i>_<key>_c<c>) and per FOWT i and case c: the snapshot right after calcTurbineConstants (``op<i>_c<c>_A_aero``
[6,6,nw,nrot], ``_B_aero``, ``_B_gyro`` [6,6,nrot], ``_f_aero0`` [6,nrot]), packer.pack_turbine_channels of the live FOWT at
that moment (``ch<i>_c<c>_coef`` / ``_avg``) and the reference's motion and Mbase statistics (``cm<i>_<key>_c<c>``), plus
array_mooring (``arr_<key>_c<c>``) where the design has one.

Designs: VolturnUS-S (rigid) with five cases -- 12 m/s one train, 8 m/s two trains, 12 m/s with another sea state (the
first case's operating point), 18 m/s, wind speed 0; the two-FOWT farm with array mooring: the first three; farm24: the first.

Usage (reference tree present):  python tests/golden/make_golden_ops.py [rigid|farm|farm24]
"""
import contextlib
import io
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg  # noqa: E402
import make_golden_rotor as mgr  # noqa: E402
import make_golden_tmoor as mgt  # noqa: E402

rh = mg.rh
MOTION = ("surge", "sway", "heave", "roll", "pitch", "yaw")
CM_KEYS = tuple(m + s for m in MOTION for s in ("_std", "_PSD")) + ("Mbase_avg", "Mbase_std", "Mbase_max", "Mbase_min", "Mbase_PSD")
ARR_KEYS = ("Tmoor_avg", "Tmoor_std", "Tmoor_max", "Tmoor_min", "Tmoor_PSD")


def five_cases():
    c = mgr.three_cases()
    c3 = dict(wave_height=3.0, wave_period=8.0, wave_heading=-20.0, wind_speed=12.0, turbulence="IIB_NTM")
    c4 = dict(wave_height=7.0, wave_period=13.0, wave_heading=15.0, wind_speed=18.0, turbulence="IIB_NTM")
    return [dict(x, turbine_status="operating") for x in (c[0], c[1], c3, c4, c[2])]


def calc_aero_stand_in(raft, seed):
    """Rotor.calcAero's results, seeded by the wind speed: a_aero / b_aero with only [0, 0] set, rotated by R_q."""
    rot6 = raft.helpers.rotateMatrix6

    def calcAero(self, case, current=False, display=0):
        U = float(case.get("wind_speed", 10.0))
        rng = np.random.default_rng([seed, int(round(U * 1000))])
        w = np.asarray(self.w)
        nw = len(w)
        a, b = np.zeros([6, 6, nw]), np.zeros([6, 6, nw])
        a[0, 0] = rng.uniform(-2e5, 2e5) * np.exp(-w)                        # aero added mass [kg]
        b[0, 0] = rng.uniform(3e5, 1.2e6) * (1.0 + 0.2 * np.sin(w * rng.uniform(1, 3)))   # aero damping [N s/m], > 0
        f = np.zeros([6, nw], dtype=complex)
        f0 = np.zeros(6)
        f0[0] = rng.uniform(1e6, 2.5e6)
        f0[:3] = self.R_q @ f0[:3]
        return f0, f, rot6(a, self.R_q), rot6(b, self.R_q)
    return calcAero


def analyze(name, design, cases, model_setup=None, seed=41):
    raft = rh.load_reference()
    mgt.set_cases(design, cases)
    model = rh.build_model(design)
    if model_setup:
        model_setup(model)
    w = np.array(model.w)
    rng = np.random.default_rng(seed)
    snaps, ops, chans = [], [], []
    saved_aero = raft.raft_rotor.Rotor.calcAero
    for f in model.fowtList:
        for rot in f.rotorList:
            rot.aeroServoMod = 2

    def statics(self, case, display=0):            # the case-by-case hook: calcTurbineConstants(case) with the stand-in
        snaps.append([[mgr.stand_in(rot, w, rng, case) for rot in f.rotorList] for f in self.fowtList])
        row_op, row_ch = [], []
        for f in self.fowtList:
            for rot in f.rotorList:
                rot.I_drivetrain = 3.2e8               # [kg m^2]: the gyroscopic term (raft_fowt.py:1569-1581)
            f.calcTurbineConstants(case, ptfm_pitch=0)
            row_op.append({k: np.array(getattr(f, k)) for k in ("A_aero", "B_aero", "B_gyro", "f_aero0")})
            row_ch.append(mg.packer.pack_turbine_channels(f))
        ops.append(row_op)
        chans.append(row_ch)
    rec = mgt.record_xi(model)
    try:
        raft.raft_rotor.Rotor.calcAero = calc_aero_stand_in(raft, seed)
        with mgt.patched(raft), contextlib.redirect_stdout(io.StringIO()):
            raft.raft_model.Model.solveStatics = statics    # restored by patched() on exit
            model.analyzeCases()
    finally:
        raft.raft_rotor.Rotor.calcAero = saved_aero
    cm = model.results["case_metrics"]
    out = dict(w=w, design_json=np.array(json.dumps(design, default=float)), cases_json=np.array(json.dumps(cases)),
               n_fowt=np.int32(model.nFOWT))
    for ic, x in enumerate(rec):
        out["Xi_c%d" % ic] = x
    for i, f in enumerate(model.fowtList):
        for k in mgr.MATS:
            out["mat%d_%s" % (i, k)] = np.array(getattr(f, k), dtype=float)
        mgr.store_fowt(out, i, f, [s[i] for s in snaps], [cm[ic][i] for ic in range(len(cases))])
        for ic in range(len(cases)):
            for k, v in ops[ic][i].items():
                out["op%d_c%d_%s" % (i, ic, k)] = v
            out["ch%d_c%d_coef" % (i, ic)] = chans[ic][i]["coef"]
            out["ch%d_c%d_avg" % (i, ic)] = chans[ic][i]["avg"]
            for k in CM_KEYS:
                if k in cm[ic][i]:
                    out["cm%d_%s_c%d" % (i, k, ic)] = np.array(cm[ic][i][k])
    for ic in range(len(cases)):
        for k in ARR_KEYS:
            if "array_mooring" in cm[ic] and k in cm[ic]["array_mooring"]:
                out["arr_%s_c%d" % (k, ic)] = np.array(cm[ic]["array_mooring"][k])
    if model.ms is not None:
        out["C_array"] = np.array(model.ms.C)
        out["arr_J"], out["arr_T0"] = np.array(model.ms.J), np.array(model.ms.T0)
    path = os.path.join(mg.OUT, "ops_%s.npz" % name)
    np.savez_compressed(path, **out)
    print("ops_%-24s %.0f KB" % (name, os.path.getsize(path) / 1024))


def rigid():
    td = os.path.join(mg.REF, "tests", "test_data")
    design = rh.load_design(os.path.join(td, "VolturnUS-S.yaml"), strip=False)
    design.pop("mooring", None)
    design["platform"]["potSecOrder"] = 0
    analyze("VolturnUS-S", design, five_cases())


def farm():
    design = mgr._farm_design(os.path.join(mg.REF, "designs", "VolturnUS-S_farm.yaml"))
    analyze("farm", design, five_cases()[:3], mgr._array_mooring(5), seed=42)


def farm24():
    import tempfile
    import yaml
    src = os.path.join(mg.REF, "designs", "VolturnUS-S_farm.yaml")
    with open(src) as fh:
        design = yaml.load(fh, Loader=yaml.FullLoader)
    ks = design["array"]["keys"]
    proto = list(design["array"]["data"][1])
    data = []
    for u in range(mgr.mf24.ROWS * mgr.mf24.COLS):
        row = list(proto)
        row[ks.index("x_location")] = mgr.mf24.SPACING * (u % mgr.mf24.COLS)
        row[ks.index("y_location")] = mgr.mf24.SPACING * (u // mgr.mf24.COLS)
        row[ks.index("heading_adjust")] = 180 if u % 5 == 0 else 0
        data.append(row)
    design["array"]["data"] = data
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "farm24.yaml")
        with open(path, "w") as fh:
            yaml.dump(design, fh)
        design = mgr._farm_design(path)
    analyze("farm24", design, five_cases()[:1], mgr._array_mooring(6), seed=43)


def main():
    only = sys.argv[1] if len(sys.argv) > 1 else None
    for k, fn in dict(rigid=rigid, farm=farm, farm24=farm24).items():
        if only in (None, k):
            fn()


if __name__ == "__main__":
    main()
