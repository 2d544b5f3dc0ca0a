#!/usr/bin/env python
"""Generate tests/golden/rotor_<name>.npz: rotor speed, generator torque and blade pitch statistics from the UNMODIFIED
reference's own output code, FOWT.saveTurbineOutputs (raft_fowt.py:2610-2679), run under oracle/ref_harness.py.

CCBlade is absent here, so Rotor.calcAero's results are stand-ins: for every case each rotor gets what calcAero would leave
on it -- a seeded complex control transfer function C [nw], turbulent-wind amplitudes V_w = sqrt(2 S dw) of the wind
spectrum S, seeded kp_beta / ki_beta, Omega_case, aero_torque, aero_power and pitch_case -- and aeroServoMod 2 (the setting
of designs/VolturnUS-S.yaml), with I_drivetrain 0.  S is the reference's own rotor-averaged Rotor.IECKaimal(case) spectrum
(IEC class IIB, normal turbulence), which runs under the harness, and V_w = sqrt(2 S dw) as calcAero forms it
(raft_rotor.py:866-869); with the wind speed 0 the rotor is inactive and V_w is left zero.  The aero loads stay those of
the harness's turbine constants (turbine off: zero A_aero, B_aero, f_aero, B_gyro), so the solve matrices do not depend on
the case and the project's solve reproduces the reference's Xi.  Ng is the turbine's own gear ratio (1: direct drive).

Rigid designs run the reference's own Model.analyzeCases (raft_model.py:264-433) as make_golden_tmoor.py does: statics are
skipped (Model.solveStatics is where calcTurbineConstants calls calcAero, so the stand-in values are set there, case by
case), lines2ss is the identity, and a farm's array mooring is a stand-in system with an injected stiffness.  The flexible
FOWT runs the reference's Model.solveDynamics and saveTurbineOutputs case by case, as make_golden_flexout.py does.

Each file stores per FOWT i: the reference's matrices for the project's Model (``mat<i>_*``) or generalised-DOF inputs
(P_*, gen_M, gen_B, gen_C), the 6 rows of fowt.T at each rotor's hub node (``hubT<i>`` [nrot, 6, nDOF]), the stand-in
inputs per case (``in<i>_C``, ``in<i>_V_w`` [nC, nrot, nw], ``in<i>_gains`` [nC, nrot, 4] = kp_tau, ki_tau, kp_beta,
ki_beta, ``in<i>_means`` [nC, nrot, 5] = Omega_case, aero_torque, Ng, aero_power, pitch_case), and every rotor key per case
(``fowt<i>_<key>_c<c>``; wind_PSD only where the reference sets it).  Also: the design (``design_json``), the cases
(``cases_json``), w, the reference's Model.Xi per case (``Xi_c<c>`` [nWaves+1, nDOF, nw]) and, for farms, C_array.

Cases: VolturnUS-S (rigid) and VolturnUS-S-flexible (150 DOFs): one wave train at 12 m/s, two wave trains at 8 m/s, and
wind_speed 0 (the rotor outputs are then all zero and wind_PSD is absent).  The two-FOWT farm: the first two of those;
farm24 (144 DOFs): the first.

Usage (build container, reference tree present):  python tests/golden/make_golden_rotor.py [rigid|farm|farm24|flexible]
"""
import contextlib
import copy
import io
import json
import os
import sys
import tempfile

import numpy as np
import yaml

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg  # noqa: E402
import make_golden_farm24 as mf24  # noqa: E402
import make_golden_tmoor as mgt  # noqa: E402

rh = mg.rh
KEYS = ("omega_avg", "omega_std", "omega_max", "omega_min", "omega_PSD", "torque_avg", "torque_std", "torque_PSD", "power_avg",
        "bPitch_avg", "bPitch_std", "bPitch_PSD", "wind_PSD")
MATS = ("M_struc", "B_struc", "C_struc", "C_hydro", "C_moor", "C_elast")


def stand_in(rot, w, rng, case):
    """What Rotor.calcAero(case) leaves on the rotor for aeroServoMod 2 (raft_rotor.py:866-945), seeded -> its snapshot."""
    nw, dw = len(w), w[1] - w[0]
    rot.aeroServoMod = 2
    rot.I_drivetrain = 0.0
    rot.C = (rng.normal(size=nw) + 1j * rng.normal(size=nw)) * 0.05 * w / (1.0 + w)
    S = rot.IECKaimal(case)[3] if float(case.get("wind_speed", 10.0)) > 0 else np.zeros(nw)   # PSD [(m/s)^2/(rad/s)]
    rot.V_w = np.array(np.sqrt(2 * S * dw), dtype=complex)
    rot.kp_beta, rot.ki_beta = -rng.uniform(0.005, 0.02), -rng.uniform(0.001, 0.004)
    rot.Omega_case = rng.uniform(5.0, 7.5)
    rot.aero_torque = rng.uniform(1.5e7, 2.2e7)
    rot.aero_power = rng.uniform(1.0e7, 1.5e7)
    rot.pitch_case = rng.uniform(0.0, 10.0)
    return (np.array(rot.C), np.array(rot.V_w), [rot.kp_tau, rot.ki_tau, rot.kp_beta, rot.ki_beta],
            [rot.Omega_case, rot.aero_torque, rot.Ng, rot.aero_power, rot.pitch_case])


def three_cases():
    c1 = dict(wave_height=6.0, wave_period=12.0, wave_heading=30.0, wind_speed=12.0, turbulence="IIB_NTM")
    c2 = dict(wave_height=[4.0, 2.0], wave_period=[10.0, 14.0], wave_heading=[0.0, 60.0], wave_spectrum=["JONSWAP"] * 2,
              wave_gamma=[0.0, 0.0], wind_speed=8.0, turbulence="IIB_NTM")
    c3 = dict(wave_height=3.5, wave_period=9.0, wave_heading=-45.0, wind_speed=0.0)
    return [c1, c2, c3]


def store_fowt(out, i, fowt, snaps, metrics):
    """Hub rows, stand-in inputs and the reference's rotor keys of FOWT i; snaps[c] = [snapshot per rotor]."""
    T = np.asarray(fowt.T, dtype=float)
    out["hubT%d" % i] = np.array([T[6 * r.nodeList[0].id:6 * r.nodeList[0].id + 6] for r in fowt.rotorList])
    for j, nm in enumerate(("C", "V_w", "gains", "means")):
        out["in%d_%s" % (i, nm)] = np.array([[s[j] for s in row] for row in snaps])
    for c, res in enumerate(metrics):
        for k in KEYS:
            if k in res:
                out["fowt%d_%s_c%d" % (i, k, c)] = np.array(res[k])


def save(name, out):
    path = os.path.join(mg.OUT, "rotor_%s.npz" % name)
    np.savez_compressed(path, **out)
    print("rotor_%-24s %.0f KB" % (name, os.path.getsize(path) / 1024))


def analyze(name, design, cases, model_setup=None, seed=31):
    """The reference's Model.analyzeCases on ``design`` with the stand-in rotors; stores what the project's Model needs."""
    raft = rh.load_reference()
    mgt.set_cases(design, cases)
    model = rh.build_model(design)
    if model_setup:
        model_setup(model)
    w = np.array(model.w)
    rng = np.random.default_rng(seed)
    snaps = []

    def statics(self, case, display=0):            # where calcTurbineConstants -> Rotor.calcAero would run for this case
        snaps.append([[stand_in(rot, w, rng, case) for rot in f.rotorList] for f in self.fowtList])
    rec = mgt.record_xi(model)
    with mgt.patched(raft), contextlib.redirect_stdout(io.StringIO()):
        raft.raft_model.Model.solveStatics = statics    # restored by patched() on exit
        model.analyzeCases()
    cm = model.results["case_metrics"]
    out = dict(w=w, design_json=np.array(json.dumps(design, default=float)), cases_json=np.array(json.dumps(cases)),
               n_fowt=np.int32(model.nFOWT))
    for ic, x in enumerate(rec):
        out["Xi_c%d" % ic] = x
    for i, f in enumerate(model.fowtList):
        for k in MATS:
            out["mat%d_%s" % (i, k)] = np.array(getattr(f, k), dtype=float)
        out["mat%d_B_struc" % i] = out["mat%d_B_struc" % i] + np.sum(f.B_gyro, axis=2)
        store_fowt(out, i, f, [s[i] for s in snaps], [cm[ic][i] for ic in range(len(cases))])
    if model.ms is not None:
        out["C_array"] = np.array(model.ms.C)
    save(name, out)


def rigid():
    td = os.path.join(mg.REF, "tests", "test_data")
    design = rh.load_design(os.path.join(td, "VolturnUS-S.yaml"), strip=False)
    design.pop("mooring", None)
    design["platform"]["potSecOrder"] = 0
    analyze("VolturnUS-S", design, three_cases())


def _farm_design(path):
    with open(path) as fh:
        design = yaml.load(fh, Loader=yaml.FullLoader)
    for k in ("mooring", "array_mooring"):
        design.pop(k, None)
    design["platform"]["potSecOrder"] = 0
    ks = design["array"]["keys"]
    for row in design["array"]["data"]:
        row[ks.index("mooringID")] = 0
    design["settings"]["max_freq"], design["settings"]["min_freq"] = 0.1024, 0.1024 / 48
    return design


def _array_mooring(seed):
    def setup(model):
        n = model.nDOF
        rng = np.random.default_rng(seed)
        A = rng.normal(size=(n, n)) * 2e4
        J, T0 = mgt.seeded_tensions(rng, 4, n)
        model.ms, model.moorMod = mgt.FakeMS(A @ A.T / n + np.diag([5e4] * n), J, T0), 0
    return setup


def farm():
    design = _farm_design(os.path.join(mg.REF, "designs", "VolturnUS-S_farm.yaml"))
    analyze("farm", design, three_cases()[:2], _array_mooring(5), seed=32)


def farm24():
    src = os.path.join(mg.REF, "designs", "VolturnUS-S_farm.yaml")
    with open(src) as fh:
        design = yaml.load(fh, Loader=yaml.FullLoader)
    ks = design["array"]["keys"]
    proto = list(design["array"]["data"][1])
    data = []
    for u in range(mf24.ROWS * mf24.COLS):
        row = list(proto)
        row[ks.index("x_location")] = mf24.SPACING * (u % mf24.COLS)
        row[ks.index("y_location")] = mf24.SPACING * (u // mf24.COLS)
        row[ks.index("heading_adjust")] = 180 if u % 5 == 0 else 0
        data.append(row)
    design["array"]["data"] = data
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "farm24.yaml")
        with open(path, "w") as fh:
            yaml.dump(design, fh)
        design = _farm_design(path)
    analyze("farm24", design, three_cases()[:1], _array_mooring(6), seed=33)


def flexible(seed=34):
    raft = rh.load_reference()
    td = os.path.join(mg.REF, "tests", "test_data")
    design = rh.load_design(os.path.join(td, "VolturnUS-S-flexible.yaml"), strip=False)
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
    P = mg.packer.pack_general_dofs(fowt)
    out = {"P_" + k: np.asarray(v) for k, v in P.items()}
    out["gen_M"] = np.sum(fowt.A_aero, axis=3)[:, :, 0] + fowt.M_struc + fowt.A_hydro_morison
    out["gen_B"] = np.sum(fowt.B_aero, axis=3)[:, :, 0] + fowt.B_struc + np.sum(fowt.B_gyro, axis=2)
    out["gen_C"] = fowt.C_struc + fowt.C_hydro + Cmoor + fowt.C_elast
    out["n_iter"], out["xi_start"] = np.int32(int(model.nIter)), np.float64(model.XiStart)
    w = np.array(model.w)
    cases = three_cases()
    out.update(w=w, cases_json=np.array(json.dumps(cases)), n_fowt=np.int32(1))
    rng = np.random.default_rng(seed)
    snaps, metrics = [], []
    for ic, c in enumerate(cases):
        case = dict(rh.make_case(), **c)
        snaps.append([stand_in(rot, w, rng, case) for rot in fowt.rotorList])
        out["Xi_c%d" % ic] = np.array(rh.solve_dynamics(model, case))
        res = {}
        with contextlib.redirect_stdout(io.StringIO()):
            fowt.saveTurbineOutputs(res, case)
        metrics.append(res)
    store_fowt(out, 0, fowt, snaps, metrics)
    save("VolturnUS-S-flexible", out)


def main():
    only = sys.argv[1] if len(sys.argv) > 1 else None
    for k, fn in dict(rigid=rigid, farm=farm, farm24=farm24, flexible=flexible).items():
        if only in (None, k):
            fn()


if __name__ == "__main__":
    main()
