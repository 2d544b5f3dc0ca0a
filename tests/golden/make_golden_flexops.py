#!/usr/bin/env python
"""Generate tests/golden/flexops_<design>_VolturnUS-S-flexible.npz: a flexible FOWT (150 DOFs) whose every load case is
solved at its own turbine operating point by the UNMODIFIED reference, run under oracle/ref_harness.py.

Set-up: VolturnUS-S-flexible as make_golden_rotor.flexible() builds it ("strip": strip theory only, so the frequency-dependent
support comes from the operating points alone) or as make_golden_flexfd.build() does without its synthetic rotor matrices
("bem": potModMaster 3 with the marin_semi WAMIT coefficients on DOFs 0-5).  For every case of make_golden_ops.five_cases()
-- 12 m/s one train, 8 m/s two trains, 12 m/s with another sea state (case 0's operating point), 18 m/s, wind speed 0 --
the reference's own FOWT.calcTurbineConstants(case) runs with Rotor.calcAero replaced by make_golden_ops.calc_aero_stand_in
(seeded by the wind speed), aeroServoMod 2 and I_drivetrain 3.2e8: the reference does its own T^T a T to the reduced DOFs,
its own gating and its own gyroscopic term.  Then Model.solveDynamics(case) and FOWT.saveTurbineOutputs(case), with the
rotor outputs' stand-ins of make_golden_rotor.stand_in set in the same step, so that the rotor keys are checked too.

Stored: the packed tables that differ from flex_VolturnUS-S-flexible.npz (``P_*``, ``P_keys`` as in make_golden_flexfd.py);
packer.pack_general_matrices(fowt, states=...) (``M``, ``B``, ``C``, ``fd_*``); per case c the snapshot right after
calcTurbineConstants restricted to its nonzero support (``op_c<c>_idx`` and ``op_c<c>_A_aero`` [k,k,nw,nrot], ``_B_aero``,
``_B_gyro`` [k,k,nrot]; everything off the support is asserted exactly zero here), Model.Xi of every train
(``ref_run_case<c>_Xi``), the trains, the pass count, the motion and tower-base entries of saveTurbineOutputs
(``ref_run_case<c>_<key>``) and its rotor keys (``fowt0_<key>_c<c>``, with the stand-in inputs ``in0_*`` and hub rows
``hubT0`` as make_golden_rotor.py stores them); the output channels (``ch_*``, packer.pack_general_channels); cases_json.

Usage (reference tree present):  python tests/golden/make_golden_flexops.py [strip|bem]
"""
import contextlib
import copy
import io
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg  # noqa: E402
import make_golden_flexfd as mgf  # noqa: E402
import make_golden_ops as mgo  # noqa: E402
import make_golden_rotor as mgr  # noqa: E402

rh = mg.rh
CHANS = ["surge", "sway", "heave", "roll", "pitch", "yaw", "AxRNA", "AyRNA", "AzRNA",
         "FbaseX", "FbaseY", "FbaseZ", "MbaseX", "MbaseY", "MbaseZ", "Mbase"]
KEYS = [c + s for c in CHANS for s in ("_avg", "_std", "_max", "_min", "_PSD")]
YAML = ("tests", "test_data", "VolturnUS-S-flexible.yaml")


def build_strip():
    """make_golden_rotor.flexible()'s model: strip theory only, mooring stripped, synthetic C_moor on DOFs 0-5."""
    raft = rh.load_reference()
    design = rh.load_design(os.path.join(mg.REF, *YAML), strip=False)
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
    return model, fowt


def build_bem():
    """make_golden_flexfd.build() without its synthetic rotor matrices: marin_semi BEM coefficients on DOFs 0-5."""
    return mgf.build(os.path.join(mg.REF, *YAML), aero=False)


def support(*tabs):
    """Reduced DOFs whose rows or columns of any of the [n, n, ...] tables hold a nonzero entry."""
    nz = np.zeros(tabs[0].shape[:2], dtype=bool)
    for t in tabs:
        nz |= np.any(t.reshape(t.shape[0], t.shape[1], -1) != 0, axis=2)
    return np.nonzero(nz.any(axis=0) | nz.any(axis=1))[0].astype(np.int32)


def fixture(name, model, fowt, seed=44):
    t0 = time.time()
    raft = rh.load_reference()
    w = np.array(model.w)
    cases = mgo.five_cases()
    rng = np.random.default_rng(seed)
    saved = raft.raft_rotor.Rotor.calcAero
    cnt, orig = mg.count_passes(fowt)
    out, snaps, states, metrics = {}, [], [], []
    try:
        raft.raft_rotor.Rotor.calcAero = mgo.calc_aero_stand_in(raft, seed)
        for ic, c in enumerate(cases):
            case = dict(rh.make_case(), **c)
            snaps.append([mgr.stand_in(rot, w, rng, case) for rot in fowt.rotorList])   # the rotor outputs' calcAero results
            for rot in fowt.rotorList:
                rot.aeroServoMod = 2
                rot.I_drivetrain = 3.2e8               # [kg m^2]: the gyroscopic term (raft_fowt.py:1569-1581)
            with contextlib.redirect_stdout(io.StringIO()):
                fowt.calcTurbineConstants(case, ptfm_pitch=0)
            s = {k: np.array(getattr(fowt, k), dtype=float) for k in ("A_aero", "B_aero", "B_gyro")}
            states.append(s)
            idx = support(s["A_aero"], s["B_aero"], s["B_gyro"])
            off = np.ones(fowt.nDOF, dtype=bool)
            off[idx] = False
            for k, v in s.items():
                assert not np.any(v[off]) and not np.any(v[:, off]), (ic, k)
                out["op_c%d_%s" % (ic, k)] = np.ascontiguousarray(v[np.ix_(idx, idx)])
            out["op_c%d_idx" % ic] = idx
            cnt[0] = 0
            x = rh.solve_dynamics(model, case)
            nT = len(np.atleast_1d(case["wave_height"]))
            out["ref_run_case%d_Xi" % ic] = np.array(x)[:nT]
            out["ref_run_case%d_passes" % ic] = np.int32(cnt[0])
            out["ref_run_case%d_trains" % ic] = np.array([np.atleast_1d(case[k]) for k in ("wave_height", "wave_period", "wave_heading")],
                                                         dtype=float).T
            res = {}
            with contextlib.redirect_stdout(io.StringIO()):
                fowt.saveTurbineOutputs(res, case)
            for k in KEYS:
                out["ref_run_case%d_%s" % (ic, k)] = np.array(res[k])
            metrics.append(res)
    finally:
        raft.raft_rotor.Rotor.calcAero = saved
        fowt.calcHydroLinearization = orig
    # the packer on the live FOWT with these states
    P = mg.packer.pack_general_dofs(fowt)
    G = mg.packer.pack_general_matrices(fowt, states=states)
    base = np.load(os.path.join(mg.OUT, "flex_VolturnUS-S-flexible.npz"))
    for k, v in P.items():
        v = np.asarray(v)
        old = base["P_" + k] if "P_" + k in base.files else None
        if old is None or old.shape != v.shape or not np.array_equal(old, v):
            out["P_" + k] = v
    out["P_keys"] = np.array(sorted(P))
    out["M"], out["B"], out["C"] = G["M"], G["B"], G["C"]
    for k, v in G["fd"].items():
        out["fd_" + k] = np.asarray(v)
    ch = mg.packer.pack_general_channels(fowt)
    out["ch_names"] = np.array(["%s:%s" % (nm, "" if ir is None else ir) for nm, ir in ch["names"]])
    out["ch_R"], out["ch_wpow"], out["ch_avg"] = ch["R"], ch["wpow"], ch["avg"]
    mgr.store_fowt(out, 0, fowt, snaps, metrics)
    out.update(w=w, cases_json=np.array(json.dumps(cases)), n_cases=np.int32(len(cases)), n_iter=np.int32(int(model.nIter)),
               xi_start=np.float64(model.XiStart))
    path = os.path.join(mg.OUT, "flexops_%s_VolturnUS-S-flexible.npz" % name)
    np.savez_compressed(path, **out)
    print("flexops_%-5s fd support %s, op %s, passes %s, %.1f s, %.0f KB"
          % (name, G["fd"]["fd_idx"].tolist(), G["ops"]["op"].tolist(), [int(out["ref_run_case%d_passes" % c]) for c in range(len(cases))],
             time.time() - t0, os.path.getsize(path) / 1024))


def main():
    only = sys.argv[1] if len(sys.argv) > 1 else None
    for k, fn in dict(strip=build_strip, bem=build_bem).items():
        if only in (None, k):
            fixture(k, *fn())


if __name__ == "__main__":
    main()
