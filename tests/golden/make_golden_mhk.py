#!/usr/bin/env python
"""Generate tests/golden/mhk_VolturnUS-S.npz: the inertial wave excitation of a submerged rotor (raft_fowt.py:1859-1888) and
the response it drives, from the UNMODIFIED reference run under oracle/ref_harness.py.

RM1_Floating.yaml (the reference's MHK design) cannot be built by this reference: a rotor whose blades lie wholly below the
waterline gets blade members (raft_rotor.py:384-386, bladeGeometry2Member) of type 3, which Member stores as the string "3"
and then refuses ("RAFT Members cannot start or end on the waterplane", raft_member.py:44, or "Member type 3 not
supported", :286, with a shaft tilt).  The script tries it, prints why it fails, and falls back to what the issue names:
VolturnUS-S with its turbine kept and the hub moved below the waterline (hHub = -18 m; the blades still cross the waterline,
so the reference builds no blade members and leaves I_hydro zero).  A seeded I_hydro [6,6] (with nonzero off-diagonal
blocks) is then set on the reference's rotor -- an injected input, like C_moor -- and everything else is the reference's
own: r3 from its setPosition, R_q, the hub node's id, fowt.T, getWaveKin, rotateMatrix6, the force loop after the train loop,
T^T.  CCBlade is stubbed and turbine_status is off; statics run without mooring (C_moor injected).

Stored: P_* (packer.pack_fowt on the live reference FOWT, rotor table included), I_hydro, R_q, r3, r6, hub_id, T_hub [6,6];
for a one-train and a two-train case the reference's F_hydro_iner [nWaves,6,nw] with the rotor and with I_hydro = 0, and the
hub kinematics rot.ud [nWaves,3,nw]; solveDynamics Xi [nCases,6,nw] and pass counts for seeded sea states.

Usage (build container, reference tree present):  python tests/golden/make_golden_mhk.py
"""
import copy
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402

rh = mg.rh
OUT = HERE


def try_rm1():
    design = rh.load_design(os.path.join(rh.REF_ROOT, "designs", "RM1_Floating.yaml"), nw=48, max_freq=0.4, strip=False)
    design.pop("mooring", None)
    design["platform"]["potModMaster"] = 1
    try:
        rh.build_model(design)
        return True
    except Exception as e:                                      # noqa: BLE001 -- reported and replaced, see the docstring
        print("RM1_Floating.yaml cannot be built by the reference: %s: %s" % (type(e).__name__, e))
        return False


def main():
    if try_rm1():
        raise SystemExit("RM1_Floating.yaml now builds: make this fixture from it")
    design = rh.load_design(os.path.join(rh.REF_ROOT, "designs", "VolturnUS-S.yaml"), nw=48, max_freq=0.4, strip=False)
    design.pop("mooring", None)
    design["platform"]["potModMaster"] = 1
    design["turbine"]["hHub"] = -18.0
    design["turbine"]["Zhub"] = -18.0
    model = rh.build_model(design)
    fowt = model.fowtList[0]
    rot = fowt.rotorList[0]
    assert rot.r3[2] < 0 and not rot.bladeMemberList
    rng = np.random.default_rng(7)
    A = rng.normal(size=(6, 6))
    rot.I_hydro = A @ A.T * 3e4 + np.diag([4e5, 1e5, 1e5, 3e6, 2e6, 2e6])
    P = mg.packer.pack_fowt(fowt)
    out = {"P_" + k: np.asarray(v) for k, v in P.items()}
    out.update(n_iter=np.int32(int(model.nIter)), xi_start=np.float64(model.XiStart), I_hydro=rot.I_hydro, R_q=np.array(rot.R_q),
               r3=np.array(rot.r3), r6=np.array(fowt.r6), hub_id=np.int32(rot.nodeList[0].id),
               T_hub=np.array(fowt.T[6 * rot.nodeList[0].id:6 * rot.nodeList[0].id + 6]))
    two = rh.make_case()
    two.update(wave_heading=[20.0, -65.0], wave_period=[10.0, 13.0], wave_height=[4.0, 2.5], wave_spectrum=["JONSWAP"] * 2,
               wave_gamma=[0.0, 0.0])
    I_keep = rot.I_hydro
    for name, case in (("one", rh.make_case(5.0, 11.0, 35.0)), ("two", two)):
        out["exc_%s_trains" % name] = np.array([np.atleast_1d(case[k]) for k in ("wave_height", "wave_period", "wave_heading")], dtype=float).T
        for tag, I in (("rot", I_keep), ("plain", np.zeros([6, 6]))):
            rot.I_hydro = I
            fowt.calcHydroExcitation(copy.deepcopy(case), memberList=fowt.memberList)
            out["exc_%s_F_hydro_iner_%s" % (name, tag)] = np.array(fowt.F_hydro_iner)
        out["exc_%s_ud" % name] = np.array(rot.ud[:fowt.nWaves])
        out["exc_%s_zeta" % name] = np.array(fowt.zeta)
    rot.I_hydro = I_keep
    Hs, Tp, beta = mg.seeded_cases(31, 4)
    cases = list(zip(Hs, Tp, beta))
    Xi, passes = mg.run_solves(model, cases)
    out.update(ref_run_solve_cases=np.array(cases, dtype=float), ref_run_solve_Xi=Xi, ref_run_solve_passes=passes)
    path = os.path.join(OUT, "mhk_VolturnUS-S.npz")
    np.savez_compressed(path, **out)
    print("mhk_VolturnUS-S: r3 %s, hub node %d, passes %s, %.0f KB" % (rot.r3, rot.nodeList[0].id, passes.tolist(), os.path.getsize(path) / 1024))


if __name__ == "__main__":
    main()
