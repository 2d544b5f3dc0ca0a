#!/usr/bin/env python
"""Generate tests/golden/flexfd_VolturnUS-S-flexible.npz (run in the BUILD CONTAINER only, like make_golden.py, whose
harness and helpers it uses): a flexible FOWT with an operating rotor and potential-flow coefficients through the unmodified
reference's Model.solveDynamics.

Set-up: VolturnUS-S-flexible as in make_golden_flexout.py (turbine kept, CCBlade stubbed, mooring stripped, synthetic C_moor
on DOFs 0-5), plus ``potModMaster 3``, ``potFirstOrder 1`` and the marin_semi WAMIT coefficients read by the reference's own
readHydro (A_BEM, B_BEM lumped on DOFs 0-5, X_BEM on 37 headings).  The rotor's aero-servo matrices are synthetic: a seeded,
smooth 6 x 6 a_aero(w), b_aero(w) about the hub node, mapped to the reduced DOFs as raft_fowt.py:1559-1561 does
(T^T a T with T = rot.nodeList[0].T), written into fowt.A_aero / B_aero after calcTurbineConstants.  Measured effect: with
them, the response of the first case moves by 17 % of its largest entry against the same run without them (printed
below as ``aero effect``).

Stored: the packed tables that differ from flex_VolturnUS-S-flexible.npz (``P_*``; the rest are taken from that file, and
``P_keys`` names the tables the design has: the flexible fixture's MacCamy-Fuchs tables are not among them),
packer.pack_general_matrices (``M``, ``B``, ``C``, ``fd_*``), and per case Model.Xi of every train, the pass count and every
train's F_BEM (reduced DOFs) and zeta.

Usage:  python tests/golden/make_golden_flexfd.py
"""
import contextlib
import copy
import io
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import OUT, count_passes, packer, rh  # noqa: E402

CASES = [  # (Hs, Tp, heading) per train
    [(6.0, 12.0, 30.0)],
    [(3.0, 9.0, 355.0)],          # BEM headings end at 350 deg: bracket wraps to 0 deg
    [(2.0, 8.0, -60.0)],
    [(4.0, 10.0, 0.0), (2.0, 14.0, 60.0)],
]


def synthetic_aero(w, seed=11):
    """Smooth 6 x 6 rotor added mass and damping [6,6,nw] about the hub: seeded symmetric positive parts, scaled per DOF
    (force rows ~1e5, moment rows ~1e7 in SI units), each entry modulated smoothly in w."""
    rng = np.random.default_rng(seed)
    s = np.sqrt(np.array([1e5, 1e5, 1e5, 1e7, 1e7, 1e7]))
    out = []
    for base in (2e-1, 6e-1):
        G = rng.standard_normal([6, 6])
        S = (G @ G.T / 6.0 + np.eye(6)) * np.outer(s, s) * base
        ph = rng.uniform(0, np.pi, [6, 6])
        ph = 0.5 * (ph + ph.T)
        out.append(S[:, :, None] * (1.0 + 0.5 * np.sin(w[None, None, :] + ph[:, :, None])) / (1.0 + 0.3 * w[None, None, :] ** 2))
    return out


def build(yaml_path, aero=True):
    raft = rh.load_reference()
    design = rh.load_design(yaml_path, strip=False)
    design.pop("mooring", None)
    pf = design["platform"]
    pf.update(potSecOrder=0, potModMaster=3, potFirstOrder=1,
              hydroPath=os.path.join(rh.REF_ROOT, "examples", "OC4semi-WAMIT_Coefs", "marin_semi"))
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
    if aero:
        a_aero, b_aero = synthetic_aero(np.asarray(fowt.w, dtype=float))
        T = fowt.rotorList[0].nodeList[0].T
        for iw in range(fowt.nw):                                     # raft_fowt.py:1559-1561
            fowt.A_aero[:, :, iw, 0] = T.T @ a_aero[:, :, iw] @ T
            fowt.B_aero[:, :, iw, 0] = T.T @ b_aero[:, :, iw] @ T
    return model, fowt


def run(model, fowt, cases):
    cnt, orig = count_passes(fowt)
    res = []
    for trains in cases:
        case = rh.make_case()
        tr = np.array(trains, dtype=float)
        if len(trains) == 1:
            case.update(wave_height=tr[0, 0], wave_period=tr[0, 1], wave_heading=tr[0, 2])
        else:
            case.update(wave_height=list(tr[:, 0]), wave_period=list(tr[:, 1]), wave_heading=list(tr[:, 2]),
                        wave_spectrum=["JONSWAP"] * len(trains), wave_gamma=[0.0] * len(trains))
        cnt[0] = 0
        x = rh.solve_dynamics(model, case)
        res.append(dict(Xi=np.array(x)[:len(trains)], passes=np.int32(cnt[0]), trains=tr,
                        F_BEM=np.array(fowt.F_BEM)[:len(trains)], zeta=np.array(fowt.zeta)[:len(trains)]))
    fowt.calcHydroLinearization = orig
    return res


def fixture_flexfd(name, yaml_path):
    t0 = time.time()
    model, fowt = build(yaml_path)
    P = packer.pack_general_dofs(fowt)
    G = packer.pack_general_matrices(fowt)
    base = np.load(os.path.join(OUT, "flex_VolturnUS-S-flexible.npz"))
    out = {}
    for k, v in P.items():
        v = np.asarray(v)
        old = base["P_" + k] if "P_" + k in base.files else None
        if old is None or old.shape != v.shape or not np.array_equal(old, v):
            out["P_" + k] = v
    out["P_keys"] = np.array(sorted(P))                               # keys of the flex fixture this design does not have are dropped
    out["M"], out["B"], out["C"] = G["M"], G["B"], G["C"]
    for k, v in G["fd"].items():
        out["fd_" + k] = np.asarray(v)
    out["n_iter"], out["xi_start"] = np.int32(int(model.nIter)), np.float64(model.XiStart)
    res = run(model, fowt, CASES)
    for ic, r in enumerate(res):
        for k, v in r.items():
            out["ref_run_case%d_%s" % (ic, k)] = v
    out["n_cases"] = np.int32(len(res))
    # measured effect of the synthetic rotor matrices (docstring): same run without them
    m0, f0 = build(yaml_path, aero=False)
    r0 = run(m0, f0, CASES[:1])[0]["Xi"][0]
    x1 = res[0]["Xi"][0]
    print("aero effect on case 0: %.3g of max|Xi|" % (np.abs(x1 - r0).max() / np.abs(x1).max()))
    print("fd support:", G["fd"]["fd_idx"].tolist(), " headings:", len(G["fd"].get("bem_headings", [])),
          " passes:", [int(r["passes"]) for r in res])
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **out)
    print("%-28s nDOF=%3d nw=%3d  %.1f s  %.0f KB  keys P_: %s" % (name, int(P["gen_nDOF"]), len(P["w"]), time.time() - t0,
                                                                  os.path.getsize(path) / 1024, [k for k in out if k.startswith("P_")]))


if __name__ == "__main__":
    fixture_flexfd("flexfd_VolturnUS-S-flexible", os.path.join(rh.REF_ROOT, "tests", "test_data", "VolturnUS-S-flexible.yaml"))
