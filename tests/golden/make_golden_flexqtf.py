#!/usr/bin/env python
"""Generate tests/golden/flexqtf_VolturnUS-S-flexible.npz (run in the BUILD CONTAINER only, like make_golden.py, whose
harness and helpers it uses): a flexible FOWT with second-order wave loads from an external QTF (potSecOrder 2) through the
unmodified reference's Model.solveDynamics.

Set-up: make_golden_flexfd.py's (VolturnUS-S-flexible, operating rotor with the seeded synthetic a_aero / b_aero,
potModMaster 3 with the marin_semi WAMIT coefficients) with ``potSecOrder 2``.  ``hydroPath`` already names marin_semi, so the
reference's own readQTF reads marin_semi.12d (56 frequencies, one heading) into fowt.qtf [56, 56, 1, nDOF], DOFs 0-5 filled.
The packed tables, matrices and frequency-dependent terms are those of flexfd_VolturnUS-S-flexible.npz (checked equal
here, not stored again), and the QTF table is not stored either: the tests rebuild it from wamit_marin_semi.npz's
``qtf_rows`` with bem.read_qtf, which tests/test_bem.py pins to the reference's readQTF.

Stored per case: Model.Xi of every train, the pass count, and every train's fowt.Fhydro_2nd[:, :6] (real; the imaginary part
and rows 6 and up are exactly zero, checked here) and Fhydro_2nd_mean[:, :6].  Cases: the four of flexfd plus one
single-train case at 180 deg.  Printed: the effect of the second-order force on case 0, max|Xi - Xi_noqtf| / max|Xi| against
the same run with potSecOrder 0 (``qtf effect``).

Usage:  python tests/golden/make_golden_flexqtf.py
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
from make_golden_flexfd import CASES as FD_CASES, synthetic_aero  # noqa: E402

CASES = FD_CASES + [[(5.0, 11.0, 180.0)]]


def build(yaml_path, sec_order=2):
    """make_golden_flexfd.build with potSecOrder ``sec_order`` (the rotor's synthetic matrices always on)."""
    raft = rh.load_reference()
    design = rh.load_design(yaml_path, strip=False)
    design.pop("mooring", None)
    pf = design["platform"]
    pf.update(potSecOrder=sec_order, potModMaster=3, potFirstOrder=1,
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
    a_aero, b_aero = synthetic_aero(np.asarray(fowt.w, dtype=float))
    T = fowt.rotorList[0].nodeList[0].T
    for iw in range(fowt.nw):                                         # raft_fowt.py:1559-1561
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
        r = dict(Xi=np.array(x)[:len(trains)], passes=np.int32(cnt[0]), trains=tr)
        if int(fowt.potSecOrder) == 2:
            F2 = np.array(fowt.Fhydro_2nd)[:len(trains)]
            F2m = np.array(fowt.Fhydro_2nd_mean)[:len(trains)]
            assert not F2.imag.any() and not F2[:, 6:].any() and not F2m[:, 6:].any()
            r.update(F2nd=np.ascontiguousarray(F2[:, :6].real), F2nd_mean=np.ascontiguousarray(F2m[:, :6]))
        res.append(r)
    fowt.calcHydroLinearization = orig
    return res


def fixture_flexqtf(name, yaml_path):
    t0 = time.time()
    model, fowt = build(yaml_path)
    assert fowt.potSecOrder == 2 and fowt.qtf.shape[3] == fowt.nDOF
    # same packed design and matrices as the flexfd fixture: the tests load those
    P = packer.pack_general_dofs(fowt)
    G = packer.pack_general_matrices(fowt)
    fdz = np.load(os.path.join(OUT, "flexfd_VolturnUS-S-flexible.npz"))
    base = np.load(os.path.join(OUT, "flex_VolturnUS-S-flexible.npz"))
    for k, v in P.items():
        ref = fdz["P_" + k] if "P_" + k in fdz.files else base["P_" + k]
        assert np.array_equal(np.asarray(v), ref), k
    for k in ("M", "B", "C"):
        assert np.array_equal(G[k], fdz[k]), k
    for k, v in G["fd"].items():
        assert np.array_equal(np.asarray(v), fdz["fd_" + k]), k
    Q = packer.pack_general_qtf(fowt)
    out = dict(n_iter=np.int32(int(model.nIter)), xi_start=np.float64(model.XiStart),
               qtf_shape=np.array(Q["qtf"].shape, dtype=np.int32))
    res = run(model, fowt, CASES)
    for ic, r in enumerate(res):
        for k, v in r.items():
            out["ref_run_case%d_%s" % (ic, k)] = v
    out["n_cases"] = np.int32(len(res))
    # measured effect of the second-order force (docstring): the same run without it
    m0, f0 = build(yaml_path, sec_order=0)
    r0 = run(m0, f0, CASES[:1])[0]["Xi"][0]
    x1 = res[0]["Xi"][0]
    eff = np.abs(x1 - r0).max() / np.abs(x1).max()
    out["qtf_effect_case0"] = np.float64(eff)
    print("qtf effect on case 0: %.3g of max|Xi|" % eff)
    print("passes:", [int(r["passes"]) for r in res])
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **out)
    print("%-28s nDOF=%3d nw=%3d  %.1f s  %.0f KB" % (name, int(P["gen_nDOF"]), len(P["w"]), time.time() - t0, os.path.getsize(path) / 1024))


if __name__ == "__main__":
    fixture_flexqtf("flexqtf_VolturnUS-S-flexible", os.path.join(rh.REF_ROOT, "tests", "test_data", "VolturnUS-S-flexible.yaml"))
