"""Frequency-dependent terms of the generalised-DOF solve on the CPU: the checker (tests/general_fd_checker.py, built on the C
checker's pinned generalised-DOF and BEM routines) against the reference's own run of a flexible FOWT with an operating rotor and
BEM coefficients (fixture flexfd_VolturnUS-S-flexible, tests/golden/make_golden_flexfd.py), packer.pack_general_matrices on the
reference's FOWT, and the argument checks of raftk_general_solve_dynamics_fd_* (no device needed: every rejection happens
before any launch).

Grouping of the impedance: the checker and the CUDA kernels form M + A_w and (B + B_w) + B_drag on the support, where the
reference sums ((M_turb + M_struc) + A_BEM) + A_hydro_morison (raft_model.py:1045-1046, 1086).  Against the fixture the
checker's largest relative error over every case and train is 5.6e-11 (measured), so the grouping and the two LUs of this
cond ~1e6 impedance together use about half of the 1e-10 budget; on the constant-matrix fixture, where the grouping is the
same as the reference's, the two LUs alone differ by ~2e-11 (tests/test_general_dofs.py).  The two groupings were not run
side by side: the fixture stores the sums, not their parts."""
import ctypes as C
import os

import numpy as np
import pytest

import general_fd_checker as gfc
from conftest import GOLDEN, relerr

FLEX = os.path.join(GOLDEN, "flex_VolturnUS-S-flexible.npz")
FLEXFD = os.path.join(GOLDEN, "flexfd_VolturnUS-S-flexible.npz")


def load_flexfd():
    """-> (P, M, B, C, fd, z): the packed design (flex fixture's tables overlaid with the flexfd ones), the constant matrices,
    the fd dict of packer.pack_general_matrices and the fixture itself."""
    base, z = np.load(FLEX), np.load(FLEXFD)
    keys = set(z["P_keys"].tolist())
    P = {k[2:]: base[k] for k in base.files if k.startswith("P_") and k[2:] in keys}
    P.update({k[2:]: z[k] for k in z.files if k.startswith("P_") and k != "P_keys"})
    fd = {k[3:]: z[k] for k in z.files if k.startswith("fd_")}
    return P, z["M"], z["B"], z["C"], fd, z


def test_checker_vs_reference_run_flexfd(oracle):
    P, M, B, Cm, fd, z = load_flexfd()
    worst = 0.0
    for ic in range(int(z["n_cases"])):
        tr = z["ref_run_case%d_trains" % ic]
        Xi, st, Fb = gfc.solve_trains_fd(oracle, P, M, B, Cm, fd, tr, nIter=int(z["n_iter"]), XiStart=float(z["xi_start"]))
        assert st[0] == int(z["ref_run_case%d_passes" % ic]) and st[2] == 0, (ic, st)
        for h in range(len(tr)):
            e = relerr(Xi[h], z["ref_run_case%d_Xi" % ic][h])
            worst = max(worst, e)
            assert e < 1e-10, (ic, h, e)
            assert relerr(Fb[h], z["ref_run_case%d_F_BEM" % ic][h]) < 1e-12, (ic, h)
    print("largest relative Xi error against the reference run: %.2e" % worst)


def test_checker_without_fd_is_the_constant_solve(oracle):
    """fd = None: the checker reproduces the C checker's single-train constant-matrix solve (same passes, 1e-12) and returns
    a zero F_BEM."""
    z = np.load(FLEX)
    P = {k[2:]: z[k] for k in z.files if k.startswith("P_")}
    cs = z["ref_run_solve_cases"]
    gd = oracle.GeneralDesign(P)
    X0, s0 = oracle.general_solve_dynamics(gd, z["gen_M"], z["gen_B"], z["gen_C"], 0, cs[0, 0], cs[0, 1], 0.0, cs[0, 2],
                                           nIter=int(z["n_iter"]), XiStart=float(z["xi_start"]))
    X1, s1, Fb = gfc.solve_trains_fd(oracle, P, z["gen_M"], z["gen_B"], z["gen_C"], None, cs[:1], nIter=int(z["n_iter"]),
                                     XiStart=float(z["xi_start"]))
    assert relerr(X1[0], X0) < 1e-12 and np.array_equal(s1, s0) and not Fb.any()


def test_checker_bem_on_rigid_design_matches_rigid_checker(oracle):
    """With T0 = I on the cfg3 OC4semi BEM design the checker's F_BEM is the rigid checker's, bit for bit, at headings that
    use the wrap-around bracket."""
    z = np.load(os.path.join(GOLDEN, "cfg3_OC4semi-WAMIT_nw128.npz"))
    P = {k[2:]: z[k] for k in z.files if k.startswith("P_")}
    G = dict(P, gen_nDOF=6)
    fd = dict(X_BEM=P["X_BEM"], bem_headings=P["bem_headings"], heading_adjust=P["heading_adjust"], T0=np.eye(6),
              x_ref=P["x_ref"], y_ref=P["y_ref"])
    od = oracle.OracleDesign(P)
    for beta in (0.0, 175.0, 355.0, -60.0):
        _, f6, _, _ = oracle.calc_hydro_excitation(od, 0, 4.0, 10.0, 0.0, beta)
        assert np.array_equal(gfc.bem_excitation(oracle, G, fd, 4.0, 10.0, beta), f6), beta


def test_fixture_support_and_tables():
    """The fixture's fd support is the PRP node and the rotor node, and scattering the restricted tables back reproduces the
    dense matrices exactly on the support (every entry off it is zero by construction)."""
    P, M, B, Cm, fd, z = load_flexfd()
    assert fd["fd_idx"].tolist() == list(range(6)) + list(range(144, 150))
    n, nw = int(P["gen_nDOF"]), len(P["w"])
    assert fd["A_w"].shape == (12, 12, nw) and fd["X_BEM"].shape[1:] == (6, nw) and fd["T0"].shape == (6, n)
    assert np.all(np.diff(fd["bem_headings"]) >= 0) and fd["bem_headings"][0] >= 0 and fd["bem_headings"][-1] < 360
    assert not np.any(fd["T0"][:, 6:])


def _ref():
    from oracle import ref_harness as rh
    if not rh.reference_available():
        pytest.skip("the reference tree is not available")
    import sys
    sys.path.insert(0, GOLDEN)
    import make_golden_flexfd
    return rh, make_golden_flexfd


def test_pack_general_matrices_on_reference_fowt():
    rh, mk = _ref()
    from raft_b200 import packer
    _, fowt = mk.build(os.path.join(rh.REF_ROOT, "tests", "test_data", "VolturnUS-S-flexible.yaml"))
    G = packer.pack_general_matrices(fowt)
    fd, idx = G["fd"], G["fd"]["fd_idx"]
    assert idx.tolist() == list(range(6)) + list(range(144, 150))
    n, nw = fowt.nDOF, fowt.nw
    for key, dense in (("A_w", np.sum(fowt.A_aero, axis=3) + fowt.A_BEM), ("B_w", np.sum(fowt.B_aero, axis=3) + fowt.B_BEM)):
        back = np.zeros([n, n, nw])
        back[np.ix_(idx, idx)] = fd[key]
        assert np.array_equal(back, dense), key
    assert np.array_equal(fd["T0"], np.asarray(fowt.T)[:6])
    z = np.load(FLEXFD)
    for k in ("M", "B", "C"):
        assert np.array_equal(G[k], z[k]), k


def test_pack_general_matrices_without_rotor_or_bem():
    """A parked turbine and no BEM coefficients: n_fd = 0 and the constant matrices the flex fixtures were made with."""
    rh, _ = _ref()
    import contextlib
    import copy
    import io
    from raft_b200 import packer
    raft = rh.load_reference()
    design = rh.load_design(os.path.join(rh.REF_ROOT, "tests", "test_data", "VolturnUS-S-flexible.yaml"), strip=False)
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
    G = packer.pack_general_matrices(fowt)
    assert len(G["fd"]["fd_idx"]) == 0 and "X_BEM" not in G["fd"]
    z = np.load(FLEX)
    for k in ("M", "B", "C"):
        assert np.array_equal(G[k], z["gen_" + k]), k


# ---- argument checks of the C ABI (host entry; nothing is launched) -------------------------------------------------------
def _rejects(fd_kw, msg):
    from raft_b200 import _lib, solver
    P, M, B, Cm, fd, z = load_flexfd()
    fd = dict(fd)
    fd.update(fd_kw)
    n, nw = int(P["gen_nDOF"]), len(P["w"])
    keep = {}

    def ptr(name, a):
        keep[name] = a
        return a.ctypes.data
    g = solver._general_struct(P, M, B, Cm, ptr)
    f = solver._general_fd_struct(fd, n, nw, ptr) if "raw" not in fd else fd["raw"]
    cs = solver.CaseTable(dict(Hs=np.array([6.0]), Tp=np.array([12.0]), gamma=np.zeros(1), beta_deg=np.zeros(1), spec=np.zeros(1, dtype=np.int32)))
    c = cs.struct(solver._host_ptr(cs.arrays))
    o = _lib.RaftkSolveOpts(10, 0, 0.01, 0.0, 0, 0)
    Xi = np.zeros([1, n, nw], dtype=np.complex128)
    st = np.zeros([1, 4], dtype=np.int32)
    rc = _lib.lib.raftk_general_solve_dynamics_fd_host(C.byref(g), C.byref(f), C.byref(c), C.byref(o), Xi.ctypes.data, st.ctypes.data, None)
    assert rc == -1, rc
    err = _lib.lib.raftk_last_error().decode()
    assert msg in err, err
    assert solver.last_dispatch()["kernel"] == "none"


def test_fd_rejects_index_out_of_range():
    _rejects(dict(fd_idx=np.array([0, 1, 2, 3, 4, 5, 144, 145, 146, 147, 148, 150])), "out of range")


def test_fd_rejects_repeated_and_unsorted_indices():
    _rejects(dict(fd_idx=np.array([0, 1, 2, 3, 4, 5, 144, 145, 146, 147, 149, 149])), "strictly increasing")
    _rejects(dict(fd_idx=np.array([0, 1, 2, 3, 4, 5, 144, 145, 146, 147, 149, 148])), "strictly increasing")


def test_fd_rejects_headings_out_of_order_or_range():
    _, _, _, _, fd, _ = load_flexfd()
    hd = fd["bem_headings"].copy()
    dec = hd.copy()
    dec[3], dec[4] = hd[4], hd[3]
    _rejects(dict(bem_headings=dec), "non-decreasing")
    hi = hd.copy()
    hi[-1] = 360.0
    _rejects(dict(bem_headings=hi), "[0, 360)")
    lo = hd.copy()
    lo[0] = -10.0
    _rejects(dict(bem_headings=lo), "[0, 360)")


def test_fd_rejects_counts_and_missing_tables():
    from raft_b200 import _lib
    _, _, _, _, fd, _ = load_flexfd()
    too_many = _lib.RaftkGeneralFd()
    too_many.n_fd = 151
    _rejects(dict(raw=too_many), "n_fd must be in [0, n_dof]")
    neg = _lib.RaftkGeneralFd()
    neg.n_bem_head = -1
    _rejects(dict(raw=neg), "n_bem_head must be >= 0")
    no_tab = _lib.RaftkGeneralFd()
    no_tab.n_fd = 12
    idx = np.ascontiguousarray(fd["fd_idx"], dtype=np.int32)
    no_tab.fd_idx = idx.ctypes.data
    _rejects(dict(raw=no_tab), "needs fd_idx, A_w and B_w")
    no_x = _lib.RaftkGeneralFd()
    no_x.n_bem_head = 2
    hd = np.array([0.0, 10.0])
    no_x.bem_headings = hd.ctypes.data
    _rejects(dict(raw=no_x), "needs bem_headings, X_BEM and T0")


def test_fd_workspace_query_without_device():
    """raftk_general_fd_workspace_bytes: fd = NULL and n_fd = 0 give the constant solve's size; BEM tables add the force buffers."""
    from raft_b200 import _lib, solver
    P, M, B, Cm, fd, z = load_flexfd()
    n, nw = int(P["gen_nDOF"]), len(P["w"])
    keep = {}

    def ptr(name, a):
        keep[name] = a
        return a.ctypes.data
    g = solver._general_struct(P, M, B, Cm, ptr)
    base = _lib.lib.raftk_general_workspace_bytes(C.byref(g), 4)
    assert _lib.lib.raftk_general_fd_workspace_bytes(C.byref(g), None, 4) == base
    empty = solver._general_fd_struct(dict(fd_idx=np.zeros(0, dtype=np.int32)), n, nw, ptr)
    assert _lib.lib.raftk_general_fd_workspace_bytes(C.byref(g), C.byref(empty), 4) == base
    full = solver._general_fd_struct(fd, n, nw, ptr)
    extra = _lib.lib.raftk_general_fd_workspace_bytes(C.byref(g), C.byref(full), 4) - base
    assert extra == (4 * 6 * nw * 16 + 255) // 256 * 256 + (4 * n * nw * 16 + 255) // 256 * 256
