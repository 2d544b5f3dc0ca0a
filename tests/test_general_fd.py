"""Frequency-dependent added mass, damping and BEM excitation on the generalised-DOF GPU path
(raftk_general_solve_dynamics_fd_*, raft_b200/csrc/raftk_general.cuh) against the unmodified reference's run of a flexible FOWT
with an operating rotor and potential-flow coefficients (fixture flexfd_VolturnUS-S-flexible) and the checker
(tests/general_fd_checker.py): both LU kernels, every case and wave train, F_BEM.  Also: fd = NULL and n_fd = 0 give the
constant-matrix solve bit for bit, and at n = 6 with T = I the path reproduces the rigid solver on the cfg3 OC4semi BEM design."""
import os

import numpy as np
import pytest

import general_fd_checker as gfc
from conftest import GOLDEN, relerr
from test_general_fd_oracle import load_flexfd

pytestmark = [pytest.mark.gpu]

RTOL = 1e-10


def _cases(z):
    from raft_b200 import packer
    cases = []
    for ic in range(int(z["n_cases"])):
        tr = z["ref_run_case%d_trains" % ic]
        cases.append(dict(wave_spectrum=["JONSWAP"] * len(tr), wave_height=list(tr[:, 0]), wave_period=list(tr[:, 1]),
                          wave_heading=list(tr[:, 2]), wave_gamma=[0.0] * len(tr)))
    table, owner, first = packer.pack_case_trains(cases)
    return cases, table, owner, first


def test_fd_vs_reference_run_and_oracle(oracle):
    from raft_b200 import solver
    P, M, B, Cm, fd, z = load_flexfd()
    _, table, owner, first = _cases(z)
    Xi, st, Fb = solver.general_solve_dynamics(P, M, B, Cm, solver.CaseTable(table), n_iter=int(z["n_iter"]), xi_start=float(z["xi_start"]),
                                               fd=fd, F_BEM=True)
    rec = solver.last_dispatch()
    assert rec["family"] == "general" and rec["kernel"] == "gen-blocked" and rec["trains"]
    for ic in range(int(z["n_cases"])):
        idx = np.nonzero(owner == ic)[0]
        assert st[first[ic], 0] == int(z["ref_run_case%d_passes" % ic]) and st[first[ic], 2] == 0
        Xo, so, Fo = gfc.solve_trains_fd(oracle, P, M, B, Cm, fd, z["ref_run_case%d_trains" % ic], nIter=int(z["n_iter"]),
                                         XiStart=float(z["xi_start"]))
        assert st[first[ic], 0] == so[0] and st[first[ic], 1] == so[1]
        for h, t in enumerate(idx):
            ref = z["ref_run_case%d_Xi" % ic][h]
            assert relerr(Xi[t], ref) < RTOL, (ic, h, relerr(Xi[t], ref))
            assert relerr(Xi[t], Xo[h]) < RTOL, (ic, h, relerr(Xi[t], Xo[h]))
            assert relerr(Fb[t], z["ref_run_case%d_F_BEM" % ic][h]) < 1e-12 and relerr(Fb[t], Fo[h]) < 1e-12, (ic, h)


def test_fd_null_and_empty_are_bit_identical_to_constant_solve():
    """fd = None and an fd with n_fd = 0 and no BEM table give np.array_equal results against raftk_general_solve_dynamics_*
    on the existing 150-DOF fixture, trains included; the F_BEM output is zero there."""
    from raft_b200 import packer, solver
    z = np.load(os.path.join(GOLDEN, "flexout_VolturnUS-S-flexible.npz"))
    P = {k[2:]: z[k] for k in z.files if k.startswith("P_")}
    cases = []
    for ic in range(3):
        tr = z["ref_run_case%d_trains" % ic]
        cases.append(dict(wave_spectrum=["JONSWAP"] * len(tr), wave_height=list(tr[:, 0]), wave_period=list(tr[:, 1]),
                          wave_heading=list(tr[:, 2]), wave_gamma=[0.0] * len(tr)))
    table, _, _ = packer.pack_case_trains(cases)
    kw = dict(n_iter=int(z["n_iter"]), xi_start=float(z["xi_start"]))
    X0, s0 = solver.general_solve_dynamics(P, z["gen_M"], z["gen_B"], z["gen_C"], solver.CaseTable(table), **kw)
    X1, s1 = solver.general_solve_dynamics(P, z["gen_M"], z["gen_B"], z["gen_C"], solver.CaseTable(table), fd=None, **kw)
    X2, s2, F2 = solver.general_solve_dynamics(P, z["gen_M"], z["gen_B"], z["gen_C"], solver.CaseTable(table),
                                               fd=dict(fd_idx=np.zeros(0, dtype=np.int32)), F_BEM=True, **kw)
    assert np.array_equal(X0, X1) and np.array_equal(s0, s1)
    assert np.array_equal(X0, X2) and np.array_equal(s0, s2) and not F2.any()
    # the device session, same bits
    S = solver.GeneralSession(P, z["gen_M"], z["gen_B"], z["gen_C"], solver.CaseTable(table), fd=dict(fd_idx=np.zeros(0, dtype=np.int32)))
    Xs, ss = S.solve(**kw)
    assert np.array_equal(Xs.cpu().numpy(), X0) and np.array_equal(ss.cpu().numpy(), s0)


def test_session_and_analyze_cases_match_host_call():
    from raft_b200 import solver
    P, M, B, Cm, fd, z = load_flexfd()
    cases, table, owner, first = _cases(z)
    kw = dict(n_iter=int(z["n_iter"]), xi_start=float(z["xi_start"]))
    Xh, sh, Fh = solver.general_solve_dynamics(P, M, B, Cm, solver.CaseTable(table), fd=fd, F_BEM=True, **kw)
    S = solver.GeneralSession(P, M, B, Cm, solver.CaseTable(table), fd=fd, F_BEM=True)
    Xs, ss, Fs = S.solve(**kw)
    assert np.array_equal(Xs.cpu().numpy(), Xh) and np.array_equal(ss.cpu().numpy(), sh) and np.array_equal(Fs.cpu().numpy(), Fh)
    Xs2, _, _ = S.solve(**kw)                              # a second solve on the same workspace
    assert np.array_equal(Xs2.cpu().numpy(), Xh)
    out = solver.general_analyze_cases(P, M, B, Cm, cases, fd=fd, **kw)
    for ic in range(len(cases)):
        assert np.array_equal(out["Xi_trains"][ic], Xh[owner == ic])
    assert np.array_equal(out["status"], sh[first])


def _rigid_as_general():
    """The cfg3 OC4semi BEM design as an n = 6 generalised design: gen_Tn = I6, gen_rr = node offset from the PRP; its constant
    matrices are M, B, C and its A_w, B_w, X_BEM become fd with fd_idx = 0..5 and T0 = I."""
    z = np.load(os.path.join(GOLDEN, "cfg3_OC4semi-WAMIT_nw128.npz"))
    P = {k[2:]: z[k] for k in z.files if k.startswith("P_")}
    r = np.asarray(P["node_r"], dtype=float)
    G = dict(P)
    G["gen_nDOF"] = 6
    G["gen_Tn"] = np.ascontiguousarray(np.repeat(np.eye(6)[None], len(r), axis=0))
    G["gen_rr"] = np.ascontiguousarray(r - np.asarray(P["prp"], dtype=float)[None, :])
    M, B, C = (np.asarray(P[k], dtype=float).reshape(6, 6) for k in ("M0", "B0", "C0"))
    fd = dict(fd_idx=np.arange(6, dtype=np.int32), A_w=P["A_w"], B_w=P["B_w"], X_BEM=P["X_BEM"], bem_headings=P["bem_headings"],
              heading_adjust=P["heading_adjust"], T0=np.eye(6), x_ref=P.get("x_ref", 0.0), y_ref=P.get("y_ref", 0.0))
    return P, G, M, B, C, fd, z


def test_n6_reproduces_rigid_solver_on_bem_design():
    """The new impedance and BEM code against the validated rigid path: same design, headings 0, 30, 175, 180, 355 (between
    the last BEM heading, 350, and the first) and -60 deg."""
    from raft_b200 import solver
    P, G, M, B, C, fd, z = _rigid_as_general()
    beta = np.array([0.0, 30.0, 175.0, 180.0, 355.0, -60.0])
    n = len(beta)
    cs = dict(Hs=np.linspace(2.0, 8.0, n), Tp=np.linspace(7.0, 15.0, n), gamma=np.zeros(n), beta_deg=beta, spec=np.zeros(n, dtype=np.int32))
    ni = int(z["n_iter"])
    rig = solver.solve_dynamics(solver.DesignBatch(P), solver.CaseTable(cs), n_iter=ni, want=("Xi", "status", "F_BEM"))
    Xg, sg, Fg = solver.general_solve_dynamics(G, M, B, C, solver.CaseTable(cs), n_iter=ni, fd=fd, F_BEM=True)
    assert solver.last_dispatch()["kernel"] == "gen-blocked"
    assert np.array_equal(sg[:, 0], rig["status"][0, :, 0])
    for c in range(n):
        assert relerr(Xg[c], rig["Xi"][0, c]) < RTOL, (beta[c], relerr(Xg[c], rig["Xi"][0, c]))
        assert relerr(Fg[c], rig["F_BEM"][0, c]) < 1e-12, beta[c]


def test_fd_dev_rejects_bad_tables_before_launch():
    """The device entry reads fd_idx and the headings back and refuses malformed ones with RAFTK_EINVAL, launching nothing."""
    from raft_b200 import solver
    from raft_b200._lib import RaftkError
    P, M, B, Cm, fd, z = load_flexfd()
    _, table, _, _ = _cases(z)
    for bad, msg in ((dict(fd_idx=fd["fd_idx"][::-1].copy()), "strictly increasing"),
                     (dict(bem_headings=np.where(np.arange(len(fd["bem_headings"])) == 0, 360.0, fd["bem_headings"])), "[0, 360)")):
        f = dict(fd)
        f.update(bad)
        S = solver.GeneralSession(P, M, B, Cm, solver.CaseTable(table), fd=f)
        with pytest.raises(RaftkError, match=r"raftk error -1: .*" + msg.replace("[", r"\[").replace("(", r"\(").replace(")", r"\)")):
            S.solve(n_iter=int(z["n_iter"]))
        assert solver.last_dispatch()["kernel"] == "none"
