"""Second-order wave loads on the generalised-DOF GPU path (raftk_general_solve_dynamics_qtf_*: the k_qtf_* force kernels on
every case and train, k_gen_add_2nd, raft_b200/csrc/raftk_general.cuh) against the unmodified reference's run of a flexible
FOWT with an operating rotor, BEM coefficients and the marin_semi QTF (fixture flexqtf_VolturnUS-S-flexible) and the checker
(tests/general_qtf_checker.py): both LU kernels and both force kernels, every case and wave train, F_2nd and the mean drift.
Also: a 4-heading table (heading interpolation) against the checker, qtf = NULL bit for bit against the fd entry, the host
entry against GeneralSession and general_analyze_cases, and at n = 6 with T = I the rigid potSecOrder-2 solver on cfg3q.

Response tolerances: general_qtf_checker.XI_RTOL from bin LOW_BINS up and XI_RTOL_ALL over every bin (the slow-drift force
drives the nearly singular lowest bins, where any two correct solvers differ by ~1e-9; see there)."""
import ctypes as C
import os

import numpy as np
import pytest

import general_qtf_checker as gqc
from conftest import GOLDEN, relerr
from test_general_qtf_oracle import load_flexqtf

pytestmark = [pytest.mark.gpu]

D2R = 0.017453292519943295


def _cases(z):
    from raft_b200 import packer
    cases = []
    for ic in range(int(z["n_cases"])):
        tr = z["ref_run_case%d_trains" % ic]
        cases.append(dict(wave_spectrum=["JONSWAP"] * len(tr), wave_height=list(tr[:, 0]), wave_period=list(tr[:, 1]),
                          wave_heading=list(tr[:, 2]), wave_gamma=[0.0] * len(tr)))
    table, owner, first = packer.pack_case_trains(cases)
    return cases, table, owner, first


def _env(monkeypatch, diag):
    if diag:
        monkeypatch.setenv("RAFTK_QTF_DIAG", "1")
    else:
        monkeypatch.delenv("RAFTK_QTF_DIAG", raising=False)


@pytest.mark.parametrize("diag", [False, True])
def test_qtf_vs_reference_run_and_oracle(diag, monkeypatch, oracle, tmp_path):
    from raft_b200 import solver
    _env(monkeypatch, diag)
    P, M, B, Cm, fd, qtf, z = load_flexqtf(tmp_path)
    _, table, owner, first = _cases(z)
    Xi, st, F2, F2m = solver.general_solve_dynamics(P, M, B, Cm, solver.CaseTable(table), n_iter=int(z["n_iter"]), xi_start=float(z["xi_start"]),
                                                    fd=fd, qtf=qtf, F_2nd=True)
    rec = solver.last_dispatch()
    assert rec["family"] == "general" and rec["kernel"] == "gen-blocked" and rec["trains"]
    worst = [0.0, 0.0]
    for ic in range(int(z["n_cases"])):
        idx = np.nonzero(owner == ic)[0]
        assert st[first[ic], 0] == int(z["ref_run_case%d_passes" % ic]) and st[first[ic], 2] == 0
        Xo, so, _, Fo, Fmo = gqc.solve_trains_qtf(oracle, P, M, B, Cm, fd, qtf, z["ref_run_case%d_trains" % ic], nIter=int(z["n_iter"]),
                                                  XiStart=float(z["xi_start"]))
        assert st[first[ic], 0] == so[0] and st[first[ic], 1] == so[1]
        for h, t in enumerate(idx):
            for ref in (z["ref_run_case%d_Xi" % ic][h], Xo[h]):
                e_all, e = gqc.xi_errors(Xi[t], ref)
                worst = [max(worst[0], e_all), max(worst[1], e)]
                assert e_all < gqc.XI_RTOL_ALL and e < gqc.XI_RTOL, (ic, h, e_all, e)
            assert relerr(F2[t], z["ref_run_case%d_F2nd" % ic][h]) < 1e-12 and relerr(F2[t], Fo[h]) < 1e-12, (ic, h)
            assert relerr(F2m[t], z["ref_run_case%d_F2nd_mean" % ic][h]) < 1e-12 and relerr(F2m[t], Fmo[h]) < 1e-12, (ic, h)
    print("largest relative Xi error: %.2e (every bin), %.2e (from bin %d)" % (worst[0], worst[1], gqc.LOW_BINS))


def _four_headings(qtf):
    """The marin_semi table on 4 headings (-90, 0, 45, 180 deg), each a scaled and rotated copy (cfg3q's mh_scale)."""
    scale = np.array([1.0, 0.7 + 0.2j, 1.3, -0.4 + 1.0j])
    return dict(qtf=np.ascontiguousarray(np.stack([qtf["qtf"][:, :, 0, :] * s for s in scale], axis=2)),
                qtf_w=qtf["qtf_w"], qtf_heads=np.array([-90.0, 0.0, 45.0, 180.0]) * D2R)


@pytest.mark.parametrize("diag", [False, True])
def test_four_heading_table_vs_checker(diag, monkeypatch, oracle, tmp_path):
    """Headings inside the table's range (20, 100 deg), on its headings (0, 45 deg) and outside it (-120, 200, 355 deg: the
    nearest table, scipy interp1d's fill values); RAFTK_QTF_DIAG=1 runs k_qtf_force<true> (MIX)."""
    from raft_b200 import solver
    _env(monkeypatch, diag)
    P, M, B, Cm, fd, qtf, z = load_flexqtf(tmp_path)
    q4 = _four_headings(qtf)
    beta = np.array([20.0, 100.0, 0.0, 45.0, -120.0, 200.0, 355.0])
    n = len(beta)
    cs = dict(Hs=np.linspace(2.0, 7.0, n), Tp=np.linspace(7.0, 14.0, n), gamma=np.zeros(n), beta_deg=beta, spec=np.zeros(n, dtype=np.int32))
    Xi, st, F2, F2m = solver.general_solve_dynamics(P, M, B, Cm, solver.CaseTable(cs), n_iter=int(z["n_iter"]), fd=fd, qtf=q4, F_2nd=True)
    for c in range(n):
        Xo, so, _, Fo, Fmo = gqc.solve_trains_qtf(oracle, P, M, B, Cm, fd, q4, [(cs["Hs"][c], cs["Tp"][c], beta[c])], nIter=int(z["n_iter"]))
        assert st[c, 0] == so[0] and st[c, 1] == so[1], beta[c]
        assert relerr(F2[c], Fo[0]) < 1e-12 and relerr(F2m[c], Fmo[0]) < 1e-12, beta[c]
        e_all, e = gqc.xi_errors(Xi[c], Xo[0])
        assert e_all < gqc.XI_RTOL_ALL and e < gqc.XI_RTOL, (beta[c], e_all, e)
    # the interpolation is live: a heading between two tables differs from both neighbours
    assert not np.allclose(F2[0], F2[2]) and not np.allclose(F2[0], F2[3])


def test_qtf_null_is_bit_identical_to_fd_entry(tmp_path):
    """qtf = None (and the empty dict of potSecOrder 0) through raftk_general_solve_dynamics_qtf_host / _dev give np.array_equal
    results against raftk_general_solve_dynamics_fd_host, trains included."""
    from raft_b200 import _lib, solver
    P, M, B, Cm, fd, _, z = load_flexqtf(tmp_path)
    _, table, _, _ = _cases(z)
    kw = dict(n_iter=int(z["n_iter"]), xi_start=float(z["xi_start"]))
    n, nw = int(P["gen_nDOF"]), len(P["w"])
    keep = {}

    def ptr(name, a):
        keep[name] = a
        return a.ctypes.data
    g = solver._general_struct(P, M, B, Cm, ptr)
    f = solver._general_fd_struct(fd, n, nw, ptr)
    ct = solver.CaseTable(table)
    c = ct.struct(solver._host_ptr(ct.arrays))
    o = _lib.RaftkSolveOpts(int(z["n_iter"]), 0, 0.01, float(z["xi_start"]), 0, 0)
    X0 = np.zeros([ct.n_cases, n, nw], dtype=np.complex128)
    s0 = np.zeros([ct.n_cases, 4], dtype=np.int32)
    F0 = np.zeros([ct.n_cases, n, nw], dtype=np.complex128)
    _lib.check(_lib.lib.raftk_general_solve_dynamics_fd_host(C.byref(g), C.byref(f), C.byref(c), C.byref(o), X0.ctypes.data, s0.ctypes.data,
                                                             F0.ctypes.data))
    for q in (None, {}):
        X1, s1, F1 = solver.general_solve_dynamics(P, M, B, Cm, solver.CaseTable(table), fd=fd, qtf=q, F_BEM=True, **kw)
        assert np.array_equal(X1, X0) and np.array_equal(s1, s0) and np.array_equal(F1, F0)
    S = solver.GeneralSession(P, M, B, Cm, solver.CaseTable(table), fd=fd, qtf=None)
    Xs, ss = S.solve(**kw)
    assert S.F_2nd is None and np.array_equal(Xs.cpu().numpy(), X0) and np.array_equal(ss.cpu().numpy(), s0)


def test_host_session_and_analyze_cases_agree(monkeypatch, tmp_path):
    """With the reproducible force kernel (RAFTK_QTF_DIAG=1): the host entry, GeneralSession (F_2nd, F_2nd_mean kept on the
    device) and general_analyze_cases (per case Fhydro_2nd [nTrains,nDOF,nw], Fhydro_2nd_mean [nTrains,nDOF], zero from row
    6) give the same bits."""
    from raft_b200 import solver
    _env(monkeypatch, True)
    P, M, B, Cm, fd, qtf, z = load_flexqtf(tmp_path)
    cases, table, owner, first = _cases(z)
    kw = dict(n_iter=int(z["n_iter"]), xi_start=float(z["xi_start"]))
    Xh, sh, Fbh, F2h, F2mh = solver.general_solve_dynamics(P, M, B, Cm, solver.CaseTable(table), fd=fd, F_BEM=True, qtf=qtf, F_2nd=True, **kw)
    S = solver.GeneralSession(P, M, B, Cm, solver.CaseTable(table), fd=fd, F_BEM=True, qtf=qtf)
    for _ in range(2):                                         # a second solve on the same workspace
        Xs, ss, Fbs = S.solve(**kw)
        assert np.array_equal(Xs.cpu().numpy(), Xh) and np.array_equal(ss.cpu().numpy(), sh) and np.array_equal(Fbs.cpu().numpy(), Fbh)
        assert S.F_2nd.is_cuda and np.array_equal(S.F_2nd.cpu().numpy(), F2h) and np.array_equal(S.F_2nd_mean.cpu().numpy(), F2mh)
    assert solver.last_dispatch()["kernel"] == "gen-blocked"
    out = solver.general_analyze_cases(P, M, B, Cm, cases, fd=fd, qtf=qtf, **kw)
    n, nw = Xh.shape[1:]
    for ic in range(len(cases)):
        sel = owner == ic
        assert np.array_equal(out["Xi_trains"][ic], Xh[sel])
        F2, F2m = out["Fhydro_2nd"][ic], out["Fhydro_2nd_mean"][ic]
        assert F2.shape == (sel.sum(), n, nw) and F2m.shape == (sel.sum(), n)
        assert np.array_equal(F2[:, :6].real, F2h[sel]) and not F2.imag.any() and not F2[:, 6:].any()
        assert np.array_equal(F2m[:, :6], F2mh[sel]) and not F2m[:, 6:].any()
    assert np.array_equal(out["status"], sh[first])
    plain = solver.general_analyze_cases(P, M, B, Cm, cases, fd=fd, **kw)
    assert "Fhydro_2nd" not in plain


def test_n6_reproduces_rigid_potsecorder2_solver():
    """The cfg3q OC4semi-QTF design (BEM + the marin_semi .12d) as an n = 6 generalised design with T = I against the rigid
    potSecOrder-2 solver: Xi and F_2nd at 1e-10, headings inside and outside the one-heading table."""
    from raft_b200 import solver
    z = np.load(os.path.join(GOLDEN, "cfg3q_OC4semi-QTF_nw96.npz"))
    P = {k[2:]: z[k] for k in z.files if k.startswith("P_")}
    r = np.asarray(P["node_r"], dtype=float)
    G = dict(P, gen_nDOF=6, gen_Tn=np.ascontiguousarray(np.repeat(np.eye(6)[None], len(r), axis=0)),
             gen_rr=np.ascontiguousarray(r - np.asarray(P["prp"], dtype=float)[None, :]))
    M, B, Cm = (np.asarray(P[k], dtype=float).reshape(6, 6) for k in ("M0", "B0", "C0"))
    fd = dict(fd_idx=np.arange(6, dtype=np.int32), A_w=P["A_w"], B_w=P["B_w"], X_BEM=P["X_BEM"], bem_headings=P["bem_headings"],
              heading_adjust=P["heading_adjust"], T0=np.eye(6), x_ref=P["x_ref"], y_ref=P["y_ref"])
    qtf = dict(qtf=P["qtf"], qtf_w=P["qtf_w"], qtf_heads=P["qtf_heads"])
    beta = np.array([0.0, 30.0, 175.0, 355.0, -60.0])
    n = len(beta)
    cs = dict(Hs=np.linspace(2.0, 8.0, n), Tp=np.linspace(7.0, 15.0, n), gamma=np.zeros(n), beta_deg=beta, spec=np.zeros(n, dtype=np.int32))
    ni = int(z["n_iter"])
    rig = solver.solve_dynamics(solver.DesignBatch(P), solver.CaseTable(cs), n_iter=ni, want=("Xi", "status", "F_2nd", "F_2nd_mean"))
    Xg, sg, F2, F2m = solver.general_solve_dynamics(G, M, B, Cm, solver.CaseTable(cs), n_iter=ni, fd=fd, qtf=qtf, F_2nd=True)
    assert np.array_equal(sg[:, 0], rig["status"][0, :, 0])
    for c in range(n):
        assert relerr(Xg[c], rig["Xi"][0, c]) < 1e-10, (beta[c], relerr(Xg[c], rig["Xi"][0, c]))
        assert relerr(F2[c], rig["F_2nd"][0, c]) < 1e-10 and relerr(F2m[c], rig["F_2nd_mean"][0, c]) < 1e-10, beta[c]
