"""The generalised-DOF GPU path (raft_b200/csrc/raftk_general.cuh) and the statistics kernels at the shapes the one flexible
fixture (VolturnUS-S-flexible: n = 150, nw = 40, fd support {0..5, 144..149}, T0 = [I6 | 0]) never reaches, against the
checkers (tests/general_fd_checker.py, tests/general_qtf_checker.py) on synthetic seeded inputs (tests/general_synth.py):

* more than 128 bins, so the second x-block of k_gen_wave, k_gen_bem, k_gen_project, k_gen_add_2nd and a second trip of
  k_gen_node_pass's RMS loop run;
* fd supports that cross the blocked LU's 8-column panels, end on the last DOF, hold only modal DOFs, a single DOF, every
  DOF, or straddle the 128-thread stride of gen_fd_map (n = 256); A_w and B_w with a 20 %+ antisymmetric part;
* rotor tables without BEM, BEM without rotor tables (k_gen_solve_blocked<false> with the BEM projection), a dense T0;
* wave trains at n = 7 .. 256 (k_gen_train_solve's b[256] full at n = 256), second-order loads at n = 6 .. 64;
* BEM heading tables of one and of four headings with heading_adjust and x_ref / y_ref;
* output-channel statistics (every wpow, 0, 1 and 2) and the response / channel statistics at 1, 127, 128, 129 and more bins.

Every solve goes through solver.general_solve_dynamics (both force
kernels with a QTF: tiles and RAFTK_QTF_DIAG=1) and asserts the kernel it ran.  Pass counts and the converged flag equal
the checker's; Xi is held per train to RTOL over the whole array and, per DOF row with a peak >= 1e-6 of the train's, to
ROW_RTOL of that row's own peak (an array-level bound alone would hide a wrong modal row at 1 % of the peak); measured
on an H100, the largest errors over the whole matrix are 5.1e-13 (array) and 7.1e-13 (per row).  F_BEM,
F_2nd and F_2nd_mean are held to 1e-12 (k_qtf_tiles adds with atomics, so nothing is compared bit for bit).  Every
synthetic impedance has cond(Z) <= 1e8 (tests/test_general_edges_oracle.py), so no bin needs the two-level tolerance of
the flexqtf fixture."""
import numpy as np
import pytest

import general_qtf_checker as gqc
import general_synth as gs
from conftest import relerr

pytestmark = [pytest.mark.gpu]

RTOL = 1e-10
ROW_RTOL = 1e-11              # measured on an H100: 7.1e-13 per row, 5.1e-13 per array (largest over every row below)
STATS_RTOL = 1e-13            # measured on an H100: <= 7.8e-15 (std, PSD, amp; n = 256, nw = 1)
_WORST = {"array": 0.0, "row": 0.0}
_CHECKER = {}


def _env(monkeypatch, diag=False):
    if diag:
        monkeypatch.setenv("RAFTK_QTF_DIAG", "1")
    else:
        monkeypatch.delenv("RAFTK_QTF_DIAG", raising=False)


def _checker(key, oracle, P, M, B, Cm, fd, qtf, trains, n_iter):
    """Checker results per case (cached: both LU kernels run on the same inputs)."""
    if key not in _CHECKER:
        _CHECKER[key] = [gqc.solve_trains_qtf(oracle, P, M, B, Cm, fd, qtf, tr, nIter=n_iter) for tr in trains]
    return _CHECKER[key]


def _solve_and_check(monkeypatch, oracle, name, arg=None, diag=False):
    from raft_b200 import solver
    r = gs.row(name, arg)
    P, M, B, Cm, fd, qtf, n_iter = r["P"], r["M"], r["B"], r["Cm"], r["fd"], r["qtf"], r["n_iter"]
    table, owner, first, trains = r["ct"]
    _env(monkeypatch, diag)
    bem = fd.get("X_BEM") is not None
    out = solver.general_solve_dynamics(P, M, B, Cm, solver.CaseTable(table), n_iter=n_iter, fd=fd, F_BEM=True, qtf=qtf, F_2nd=qtf is not None)
    Xi, st, Fb = out[:3]
    rec = solver.last_dispatch()
    assert rec["family"] == "general" and rec["kernel"] == "gen-blocked", rec
    assert rec["trains"] == (len(owner) > len(first)), rec
    ref = _checker((name, arg), oracle, P, M, B, Cm, fd, qtf, trains, n_iter)
    for ic, (Xo, so, Fo, F2o, F2mo) in enumerate(ref):
        idx = np.nonzero(owner == ic)[0]
        f = first[ic]
        assert st[f, 0] == so[0] and st[f, 1] == so[1] and st[f, 2] == so[2] == 0 and st[f, 3] == 0, (ic, st[f], so)
        for h, t in enumerate(idx):
            if h:
                assert st[t].tolist() == [0, 1, 0, f + 1], (ic, h, st[t])
            e, er = relerr(Xi[t], Xo[h]), gs.row_errors(Xi[t], Xo[h])
            _WORST["array"], _WORST["row"] = max(_WORST["array"], e), max(_WORST["row"], er)
            assert e < RTOL and er < ROW_RTOL, (ic, h, e, er)
            if bem:
                assert relerr(Fb[t], Fo[h]) < 1e-12, (ic, h, relerr(Fb[t], Fo[h]))
            else:
                assert not Fb[t].any()
            if qtf is not None:
                assert relerr(out[3][t], F2o[h]) < 1e-12 and relerr(out[4][t], F2mo[h]) < 1e-12, (ic, h)
    print("%s %s: largest Xi error so far %.2e (array), %.2e (per row)" % (name, arg, _WORST["array"], _WORST["row"]))


@pytest.mark.parametrize("n", [7, 9, 17])
def test_a_panel_crossing_support_with_trains(n, monkeypatch, oracle):
    """fd support {0, 3, 7, 8, 15, 16} & [0, n) | {n - 1}, rotor and BEM tables, dense T0, 129 bins, trains."""
    _solve_and_check(monkeypatch, oracle, "a", n)


def test_b_modal_support_rotor_only(monkeypatch, oracle):
    """n = 64, 257 bins, support {6, 31, 32, 63} (no platform DOF), rotor tables without BEM, trains."""
    _solve_and_check(monkeypatch, oracle, "b")


@pytest.mark.parametrize("nw", [128, 129])
def test_c_bem_only(nw, monkeypatch, oracle):
    """BEM table with n_fd = 0 (the constant-matrix LU with the BEM projection), dense T0, 128 and 129 bins."""
    _solve_and_check(monkeypatch, oracle, "c", nw)


@pytest.mark.parametrize("which", ["full", "last"])
def test_d_full_and_single_dof_support(which, monkeypatch, oracle):
    """n = 17, 33 bins: every DOF on the support (with BEM), or only the last one."""
    _solve_and_check(monkeypatch, oracle, "d", which)


@pytest.mark.parametrize("which", ["stride", "full"])
def test_e_256_dofs(which, monkeypatch, oracle):
    """n = 256 (k_gen_train_solve's b[256] full), support {0..5, 127, 128, 255} across the 128-thread stride of gen_fd_map,
    or all 256 DOFs; trains; n_iter 4 as in test_dispatch_general."""
    _solve_and_check(monkeypatch, oracle, "e", which)


QTF_ROWS = [(6, 33, False), (9, 129, True), (17, 129, False), (64, 257, False), (64, 257, True)]


@pytest.mark.parametrize("n,nw,diag", QTF_ROWS)
def test_f_second_order_loads(n, nw, diag, monkeypatch, oracle):
    """Second-order loads with a 3-heading QTF that covers bins nw/6 .. 2 nw/3; both force kernels; trains."""
    _solve_and_check(monkeypatch, oracle, "f", (n, nw), diag=diag)


def test_f_session_is_bit_identical_to_host_entry(monkeypatch):
    """With the reproducible force kernel (RAFTK_QTF_DIAG=1) at 129 bins: GeneralSession gives the host entry's bits."""
    from raft_b200 import solver
    _env(monkeypatch, True)
    r = gs.row("f", (17, 129))
    P, M, B, Cm, fd, qtf = r["P"], r["M"], r["B"], r["Cm"], r["fd"], r["qtf"]
    table = solver.CaseTable(r["ct"][0])
    Xh, sh, Fbh, F2h, F2mh = solver.general_solve_dynamics(P, M, B, Cm, table, fd=fd, F_BEM=True, qtf=qtf, F_2nd=True)
    S = solver.GeneralSession(P, M, B, Cm, table, fd=fd, F_BEM=True, qtf=qtf)
    Xs, ss, Fbs = S.solve()
    assert solver.last_dispatch()["kernel"] == "gen-blocked"
    assert np.array_equal(Xs.cpu().numpy(), Xh) and np.array_equal(ss.cpu().numpy(), sh) and np.array_equal(Fbs.cpu().numpy(), Fbh)
    assert np.array_equal(S.F_2nd.cpu().numpy(), F2h) and np.array_equal(S.F_2nd_mean.cpu().numpy(), F2mh)


@pytest.mark.parametrize("heads", [(40.0,), (20.0, 95.0, 200.0, 290.0)])
def test_g_bem_headings(heads, monkeypatch, oracle):
    """One BEM heading, or four; case headings 0, 20, 300, 355 (between the last table heading and the first) and -45 deg;
    heading_adjust 12.5 deg, x_ref 3 m, y_ref -2 m."""
    _solve_and_check(monkeypatch, oracle, "g", heads)


# ---- statistics kernels at the bin-count edges, against long-double references ------------------------------------------
def _rel_rows(a, ref):
    """max over rows (last axis = bins) of max|a - ref| / max|ref|."""
    a, ref = np.asarray(a, dtype=np.clongdouble), np.asarray(ref)
    return float((np.abs(a - ref).max(axis=-1) / np.maximum(np.abs(ref).max(axis=-1), 1e-300)).max())


def _general_ref(R, wpow, w, Xi, dw):
    L = np.longdouble
    Y = np.einsum("kb,ubw->ukw", R.astype(L), Xi.real.astype(L)) + 1j * np.einsum("kb,ubw->ukw", R.astype(L), Xi.imag.astype(L))
    Y = Y * (w.astype(L)[None, None, :] ** wpow.astype(L)[None, :, None])
    a2 = Y.real ** 2 + Y.imag ** 2
    return np.sqrt(L(0.5) * a2.sum(axis=-1)), L(0.5) * a2 / L(dw), Y


@pytest.mark.parametrize("nw", [1, 2, 127, 128, 129, 1000])
@pytest.mark.parametrize("n", [6, 150, 256])
def test_general_channel_stats_vs_longdouble(n, nw):
    """solver.general_channel_stats and GeneralSession.stats: 40 channels (wpow 0, 1, 2 mixed), 3 units."""
    import torch
    from raft_b200 import solver
    rng = np.random.default_rng(n * 1000 + nw)
    P, M, B, Cm = gs.design(n, 16)
    dw = 1.5 / nw                                      # the session's grid: nw bins up to 1.5 rad/s
    w = dw * np.arange(1, nw + 1)
    P = dict(P, w=w, k=w * w / 9.81, dw=dw)
    nch = 40
    R = rng.normal(size=(nch, n))
    wpow = np.resize(np.array([0, 1, 2, 1, 0, 2, 2], dtype=np.int32), nch)
    Xi = (rng.normal(size=(3, n, nw)) + 1j * rng.normal(size=(3, n, nw))) * rng.uniform(0.1, 10.0, (1, n, 1))
    sd_r, ps_r, Y_r = _general_ref(R, wpow, w, Xi, dw)
    S = solver.GeneralSession(P, M, B, Cm, solver.CaseTable(dict(Hs=np.full(3, 4.0), Tp=np.full(3, 10.0), gamma=np.zeros(3),
                                                                  beta_deg=np.zeros(3), spec=np.zeros(3, dtype=np.int32))))
    S.Xi.copy_(torch.from_numpy(Xi))
    sd_s, ps_s, amp_s = S.stats(R, wpow, psd=True, amp=True)
    got = [solver.general_channel_stats(R, wpow, w, Xi, dw, psd=True, amp=True),
           (sd_s.cpu().numpy(), ps_s.cpu().numpy(), amp_s.cpu().numpy())]
    for sd, ps, amp in got:
        e = (float(np.abs((sd - sd_r) / sd_r).max()), _rel_rows(ps, ps_r), _rel_rows(amp, Y_r))
        assert max(e) < STATS_RTOL, (n, nw, e)
        print("n %d nw %d: std %.1e, PSD %.1e, amp %.1e" % ((n, nw) + e))
    assert np.array_equal(got[0][0], got[1][0]) and np.array_equal(got[0][1], got[1][1])


def test_general_channel_stats_refuses_other_powers():
    """wpow outside {0, 1, 2}: ValueError from both Python entries, RAFTK_EINVAL from the device entry (read back)."""
    import torch
    from raft_b200 import _lib, solver
    P, M, B, Cm = gs.design(6, 8)
    S = solver.GeneralSession(P, M, B, Cm, solver.CaseTable(dict(Hs=np.full(1, 4.0), Tp=np.full(1, 10.0), gamma=np.zeros(1),
                                                                  beta_deg=np.zeros(1), spec=np.zeros(1, dtype=np.int32))))
    R = np.ones((2, 6))
    for bad in ([0, 3], [-1, 2]):
        with pytest.raises(ValueError, match="wpow must be 0, 1 or 2"):
            S.stats(R, np.array(bad))
    dR = torch.ones((2, 6), dtype=torch.float64, device=S.device)
    dp = torch.tensor([2, 3], dtype=torch.int32, device=S.device)
    sd = torch.zeros(2, dtype=torch.float64, device=S.device)
    rc = _lib.lib.raftk_general_channel_stats_dev(1, 6, 2, 8, S.dw, S.keep["w"].data_ptr(), dR.data_ptr(), dp.data_ptr(), S.Xi.data_ptr(),
                                                  sd.data_ptr(), None, None, torch.cuda.current_stream().cuda_stream)
    assert rc == -1 and b"wpow must be 0, 1 or 2" in _lib.lib.raftk_last_error()
    assert not sd.any()


@pytest.mark.parametrize("nw", [1, 127, 128, 129])
@pytest.mark.parametrize("rot_deg", [False, True])
def test_response_stats_vs_longdouble(nw, rot_deg):
    from raft_b200 import solver
    rng = np.random.default_rng(nw + 7 * rot_deg)
    Xi = rng.normal(size=(3, 2, 6, nw)) + 1j * rng.normal(size=(3, 2, 6, nw))
    dw = 0.037
    sd, ps = solver.response_stats(Xi, dw, psd=True, rot_deg=rot_deg)
    L = np.longdouble
    scale = np.array([1, 1, 1] + [L(180) / L(np.pi) if rot_deg else 1] * 3, dtype=L)[:, None]
    a2 = (Xi.real.astype(L) * scale) ** 2 + (Xi.imag.astype(L) * scale) ** 2
    e = (float(np.abs((sd - np.sqrt(L(0.5) * a2.sum(-1))) / np.sqrt(L(0.5) * a2.sum(-1))).max()), _rel_rows(ps, L(0.5) * a2 / L(dw)))
    assert max(e) < STATS_RTOL, (nw, rot_deg, e)


@pytest.mark.parametrize("nw", [1, 127, 128, 129])
def test_channel_stats_vs_longdouble(nw):
    """3 designs x 2 cases x 5 channels: the (design, case, channel) row mapping of k_channel_stats."""
    from raft_b200 import solver
    rng = np.random.default_rng(100 + nw)
    coef = (rng.normal(size=(3, 5, 6, nw)) + 1j * rng.normal(size=(3, 5, 6, nw))) * rng.uniform(0.5, 5.0, (3, 5, 1, 1))
    Xi = (rng.normal(size=(3, 2, 6, nw)) + 1j * rng.normal(size=(3, 2, 6, nw))) * rng.uniform(0.5, 5.0, (3, 2, 1, 1))
    dw = 0.05
    sd, ps, amp = solver.channel_stats(coef, Xi, dw, psd=True, amp=True)
    L = np.longdouble
    Y = np.einsum("dkaw,dcaw->dckw", coef.astype(np.clongdouble), Xi.astype(np.clongdouble))
    a2 = Y.real ** 2 + Y.imag ** 2
    sd_r = np.sqrt(L(0.5) * a2.sum(-1))
    e = (float(np.abs((sd - sd_r) / sd_r).max()), _rel_rows(ps, L(0.5) * a2 / L(dw)), _rel_rows(amp, Y))
    assert max(e) < STATS_RTOL, (nw, e)
