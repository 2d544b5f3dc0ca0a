"""Generalised degrees of freedom: the LU kernel of raftk_general_solve_dynamics, k_gen_solve_blocked, at sizes around its
panel width (8) and up to the limit of 256 DOFs, against oracle.general_solve_dynamics, asserted through solver.last_dispatch().

The designs are synthetic: the rigid OC3spar on a small grid, with n - 6 seeded smooth mode shapes added to the node
transformation (gen_Tn = [I6 | modes], gen_rr = node offset from the reference point) and modal blocks in M, B, C.  The
modal stiffness couples each mode to the next (a cyclic shift of weight 3), so partial pivoting swaps rows.  At n = 6 the
construction is the rigid design itself: the CPU test below checks that the oracle's generalised solve reproduces its rigid
solve there."""

import numpy as np
import pytest

from conftest import GOLDEN, load_golden, relerr, response_err

RTOL = 1e-10


def _rigid(nw):
    from raft_b200 import grid
    return grid.regrid(load_golden("cfg1_OC3spar")[1], nw, 0.25)


def general_design(n, nw, seed=0):
    """-> (P, M, B, C) of a synthetic n-DOF design built on the rigid OC3spar (see the module docstring)."""
    P = dict(_rigid(nw))
    rng = np.random.default_rng(seed + n)
    r = np.asarray(P["node_r"], dtype=float)
    Ns, m = len(r), n - 6
    Tn = np.zeros([Ns, 6, n])
    Tn[:, :, :6] = np.eye(6)[None]
    z = r[:, 2]
    L = max(np.ptp(z), 1.0)
    for j in range(m):
        kz, ph = (j % 7 + 1) * np.pi / L, rng.uniform(0, 2 * np.pi, 5)
        amp = rng.uniform(0.5, 1.5)
        Tn[:, 0, 6 + j] = amp * np.sin(kz * z + ph[0])
        Tn[:, 1, 6 + j] = amp * np.cos(kz * z + ph[1])
        Tn[:, 2, 6 + j] = 0.2 * amp * np.sin(kz * z + ph[2])
        Tn[:, 3, 6 + j] = 0.01 * amp * kz * np.cos(kz * z + ph[3])
        Tn[:, 4, 6 + j] = 0.01 * amp * kz * np.sin(kz * z + ph[4])
    P["gen_nDOF"] = n
    P["gen_Tn"] = np.ascontiguousarray(Tn)
    P["gen_rr"] = np.ascontiguousarray(r - np.asarray(P["prp"], dtype=float)[None, :])
    M, B, C = (np.zeros([n, n]) for _ in range(3))
    M[:6, :6], B[:6, :6], C[:6, :6] = (np.asarray(P[k]).reshape(6, 6) for k in ("M0", "B0", "C0"))
    if m:
        mm = rng.uniform(0.5, 2.0, m) * 1e6
        om = rng.uniform(0.6, 2.5, m)
        shift = np.roll(np.eye(m), 1, axis=1) if m > 1 else np.zeros([1, 1])
        M[6:, 6:] = np.diag(mm)
        C[6:, 6:] = np.diag(mm * om ** 2) + 3.0 * shift * (mm * om ** 2)[:, None]
        B[6:, 6:] = np.diag(2 * 0.05 * mm * om)
    return P, M, B, C


def _sea(n=2, seed=5):
    rng = np.random.default_rng(seed)
    return dict(Hs=rng.uniform(2, 8, n), Tp=rng.uniform(6, 16, n), gamma=np.zeros(n), beta_deg=rng.uniform(-90, 90, n),
                spec=np.zeros(n, dtype=np.int32))


def test_construction_at_six_dofs_is_the_rigid_design(oracle):
    """CPU: with n = 6 the generalised oracle reproduces the rigid oracle on the same design."""
    P, M, B, C = general_design(6, 48)
    cs = _sea(3)
    Xr, sr, _ = oracle.solve_cases(oracle.OracleDesign(P), cs, nIter=10)
    gd = oracle.GeneralDesign(P)
    for c in range(3):
        Xg, sg = oracle.general_solve_dynamics(gd, M, B, C, 0, cs["Hs"][c], cs["Tp"][c], 0.0, cs["beta_deg"][c], nIter=10)
        assert sg[0] == sr[c, 0] and sg[1] == sr[c, 1]
        assert response_err(Xg, Xr[c]) < 1e-10


def test_construction_pivots_and_couples(oracle):
    """CPU: the synthetic impedance needs row swaps (partial pivoting picks an off-diagonal row) and the modes carry load."""
    P, M, B, C = general_design(9, 24)
    w = P["w"][len(P["w"]) // 2]
    Z = -w * w * M + 1j * w * B + C
    sub = np.abs(Z[6:, 6:])
    assert np.any(sub.max(axis=0) > np.diag(sub))
    gd = oracle.GeneralDesign(P)
    _, F, _ = oracle.general_excitation(gd, 0, 6.0, 10.0, 0.0, 30.0)
    assert np.abs(F[6:]).max() > 1e-3 * np.abs(F[:6]).max()


def _gpu_solve(P, M, B, C, cs, n_iter):
    from raft_b200 import solver
    Xi, st = solver.general_solve_dynamics(P, M, B, C, solver.CaseTable(cs), n_iter=n_iter)
    return Xi, st, solver.last_dispatch()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [6, 7, 8, 9, 16, 17, 64, 256])
def test_lu_kernels_vs_oracle(n, oracle):
    nw = 12 if n > 64 else 32
    n_iter = 4 if n > 64 else 10
    P, M, B, C = general_design(n, nw)
    cs = _sea()
    gd = oracle.GeneralDesign(P)
    ref = [oracle.general_solve_dynamics(gd, M, B, C, 0, cs["Hs"][c], cs["Tp"][c], 0.0, cs["beta_deg"][c], nIter=n_iter) for c in range(2)]
    Xi, st, rec = _gpu_solve(P, M, B, C, cs, n_iter)
    assert rec["family"] == "general" and rec["kernel"] == "gen-blocked", rec
    for c, (Xo, so) in enumerate(ref):
        assert st[c, 0] == so[0] and st[c, 1] == so[1] and st[c, 2] == 0, (c, st[c], so)
        assert relerr(Xi[c], Xo) < RTOL, (c, relerr(Xi[c], Xo))


@pytest.mark.gpu
def test_more_than_256_dofs_is_rejected():
    from raft_b200 import _lib, solver
    P, M, B, C = general_design(257, 8)
    with pytest.raises(_lib.RaftkError, match="n_dof <= 256"):
        solver.general_solve_dynamics(P, M, B, C, solver.CaseTable(_sea(1)), n_iter=2)
    assert solver.last_dispatch()["kernel"] == "none"
