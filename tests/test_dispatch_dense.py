"""Dense complex solves: k_system_solve on both sides of its switch at n = 24 (column-at-a-time LU up to 24, blocked LU with
8-column panels above), including sizes that are not a multiple of the panel width and an exactly singular frequency, and
the farm's shared-memory warp kernel at 6N = 12 (RAFTK_FARM_SMEM=1), all against the oracle's explicit-inverse response
(raft_model.py:1189-1216), with the kernel asserted through solver.last_dispatch()."""
import numpy as np
import pytest

from conftest import relerr, response_err

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n", [1, 2, 5, 23, 24, 25, 31, 33, 49])
@pytest.mark.parametrize("nrhs", [1, 3])
def test_system_solve_around_the_switch(n, nrhs, oracle):
    from raft_b200 import solver
    rng = np.random.default_rng(100 * n + nrhs)
    nw = 21
    A = rng.normal(size=(nw, n, n)) + 1j * rng.normal(size=(nw, n, n))
    A[1::2] += 2 * np.sqrt(n) * np.eye(n)[None]                             # half the frequencies diagonally dominant, half pivoting
    F = rng.normal(size=(nw, n, nrhs)) + 1j * rng.normal(size=(nw, n, nrhs))
    X, info = solver.system_solve(A, F)
    rec = solver.last_dispatch()
    assert rec["family"] == "system" and rec["kernel"] == ("sys-blocked" if n > 24 else "sys-unblocked"), rec
    assert np.all(info == 0)
    for r in range(nrhs):
        assert relerr(X[:, :, r], oracle.system_response(A, F[:, :, r])) < 1e-11


@pytest.mark.parametrize("n", [5, 25])
def test_system_solve_singular_frequency(n, oracle):
    """One frequency's matrix has an all-zero column 3: info there is 4 (k+1 of the first zero pivot); the other frequencies
    are unaffected."""
    from raft_b200 import solver
    rng = np.random.default_rng(n)
    nw, bad = 9, 4
    A = rng.normal(size=(nw, n, n)) + 1j * rng.normal(size=(nw, n, n)) + 3 * np.eye(n)[None]
    A[bad, :, 3] = 0.0
    F = rng.normal(size=(nw, n)) + 1j * rng.normal(size=(nw, n))
    X, info = solver.system_solve(A, F)
    assert info[bad] == 4 and np.count_nonzero(info) == 1
    ok = np.arange(nw) != bad
    assert relerr(X[ok], oracle.system_response(A[ok], F[ok])) < 1e-11
    with pytest.raises(np.linalg.LinAlgError):
        oracle.system_response(A, F)


@pytest.mark.parametrize("smem", [False, True])
def test_farm_two_fowts_kernels_vs_oracle(smem, monkeypatch, oracle):
    """N = 2: the register-row kernel (default) and the shared-memory warp kernel (RAFTK_FARM_SMEM=1) against the oracle's
    per-FOWT solves and explicit-inverse system response, as test_farm.test_farm_baseline_size_vs_oracle."""
    from test_farm import _cases, _farm_fixture
    from raft_b200 import grid, solver
    if smem:
        monkeypatch.setenv("RAFTK_FARM_SMEM", "1")
    else:
        monkeypatch.delenv("RAFTK_FARM_SMEM", raising=False)
    z, packs = _farm_fixture()
    nw = 301
    Q = [grid.regrid(P, nw, 0.1024) for P in packs]
    cs = _cases(np.array([[6.0, 12.0, 0.0], [4.0, 9.0, 35.0], [2.5, 7.0, -120.0]]))
    out = solver.solve_dynamics_farm(solver.DesignBatch(Q), solver.CaseTable(cs), C_arr=z["C_array"], n_iter=10)
    rec = solver.last_dispatch()
    assert rec["family"] == "farm" and rec["kernel"] == ("farm-warp" if smem else "farm-rows12"), rec
    assert not np.any(out["info"])
    for c in range(3):
        Zs = np.zeros([nw, 12, 12], dtype=complex)
        F = np.zeros([nw, 12], dtype=complex)
        for i, P in enumerate(Q):
            Xi_i, st, Z_i, _ = oracle.solve_dynamics(oracle.OracleDesign(P), 0, cs["Hs"][c], cs["Tp"][c], 0.0, cs["beta_deg"][c], nIter=10, want_Z=True)
            assert st[0] == out["status"][i, c, 0]
            Zs[:, 6 * i:6 * i + 6, 6 * i:6 * i + 6] = Z_i
            F[:, 6 * i:6 * i + 6] = np.einsum("wab,bw->wa", Z_i, Xi_i)
        Xo = oracle.system_response(Zs + z["C_array"][None], F).T
        err = max(response_err(out["Xi_sys"][c, 6 * i:6 * i + 6], Xo[6 * i:6 * i + 6]) for i in range(2))
        assert err < 1e-9, err
