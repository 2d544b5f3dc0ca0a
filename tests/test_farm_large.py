"""Farms whose coupled 6N x 6N system does not fit in one CTA's shared memory (k_farm_response_global), and dense system
solves of any size (k_system_solve_global): against a run of the UNMODIFIED reference on a 24-FOWT array (fixture
farm24_VolturnUS-S_farm_nw48, tests/golden/make_golden_farm24.py), against the oracle's per-FOWT solves + explicit-inverse
system response, against a NumPy assembly of the same call's inputs, and across workspace sizes."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN, relerr, response_err

RTOL = 1e-10
gpu = pytest.mark.gpu


def _cases(rows, primary=None):
    n = len(rows)
    d = dict(Hs=rows[:, 0], Tp=rows[:, 1], gamma=np.zeros(n), beta_deg=rows[:, 2], spec=np.zeros(n, dtype=np.int32))
    if primary is not None:
        d["primary"] = np.asarray(primary, dtype=np.int32)
    return d


def _fixture24():
    z = np.load(os.path.join(GOLDEN, "farm24_VolturnUS-S_farm_nw48.npz"))
    N = int(z["n_fowt"])
    packs = [{k[len("P%d_" % i):]: z[k] for k in z.files if k.startswith("P%d_" % i)} for i in range(N)]
    return z, packs


def _block_err(Xi_sys, ref, N):
    return max(response_err(Xi_sys[..., 6 * i:6 * i + 6, :], ref[..., 6 * i:6 * i + 6, :]) for i in range(N))


def test_farm_workspace_query_without_gpu():
    """raftk_farm_workspace_bytes: 0 while the shared-memory kernels keep the farm, one [6N][6N+1] slab per resident CTA
    above (never more slabs than systems)."""
    from raft_b200 import solver
    for N in range(1, 20):
        assert solver.farm_workspace_bytes(N, 64, 1024) == 0, N
    for N in (21, 24, 32, 64, 100):
        slab = 6 * N * (6 * N + 1) * 16
        b = solver.farm_workspace_bytes(N, 64, 1024)
        assert b > 0 and b % slab == 0 and 1 <= b // slab <= 64 * 1024, (N, b)
        assert solver.farm_workspace_bytes(N, 1, 3) == 3 * slab
        assert solver.farm_workspace_bytes(N, 2, 1) == 2 * slab


@gpu
def test_farm24_vs_reference_run():
    """24 FOWTs (144 DOFs) through the host entry and the Model API against the reference's own run."""
    from raft_b200 import solver
    from raft_b200.model import Model
    z, packs = _fixture24()
    N = len(packs)
    cs = _cases(z["cases"])
    out = solver.solve_dynamics_farm(solver.DesignBatch(packs), solver.CaseTable(cs), C_arr=z["C_array"],
                                     n_iter=int(z["n_iter"]), xi_start=float(z["xi_start"]))
    rec = solver.last_dispatch()
    assert rec["family"] == "farm" and rec["kernel"] == "farm-global", rec
    assert not np.any(out["info"]) and np.all(out["status"][..., 2] == 0)
    assert np.array_equal(out["status"][:, :, 0].T, z["ref_run_passes"])
    ref = z["ref_run_Xi"][:, 0]                                                             # [nCases, 144, nw]
    err = _block_err(out["Xi_sys"], ref, N)
    assert err < RTOL, err
    D = json.loads(str(z["design_json"]))
    design = dict(settings=D["settings"], site=D["site"], platform=D["platform"], array=D["array"])
    mats = [dict(M_struc=P["M0"] - z["A_hydro_morison%d" % i], C_struc=P["C0"] - z["C_moor%d" % i], C_moor=z["C_moor%d" % i])
            for i, P in enumerate(packs)]
    model = Model(design, matrices=mats, array_stiffness=z["C_array"])
    assert model.nFOWT == N and model.nDOF == 6 * N and model.nw == 48
    case_dicts = [dict(wave_spectrum="JONSWAP", wave_height=Hs, wave_period=Tp, wave_heading=beta) for Hs, Tp, beta in z["cases"]]
    for ic, case in enumerate(case_dicts):
        Xi = model.solveDynamics(case)
        assert Xi.shape == z["ref_run_Xi"][ic].shape and np.all(Xi[-1] == 0)
        assert _block_err(Xi[0], z["ref_run_Xi"][ic, 0], N) < RTOL
        assert solver.last_dispatch()["kernel"] == "farm-global"
    model.analyzeCases(cases=case_dicts)
    assert _block_err(model.results["Xi"], ref, N) < RTOL
    assert np.array_equal(model.results["status"][:, :, 0], z["ref_run_passes"])


@gpu
@pytest.mark.parametrize("N", [20, 21, 32, 64])
def test_farm_large_arrays_vs_oracle(N, oracle):
    """N = 20 on whichever kernel the fit rule picks (the shared-memory block kernel when 120 x 121 x 16 B plus its static
    shared memory fits the device's opt-in maximum), N >= 21 on the global-memory kernel."""
    import bench_extra
    from raft_b200 import solver
    packs, C_arr, _ = bench_extra.farm_designs(N, nw=96, max_freq=0.1024)
    cs = _cases(np.array([[6.0, 12.0, 0.0], [3.0, 8.0, -70.0]]))
    out = solver.solve_dynamics_farm(solver.DesignBatch(packs), solver.CaseTable(cs), C_arr=C_arr, n_iter=10)
    rec = solver.last_dispatch()
    fits = solver.farm_workspace_bytes(N, 2, 96) == 0
    assert rec["family"] == "farm" and rec["kernel"] == ("farm-block" if fits else "farm-global"), rec
    if N > 20:
        assert not fits
    print("N = %d: %s" % (N, rec["kernel"]))
    Xo, passes = bench_extra._oracle_farm(packs, C_arr, cs)
    assert np.array_equal(passes, out["status"][:, :, 0]) and not np.any(out["info"])
    err = _block_err(out["Xi_sys"], Xo, N)
    assert err < 1e-9, err


@gpu
def test_farm_global_assembly_inputs():
    """M_arr, B_arr and C_arr together, and a case with two wave trains (the secondary uses its primary's B_drag): Xi_sys
    against a NumPy assembly of the same call's per-FOWT outputs solved by numpy.linalg.solve; without array matrices
    Xi_sys is the stacked per-FOWT response."""
    import bench_extra
    from raft_b200 import solver
    N, nw = 22, 40
    n = 6 * N
    packs, C_arr, _ = bench_extra.farm_designs(N, nw=nw, max_freq=0.1024)
    rng = np.random.default_rng(22)
    G = rng.normal(size=(n, n))
    M_arr = (G @ G.T) * 2e3 / n
    B_arr = (G + G.T) * 1e3
    rows = np.array([[6.0, 12.0, 0.0], [2.0, 7.0, 60.0], [4.0, 10.0, -30.0]])
    cs = _cases(rows, primary=[0, 0, 2])
    batch, cases = solver.DesignBatch(packs), solver.CaseTable(cs)
    out = solver.solve_dynamics_farm(batch, cases, C_arr=C_arr, M_arr=M_arr, B_arr=B_arr, n_iter=10,
                                     want=("Xi", "status", "B_drag", "F_drag", "F_iner"))
    assert solver.last_dispatch()["kernel"] == "farm-global" and not np.any(out["info"])
    w = packs[0]["w"]
    for c, cp in enumerate(cs["primary"]):
        for iw in range(nw):
            Z = -w[iw] ** 2 * M_arr + 1j * w[iw] * B_arr + C_arr
            F = np.zeros(n, dtype=complex)
            for i, P in enumerate(packs):
                s = slice(6 * i, 6 * i + 6)
                Z[s, s] += -w[iw] ** 2 * P["M0"] + 1j * w[iw] * (P["B0"] + out["B_drag"][i, cp]) + P["C0"]
                F[s] = out["F_drag"][i, c, :, iw] + out["F_iner"][i, c, :, iw]
            x = np.linalg.solve(Z, F)
            assert relerr(out["Xi_sys"][c, :, iw], x) < 1e-11, (c, iw)
    unc = solver.solve_dynamics_farm(batch, cases, n_iter=10)
    assert solver.last_dispatch()["kernel"] == "farm-global"
    per = np.concatenate([unc["Xi"][i] for i in range(N)], axis=1)                          # [nC, 6N, nw]
    assert _block_err(unc["Xi_sys"], per, N) < RTOL


@gpu
def test_farm_global_workspace_sizes():
    """The queried workspace and exactly one slab give bit-identical Xi_sys and info; one byte less than a slab is refused
    before any launch; the host entry and DeviceSession.farm_response agree bit for bit."""
    import torch
    import bench_extra
    from raft_b200 import _lib, solver
    N, nw = 21, 64
    n = 6 * N
    packs, C_arr, _ = bench_extra.farm_designs(N, nw=nw, max_freq=0.1024)
    cs = _cases(np.array([[6.0, 12.0, 0.0], [3.0, 8.0, -70.0], [9.0, 15.0, 150.0]]))
    batch, cases = solver.DesignBatch(packs), solver.CaseTable(cs)
    sess = solver.DeviceSession(batch, cases, device="cuda:0", want=("Xi", "status", "B_drag", "F_drag", "F_iner"))
    sess.solve(n_iter=10)
    xi, info = sess.farm_response(C_arr=C_arr)
    assert solver.last_dispatch()["kernel"] == "farm-global"
    full_xi, full_info = xi.cpu().numpy().copy(), info.cpu().numpy().copy()
    f, _, _, _, _, wsb = sess._farm
    slab = n * (n + 1) * 16
    assert wsb == solver.farm_workspace_bytes(N, 3, nw) and wsb > slab
    one = torch.empty(slab, dtype=torch.uint8, device="cuda:0")
    xi.zero_()
    info.fill_(-7)
    args = (C.byref(sess.d_struct), C.byref(sess.c_struct), C.byref(sess.o_struct), C.byref(f))
    stream = torch.cuda.current_stream().cuda_stream
    assert _lib.lib.raftk_farm_response_ws_dev(*args, one.data_ptr(), slab, stream) == 0
    rec = solver.last_dispatch()
    assert rec["kernel"] == "farm-global" and rec["threads_per_cta"] > 0
    torch.cuda.synchronize()
    assert np.array_equal(xi.cpu().numpy(), full_xi) and np.array_equal(info.cpu().numpy(), full_info)
    assert _lib.lib.raftk_farm_response_ws_dev(*args, one.data_ptr(), slab - 1, stream) == -1
    assert solver.last_dispatch()["kernel"] == "none"
    assert _lib.lib.raftk_farm_response_dev(*args, stream) == -1                            # no workspace: refused
    assert solver.last_dispatch()["kernel"] == "none"
    host = solver.solve_dynamics_farm(batch, cases, C_arr=C_arr, n_iter=10)
    assert np.array_equal(host["Xi_sys"], full_xi) and np.array_equal(host["info"], full_info)
    assert np.array_equal(host["Xi"], sess.out["Xi"].cpu().numpy())


@gpu
@pytest.mark.parametrize("n", [121, 150, 197, 385])
@pytest.mark.parametrize("nrhs", [1, 3])
def test_system_solve_global_vs_oracle(n, nrhs, oracle):
    """Systems whose [n][n+nrhs] matrix does not fit in shared memory, including sizes that are not a multiple of the panel
    width, half of the frequencies diagonally dominant and half pivoting."""
    from raft_b200 import solver
    rng = np.random.default_rng(1000 * n + nrhs)
    nw = 7
    A = rng.normal(size=(nw, n, n)) + 1j * rng.normal(size=(nw, n, n))
    A[1::2] += 2 * np.sqrt(n) * np.eye(n)[None]
    F = rng.normal(size=(nw, n, nrhs)) + 1j * rng.normal(size=(nw, n, nrhs))
    X, info = solver.system_solve(A, F)
    rec = solver.last_dispatch()
    assert rec["family"] == "system" and rec["kernel"] == "sys-global", rec
    assert np.all(info == 0)
    for r in range(nrhs):
        assert relerr(X[:, :, r], oracle.system_response(A, F[:, :, r])) < 1e-11


@gpu
def test_system_solve_global_singular_frequency(oracle):
    """n = 150: one frequency with an all-zero column 3 gives info = 4 there; the other frequencies are unaffected."""
    from raft_b200 import solver
    n, nw, bad = 150, 6, 2
    rng = np.random.default_rng(150)
    A = rng.normal(size=(nw, n, n)) + 1j * rng.normal(size=(nw, n, n)) + 3 * np.eye(n)[None]
    A[bad, :, 3] = 0.0
    F = rng.normal(size=(nw, n)) + 1j * rng.normal(size=(nw, n))
    X, info = solver.system_solve(A, F)
    assert solver.last_dispatch()["kernel"] == "sys-global"
    assert info[bad] == 4 and np.count_nonzero(info) == 1
    ok = np.arange(nw) != bad
    assert relerr(X[ok], oracle.system_response(A[ok], F[ok])) < 1e-11
