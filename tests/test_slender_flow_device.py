"""potSecOrder 1 on the device in one call (raftk_solve_dynamics_slender_*, solver.SlenderSession): loop A, RAOs on the
second-order grid (k_slender_rao), batched slender-body QTF, second-order force and loop B, merged per unit (k_slender_merge).
The host flow ``solver.solve_dynamics_slender`` (pinned to the reference run) is the checker."""
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN, relerr, response_err

pytestmark = pytest.mark.gpu
RTOL = 1e-10
OUTS = ("Xi", "status", "B_drag", "F_drag", "F_iner", "F_BEM", "zeta", "F_2nd", "F_2nd_mean", "Xi_last", "qtf", "Xi_rao")


@pytest.fixture(scope="module")
def solver():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from raft_b200 import solver as s
    return s


def _golden(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    return z, {k[2:]: z[k] for k in z.files if k.startswith("P_")}


def _random_design(Pa, seed):
    """A strip-theory design of random members on the VolturnUS-S fixture's grids (potSecOrder 1)."""
    from raft_b200.fowt import FOWT
    from test_slender_qtf import _member
    rng = np.random.default_rng(seed)
    members = [_member(rng, i, 30.0, 3.0) for i in range(5)]
    plat = dict(potModMaster=0, dlsMax=5.0, members=members, potSecOrder=1, min_freq2nd=0.04, df_freq2nd=0.008, max_freq2nd=0.2)
    mats = dict(M_struc=np.diag([2e7, 2e7, 2e7, 1.8e10, 1.8e10, 3e10]), C_hydro=np.diag([0, 0, 4e6, 2e9, 2e9, 0.0]),
                C_moor=np.diag([7e4, 7e4, 0, 0, 0, 1.2e8]))
    f = FOWT(dict(site=dict(water_depth=float(Pa["depth"]), rho_water=float(Pa["rho"]), g=float(Pa["g"])), platform=plat), Pa["w"],
             depth=float(Pa["depth"]), matrices=mats)
    f.calcHydroConstants()
    P = f.pack()
    assert np.array_equal(P["qs_w"], Pa["qs_w"]) and np.array_equal(P["w"], Pa["w"])
    return P


def _cases(seed, n, zeta=None):
    rng = np.random.default_rng(seed)
    return dict(Hs=rng.uniform(1.5, 9.0, n), Tp=rng.uniform(6.0, 17.0, n), gamma=np.zeros(n), beta_deg=rng.uniform(-180, 180, n),
                spec=np.zeros(n, dtype=np.int32))


def _session(solver, packed, ct, want=OUTS, qtf_chunk=0, **kw):
    import torch
    s = solver.SlenderSession(packed, ct, want=want, qtf_chunk=qtf_chunk)
    out = s.solve(**kw)
    torch.cuda.synchronize()
    return s, {k: v.cpu().numpy() for k, v in out.items()}


@pytest.fixture(scope="module")
def designs():
    _, Pa = _golden("slender_VolturnUS-S")
    return [Pa, _random_design(Pa, 9), _random_design(Pa, 13)]


def test_reference_run_through_session(solver):
    """The reference's own potSecOrder 1 run: pass counts identical, Xi, F_2nd, F_2nd_mean and qtf within RTOL."""
    z, P = _golden("slender_VolturnUS-S")
    cs = z["ref_run_solve_cases"]
    n = len(cs)
    ct = solver.CaseTable(dict(Hs=cs[:, 0], Tp=cs[:, 1], gamma=np.zeros(n), beta_deg=cs[:, 2], spec=np.zeros(n, dtype=np.int32)))
    _, out = _session(solver, P, ct, n_iter=int(z["n_iter"]), xi_start=float(z["xi_start"]))
    assert np.array_equal(out["status"][0, :, 0], z["ref_run_solve_passes"])
    assert response_err(out["Xi"][0], z["ref_run_solve_Xi"]) < RTOL
    assert relerr(out["F_2nd"][0], z["ref_run_solve_F2nd"]) < RTOL and relerr(out["F_2nd_mean"][0], z["ref_run_solve_F2nd_mean"]) < RTOL
    for i in range(n):
        assert relerr(out["qtf"][0, i], z["ref_run_solve_qtf"][i]) < RTOL


@pytest.mark.parametrize("n_iter", [4, 5, 10])
def test_multi_design_batch_vs_host_flow(solver, designs, n_iter, monkeypatch):
    """Three designs x 16 cases against solve_dynamics_slender: with the diagonal force kernel every output is bit-identical;
    with the default tile kernel (atomic sums) the status words are identical and Xi within 1e-12.  Small n_iter leaves some
    units unconverged after loop A: they keep loop A's result with zero force and QTF."""
    ct = solver.CaseTable(_cases(n_iter, 16))
    want = tuple(k for k in OUTS if k not in ("qtf", "Xi_rao"))
    monkeypatch.setenv("RAFTK_QTF_DIAG", "1")
    ref = solver.solve_dynamics_slender(designs, ct, n_iter=n_iter, want=want)
    _, out = _session(solver, designs, ct, n_iter=n_iter)
    plain = solver.DesignBatch([{k: v for k, v in P.items() if not k.startswith("qs_")} for P in designs])
    conv = solver.solve_dynamics(plain, ct, n_iter=n_iter)["status"][..., 1] == 1          # loop A alone
    assert conv.any(), conv
    if n_iter == 4:
        assert (~conv).any(), conv
    for k in want + ("qtf",):
        assert np.array_equal(out[k], ref[k]), k
    assert np.all(out["F_2nd"][~conv] == 0) and np.all(out["qtf"][~conv] == 0) and np.all(out["Xi_rao"][~conv] == 0)
    monkeypatch.delenv("RAFTK_QTF_DIAG")
    ref = solver.solve_dynamics_slender(designs, ct, n_iter=n_iter, want=want)
    _, out = _session(solver, designs, ct, n_iter=n_iter)
    assert np.array_equal(out["status"], ref["status"])
    assert response_err(out["Xi"], ref["Xi"]) < 1e-12
    assert relerr(out["F_2nd"], ref["F_2nd"]) < 1e-14 and relerr(out["qtf"], ref["qtf"]) < 1e-14


def test_rao_kernel_bits_and_batched_qtf(solver, designs):
    """k_slender_rao against getRAO + np.interp bit for bit, on a second-order grid reaching past the first-order grid on both
    sides and with explicit wave amplitudes at or below 1e-6 in some bins; each unit's QTF against qtf_slender on its own
    design, bit for bit."""
    Pa, Pb = designs[0], designs[1]
    w = Pa["w"]
    qw = np.linspace(0.5 * w[0], 1.3 * w[-1], 17)
    grids = [dict(P, qs_w=qw, qs_k=qw ** 2 / float(P["g"])) for P in (Pa, Pb)]
    rng = np.random.default_rng(4)
    nC = 6
    zeta = rng.uniform(0.05, 0.6, (nC, len(w)))
    zeta[:, ::5] = rng.uniform(0, 1e-6, zeta[:, ::5].shape)
    zeta[:, 1::7] = 1e-6
    cs = _cases(3, nC)
    ct = solver.CaseTable(cs, zeta=zeta)
    _, out = _session(solver, grids, ct, n_iter=10)
    plain = solver.DesignBatch([{k: v for k, v in P.items() if not k.startswith("qs_")} for P in grids])
    A = solver.solve_dynamics(plain, solver.CaseTable(cs, zeta=zeta), n_iter=10, want=("Xi", "status", "zeta"))
    conv = A["status"][..., 1] == 1
    assert conv.sum() >= 4
    beta = cs["beta_deg"] * 0.017453292519943295
    for d, P in enumerate(grids):
        for c in range(nC):
            if not conv[d, c]:
                assert np.all(out["Xi_rao"][d, c] == 0)
                continue
            r = solver.get_rao(A["Xi"][d, c], A["zeta"][c])
            want = np.array([np.interp(qw, w, r[a], left=0, right=0) for a in range(6)])
            assert np.array_equal(out["Xi_rao"][d, c].view(np.int64), want.view(np.int64)), (d, c)
            q = solver.qtf_slender(P, beta[c:c + 1], out["Xi_rao"][d, c][None])[0]
            assert np.array_equal(out["qtf"][d, c], q), (d, c)


def test_results_independent_of_qtf_chunk(solver, designs, monkeypatch):
    """QTF chunks of 1, 7 (straddling design boundaries) and all units: bit-identical with the diagonal force kernel, within
    1e-14 (F_2nd; Xi within 1e-12 after loop B) with the tile kernel; the host entry point gives the same bits."""
    ct = solver.CaseTable(_cases(7, 16))
    monkeypatch.setenv("RAFTK_QTF_DIAG", "1")
    runs = [_session(solver, designs, ct, qtf_chunk=k, n_iter=4) for k in (0, 1, 7)]
    for s, o in runs[1:]:
        for k in OUTS:
            assert np.array_equal(o[k], runs[0][1][k]), (s.qtf_chunk, k)
    assert runs[1][0].workspace_bytes < runs[2][0].workspace_bytes < runs[0][0].workspace_bytes
    host = solver.slender_flow_host(designs, ct, n_iter=4, want=OUTS, qtf_chunk=5)
    for k in OUTS:
        assert np.array_equal(host[k], runs[0][1][k]), k
    monkeypatch.delenv("RAFTK_QTF_DIAG")
    a = _session(solver, designs, ct, qtf_chunk=1, n_iter=4)[1]
    b = _session(solver, designs, ct, qtf_chunk=0, n_iter=4)[1]
    assert np.array_equal(a["status"], b["status"]) and np.array_equal(a["qtf"], b["qtf"])
    assert relerr(a["F_2nd"], b["F_2nd"]) < 1e-14 and response_err(a["Xi"], b["Xi"]) < 1e-12


def test_device_farm_vs_couple_route(solver, designs, monkeypatch):
    """Two FOWTs with potSecOrder 1 coupled by a mooring stiffness: SlenderSession.farm_response against Model._couple on
    the host flow's outputs (the route Model takes for potSecOrder 1 arrays)."""
    from raft_b200.model import Model
    monkeypatch.setenv("RAFTK_QTF_DIAG", "1")
    packs = designs[:2]
    ct = solver.CaseTable(_cases(11, 5))
    want = ("Xi", "status", "B_drag", "F_drag", "F_iner", "F_BEM", "zeta")
    o = solver.solve_dynamics_slender(packs, ct, n_iter=10, want=want)
    n, n_w = 12, len(packs[0]["w"])
    Ca = np.zeros([n, n])
    k = np.diag([8e4, 8e4, 0, 0, 0, 5e7])
    Ca[:6, :6] += k; Ca[6:, 6:] += k; Ca[:6, 6:] -= k; Ca[6:, :6] -= k

    class _F:
        def __init__(self, P):
            self.P = P

        def pack(self):
            return self.P

    class _M:
        nDOF, nw, w, C_array = n, n_w, packs[0]["w"], Ca
        fowtList = [_F(P) for P in packs]
    ref = Model._couple(_M(), o, ct.n_cases)
    s, out = _session(solver, packs, ct, want=want + ("F_2nd",), n_iter=10)
    xi, info = s.farm_response(C_arr=Ca)
    assert not info.cpu().numpy().any()
    assert response_err(xi.cpu().numpy(), ref) < 1e-10


def test_sweep_on_one_rank(solver, designs):
    """solve_sweep_slender on one rank against the host flow per design."""
    from raft_b200 import sweep
    cs = _cases(21, 16)
    Xi, st = sweep.solve_sweep_slender(designs, cs, n_iter=10)
    Xi, st = Xi.cpu().numpy(), st.cpu().numpy()
    for d, P in enumerate(designs):
        ref = solver.solve_dynamics_slender(P, solver.CaseTable(cs), n_iter=10)
        assert np.array_equal(st[d], ref["status"][0]) and response_err(Xi[d], ref["Xi"][0]) < 1e-12, d


def test_build_variants_family(solver):
    """Seeded build_variants VolturnUS-S variants with potSecOrder 1, 16 cases: status identical to the host flow, Xi within
    1e-12."""
    from raft_b200 import sweep
    D = json.load(open(os.path.join(GOLDEN, "designs.json")))["test_VolturnUS-S"]
    z, P = _golden("slender_VolturnUS-S")
    base = dict(D, platform=dict(D["platform"], potSecOrder=1), site=dict(D["site"], water_depth=float(P["depth"])))
    mats = dict(M_struc=P["M0"] - z["A_hydro_morison"], C_struc=P["C0"] - z["C_moor"], C_moor=z["C_moor"])
    packed = sweep.build_variants(base, mats, sweep.sample_factors(4, seed=3), len(P["w"]), float(P["w"][-1]) / (2 * np.pi), float(P["depth"]))
    assert all("qs_w" in Q for Q in packed)
    ct = solver.CaseTable(_cases(5, 16))
    ref = solver.solve_dynamics_slender(packed, ct, n_iter=4)
    _, out = _session(solver, packed, ct, want=("Xi", "status"), n_iter=4)
    assert np.array_equal(out["status"], ref["status"]) and response_err(out["Xi"], ref["Xi"]) < 1e-12


def test_rejected_inputs(solver, designs):
    """The host flow's rejections, with its exception types: several wave trains, different second-order grids, n_iter < 1."""
    cs = _cases(1, 4)
    tr = solver.CaseTable(dict(cs, primary=np.array([0, 0, 2, 2], dtype=np.int32)))
    for fn in (lambda p, c: solver.solve_dynamics_slender(p, c), lambda p, c: solver.SlenderSession(p, c)):
        with pytest.raises(NotImplementedError):
            fn(designs[:1], tr)
        with pytest.raises(ValueError):
            fn([designs[0], dict(designs[1], qs_w=designs[1]["qs_w"] * 1.01)], solver.CaseTable(cs))
    with pytest.raises(ValueError):
        solver.solve_dynamics_slender(designs[:1], solver.CaseTable(cs), n_iter=0)
    with pytest.raises(ValueError):
        solver.SlenderSession(designs[:1], solver.CaseTable(cs)).solve(n_iter=0)
    with pytest.raises(ValueError):
        solver.slender_flow_host(designs[:1], solver.CaseTable(cs), n_iter=0)


def test_no_device_to_host_copy_inside_solve(solver, designs):
    """torch.profiler records no device-to-host copy (and no host-to-device one) while SlenderSession.solve() runs."""
    import tempfile
    import torch
    from torch.profiler import ProfilerActivity, profile
    s = solver.SlenderSession(designs, solver.CaseTable(_cases(2, 16)), want=OUTS, qtf_chunk=7)
    s.solve(n_iter=4)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        s.solve(n_iter=4)
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        ev = json.load(open(path))["traceEvents"]
    copies = [e["name"] for e in ev if e.get("cat") == "gpu_memcpy"]
    kernels = [e["name"] for e in ev if e.get("cat") == "kernel"]
    assert not copies, copies
    assert any("k_slender_merge" in k for k in kernels) and any("k_slender_rao" in k for k in kernels)
