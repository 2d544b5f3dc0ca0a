"""The *_host entry points stage their inputs through one device arena per device (raftk.cu, "host-pointer front ends"):
every one of them against its *_dev twin on the same inputs, bit for bit; a call whose small inputs overflow the pinned
staging block; one arena shared by the solve and the small wrappers; and inputs passed as NULL, or with no elements,
reaching the kernels as NULL."""
import ctypes as C

import numpy as np
import pytest

from conftest import load_golden

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def env():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from raft_b200 import _lib, solver
    return torch, _lib.lib, solver


def _cases(n, seed):
    rng = np.random.default_rng(seed)
    return dict(Hs=rng.uniform(2.0, 8.0, n), Tp=rng.uniform(6.0, 14.0, n), gamma=np.zeros(n), beta_deg=rng.uniform(-90.0, 90.0, n),
                spec=np.zeros(n, dtype=np.int32))


def _same(host, dev, keys):
    for k in keys:
        d = dev[k].cpu().numpy() if hasattr(dev[k], "cpu") else dev[k]
        assert np.array_equal(host[k], d), k


def _to_dev(torch, a):
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.float64) if a.dtype == np.complex128 else a).cuda()


# ---- rigid solve, excitation, linearisation, second-order force, farm ----------------------------------------------------

@pytest.mark.parametrize("name", ["cfg2_VolturnUS-S_nw64", "cfg3_OC4semi-WAMIT_nw128"])
def test_rigid_host_equals_dev(name, env):
    torch, _, solver = env
    G, P = load_golden(name)
    batch, ct, ni = solver.DesignBatch(P), solver.CaseTable(_cases(5, 1)), int(G["n_iter"])
    bem = ("F_BEM",) if batch.n_bem_head else ()
    want = ("Xi", "status", "B_drag", "F_drag", "F_iner", "zeta") + bem
    h = solver.solve_dynamics(batch, ct, n_iter=ni, want=want)
    d = solver.DeviceSession(batch, ct, want=want).solve(n_iter=ni)
    torch.cuda.synchronize()
    _same(h, d, want)
    ex = ("F_iner", "zeta") + bem
    he = solver.hydro_excitation(batch, ct, want=ex)
    S = solver.DeviceSession(batch, ct, want=ex + ("B_drag", "F_drag"), tables=True)
    de = S.excitation()
    torch.cuda.synchronize()
    _same(he, de, ex)
    hl = solver.hydro_linearization(batch, ct, h["Xi"], want=("B_drag", "F_drag"))
    dl = S.linearization(_to_dev(torch, h["Xi"]).view(torch.complex128))
    torch.cuda.synchronize()
    _same(hl, dl, ("B_drag", "F_drag"))


def test_second_order_force_and_qtf_solve_host_equal_dev(env):
    """k_qtf_tiles sums into F_2nd with atomics, so two runs agree to rounding, not bit for bit: F_2nd and the response it
    drives are compared at 1e-13, the pass counts exactly."""
    from conftest import relerr
    torch, _, solver = env
    G, P = load_golden("cfg3q_OC4semi-QTF_nw96")
    batch, ct, ni = solver.DesignBatch(P), solver.CaseTable(_cases(3, 2)), int(G["n_iter"])
    h = solver.second_order_force(batch, ct)
    S = solver.DeviceSession(batch, ct, want=("Xi", "status"))
    d = S.second_order_force()
    torch.cuda.synchronize()
    for k in ("F_2nd", "F_2nd_mean"):
        assert relerr(d[k].cpu().numpy(), h[k]) < 1e-13, k
    want = ("Xi", "status", "F_2nd", "F_2nd_mean")
    hs = solver.solve_dynamics(batch, ct, n_iter=ni, want=want)         # potSecOrder 2: the force is computed first
    ds = S.solve(n_iter=ni)
    torch.cuda.synchronize()
    _same(hs, ds, ("status",))
    for k in ("Xi", "F_2nd", "F_2nd_mean"):
        assert relerr(ds[k].cpu().numpy(), hs[k]) < 1e-13, k


@pytest.mark.parametrize("N", [2, 21])
def test_farm_host_equals_dev(N, env):
    """N = 2 on a shared-memory kernel; N = 21 on the global-memory one, whose workspace the host call stages itself."""
    import bench_extra
    torch, _, solver = env
    packs, C_arr, _ = bench_extra.farm_designs(N, nw=48, max_freq=0.1024)
    batch, ct = solver.DesignBatch(packs), solver.CaseTable(_cases(2, 3))
    want = ("Xi", "status", "B_drag", "F_drag", "F_iner")
    h = solver.solve_dynamics_farm(batch, ct, C_arr=C_arr, n_iter=10, want=want)
    if N > 20:
        assert solver.last_dispatch()["kernel"] == "farm-global"
    S = solver.DeviceSession(batch, ct, want=want)
    d = dict(S.solve(n_iter=10))
    d["Xi_sys"], d["info"] = S.farm_response(C_arr=C_arr)
    torch.cuda.synchronize()
    _same(h, d, want + ("Xi_sys", "info"))


def test_small_inputs_overflowing_the_pinned_block(env):
    """60 VolturnUS-S designs: their node, member and matrix tables (each under 64 KB) add up to more than the 256 KB pinned
    block, so the ones that do not fit are copied one by one."""
    torch, _, solver = env
    G, P = load_golden("cfg2_VolturnUS-S_nw64")
    batch, ct = solver.DesignBatch([P] * 60), solver.CaseTable(_cases(2, 4))
    small = sum((v.nbytes + 255) // 256 * 256 for a in (batch.arrays, ct.arrays) for v in a.values() if v.nbytes <= 64 << 10)
    assert small > 256 << 10, small
    want = ("Xi", "status", "B_drag", "F_iner")
    h = solver.solve_dynamics(batch, ct, n_iter=int(G["n_iter"]), want=want)
    d = solver.DeviceSession(batch, ct, want=want).solve(n_iter=int(G["n_iter"]))
    torch.cuda.synchronize()
    _same(h, d, want)


# ---- generalised DOFs, slender-body QTF, system solve, statistics --------------------------------------------------------

def test_general_host_equals_session(env):
    """The flexfd fixture's cases after the first (wave trains included) with F_BEM, then its channel statistics with and
    without the optional PSD and amplitude outputs."""
    torch, _, solver = env
    from raft_b200 import packer
    from test_general_fd_oracle import load_flexfd
    P, M, B, Cm, fd, z = load_flexfd()
    cases = []
    for ic in range(1, int(z["n_cases"])):
        tr = z["ref_run_case%d_trains" % ic]
        cases.append(dict(wave_spectrum=["JONSWAP"] * len(tr), wave_height=list(tr[:, 0]), wave_period=list(tr[:, 1]),
                          wave_heading=list(tr[:, 2]), wave_gamma=[0.0] * len(tr)))
    table, _, _ = packer.pack_case_trains(cases)
    assert len(table["Hs"]) > len(cases)
    ct, kw = solver.CaseTable(table), dict(n_iter=int(z["n_iter"]), xi_start=float(z["xi_start"]))
    Xh, sh, Fh = solver.general_solve_dynamics(P, M, B, Cm, ct, fd=fd, F_BEM=True, **kw)
    S = solver.GeneralSession(P, M, B, Cm, ct, fd=fd, F_BEM=True)
    Xs, ss, Fs = S.solve(**kw)
    torch.cuda.synchronize()
    _same(dict(Xi=Xh, status=sh, F_BEM=Fh), dict(Xi=Xs, status=ss, F_BEM=Fs), ("Xi", "status", "F_BEM"))
    rng = np.random.default_rng(5)
    R, wpow = rng.normal(size=(4, S.n)), np.array([0, 1, 2, 0], dtype=np.int32)
    for psd, amp in ((True, True), (False, False), (True, False)):
        hs = solver.general_channel_stats(R, wpow, P["w"], Xh, float(P["dw"]), psd=psd, amp=amp)
        ds = S.stats(R, wpow, psd=psd, amp=amp)
        torch.cuda.synchronize()
        for a, b in zip(hs, ds):
            assert (a is None) == (b is None) and (a is None or np.array_equal(a, b.cpu().numpy())), (psd, amp)


def _slender_dev(env, P, beta, Xi):
    torch, lib, solver = env
    keep = {}

    def to_dev(name, a):
        keep[name] = torch.from_numpy(a).cuda()
        return keep[name].data_ptr() if a.size else None
    s = solver._slender_struct(P, to_dev)
    n, nw2 = len(beta), s.nw
    b, X = _to_dev(torch, np.asarray(beta, dtype=float)), _to_dev(torch, Xi)
    q = torch.empty(n * nw2 * nw2 * 12, dtype=torch.float64, device="cuda")
    wb = int(lib.raftk_qtf_slender_workspace_bytes(C.byref(s), n))
    ws = torch.empty(wb, dtype=torch.uint8, device="cuda")
    assert lib.raftk_qtf_slender_dev(C.byref(s), n, b.data_ptr(), X.data_ptr(), q.data_ptr(), ws.data_ptr(), wb, None) == 0
    torch.cuda.synchronize()
    return q.cpu().numpy().view(np.complex128).reshape(n, nw2, nw2, 6)


def _slender_case(P, n, seed):
    rng = np.random.default_rng(seed)
    nw2 = len(P["qs_w"])
    return rng.uniform(-np.pi, np.pi, n), (rng.normal(size=(n, 6, nw2)) + 1j * rng.normal(size=(n, 6, nw2))) * 0.02


def test_slender_host_equals_dev(env):
    _, _, solver = env
    _, P = load_golden("slender_VolturnUS-S")
    beta, Xi = _slender_case(P, 3, 6)
    assert np.array_equal(solver.qtf_slender(P, beta, Xi), _slender_dev(env, P, beta, Xi))


def _dev_call(torch, fn, host_in, out_shapes):
    """fn(*device input pointers, *device output pointers or None) on torch tensors -> host copies of the outputs."""
    ins = [_to_dev(torch, a) for a in host_in]
    outs = [torch.zeros(int(np.prod(s)) * (2 if dt == np.complex128 else 1), dtype=torch.int32 if dt == np.int32 else torch.float64,
                        device="cuda") if s is not None else None for s, dt in out_shapes]
    assert fn(*[t.data_ptr() for t in ins], *[t.data_ptr() if t is not None else None for t in outs]) == 0
    torch.cuda.synchronize()
    return [o.cpu().numpy().view(dt).reshape(s) if o is not None else None for o, (s, dt) in zip(outs, out_shapes)]


@pytest.mark.parametrize("n", [12, 150])
def test_system_solve_host_equals_dev(n, env):
    """n = 12 in shared memory, n = 150 on the global-memory kernel."""
    torch, lib, solver = env
    rng = np.random.default_rng(n)
    nw, nrhs = 5, 2
    Z = rng.normal(size=(nw, n, n)) + 1j * rng.normal(size=(nw, n, n)) + 4 * n * np.eye(n)
    F = rng.normal(size=(nw, n, nrhs)) + 1j * rng.normal(size=(nw, n, nrhs))
    Xh, ih = solver.system_solve(Z, F)
    Zd, Fd = _to_dev(torch, Z), _to_dev(torch, F)
    info = torch.zeros(nw, dtype=torch.int32, device="cuda")
    assert lib.raftk_system_solve_dev(n, nw, nrhs, Zd.data_ptr(), Fd.data_ptr(), info.data_ptr(), None) == 0
    torch.cuda.synchronize()
    if n > 120:
        assert solver.last_dispatch()["kernel"] == "sys-global"
    assert np.array_equal(Xh, Fd.cpu().numpy().view(np.complex128).reshape(nw, n, nrhs)) and np.array_equal(ih, info.cpu().numpy())


@pytest.mark.parametrize("psd,amp", [(True, True), (False, False), (True, False)])
def test_statistics_host_equal_dev(psd, amp, env):
    torch, lib, solver = env
    rng = np.random.default_rng(7)
    nD, nC, nch, nw, dw = 2, 3, 4, 40, 0.05
    Xi = rng.normal(size=(nD, nC, 6, nw)) + 1j * rng.normal(size=(nD, nC, 6, nw))
    sd, P = solver.response_stats(Xi, dw, psd=psd)
    n = nD * nC
    d_sd, d_P = _dev_call(torch, lambda x, s, p: lib.raftk_response_stats_dev(n, nw, dw, 1, x, s, p, None), [Xi],
                          [((nD, nC, 6), np.float64), ((nD, nC, 6, nw) if psd else None, np.float64)])
    assert np.array_equal(sd, d_sd) and (P is None) == (d_P is None) and (P is None or np.array_equal(P, d_P))
    coef = rng.normal(size=(nD, nch, 6, nw)) + 1j * rng.normal(size=(nD, nch, 6, nw))
    host = solver.channel_stats(coef, Xi, dw, psd=psd, amp=amp)
    dev = _dev_call(torch, lambda c, x, s, p, a: lib.raftk_channel_stats_dev(nD, nC, nch, nw, dw, c, x, s, p, a, None), [coef, Xi],
                    [((nD, nC, nch), np.float64), ((nD, nC, nch, nw) if psd else None, np.float64),
                     ((nD, nC, nch, nw) if amp else None, np.complex128)])
    for a, b in zip(host, dev):
        assert (a is None) == (b is None) and (a is None or np.array_equal(a, b))


# ---- one arena ----------------------------------------------------------------------------------------------------------

def test_one_arena_for_every_host_call(env):
    """After a large solve, the small wrappers at sizes above their warm-up run in the arena the solve left: the device's free
    memory does not move.  The warm-up calls use the same kernels, so that lazily loaded modules are already resident."""
    torch, _, solver = env
    from raft_b200 import grid
    from test_general_fd import _rigid_as_general
    _, P2 = load_golden("cfg2_VolturnUS-S_nw64")
    _, Pq = load_golden("cfg3q_OC4semi-QTF_nw96")
    _, Ps = load_golden("slender_VolturnUS-S")
    _, Gg, Mg, Bg, Cg, fdg, _ = _rigid_as_general()
    rng = np.random.default_rng(9)
    b2, bq = solver.DesignBatch(P2), solver.DesignBatch(Pq)
    nw2 = len(Ps["qs_w"])

    def small_calls(k):
        ct = solver.CaseTable(_cases(k, 10))
        solver.hydro_excitation(b2, ct)
        solver.hydro_linearization(b2, ct, np.zeros([1, k, 6, b2.nw], dtype=complex))
        solver.second_order_force(bq, ct)
        solver.general_solve_dynamics(Gg, Mg, Bg, Cg, ct, fd=fdg, F_BEM=True)
        solver.qtf_slender(Ps, np.zeros(k), np.zeros([k, 6, nw2], dtype=complex))
        solver.system_solve(np.tile(np.eye(12, dtype=complex), (64 * k, 1, 1)), np.ones([64 * k, 12], dtype=complex))
        Xi = rng.normal(size=(k, 6, 1024)) + 0j
        solver.response_stats(Xi, 0.01)
        solver.channel_stats(rng.normal(size=(2, 6, 1024)) + 0j, Xi, 0.01, psd=True, amp=True)
        solver.general_channel_stats(np.ones([2, 6]), np.zeros(2, dtype=np.int32), np.linspace(0.01, 1, 1024), Xi, 0.01, amp=True)

    small_calls(1)
    P = grid.regrid(P2, 1024, 0.512)
    solver.solve_dynamics(solver.DesignBatch(P), solver.CaseTable(_cases(256, 11)), want=("Xi", "status", "F_iner", "F_drag"))
    torch.cuda.synchronize()
    free = torch.cuda.mem_get_info()[0]
    small_calls(32)
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info()[0] == free


# ---- NULL inputs --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("what", ["no_strip_nodes", "no_segments"])
def test_slender_empty_tables_vs_oracle(what, env, oracle):
    """Tables with no elements reach the kernels as NULL: a design without strip nodes, and one without Kim & Yue segments."""
    _, _, solver = env
    from test_slender_qtf import BOUND, dof_err, nodeless_tables
    if what == "no_strip_nodes":
        mem = dict(q=[0.35, -0.2, 0.9], mcf=1, wl=1, r_int=[1.0, 0.5, 0.0], a_wl=30.0, rwl=[3.0, -2.0, 0.0], R_wl=4.0,
                   segs=[(-9.0, 0.0, 4.0, [-0.5, 1.0, -4.5])])
        P = nodeless_tables(60.0, np.geomspace(0.01, 1.5, 12), [mem], np.random.default_rng(12))
    else:
        _, P = load_golden("slender_VolturnUS-S")
        P = dict(P, qs_seg_mem=np.zeros(0, dtype=np.int32), qs_seg_z1=np.zeros(0), qs_seg_z2=np.zeros(0), qs_seg_R=np.zeros(0),
                 qs_seg_rmid=np.zeros([0, 3]))
    beta, Xi = _slender_case(P, 2, 13)
    q = solver.qtf_slender(P, beta, Xi)
    assert np.array_equal(q, _slender_dev(env, P, beta, Xi))
    od = oracle.OracleDesign(P)
    for c in range(2):
        assert dof_err(q[c], oracle.qtf_slender(od, beta[c], Xi[c])) < BOUND


def test_general_without_nodes(env):
    """A generalised design with n_nodes = 0 (the cfg3 OC4semi BEM design as six rigid DOFs, its strip nodes removed): host
    and device calls agree bit for bit, and the BEM force is the rigid solver's, which no node enters."""
    torch, _, solver = env
    from conftest import relerr
    from test_general_fd import _rigid_as_general
    P, G, M, B, Cm, fd, z = _rigid_as_general()
    G = dict(G, node_r=np.zeros([0, 3]), node_mem=np.zeros(0, dtype=np.int64), node_Imat=np.zeros([0, 3, 3]), node_a_i=np.zeros(0),
             gen_Tn=np.zeros([0, 6, 6]), gen_rr=np.zeros([0, 3]), node_Imat_w=None,
             **{"node_" + k: np.zeros(0) for k in ("ls", "a_q", "a_p1", "a_p2", "a_End", "Cd_q", "Cd_p1", "Cd_p2", "Cd_End")})
    ct = solver.CaseTable(_cases(3, 14))
    Xh, sh, Fh = solver.general_solve_dynamics(G, M, B, Cm, ct, n_iter=int(z["n_iter"]), fd=fd, F_BEM=True)
    Xs, ss, Fs = solver.GeneralSession(G, M, B, Cm, ct, fd=fd, F_BEM=True).solve(n_iter=int(z["n_iter"]))
    torch.cuda.synchronize()
    _same(dict(Xi=Xh, status=sh, F_BEM=Fh), dict(Xi=Xs, status=ss, F_BEM=Fs), ("Xi", "status", "F_BEM"))
    assert np.all(np.isfinite(Xh)) and np.any(Xh)
    rig = solver.solve_dynamics(solver.DesignBatch(P), ct, n_iter=int(z["n_iter"]), want=("Xi", "status", "F_BEM"))
    assert relerr(Fh, rig["F_BEM"][0]) < 1e-12
