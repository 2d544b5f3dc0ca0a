"""k_rao_fused2's two exchanges between the CTAs of a unit: through distributed shared memory inside a thread-block cluster
(RAFTK_FUSED2_XCHG=cluster) or through the L2-resident workspace in a cooperative launch (RAFTK_FUSED2_XCHG=grid).  Both sum
the ranks' partials in the same order, so every output must be bit-identical, on every route into the solver."""
import ctypes as C

import numpy as np
import pytest

from conftest import load_golden

pytestmark = pytest.mark.gpu

KEYS = ("Xi", "status", "B_drag", "F_drag")


def sea_states(seed, n):
    rng = np.random.default_rng(seed)
    return dict(Hs=rng.uniform(1, 10, n), Tp=rng.uniform(5, 18, n), gamma=np.zeros(n), beta_deg=rng.uniform(-180, 180, n),
                spec=np.zeros(n, dtype=np.int32))


def design(nw):
    from raft_b200 import grid
    _, P = load_golden("cfg2_VolturnUS-S_nw64")
    return grid.regrid(P, nw, 0.512)


def both(monkeypatch, run):
    """run() under each exchange -> (cluster outputs, grid outputs) as host arrays"""
    got = []
    for x in ("cluster", "grid"):
        monkeypatch.setenv("RAFTK_FUSED2_XCHG", x)
        got.append({k: np.array(v) for k, v in run().items()})
    return got


def assert_bit_equal(a, b, keys=KEYS):
    for k in keys:
        assert a[k].shape == b[k].shape and np.array_equal(a[k], b[k]), "%s differs between the cluster and grid exchanges" % k


def test_cfg2_bench_shape(monkeypatch):
    """bench.py's cfg2: 1024 bins x 64 sea states, 4 CTAs per unit"""
    from raft_b200 import solver
    b, c = solver.DesignBatch(design(1024)), solver.CaseTable(sea_states(2, 64))
    cl, gr = both(monkeypatch, lambda: solver.solve_dynamics(b, c, n_iter=10, want=KEYS))
    assert_bit_equal(cl, gr)
    assert np.all(cl["status"][0, :, 2] == 0) and np.all(cl["status"][0, :, 1] == 1)


@pytest.mark.parametrize("nw", [1000, 1001, 777])
def test_partial_last_cta(monkeypatch, nw):
    from raft_b200 import solver
    b, c = solver.DesignBatch(design(nw)), solver.CaseTable(sea_states(31, 7))
    cl, gr = both(monkeypatch, lambda: solver.solve_dynamics(b, c, n_iter=10, want=KEYS))
    assert_bit_equal(cl, gr)


def test_wave_train_table(monkeypatch):
    from raft_b200 import packer, solver
    tr = np.array([[6.0, 12.0, 30.0], [2.5, 7.0, -100.0], [1.0, 16.0, 170.0]])
    case = dict(wave_spectrum=["JONSWAP"] * 3, wave_height=list(tr[:, 0]), wave_period=list(tr[:, 1]), wave_heading=list(tr[:, 2]),
                wave_gamma=[0.0] * 3)
    cases = [dict(wave_spectrum="JONSWAP", wave_height=2.0, wave_period=9.0, wave_heading=10.0), case]
    table, _, _ = packer.pack_case_trains(cases)
    b, c = solver.DesignBatch(design(1024)), solver.CaseTable(table)
    cl, gr = both(monkeypatch, lambda: solver.solve_dynamics(b, c, n_iter=10, want=KEYS))
    assert_bit_equal(cl, gr)
    assert np.array_equal(cl["status"][0, 2:4, 3], [2, 2])


def test_xi_init_continuation(monkeypatch):
    from raft_b200 import solver
    b, cs = solver.DesignBatch(design(1024)), sea_states(23, 5)
    a = solver.solve_dynamics(b, solver.CaseTable(cs), n_iter=1, want=("Xi", "status", "Xi_last"))
    nxt = 0.2 * a["Xi_last"] + 0.8 * a["Xi"]
    c = solver.CaseTable(cs, Xi_init=nxt)
    cl, gr = both(monkeypatch, lambda: solver.solve_dynamics(b, c, n_iter=8, want=KEYS + ("Xi_last",)))
    assert_bit_equal(cl, gr, KEYS + ("Xi_last",))


def test_device_session_reuses_its_plan(monkeypatch):
    """the second solve of a session skips k_fused_plan (RAFTK_SOLVE_REUSE_PLAN); the exchange counters are reset per launch"""
    import torch
    from raft_b200 import solver
    b, c = solver.DesignBatch(design(1024)), solver.CaseTable(sea_states(2, 64))

    def run():
        sess = solver.DeviceSession(b, c, want=KEYS)
        first = {k: v.cpu().numpy() for k, v in sess.solve(n_iter=10).items()}
        for v in sess.out.values():
            v.zero_()
        second = {k: v.cpu().numpy() for k, v in sess.solve(n_iter=10).items()}
        torch.cuda.synchronize()
        assert_bit_equal(first, second)
        return second

    cl, gr = both(monkeypatch, run)
    assert_bit_equal(cl, gr)


def test_two_emulated_ranks(monkeypatch):
    """the fused multi-GPU exchange of tests/test_exchange.py (two ranks on two streams of one GPU) at 4 CTAs per unit"""
    import torch
    from raft_b200 import solver, sweep
    from raft_b200._lib import RaftkPeers, check, lib
    Q = design(1024)
    world, nC, nw = 2, 6, 1024
    cs_all = sea_states(5, world * nC)
    monkeypatch.setenv("RAFTK_FUSED2_XCHG", "cluster")
    ref = solver.solve_dynamics(solver.DesignBatch(Q), solver.CaseTable(cs_all), n_iter=10)
    dev = torch.device("cuda", 0)
    block = nC * 6 * nw
    xi_bytes = world * block * 16
    off_flags = (xi_bytes + 255) // 256 * 256
    off_status = off_flags + 256
    total = off_status + world * nC * 16
    ptrs = []
    for _ in range(world):
        p, h = C.c_void_p(), C.create_string_buffer(64)
        check(lib.raftk_peer_alloc(total, C.byref(p), h))
        ptrs.append(p.value)
    try:
        streams = [torch.cuda.Stream(device=dev) for _ in range(world)]
        timeout = torch.zeros(1, dtype=torch.int32, device=dev)
        views, sessions = [], []
        for r in range(world):
            raw = torch.as_tensor(sweep._DevMem(ptrs[r], total), device=dev)
            g = torch.view_as_complex(raw[:xi_bytes].view(torch.float64).view(-1, 2)).view(world, 1, nC, 6, nw)
            s = raw[off_status:off_status + world * nC * 16].view(torch.int32).view(world, 1, nC, 4)
            views.append((g, s))
            cs = {k: v[r * nC:(r + 1) * nC] for k, v in cs_all.items()}
            sessions.append(solver.DeviceSession(solver.DesignBatch(Q), solver.CaseTable(cs), device=dev,
                                                 out_tensors=dict(Xi=g[r], status=s[r])))
        for epoch, x in ((1, "grid"), (2, "cluster"), (3, "grid")):
            monkeypatch.setenv("RAFTK_FUSED2_XCHG", x)
            for r in range(world):
                pr = RaftkPeers()
                pr.n_ranks, pr.rank, pr.epoch, pr.block_elems = world, r, epoch, block
                for q in range(world):
                    pr.gathered[q], pr.flags[q], pr.status[q] = ptrs[q], ptrs[q] + off_flags, ptrs[q] + off_status
                with torch.cuda.stream(streams[r]):
                    sessions[r].solve_gather(pr, n_iter=10, timeout_flag=timeout.data_ptr())
            torch.cuda.synchronize()
            assert timeout.item() == 0
            for r in range(world):
                g, s = views[r]
                assert np.array_equal(g.cpu().numpy().reshape(world * nC, 6, nw), ref["Xi"][0]), "%s exchange: copy of rank %d" % (x, r)
                assert np.array_equal(s.cpu().numpy().reshape(world * nC, 4), ref["status"][0])
            for g, s in views:
                g.zero_(); s.zero_()
            torch.cuda.synchronize()
        del views, sessions
    finally:
        for p in ptrs:
            check(lib.raftk_peer_free(p))


def test_grid_override_needs_a_resident_launch(monkeypatch):
    """RAFTK_FUSED2_XCHG=grid on a batch whose CTAs cannot all be resident is an error, not a hang or a silent switch"""
    from raft_b200 import solver
    from raft_b200._lib import RaftkError
    b, c = solver.DesignBatch(design(1024)), solver.CaseTable(sea_states(3, 600))
    monkeypatch.setenv("RAFTK_FUSED2_XCHG", "grid")
    with pytest.raises(RaftkError, match="resident"):
        solver.solve_dynamics(b, c, n_iter=10)
    monkeypatch.setenv("RAFTK_FUSED2_XCHG", "bogus")
    with pytest.raises(RaftkError, match="RAFTK_FUSED2_XCHG"):
        solver.solve_dynamics(b, c, n_iter=10)
