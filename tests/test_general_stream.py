"""The generalised-DOF solve streamed through a bounded workspace (raftk_general_solve_dynamics_stream_*) and sharded over
ranks (raftk_general_publish_dev, sweep.ShardedGeneralSolve), on the GPU.

* Chunks of 1, 2, 3 and all cases give the single-table entry's Xi, status, F_BEM, F_2nd and F_2nd_mean bit for bit on the
  flexout, flexfd and flexqtf fixtures (the QTF fixture with RAFTK_QTF_DIAG=1: k_qtf_tiles sums with atomics; without it,
  to 1e-12), through the host entry and GeneralSession.  Tables with a two-train case do not run at chunk 1 (refused: the
  group does not fit), so chunk 1 runs the single-train rows.
* A synthetic table whose single-table workspace exceeds a 32 MB budget runs within it, a sample of its cases within 1e-10 of
  tests/general_trains_checker.py.
* Two emulated ranks on two streams of one GPU, as tests/test_exchange.py: every rank's gathered Xi and status equal the
  single-GPU streamed result bit for bit, with ragged train groups that split the table 4 / 5."""
import ctypes as C
import os

import numpy as np
import pytest

import general_synth as gs
import general_trains_checker as gtc
from conftest import GOLDEN, relerr
from test_general_fd_oracle import load_flexfd
from test_general_qtf_oracle import load_flexqtf

pytestmark = [pytest.mark.gpu]


def _case_dicts(z, order=None):
    cases = []
    for ic in range(int(z["n_cases"]) if "n_cases" in z else 3):
        tr = z["ref_run_case%d_trains" % ic]
        cases.append(dict(wave_spectrum=["JONSWAP"] * len(tr), wave_height=list(tr[:, 0]), wave_period=list(tr[:, 1]),
                          wave_heading=list(tr[:, 2]), wave_gamma=[0.0] * len(tr)))
    return cases if order is None else [cases[i] for i in order]


def _flexout():
    z = np.load(os.path.join(GOLDEN, "flexout_VolturnUS-S-flexible.npz"))
    G = {k: z[k] for k in z.files}
    P = {k[2:]: v for k, v in G.items() if k.startswith("P_")}
    return P, G["gen_M"], G["gen_B"], G["gen_C"], None, None, G


def _inputs(name, tmp_path):
    if name == "flexout":
        return _flexout()
    if name == "flexfd":
        P, M, B, Cm, fd, z = load_flexfd()
        return P, M, B, Cm, fd, None, z
    P, M, B, Cm, fd, qtf, z = load_flexqtf(tmp_path)
    return P, M, B, Cm, fd, qtf, z


def _table(z, order):
    from raft_b200 import packer, solver
    table, _, _ = packer.pack_case_trains(_case_dicts(z, order))
    return solver.CaseTable(table)


def _groups(ct):
    pr = ct.arrays.get("primary")
    return 1 if pr is None else max(np.bincount(pr))


@pytest.mark.parametrize("name", ["flexout", "flexfd", "flexqtf"])
def test_streamed_equals_single_table(name, monkeypatch, tmp_path):
    from raft_b200 import solver
    monkeypatch.setenv("RAFTK_QTF_DIAG", "1")
    P, M, B, Cm, fd, qtf, z = _inputs(name, tmp_path)
    n_iter, xs = int(z["n_iter"]), float(z["xi_start"])
    nc = int(z["n_cases"]) if "n_cases" in z else 3
    kw = dict(n_iter=n_iter, xi_start=xs, fd=fd, F_BEM=fd is not None, qtf=qtf, F_2nd=qtf is not None)
    mixed = list(range(nc)) + list(range(nc))[::-1]    # every case twice: groups on both sides of the chunk boundaries
    singles = [i for i in range(nc) if len(z["ref_run_case%d_trains" % i]) == 1]
    for order in [o for o in (mixed, singles) if o]:
        ct = _table(z, order)
        ref = solver.general_solve_dynamics(P, M, B, Cm, ct, **kw)
        big = _groups(ct)
        for K in (1, 2, 3, 0):
            if K and K < big:
                with pytest.raises(solver._lib.RaftkError, match="more cases than max_chunk_cases"):
                    solver.general_solve_dynamics(P, M, B, Cm, ct, max_chunk_cases=K, **kw)
                continue
            plan = solver.general_chunk_plan(ct.arrays.get("primary"), ct.n_cases, K)
            got = solver.general_solve_dynamics(P, M, B, Cm, ct, max_chunk_cases=K, **kw)
            assert solver.last_dispatch()["chunks"] == len(plan) - 1
            for a, b in zip(got, ref):
                assert np.array_equal(a, b), (name, order, K)
            sess = solver.GeneralSession(P, M, B, Cm, ct, fd=fd, F_BEM=fd is not None, qtf=qtf, max_chunk_cases=K)
            out = sess.solve(n_iter=n_iter, xi_start=xs)
            dev = [t.cpu().numpy() for t in out] + ([sess.F_2nd.cpu().numpy(), sess.F_2nd_mean.cpu().numpy()] if qtf else [])
            for a, b in zip(dev, ref):
                assert np.array_equal(a, b), (name, order, K, "session")


def test_streamed_qtf_tiles_within_1e12(monkeypatch, tmp_path):
    from raft_b200 import solver
    monkeypatch.delenv("RAFTK_QTF_DIAG", raising=False)
    P, M, B, Cm, fd, qtf, z = _inputs("flexqtf", tmp_path)
    ct = _table(z, None)
    kw = dict(n_iter=int(z["n_iter"]), xi_start=float(z["xi_start"]), fd=fd, qtf=qtf, F_2nd=True)
    ref = solver.general_solve_dynamics(P, M, B, Cm, ct, **kw)
    got = solver.general_solve_dynamics(P, M, B, Cm, ct, max_chunk_cases=2, **kw)
    assert np.array_equal(got[1], ref[1])
    for a, b in zip((got[0], got[2], got[3]), (ref[0], ref[2], ref[3])):
        assert relerr(a, b) < 1e-12


def test_table_beyond_the_budget(oracle):
    """A synthetic 17-DOF design on 129 bins, 160 cases (280 trains): the single-table workspace is several times the budget."""
    import torch
    from raft_b200 import solver
    P, M, B, Cm = gs.design(17, 129)
    table, owner, first, trains = gs.cases((1, 3, 1, 2) * 40, seed=11)
    ct = solver.CaseTable(table)
    budget = 32 << 20
    single = solver.general_stream_workspace_bytes(P, None, None, ct.n_cases, 0)
    assert single > 4 * budget
    K = solver.general_chunk_for_budget(P, None, None, ct.n_cases, budget)
    sess = solver.GeneralSession(P, M, B, Cm, ct, max_chunk_cases=K)
    assert sess.workspace_bytes <= budget and 3 <= K < ct.n_cases
    Xi, st = sess.solve(n_iter=10)
    torch.cuda.synchronize()
    Xi, st = Xi.cpu().numpy(), st.cpu().numpy()
    assert solver.last_dispatch()["chunks"] == len(solver.general_chunk_plan(table["primary"], ct.n_cases, K)) - 1 > 4
    Xh, sh = solver.general_solve_dynamics(P, M, B, Cm, ct, n_iter=10)
    assert np.array_equal(Xi, Xh) and np.array_equal(st, sh)
    for ic in (0, 1, 57, 90, 159):
        idx = np.nonzero(owner == ic)[0]
        Xo, so, _ = gtc.solve_trains(oracle, P, M, B, Cm, trains[ic], nIter=10)
        assert st[first[ic], 0] == so[0] and st[first[ic], 1] == so[1], (ic, st[first[ic]], so)
        for h, t in enumerate(idx):
            assert relerr(Xi[t], Xo[h]) < 1e-10, (ic, h, relerr(Xi[t], Xo[h]))
            if h:
                assert st[t].tolist() == [0, 1, 0, first[ic] + 1]


def _ragged(z):
    """flexout's cases in the order 0, 2, 1, 2, 2, 0: train groups 1, 2, 1, 2, 2, 1 -> shards (0, 4) and (4, 9) of 2 ranks."""
    return _table(z, [0, 2, 1, 2, 2, 0])


def test_two_emulated_ranks_gather_the_streamed_result():
    import torch
    from raft_b200 import solver, sweep
    from raft_b200._lib import RaftkPeers, check, lib
    P, M, B, Cm, _, _, G = _flexout()
    n_iter, xs = int(G["n_iter"]), float(G["xi_start"])
    ct = _ragged(G)
    world, n, nw = 2, int(P["gen_nDOF"]), len(P["w"])
    ref = solver.GeneralSession(P, M, B, Cm, ct, max_chunk_cases=2)
    rX, rS = (t.cpu().numpy() for t in ref.solve(n_iter=n_iter, xi_start=xs))
    bounds = sweep.general_shards(ct.arrays["primary"], ct.n_cases, world)
    assert bounds == [(0, 4), (4, 9)]
    rows = max(h - l for l, h in bounds)
    dev = torch.device("cuda", 0)
    block = rows * n * nw
    xi_bytes = world * block * 16
    off_flags = (xi_bytes + 255) // 256 * 256
    off_status = off_flags + 256
    total = off_status + world * rows * 16
    ptrs = []
    for _ in range(world):
        p, h = C.c_void_p(), C.create_string_buffer(64)
        check(lib.raftk_peer_alloc(total, C.byref(p), h))
        ptrs.append(p.value)
    streams = [torch.cuda.Stream(device=dev) for _ in range(world)]
    timeout = torch.zeros(1, dtype=torch.int32, device=dev)
    sessions, views = [], []
    for r, (lo, hi) in enumerate(bounds):
        sessions.append(solver.GeneralSession(P, M, B, Cm, sweep.shard_case_table(ct, lo, hi), device=dev, max_chunk_cases=2))
        raw = torch.as_tensor(sweep._DevMem(ptrs[r], total), device=dev)
        views.append((torch.view_as_complex(raw[:xi_bytes].view(torch.float64).view(-1, 2)).view(world * rows, n, nw),
                      raw[off_status:off_status + world * rows * 16].view(torch.int32).view(world * rows, 4)))
    index = torch.cat([torch.arange(h - l) + r * rows for r, (l, h) in enumerate(bounds)]).to(dev)
    torch.cuda.synchronize()
    for epoch in (1, 2):
        for r, (lo, hi) in enumerate(bounds):
            pr = RaftkPeers()
            pr.n_ranks, pr.rank, pr.epoch, pr.block_elems = world, r, epoch, block
            for q in range(world):
                pr.gathered[q], pr.flags[q], pr.status[q] = ptrs[q], ptrs[q] + off_flags, ptrs[q] + off_status
            with torch.cuda.stream(streams[r]):
                s = sessions[r]
                s.solve(n_iter=n_iter, xi_start=xs)
                st = streams[r].cuda_stream
                check(lib.raftk_general_publish_dev(C.byref(pr), s.Xi.data_ptr(), s.status.data_ptr(), r * rows, hi - lo, n, nw, lo, st))
                check(lib.raftk_peer_barrier_dev(C.byref(pr), timeout.data_ptr(), st))
        torch.cuda.synchronize()
        assert timeout.item() == 0
        for r in range(world):
            X, S = views[r]
            assert np.array_equal(X.index_select(0, index).cpu().numpy(), rX), "copy of rank %d differs from the streamed solve" % r
            assert np.array_equal(S.index_select(0, index).cpu().numpy(), rS), r
        for X, S in views:
            X.zero_(); S.zero_()
        torch.cuda.synchronize()
    assert rS[:, 3].tolist() == [0, 0, 2, 0, 0, 5, 0, 7, 0]
    del views, sessions
    for p in ptrs:
        check(lib.raftk_peer_free(p))


@pytest.mark.parametrize("exchange", ["peer", "nccl"])
def test_sharded_general_solve_single_rank(exchange):
    """ShardedGeneralSolve without a process group: the streamed solve, delivered through the exchange path."""
    import torch
    from raft_b200 import solver, sweep
    P, M, B, Cm, _, _, G = _flexout()
    ct = _ragged(G)
    kw = dict(n_iter=int(G["n_iter"]), xi_start=float(G["xi_start"]))
    rX, rS = solver.general_solve_dynamics(P, M, B, Cm, ct, **kw)
    sh = sweep.ShardedGeneralSolve(P, M, B, Cm, ct, max_chunk_cases=3, exchange=exchange)
    for _ in range(2):
        X, S = sh.step(**kw)
        torch.cuda.synchronize()
        assert np.array_equal(X.cpu().numpy(), rX) and np.array_equal(S.cpu().numpy(), rS)
    assert not sh.timed_out()
    sh.close()
