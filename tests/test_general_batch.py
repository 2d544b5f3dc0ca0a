"""Design batches of flexible FOWTs (raftk_general_batch_solve_dynamics_*, solver.GeneralBatch / GeneralBatchSession /
general_solve_dynamics_batch), on the GPU.

* Five synthetic 17-DOF designs on 129 bins with ragged node counts (two truncated, one with no submerged node), each with its
  own rotor and BEM tables (T0, x_ref, heading_adjust per design), over a train table (1, 3, 2): every design's Xi, status and
  F_BEM equal general_solve_dynamics on that design alone bit for bit; again with per-design and with shared QTF tables
  (RAFTK_QTF_DIAG=1), F_2nd and F_2nd_mean included.
* Chunks of one train group, of a size that cuts across designs, and of the whole batch are bit-identical; the launch count of
  a one-chunk call does not depend on the number of designs; more than 65535 units run through chunks.
* The flexout, flexfd and flexqtf fixtures batched with two seeded variants each (scaled M / C, scaled drag coefficients): every
  unit equals the single-design entry bit for bit, the fixture's unit meets the reference run, and every variant its checker,
  at the tolerances of the single-design tests.
* n_designs = 1 is the single-design entry bit for bit on the 150-DOF fixture; per-design channel statistics; refusals of the
  device entry before any launch."""
import numpy as np
import pytest

import general_fd_checker as gfc
import general_qtf_checker as gqc
import general_synth as gs
import general_trains_checker as gtc
from conftest import relerr
from test_general_fd_oracle import load_flexfd
from test_general_qtf_oracle import load_flexqtf
from test_general_stream import _case_dicts, _flexout

pytestmark = [pytest.mark.gpu]

NODE_KEYS = ("gen_Tn", "gen_rr")


def truncate(P, keep):
    """P with only its first ``keep`` strip nodes (every node_* table and the nodes' Tn / rr rows)."""
    Ns = len(P["node_ls"])
    Q = dict(P)
    for k, v in P.items():
        if (k.startswith("node_") or k in NODE_KEYS) and v is not None and np.ndim(v) and np.shape(v)[0] == Ns:
            Q[k] = np.asarray(v)[:keep]
    return Q


def synth(qtf=None):
    """-> (designs, CaseTable): 5 designs, nodes kept: all, half, all, none, a third; their own fd tables with BEM."""
    from raft_b200 import solver
    designs = []
    for s in range(5):
        P, M, B, Cm = gs.design(17, 129, seed=s)
        Ns = len(P["node_ls"])
        P = truncate(P, [Ns, Ns // 2, Ns, 0, Ns // 3][s])
        fd = gs.fd_tables(P, M, B, gs.support(17), seed=s, bem="table", heading_adjust=5.0 * s, x_ref=1.5 * s, y_ref=-0.5 * s)
        q = gs.qtf_table(P, 20, [0.0, 90.0, 200.0], seed=s) if qtf == "own" else None
        designs.append(dict(P=P, M=M, B=B, Cm=Cm, fd=fd, qtf=q))
    table, _, _, _ = gs.cases((1, 3, 2), seed=0)
    return designs, solver.CaseTable(table)


def _single(e, ct, qtf=None, **kw):
    from raft_b200 import solver
    return solver.general_solve_dynamics(e["P"], e["M"], e["B"], e["Cm"], ct, fd=e.get("fd"), qtf=e.get("qtf") or qtf, **kw)


@pytest.mark.parametrize("qtf", [None, "own", "shared"])
def test_batch_equals_per_design_calls(qtf, monkeypatch):
    from raft_b200 import solver
    monkeypatch.setenv("RAFTK_QTF_DIAG", "1")
    designs, ct = synth(qtf)
    shared = gs.qtf_table(designs[0]["P"], 20, [0.0, 90.0, 200.0], seed=9) if qtf == "shared" else None
    bt = solver.GeneralBatch(designs, qtf=shared)
    assert bt.node_counts.tolist()[3] == 0 and len(set(bt.node_counts.tolist())) == 4
    q = qtf is not None
    got = solver.general_solve_dynamics_batch(bt, ct, n_iter=10, F_BEM=True, F_2nd=q)
    sess = solver.GeneralBatchSession(bt, ct, F_BEM=True)
    dev = [t.cpu().numpy() for t in sess.solve(n_iter=10)] + ([sess.F_2nd.cpu().numpy(), sess.F_2nd_mean.cpu().numpy()] if q else [])
    for d, e in enumerate(designs):
        ref = _single(e, ct, n_iter=10, F_BEM=True, F_2nd=q, qtf=shared)
        assert not ref[1][:, 2].any()
        for k, r in enumerate(ref):
            assert np.array_equal(got[k][d], r), (qtf, d, k)
            assert np.array_equal(dev[k][d], r), (qtf, d, k, "session")
    assert (got[1][:, :, 3] == ref[1][:, 3]).all()               # status word 3: the primary's case index + 1 in every design


def test_chunks_and_launch_count():
    from raft_b200 import solver
    designs, ct = synth()
    bt = solver.GeneralBatch(designs)
    nC = ct.n_cases
    ref = solver.general_solve_dynamics_batch(bt, ct, n_iter=10, F_BEM=True)
    for K in (3, 8, 5 * nC):                           # one train group; across design boundaries; the whole batch
        plan = solver.general_batch_chunk_plan(ct.arrays["primary"], nC, 5, K)
        if K == 8:
            assert any(u % nC for u in plan[1:-1]) and any(u // nC != (v - 1) // nC for u, v in zip(plan[:-1], plan[1:]))
        got = solver.general_solve_dynamics_batch(bt, ct, n_iter=10, F_BEM=True, max_chunk_units=K)
        assert solver.last_dispatch()["chunks"] == len(plan) - 1
        for a, b in zip(got, ref):
            assert np.array_equal(a, b), K
        sess = solver.GeneralBatchSession(bt, ct, F_BEM=True, max_chunk_units=K)
        for a, b in zip(sess.solve(n_iter=10), ref):
            assert np.array_equal(a.cpu().numpy(), b), (K, "session")
    counts = []
    for nD in (2, 5):
        solver.general_solve_dynamics_batch(solver.GeneralBatch(designs[:nD]), ct, n_iter=10)
        n0 = solver.launch_count()
        solver.general_solve_dynamics_batch(solver.GeneralBatch(designs[:nD]), ct, n_iter=10)
        counts.append(solver.launch_count() - n0)
    assert counts[0] == counts[1], counts


def test_more_than_65535_units():
    import torch
    from raft_b200 import solver
    designs = []
    for s in range(3):
        P, M, B, Cm = gs.design(7, 16, seed=s)
        designs.append(dict(P=truncate(P, 4 + s), M=M, B=B, Cm=Cm))
    nC = 22000
    rng = np.random.default_rng(5)
    ct = solver.CaseTable(dict(Hs=rng.uniform(2, 6, nC), Tp=rng.uniform(7, 14, nC), gamma=np.zeros(nC), beta_deg=rng.uniform(-90, 90, nC),
                               spec=np.zeros(nC, dtype=np.int32)))
    bt = solver.GeneralBatch(designs)
    sess = solver.GeneralBatchSession(bt, ct, max_chunk_units=30000)
    Xi, st = sess.solve(n_iter=10)
    torch.cuda.synchronize()
    assert solver.last_dispatch()["chunks"] == 3
    Xi, st = Xi.cpu().numpy(), st.cpu().numpy()
    for d, e in enumerate(designs):
        X1, s1 = _single(e, ct, n_iter=10)
        assert np.array_equal(Xi[d], X1) and np.array_equal(st[d], s1), d


def _variants(P, M, B, Cm, fd, seed):
    """Two seeded variants of a fixture design: scaled M / C entries, and scaled drag coefficients."""
    rng = np.random.default_rng(seed)
    M1 = M * (1.0 + 0.01 * rng.uniform(-1, 1, M.shape))
    M1 = 0.5 * (M1 + M1.T)
    C1 = Cm * (1.0 + 0.01 * rng.uniform(-1, 1, Cm.shape))
    C1 = 0.5 * (C1 + C1.T)
    P2 = dict(P)
    for k in ("node_Cd_q", "node_Cd_p1", "node_Cd_p2", "node_Cd_End"):
        P2[k] = np.asarray(P[k]) * rng.uniform(0.9, 1.1, np.shape(P[k]))
    return [dict(P=P, M=M1, B=B, Cm=C1, fd=fd), dict(P=P2, M=M, B=B, Cm=Cm, fd=fd)]


@pytest.mark.parametrize("name", ["flexout", "flexfd", "flexqtf"])
def test_fixture_and_variants_against_the_reference(name, oracle, monkeypatch, tmp_path):
    from raft_b200 import packer, solver
    monkeypatch.setenv("RAFTK_QTF_DIAG", "1")
    if name == "flexout":
        P, M, B, Cm, fd, qtf, z = _flexout()
    elif name == "flexfd":
        (P, M, B, Cm, fd, z), qtf = load_flexfd(), None
    else:
        P, M, B, Cm, fd, qtf, z = load_flexqtf(tmp_path)
    n_iter, xs = int(z["n_iter"]), float(z["xi_start"])
    nc = int(z["n_cases"]) if "n_cases" in z else 3
    table, owner, first = packer.pack_case_trains(_case_dicts(z))
    designs = [dict(P=P, M=M, B=B, Cm=Cm, fd=fd)] + _variants(P, M, B, Cm, fd, seed=len(name))
    bt = solver.GeneralBatch(designs, qtf=qtf)
    res = solver.general_solve_dynamics_batch(bt, solver.CaseTable(table), n_iter=n_iter, xi_start=xs, F_2nd=qtf is not None)
    Xi, st = res[0], res[1]

    def close(X, ref):
        if qtf is None:
            return relerr(X, ref) < 1e-10, relerr(X, ref)
        e_all, e = gqc.xi_errors(X, ref)
        return e_all < gqc.XI_RTOL_ALL and e < gqc.XI_RTOL, (e_all, e)
    for d, e in enumerate(designs):                    # every unit is the single-design entry's, bit for bit
        one = solver.general_solve_dynamics(e["P"], e["M"], e["B"], e["Cm"], solver.CaseTable(table), n_iter=n_iter, xi_start=xs, fd=fd, qtf=qtf)
        assert np.array_equal(Xi[d], one[0]) and np.array_equal(st[d], one[1]), (name, d)
    for ic in range(nc):
        idx = np.nonzero(owner == ic)[0]
        tr = z["ref_run_case%d_trains" % ic]
        assert st[0, first[ic], 0] == int(z["ref_run_case%d_passes" % ic]) and st[0, first[ic], 2] == 0
        for h, t in enumerate(idx):
            ok, err = close(Xi[0, t], z["ref_run_case%d_Xi" % ic][h])
            assert ok, (name, ic, h, err)
        for d, e in enumerate(designs[1:], 1):
            if qtf is not None:
                Xo, so, _, _, _ = gqc.solve_trains_qtf(oracle, e["P"], e["M"], e["B"], e["Cm"], fd, qtf, tr, nIter=n_iter, XiStart=xs)
            elif fd is not None:
                Xo, so, _ = gfc.solve_trains_fd(oracle, e["P"], e["M"], e["B"], e["Cm"], fd, tr, nIter=n_iter, XiStart=xs)
            else:
                Xo, so, _ = gtc.solve_trains(oracle, e["P"], e["M"], e["B"], e["Cm"], tr, nIter=n_iter, XiStart=xs)
            assert st[d, first[ic], 0] == so[0] and st[d, first[ic], 1] == so[1], (name, d, ic, st[d, first[ic]], so)
            for h, t in enumerate(idx):
                ok, err = close(Xi[d, t], Xo[h])
                assert ok, (name, d, ic, h, err)
            assert not np.array_equal(Xi[d, idx], Xi[0, idx])


def test_one_design_is_the_single_entry():
    from raft_b200 import packer, solver
    P, M, B, Cm, _, _, z = _flexout()
    table, _, _ = packer.pack_case_trains(_case_dicts(z))
    ct = solver.CaseTable(table)
    kw = dict(n_iter=int(z["n_iter"]), xi_start=float(z["xi_start"]))
    ref = solver.general_solve_dynamics(P, M, B, Cm, ct, **kw)
    got = solver.general_solve_dynamics_batch([(P, M, B, Cm)], ct, **kw)
    assert np.array_equal(got[0][0], ref[0]) and np.array_equal(got[1][0], ref[1])


def test_channel_stats_per_design():
    from raft_b200 import solver
    designs, ct = synth()
    rng = np.random.default_rng(3)
    nch, n = 5, 17
    R = rng.normal(size=(5, nch, n))
    wpow = np.array([0, 1, 2, 0, 1], dtype=np.int32)
    sess = solver.GeneralBatchSession(designs, ct)
    Xi = sess.solve(n_iter=10)[0]
    sd, P, A = sess.stats(R, wpow, psd=True, amp=True)
    Xi = Xi.cpu().numpy()
    for d in range(5):
        s1, p1, a1 = solver.general_channel_stats(R[d], wpow, designs[d]["P"]["w"], Xi[d], float(designs[d]["P"]["dw"]), psd=True, amp=True)
        assert np.array_equal(sd[d].cpu().numpy(), s1) and np.array_equal(P[d].cpu().numpy(), p1) and np.array_equal(A[d].cpu().numpy(), a1)


def test_analyze_cases_batch_equals_single():
    from raft_b200 import solver
    designs, _ = synth()
    cases = [dict(wave_spectrum="JONSWAP", wave_height=3.0, wave_period=9.0, wave_heading=20.0, wave_gamma=0.0),
             dict(wave_spectrum=["JONSWAP"] * 2, wave_height=[2.0, 1.5], wave_period=[8.0, 12.0], wave_heading=[0.0, 90.0], wave_gamma=[0.0, 0.0])]
    got = solver.general_analyze_cases_batch(designs, cases)
    for d, e in enumerate(designs):
        ref = solver.general_analyze_cases(e["P"], e["M"], e["B"], e["Cm"], cases, fd=e["fd"])
        assert np.array_equal(got[d]["status"], ref["status"])
        assert all(np.array_equal(a, b) for a, b in zip(got[d]["Xi_trains"], ref["Xi_trains"]))


def test_device_entry_refusals():
    """node_offset edited on the device after the session is built; a workspace below the query; a chunk below a train group:
    refused before any launch."""
    from raft_b200 import solver
    designs, ct = synth()
    sess = solver.GeneralBatchSession(designs[:3], ct)
    off = sess.keep["node_offset"]
    good = off.clone()
    for bad, msg in (([1, 5, 9, 12], "start at 0"), ([0, 9, 5, int(good[-1])], "non-decreasing"), ([0, 2, 4, 6], "equal n_nodes")):
        off.copy_(off.new_tensor(bad))
        n0 = solver.launch_count()
        with pytest.raises(solver._lib.RaftkError, match=msg):
            sess.solve()
        assert solver.launch_count() == n0
    off.copy_(good)
    sess.workspace_bytes -= 1
    n0 = solver.launch_count()
    with pytest.raises(solver._lib.RaftkError, match="workspace smaller"):
        sess.solve()
    sess.workspace_bytes += 1
    sess.max_chunk_units = 2
    with pytest.raises(solver._lib.RaftkError, match="more cases than max_chunk_units"):
        sess.solve()
    assert solver.launch_count() == n0
    sess.max_chunk_units = 0
    sess.solve()
