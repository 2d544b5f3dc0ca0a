"""Every generalised-DOF solve entry, *_host and *_dev, one-shot, streamed and batched, given the same faulty inputs: each
refuses with RAFTK_EINVAL and its family's message, before any launch.  The count faults need no table contents, so the
*_dev entries refuse them without a device; the table faults are read back from device memory on the GPU."""
import ctypes as C

import numpy as np
import pytest

ONE = "general solve: 0 < n_dof <= 256, nw > 0, 0 < n_cases <= 65535"
MANY = "general solve: 0 < n_dof <= 256, nw > 0, n_cases > 0"
F2 = "general solve: F_2nd / Xi_init are not supported"
IDX = "general solve: fd.fd_idx must be strictly increasing (no repeats)"
QW = "general solve: qtf.qtf_w must be strictly increasing"
# fault -> message per entry family (one-shot, stream, batch); None: the family takes no such argument or table
FAULTS = [("n_dof", (ONE, MANY, MANY)),
          ("F_2nd", (F2, F2, F2)),
          ("max_chunk", (None, "general stream: max_chunk_cases must be >= 0 (0: all cases)",
                         "general batch: max_chunk_units must be >= 0 (0: all units)")),
          ("n_dof+fd_idx", (ONE, MANY, MANY)),                # the counts are checked before any table
          ("fd_idx", (IDX, IDX, IDX)),
          ("qtf_w", (QW, QW, QW)),
          ("fd_idx+qtf_w", (IDX, IDX, IDX))]                  # tables in the order fd, qtf
TABLE_FAULTS = ("fd_idx", "qtf_w", "fd_idx+qtf_w")


def _inputs(fault, ptr):
    """Structs of a synthetic 9-DOF design with fd and QTF tables and a two-design batch of it, broken by ``fault``; ``ptr``
    places each array (host or device) and returns its address."""
    import general_synth as gs
    from raft_b200 import solver
    from raft_b200._lib import RaftkSolveOpts
    n, nw, nC = 9, 12, 3
    P, M, B, Cm = gs.design(n, nw, seed=1)
    fd = gs.fd_tables(P, M, B, gs.support(n), seed=1)
    qtf = gs.qtf_table(P, 5, (0.0, 30.0), seed=1)
    faults = fault.split("+")
    if "fd_idx" in faults:
        fd = dict(fd, fd_idx=fd["fd_idx"][::-1].copy())
    if "qtf_w" in faults:
        qtf = dict(qtf, qtf_w=qtf["qtf_w"][::-1].copy())
    ct = solver.CaseTable(dict(Hs=np.ones(nC), Tp=np.full(nC, 8.0), gamma=np.zeros(nC), beta_deg=np.zeros(nC),
                               spec=np.zeros(nC, dtype=np.int32)))
    c = ct.struct(lambda k: ptr("c_" + k, ct.arrays[k]))
    g = solver._general_struct(P, M, B, Cm, lambda k, a: ptr("g_" + k, a))
    f = solver._general_fd_struct(fd, n, nw, lambda k, a: ptr("f_" + k, a))
    q = solver._general_qtf_struct(qtf, lambda k, a: ptr("q_" + k, a))
    bg, bb, bf, bq = solver.GeneralBatch([dict(P=P, M=M, B=B, Cm=Cm, fd=fd)] * 2, qtf=qtf).structs(lambda k, a: ptr("b_" + k, a))
    if "n_dof" in faults:
        g.n_dof = bg.n_dof = 300
    if "F_2nd" in faults:
        c.F_2nd = ptr("c_F_2nd", np.zeros(nC * 6 * nw))
    return g, f, q, bg, bb, bf, bq, c, RaftkSolveOpts(4, 0, 0.01, 0.0, 0, 0)


def _entries(g, f, q, bg, bb, bf, bq, c, o, out, ws, K):
    """(family, call) of the ten solve entries, *_host first; ``out``: the address of every output, ``ws``: the workspace's"""
    from raft_b200._lib import lib
    R = C.byref
    X = S = out
    return [(0, lambda: lib.raftk_general_solve_dynamics_host(R(g), R(c), R(o), X, S)),
            (0, lambda: lib.raftk_general_solve_dynamics_fd_host(R(g), R(f), R(c), R(o), X, S, None)),
            (0, lambda: lib.raftk_general_solve_dynamics_qtf_host(R(g), R(f), R(q), R(c), R(o), X, S, None, None, None)),
            (1, lambda: lib.raftk_general_solve_dynamics_stream_host(R(g), R(f), R(q), R(c), R(o), X, S, None, None, None, K)),
            (2, lambda: lib.raftk_general_batch_solve_dynamics_host(R(bg), R(bb), R(bf), R(bq), R(c), R(o), X, S, None, None, None, K)),
            (0, lambda: lib.raftk_general_solve_dynamics_dev(R(g), R(c), R(o), X, S, ws, 1 << 22, None)),
            (0, lambda: lib.raftk_general_solve_dynamics_fd_dev(R(g), R(f), R(c), R(o), X, S, None, ws, 1 << 22, None)),
            (0, lambda: lib.raftk_general_solve_dynamics_qtf_dev(R(g), R(f), R(q), R(c), R(o), X, S, None, None, None, ws, 1 << 22, None)),
            (1, lambda: lib.raftk_general_solve_dynamics_stream_dev(R(g), R(f), R(q), R(c), R(o), X, S, None, None, None, ws, 1 << 22, K,
                                                                    None)),
            (2, lambda: lib.raftk_general_batch_solve_dynamics_dev(R(bg), R(bb), R(bf), R(bq), R(c), R(o), X, S, None, None, None, ws, 1 << 22,
                                                                   K, None))]


def _check(fault, msgs, ptr, out, ws, which):
    """Every entry of ``which`` (indices into ``_entries``) that sees ``fault`` refuses it with its family's message."""
    from raft_b200._lib import lib
    K = -1 if fault == "max_chunk" else 0
    entries = _entries(*_inputs(fault, ptr), out, ws, K)
    plain = (0, 5)                                     # no fd and no QTF table: the table faults do not reach them
    fd_only = (1, 6)                                   # fd, no QTF table
    ran = 0
    before = lib.raftk_launch_count()
    for i in which:
        fam, call = entries[i]
        if msgs[fam] is None or (fault in TABLE_FAULTS and (i in plain or (fault == "qtf_w" and i in fd_only))):
            continue
        rc = call()
        assert (rc, lib.raftk_last_error().decode()) == (-1, msgs[fam]), (fault, i)
        ran += 1
    assert lib.raftk_launch_count() == before
    return ran


@pytest.mark.parametrize("fault,msgs", FAULTS)
def test_every_entry_refuses_the_same_faults(fault, msgs):
    """Host arrays: every *_host entry, and the *_dev entries for the faults found without reading a table."""
    keep = {}

    def ptr(name, a):
        keep[name] = a
        return a.ctypes.data
    buf = keep.setdefault("buf", np.zeros(1 << 16))
    which = range(5) if fault in TABLE_FAULTS else range(10)
    assert _check(fault, msgs, ptr, buf.ctypes.data, buf.ctypes.data, which) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("fault,msgs", [(f, m) for f, m in FAULTS if f in TABLE_FAULTS])
def test_dev_entries_refuse_bad_tables(fault, msgs):
    """Device arrays: the *_dev entries read the tables back and refuse them as the *_host entries do."""
    import torch
    keep = {}

    def ptr(name, a):
        keep[name] = torch.from_numpy(np.ascontiguousarray(a).view(np.uint8)).cuda()
        return keep[name].data_ptr()
    buf = torch.zeros(1 << 22, dtype=torch.uint8, device="cuda")
    assert _check(fault, msgs, ptr, buf.data_ptr(), buf.data_ptr(), range(5, 10)) > 0
    torch.cuda.synchronize()
