"""The streamed generalised-DOF solve and its shard exchange without a GPU: the new entry points' C declarations against the
ctypes bindings, the workspace query, the chunk and shard planners on primary maps, and every refusal of the streamed entry
points before anything is launched (raftk_general_solve_dynamics_stream_*, raftk_general_publish_dev; include/raftk.h)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import GOLDEN, ROOT

HEADER = os.path.join(ROOT, "include", "raftk.h")
NEW = ("raftk_general_stream_workspace_bytes", "raftk_general_solve_dynamics_stream_dev", "raftk_general_solve_dynamics_stream_host",
       "raftk_general_publish_dev")


def _prototype(name):
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    m = re.search(r"\b(\w+\s*\*?)\s*\b%s\s*\(([^)]*)\)\s*;" % name, src)
    assert m, name
    return m.group(1).strip(), [a.strip() for a in m.group(2).split(",")]


def _ctype_of(decl):
    """ctypes type the binding must use for one C parameter declaration."""
    from raft_b200 import _lib
    if "*" in decl:
        for struct, ct in (("raftk_general_fd", "RaftkGeneralFd"), ("raftk_general_qtf", "RaftkGeneralQtf"), ("raftk_general ", "RaftkGeneral"),
                           ("raftk_cases", "RaftkCases"), ("raftk_solve_opts", "RaftkSolveOpts"), ("raftk_peers", "RaftkPeers")):
            if struct in decl:
                return C.POINTER(getattr(_lib, ct))
        return C.c_void_p
    return {"int32_t": C.c_int32, "size_t": C.c_size_t}[decl.split()[0]]


@pytest.mark.parametrize("name", NEW)
def test_bindings_match_header_prototypes(name):
    from raft_b200 import _lib
    ret, params = _prototype(name)
    fn = getattr(_lib.lib, name)
    assert name in _lib.SYMBOLS
    assert len(fn.argtypes) == len(params), (name, params)
    for decl, ct in zip(params, fn.argtypes):
        assert ct is _ctype_of(decl), (name, decl, ct)
    assert fn.restype is (C.c_size_t if ret == "size_t" else C.c_int)


def _flexout():
    z = np.load(os.path.join(GOLDEN, "flexout_VolturnUS-S-flexible.npz"))
    return {k[2:]: z[k] for k in z.files if k.startswith("P_")}


def _flexfd():
    from test_general_fd_oracle import load_flexfd
    P, _, _, _, fd, _ = load_flexfd()
    return P, fd


def _qtf(nw2=12):
    w = np.linspace(0.2, 1.2, nw2)
    return dict(qtf=np.zeros([nw2, nw2, 1, 6], dtype=complex), qtf_w=w, qtf_heads=np.zeros(1))


@pytest.mark.parametrize("tables", ["plain", "fd", "fd+qtf"])
def test_stream_workspace_query(tables):
    """At max_chunk_cases >= n_cases (and 0) the query is the single-table one; below, it is the single-table query of one chunk
    plus the rebased primary map, so it grows linearly in the chunk (up to the 256-byte rounding of each region)."""
    from raft_b200 import solver
    from raft_b200._lib import lib
    if tables == "plain":
        P, fd, q = _flexout(), None, None
    else:
        P, fd = _flexfd()
        q = _qtf() if tables == "fd+qtf" else None
    g = solver._general_struct(P, np.eye(int(P["gen_nDOF"])), np.eye(int(P["gen_nDOF"])), np.eye(int(P["gen_nDOF"])), lambda n, a: None)
    nofn = lambda n, a: None          # noqa: E731
    f, qq = solver._general_fd_struct(fd, int(P["gen_nDOF"]), len(P["w"]), nofn), solver._general_qtf_struct(q, nofn)
    fp, qp = (C.byref(f) if f is not None else None), (C.byref(qq) if qq is not None else None)
    single = lambda n: int(lib.raftk_general_qtf_workspace_bytes(C.byref(g), fp, qp, n))      # noqa: E731
    for nC in (1, 7, 256):
        for K in (0, nC, nC + 5):
            assert solver.general_stream_workspace_bytes(P, fd, q, nC, K) == single(nC)
    nC = 256
    got = [solver.general_stream_workspace_bytes(P, fd, q, nC, K) for K in range(1, nC)]
    assert got == [single(K) + (K * 4 + 255) // 256 * 256 for K in range(1, nC)]
    slope = (got[-1] - got[0]) / (len(got) - 1)
    for K in range(1, nC):                             # a line through both ends, up to the rounding of 16 regions
        assert abs(got[K - 1] - got[0] - (K - 1) * slope) <= 16 * 256, K
    assert all(b > a for a, b in zip(got, got[1:]))
    assert solver.general_stream_workspace_bytes(P, fd, q, nC, 128) * 2 > solver.general_stream_workspace_bytes(P, fd, q, nC, 255)


def test_chunk_for_budget():
    from raft_b200 import solver
    P = _flexout()
    nC = 300
    full = solver.general_stream_workspace_bytes(P, None, None, nC, 0)
    assert solver.general_chunk_for_budget(P, None, None, nC, full) == nC
    for budget in (full - 1, full // 3, 64 << 20, solver.general_stream_workspace_bytes(P, None, None, nC, 1)):
        K = solver.general_chunk_for_budget(P, None, None, nC, budget)
        assert 1 <= K < nC
        assert solver.general_stream_workspace_bytes(P, None, None, nC, K) <= budget
        assert K + 1 == nC or solver.general_stream_workspace_bytes(P, None, None, nC, K + 1) > budget
    with pytest.raises(ValueError):
        solver.general_chunk_for_budget(P, None, None, nC, 1000)


def _prim(sizes):
    """Primary map of consecutive train groups of the given sizes (primary first, as packer.pack_case_trains lays them out)."""
    out, c = [], 0
    for s in sizes:
        out += [c] * s
        c += s
    return np.array(out, dtype=np.int32)


@pytest.mark.parametrize("sizes,K,want", [
    ((1,) * 7, 3, [0, 3, 6, 7]),                       # single trains
    ((1,) * 7, 0, [0, 7]),
    ((1,) * 7, 7, [0, 7]),
    ((1,) * 7, 1, list(range(8))),
    ((1, 3, 1, 2), 3, [0, 1, 4, 7]),                   # mixed sizes: a group never straddles a chunk
    ((1, 3, 1, 2), 4, [0, 4, 7]),                      # groups ending exactly on a chunk boundary
    ((2, 2, 2), 2, [0, 2, 4, 6]),
    ((2, 2, 2), 5, [0, 4, 6]),
    ((3, 1, 1, 1, 3), 3, [0, 3, 6, 9]),
    ((1, 1, 4), 4, [0, 2, 6]),
])
def test_chunk_plan(sizes, K, want):
    from raft_b200 import solver
    pr = _prim(sizes)
    assert solver.general_chunk_plan(pr, len(pr), K) == want
    if all(s == 1 for s in sizes):
        assert solver.general_chunk_plan(None, len(pr), K) == want


def test_chunk_plan_refusals():
    from raft_b200 import solver
    with pytest.raises(ValueError, match="more than max_chunk_cases"):
        solver.general_chunk_plan(_prim((1, 3, 1)), 5, 2)
    with pytest.raises(ValueError, match="interleave"):
        solver.general_chunk_plan(np.array([0, 1, 0, 1], dtype=np.int32), 4, 2)


@pytest.mark.parametrize("sizes,world,want", [
    ((1,) * 8, 2, [(0, 4), (4, 8)]),
    ((1,) * 9, 4, [(0, 2), (2, 5), (5, 7), (7, 9)]),   # cut at 4.5: the later start
    ((1, 2, 1, 2, 2, 1), 2, [(0, 4), (4, 9)]),         # ragged groups: uneven shards of whole groups
    ((4, 1), 2, [(0, 4), (4, 5)]),
    ((5,), 2, [(0, 5), (5, 5)]),                       # one group: the second rank gets nothing
    ((1, 1, 1), 1, [(0, 3)]),
])
def test_general_shards(sizes, world, want):
    from raft_b200 import sweep
    pr = _prim(sizes)
    got = sweep.general_shards(pr, len(pr), world)
    assert got == want
    starts = set(sweep.general_groups(pr, len(pr)).tolist())
    assert all(lo in starts and hi in starts for lo, hi in got)


def test_shard_case_table_rebases_primaries():
    from raft_b200 import solver, sweep
    pr = _prim((1, 2, 1, 2))
    n = len(pr)
    ct = solver.CaseTable(dict(Hs=np.arange(n) + 1.0, Tp=np.full(n, 9.0), gamma=np.zeros(n), beta_deg=np.zeros(n),
                               spec=np.zeros(n, dtype=np.int32), primary=pr))
    sub = sweep.shard_case_table(ct, 3, 6)
    assert sub.n_cases == 3 and sub.arrays["primary"].tolist() == [0, 1, 1] and sub.arrays["Hs"].tolist() == [4.0, 5.0, 6.0]


def _host_call(P, primary, K, n=None):
    """raftk_general_solve_dynamics_stream_host on a flexout case table with the given primary map -> (rc, error, launches)."""
    from raft_b200 import solver
    from raft_b200._lib import RaftkSolveOpts, lib
    nC = len(primary)
    ct = solver.CaseTable(dict(Hs=np.full(nC, 2.0), Tp=np.full(nC, 9.0), gamma=np.zeros(nC), beta_deg=np.zeros(nC),
                               spec=np.zeros(nC, dtype=np.int32), primary=primary))
    nd = int(P["gen_nDOF"])
    keep = {}

    def ptr(name, a):
        keep[name] = a
        return a.ctypes.data
    g = solver._general_struct(P, np.eye(nd), np.eye(nd), np.eye(nd), ptr)
    c = ct.struct(lambda name: ct.arrays[name].ctypes.data)
    o = RaftkSolveOpts(10, 0, 0.01, 0.0, 0, 0)
    Xi = np.zeros([nC, nd, len(P["w"])], dtype=complex)
    st = np.zeros([nC, 4], dtype=np.int32)
    before = lib.raftk_launch_count()
    rc = lib.raftk_general_solve_dynamics_stream_host(C.byref(g), None, None, C.byref(c), C.byref(o), Xi.ctypes.data, st.ctypes.data,
                                                      None, None, None, K)
    return rc, lib.raftk_last_error().decode(), lib.raftk_launch_count() - before


def test_host_entry_refuses_before_launching():
    P = _flexout()
    rc, err, nl = _host_call(P, np.array([0, 1, 0, 1], dtype=np.int32), 2)
    assert rc == -1 and "interleave" in err and nl == 0
    rc, err, nl = _host_call(P, _prim((1, 3, 1)), 2)
    assert rc == -1 and "more cases than max_chunk_cases" in err and nl == 0
    rc, err, nl = _host_call(P, _prim((1, 1)), -1)
    assert rc == -1 and "max_chunk_cases" in err and nl == 0


def test_device_entry_refuses_a_small_workspace():
    """No primary map and no fd / qtf tables: the device entry reads nothing back, so it refuses without touching a device."""
    from raft_b200 import solver
    from raft_b200._lib import RaftkCases, RaftkSolveOpts, lib
    P = _flexout()
    g = solver._general_struct(P, np.eye(int(P["gen_nDOF"])), np.eye(int(P["gen_nDOF"])), np.eye(int(P["gen_nDOF"])), lambda n, a: 0x1000)
    c = RaftkCases()
    c.n_cases = 40
    o = RaftkSolveOpts(10, 0, 0.01, 0.0, 0, 0)
    need = solver.general_stream_workspace_bytes(P, None, None, 40, 8)
    before = lib.raftk_launch_count()
    for wb in (need - 1, 0):
        rc = lib.raftk_general_solve_dynamics_stream_dev(C.byref(g), None, None, C.byref(c), C.byref(o), 0x1000, 0x1000, None, None, None,
                                                         0x1000, wb, 8, None)
        assert rc == -1 and b"workspace smaller" in lib.raftk_last_error()
    c.n_cases = 70000                                  # more than one launch grid takes, in one chunk
    rc = lib.raftk_general_solve_dynamics_stream_dev(C.byref(g), None, None, C.byref(c), C.byref(o), 0x1000, 0x1000, None, None, None,
                                                     0x1000, 1 << 40, 0, None)
    assert rc == -1 and b"65535" in lib.raftk_last_error()
    assert lib.raftk_launch_count() == before


def test_publish_refusals():
    from raft_b200._lib import RaftkPeers, lib
    pr = RaftkPeers()
    pr.n_ranks, pr.rank, pr.epoch, pr.block_elems = 2, 0, 1, 4 * 3 * 5
    for r in range(2):
        pr.gathered[r], pr.flags[r] = 0x1000, 0x2000
    before = lib.raftk_launch_count()
    assert lib.raftk_general_publish_dev(C.byref(pr), 0x3000, None, 5, 4, 3, 5, 0, None) == -1          # rows 5..9 of 8
    assert b"past the gathered array" in lib.raftk_last_error()
    assert lib.raftk_general_publish_dev(C.byref(pr), 0x3000, 0x4000, 0, 4, 3, 5, 0, None) == -1        # no status copies
    assert lib.raftk_general_publish_dev(C.byref(pr), None, None, 0, 4, 3, 5, 0, None) == -1
    assert lib.raftk_general_publish_dev(C.byref(pr), 0x3000, None, 0, 0, 3, 5, 0, None) == 0            # nothing to store
    pr.n_ranks = 0
    assert lib.raftk_general_publish_dev(C.byref(pr), 0x3000, None, 0, 1, 3, 5, 0, None) == -1
    assert lib.raftk_launch_count() == before
