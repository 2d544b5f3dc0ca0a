"""Design batches of flexible FOWTs without a GPU: the batch entry points' C declarations against the ctypes bindings, the
workspace query and the chunk plan on ragged batches, the CSR assembly of solver.GeneralBatch and its mismatch errors, and
the host entry's refusals before anything is launched (raftk_general_batch_*; include/raftk.h)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import ROOT

HEADER = os.path.join(ROOT, "include", "raftk.h")
NEW = ("raftk_general_batch_workspace_bytes", "raftk_general_batch_solve_dynamics_dev", "raftk_general_batch_solve_dynamics_host")


def _prototype(name):
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    m = re.search(r"\b(\w+\s*\*?)\s*\b%s\s*\(([^)]*)\)\s*;" % name, src)
    assert m, name
    return m.group(1).strip(), [a.strip() for a in m.group(2).split(",")]


def _ctype_of(decl):
    from raft_b200 import _lib
    if "*" in decl:
        for struct, ct in (("raftk_general_batch", "RaftkGeneralBatch"), ("raftk_general_fd", "RaftkGeneralFd"),
                           ("raftk_general_qtf", "RaftkGeneralQtf"), ("raftk_general ", "RaftkGeneral"), ("raftk_cases", "RaftkCases"),
                           ("raftk_solve_opts", "RaftkSolveOpts")):
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


def test_batch_struct_layout(tmp_path):
    import subprocess
    from raft_b200 import _lib
    src = tmp_path / "t.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "raftk.h"\nint main(void){printf("%zu %zu %zu %zu\\n", '
                   'sizeof(raftk_general_batch), offsetof(raftk_general_batch, node_offset), offsetof(raftk_general_batch, qtf_shared), '
                   'offsetof(raftk_general_batch, heading_adjust));return 0;}\n')
    exe = tmp_path / "t"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    B = _lib.RaftkGeneralBatch
    assert got == [C.sizeof(B), B.node_offset.offset, B.qtf_shared.offset, B.heading_adjust.offset]


def truncate(P, keep):
    Ns = len(P["node_ls"])
    Q = dict(P)
    for k, v in P.items():
        if (k.startswith("node_") or k in ("gen_Tn", "gen_rr")) and v is not None and np.ndim(v) and np.shape(v)[0] == Ns:
            Q[k] = np.asarray(v)[:keep]
    return Q


def _designs(keep=(None, 0.5, 0.0), fd=True, n=9, nw=33):
    import general_synth as gs
    out = []
    for s, f in enumerate(keep):
        P, M, B, Cm = gs.design(n, nw, seed=s)
        Ns = len(P["node_ls"])
        P = truncate(P, Ns if f is None else int(f * Ns))
        e = dict(P=P, M=M, B=B, Cm=Cm)
        if fd:
            e["fd"] = gs.fd_tables(P, M, B, gs.support(n), seed=s, bem="table", heading_adjust=2.0 * s, x_ref=float(s))
        out.append(e)
    return out


def test_csr_assembly():
    from raft_b200 import solver
    ds = _designs()
    bt = solver.GeneralBatch(ds)
    Ns = [len(e["P"]["node_ls"]) for e in ds]
    assert bt.node_counts.tolist() == Ns and Ns[2] == 0 and bt.max_nodes == max(Ns)
    assert bt.node_offset.tolist() == [0, Ns[0], Ns[0] + Ns[1], sum(Ns)]
    n = bt.n
    for d, e in enumerate(ds):
        got = {}
        solver._general_struct(e["P"], e["M"], e["B"], e["Cm"], lambda name, a: got.__setitem__(name, a))
        lo, hi = bt.node_offset[d], bt.node_offset[d + 1]
        assert np.array_equal(bt.arrays["Tn"].reshape(-1, 6, n)[lo:hi], got["Tn"].reshape(-1, 6, n))
        assert np.array_equal(bt.arrays["node_r"].reshape(-1, 3)[lo:hi], got["node_r"].reshape(-1, 3))
        assert np.array_equal(bt.arrays["node_cd"].reshape(-1, 4)[lo:hi], got["node_cd"].reshape(-1, 4))
        assert np.array_equal(bt.arrays["M"][d], e["M"]) and np.array_equal(bt.arrays["C"][d], e["Cm"])
        assert np.array_equal(bt.fd["fd_X_BEM"][d], e["fd"]["X_BEM"]) and np.array_equal(bt.fd["fd_T0"][d], e["fd"]["T0"])
        assert bt.fd["heading_adjust"][d] == 2.0 * d and bt.fd["x_ref"][d] == float(d)
    g, b, f, q = bt.structs(lambda name, a: None)
    assert g.n_nodes == sum(Ns) and b.n_designs == 3 and b.max_nodes == max(Ns) and f.n_fd == len(ds[0]["fd"]["fd_idx"]) and q is None


def test_mismatched_designs_raise():
    import general_synth as gs
    from raft_b200 import solver
    ds = _designs(fd=False)
    P, M, B, Cm = gs.design(7, 33, seed=4)
    with pytest.raises(ValueError, match="design 3: n_dof"):
        solver.GeneralBatch(ds + [dict(P=P, M=M, B=B, Cm=Cm)])
    P, M, B, Cm = gs.design(9, 34, seed=4)
    with pytest.raises(ValueError, match="design 1: the frequency grid"):
        solver.GeneralBatch(ds[:1] + [dict(P=P, M=M, B=B, Cm=Cm)])
    e = dict(ds[1], P=dict(ds[1]["P"], depth=float(ds[1]["P"]["depth"]) + 1.0))
    with pytest.raises(ValueError, match="design 1: depth"):
        solver.GeneralBatch([ds[0], e])
    fds = _designs()
    e = dict(fds[2], fd=dict(fds[2]["fd"], fd_idx=fds[2]["fd"]["fd_idx"][1:], A_w=fds[2]["fd"]["A_w"][1:, 1:], B_w=fds[2]["fd"]["B_w"][1:, 1:]))
    with pytest.raises(ValueError, match="design 2: n_fd"):
        solver.GeneralBatch(fds[:2] + [e])
    e = dict(fds[1], fd=dict(fds[1]["fd"], bem_headings=fds[1]["fd"]["bem_headings"][:3], X_BEM=fds[1]["fd"]["X_BEM"][:3]))
    with pytest.raises(ValueError, match="design 1: n_bem_head"):
        solver.GeneralBatch([fds[0], e])
    q0 = gs.qtf_table(ds[0]["P"], 12, [0.0, 90.0])
    q1 = gs.qtf_table(ds[0]["P"], 13, [0.0, 90.0])
    with pytest.raises(ValueError, match="design 1: the QTF grid"):
        solver.GeneralBatch([dict(ds[0], qtf=q0), dict(ds[1], qtf=q1)])
    with pytest.raises(ValueError, match="design 1: qtf"):
        solver.GeneralBatch([dict(ds[0], qtf=q0), ds[1]])
    with pytest.raises(ValueError, match="design 1: fd"):
        solver.GeneralBatch([fds[0], ds[1]])


def test_workspace_query_on_ragged_batch():
    """The batch query is the single-design query of K units of max_nodes node rows, plus the chunk's primary map (K * 4 bytes
    rounded up to 256) -- a batch of more than one design always carries it."""
    from raft_b200 import solver
    from raft_b200._lib import lib
    ds = _designs()
    bt = solver.GeneralBatch(ds)
    big = [e for e in ds if len(e["P"]["node_ls"]) == bt.max_nodes][0]
    g1 = solver._general_struct(big["P"], big["M"], big["B"], big["Cm"], lambda n, a: None)
    f1 = solver._general_fd_struct(big["fd"], bt.n, bt.nw, lambda n, a: None)
    single = lambda K: int(lib.raftk_general_qtf_workspace_bytes(C.byref(g1), C.byref(f1), None, K))      # noqa: E731
    nC = 7
    for K in (0, 1, 5, 7, 13, 21, 40):
        k = 21 if K in (0, 40) else K
        assert solver.general_batch_workspace_bytes(bt, nC, K) == single(k) + (k * 4 + 255) // 256 * 256, K
    one = solver.GeneralBatch(ds[:1])
    g0 = solver._general_struct(ds[0]["P"], ds[0]["M"], ds[0]["B"], ds[0]["Cm"], lambda n, a: None)
    f0 = solver._general_fd_struct(ds[0]["fd"], bt.n, bt.nw, lambda n, a: None)
    assert solver.general_batch_workspace_bytes(one, nC, 0) == int(lib.raftk_general_qtf_workspace_bytes(C.byref(g0), C.byref(f0), None, nC))
    budget = solver.general_batch_workspace_bytes(bt, nC, 10)
    K = solver.general_batch_chunk_for_budget(bt, nC, budget)
    assert K == 10
    with pytest.raises(ValueError):
        solver.general_batch_chunk_for_budget(bt, nC, solver.general_batch_workspace_bytes(bt, nC, 2) - 1,
                                              primary=np.array([0, 1, 1, 3, 4, 4, 4], dtype=np.int32))


def _prim(sizes):
    out, c = [], 0
    for s in sizes:
        out += [c] * s
        c += s
    return np.array(out, dtype=np.int32)


@pytest.mark.parametrize("sizes,nD,K,want", [
    ((1, 3, 2), 2, 3, [0, 1, 4, 7, 10, 12]),           # one train group per chunk where two do not fit
    ((1, 3, 2), 2, 8, [0, 7, 12]),                     # a chunk across the design boundary
    ((1, 3, 2), 2, 6, [0, 6, 12]),                     # design-aligned
    ((1, 3, 2), 3, 0, [0, 18]),
    ((1,) * 4, 3, 5, [0, 5, 10, 12]),
    ((2, 2), 3, 3, [0, 2, 4, 6, 8, 10, 12]),
])
def test_batch_chunk_plan(sizes, nD, K, want):
    from raft_b200 import solver
    pr = _prim(sizes)
    assert solver.general_batch_chunk_plan(pr, len(pr), nD, K) == want
    assert solver.general_batch_chunk_plan(pr, len(pr), 1, K if K < len(pr) else 0) == solver.general_chunk_plan(pr, len(pr), K)
    if max(sizes) > 1:
        with pytest.raises(ValueError, match="more than max_chunk_units"):
            solver.general_batch_chunk_plan(pr, len(pr), nD, max(sizes) - 1)


def _host_call(bt, primary, K, mutate=None):
    from raft_b200 import solver
    from raft_b200._lib import RaftkSolveOpts, lib
    nC = len(primary)
    ct = solver.CaseTable(dict(Hs=np.full(nC, 2.0), Tp=np.full(nC, 9.0), gamma=np.zeros(nC), beta_deg=np.zeros(nC),
                               spec=np.zeros(nC, dtype=np.int32), primary=primary))
    keep = {}

    def ptr(name, a):
        keep[name] = a.copy()                          # mutations stay out of the batch's own tables
        return keep[name].ctypes.data
    g, b, f, q = bt.structs(ptr)
    if mutate:
        mutate(keep, b)
    c = ct.struct(lambda name: ct.arrays[name].ctypes.data)
    o = RaftkSolveOpts(10, 0, 0.01, 0.0, 0, 0)
    Xi = np.zeros([bt.n_designs, nC, bt.n, bt.nw], dtype=complex)
    st = np.zeros([bt.n_designs, nC, 4], dtype=np.int32)
    before = lib.raftk_launch_count()
    rc = lib.raftk_general_batch_solve_dynamics_host(C.byref(g), C.byref(b), C.byref(f) if f else None, None, C.byref(c), C.byref(o),
                                                     Xi.ctypes.data, st.ctypes.data, None, None, None, K)
    return rc, lib.raftk_last_error().decode(), lib.raftk_launch_count() - before


def test_host_entry_refuses_before_launching():
    from raft_b200 import solver
    bt = solver.GeneralBatch(_designs())
    pr = _prim((1, 3, 2))

    def off(vals):
        def m(keep, b):
            keep["node_offset"][:] = vals
        return m
    Ns = bt.node_offset.tolist()
    for mut, msg in ((off([1, Ns[1], Ns[2], Ns[3]]), "start at 0"), (off([0, Ns[1], Ns[1] - 1, Ns[3]]), "non-decreasing"),
                     (off([0, Ns[1], Ns[2] - 1, Ns[3] - 1]), "equal n_nodes")):
        rc, err, nl = _host_call(bt, pr, 0, mut)
        assert rc == -1 and msg in err and nl == 0, err

    def fd_bad(keep, b):
        keep["fd_idx"][1, :2] = [3, 3]
    rc, err, nl = _host_call(bt, pr, 0, fd_bad)
    assert rc == -1 and "fd_idx" in err and nl == 0, err

    def shared(keep, b):
        b.qtf_shared = 2
    rc, err, nl = _host_call(bt, pr, 0, shared)
    assert rc == -1 and "qtf_shared" in err and nl == 0
    rc, err, nl = _host_call(bt, pr, 2)
    assert rc == -1 and "more cases than max_chunk_units" in err and nl == 0
    rc, err, nl = _host_call(bt, np.array([0, 1, 0, 1], dtype=np.int32), 0)
    assert rc == -1 and "interleave" in err and nl == 0
    rc, err, nl = _host_call(bt, pr, -1)
    assert rc == -1 and "max_chunk_units" in err and nl == 0
    rc, err, nl = _host_call(bt, pr, 70000)
    assert rc != -1 or "65535" not in err               # a cap above the unit count is the whole batch (18 units)


def test_device_entry_refuses_a_small_workspace():
    """No primary map and no fd / qtf tables: the device entry's only read-back is node_offset, which a bad count refuses
    before; a chunk cap over 65535 units is refused without touching a device."""
    from raft_b200 import solver
    from raft_b200._lib import RaftkCases, RaftkSolveOpts, lib
    bt = solver.GeneralBatch(_designs(fd=False))
    g, b, f, q = bt.structs(lambda n, a: 0x1000)
    c = RaftkCases()
    c.n_cases = 40000
    o = RaftkSolveOpts(10, 0, 0.01, 0.0, 0, 0)
    before = lib.raftk_launch_count()
    rc = lib.raftk_general_batch_solve_dynamics_dev(C.byref(g), C.byref(b), None, None, C.byref(c), C.byref(o), 0x1000, 0x1000, None, None,
                                                    None, 0x1000, 1 << 40, 0, None)
    assert rc == -1 and b"65535" in lib.raftk_last_error()
    b.n_designs = 0
    rc = lib.raftk_general_batch_solve_dynamics_dev(C.byref(g), C.byref(b), None, None, C.byref(c), C.byref(o), 0x1000, 0x1000, None, None,
                                                    None, 0x1000, 1 << 40, 1000, None)
    assert rc == -1 and b"n_designs" in lib.raftk_last_error()
    assert lib.raftk_launch_count() == before
