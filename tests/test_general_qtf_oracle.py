"""Second-order wave loads on the generalised-DOF path, on the CPU: the checker (tests/general_qtf_checker.py, built on the C
checker's pinned generalised-DOF, BEM and second-order force routines) against the reference's own run of a flexible FOWT with
an operating rotor, BEM coefficients and the marin_semi .12d QTF (fixture flexqtf_VolturnUS-S-flexible,
tests/golden/make_golden_flexqtf.py), packer.pack_general_qtf, the struct layout of raftk_general_qtf and the argument checks
of raftk_general_solve_dynamics_qtf_* (no device needed: every rejection happens before any launch).

The fixture stores no QTF table: it is rebuilt from wamit_marin_semi.npz's ``qtf_rows`` with bem.read_qtf, which
tests/test_bem.py pins to the state the reference's readQTF leaves.  Response tolerances: general_qtf_checker.XI_RTOL (bins from
LOW_BINS up) and XI_RTOL_ALL (every bin; the lowest bins are resonant and nearly singular, see there)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import general_fd_checker as gfc
import general_qtf_checker as gqc
from conftest import GOLDEN, ROOT, relerr
from test_general_fd_oracle import load_flexfd

FLEXQTF = os.path.join(GOLDEN, "flexqtf_VolturnUS-S-flexible.npz")


def marin_qtf(tmp_dir):
    """The marin_semi QTF table as the reference reads it: dict(qtf [56,56,1,6], qtf_w, qtf_heads) (packer.pack_general_qtf)."""
    from raft_b200 import bem
    rows = np.load(os.path.join(GOLDEN, "wamit_marin_semi.npz"))["qtf_rows"]
    path = os.path.join(str(tmp_dir), "semi.12d")
    np.savetxt(path, rows, fmt="%.5e")                     # the file carries 6 significant digits
    q, w, heads = bem.read_qtf(path, rho=1025.0, g=9.81)
    return dict(qtf=q, qtf_w=w, qtf_heads=heads)


def load_flexqtf(tmp_dir):
    """-> (P, M, B, C, fd, qtf, z): the flexfd design and matrices, the marin_semi QTF and the fixture."""
    P, M, B, Cm, fd, _ = load_flexfd()
    return P, M, B, Cm, fd, marin_qtf(tmp_dir), np.load(FLEXQTF)


def test_checker_vs_reference_run_flexqtf(oracle, tmp_path):
    P, M, B, Cm, fd, qtf, z = load_flexqtf(tmp_path)
    assert tuple(z["qtf_shape"]) == qtf["qtf"].shape
    worst = 0.0
    for ic in range(int(z["n_cases"])):
        tr = z["ref_run_case%d_trains" % ic]
        Xi, st, _, F2, F2m = gqc.solve_trains_qtf(oracle, P, M, B, Cm, fd, qtf, tr, nIter=int(z["n_iter"]), XiStart=float(z["xi_start"]))
        assert st[0] == int(z["ref_run_case%d_passes" % ic]) and st[2] == 0, (ic, st)
        for h in range(len(tr)):
            e_all, e = gqc.xi_errors(Xi[h], z["ref_run_case%d_Xi" % ic][h])
            worst = max(worst, e_all)
            assert e_all < gqc.XI_RTOL_ALL and e < gqc.XI_RTOL, (ic, h, e_all, e)
            assert relerr(F2[h], z["ref_run_case%d_F2nd" % ic][h]) < 1e-12, (ic, h)
            assert relerr(F2m[h], z["ref_run_case%d_F2nd_mean" % ic][h]) < 1e-12, (ic, h)
    print("largest relative Xi error against the reference run: %.2e" % worst)


def test_fixture_needs_the_second_order_force(oracle, tmp_path):
    """The force moves the response far beyond both response tolerances: the stored effect (the reference's run without the
    QTF, measured 1.0 of max|Xi|), and the checker without the table against the fixture."""
    P, M, B, Cm, fd, _, z = load_flexqtf(tmp_path)
    assert float(z["qtf_effect_case0"]) > 1e-6
    tr = z["ref_run_case0_trains"]
    Xi, _, _, F2, _ = gqc.solve_trains_qtf(oracle, P, M, B, Cm, fd, None, tr, nIter=int(z["n_iter"]), XiStart=float(z["xi_start"]))
    assert not F2.any()
    e_all, e = gqc.xi_errors(Xi[0], z["ref_run_case0_Xi"][0])
    assert e_all > 1e6 * gqc.XI_RTOL_ALL and e > 1e6 * gqc.XI_RTOL, (e_all, e)


def test_checker_without_qtf_is_the_fd_checker(oracle, tmp_path):
    P, M, B, Cm, fd, _, z = load_flexqtf(tmp_path)
    tr = z["ref_run_case3_trains"]
    X0, s0, F0 = gfc.solve_trains_fd(oracle, P, M, B, Cm, fd, tr, nIter=int(z["n_iter"]), XiStart=float(z["xi_start"]))
    X1, s1, F1, _, _ = gqc.solve_trains_qtf(oracle, P, M, B, Cm, fd, {}, tr, nIter=int(z["n_iter"]), XiStart=float(z["xi_start"]))
    assert np.array_equal(s0, s1) and np.array_equal(F0, F1) and relerr(X1, X0) < 1e-14


def test_fixture_trains_and_headings():
    """Case 3 has two trains (each with its own spectrum and heading), case 4 is the single train at 180 deg; -60 and 355 deg
    lie outside the one-heading table (the reference clamps to it)."""
    z = np.load(FLEXQTF)
    assert int(z["n_cases"]) == 5
    assert z["ref_run_case3_trains"].shape == (2, 3) and z["ref_run_case4_trains"].tolist() == [[5.0, 11.0, 180.0]]
    for ic in range(5):
        F2 = z["ref_run_case%d_F2nd" % ic]
        assert F2.shape[1] == 6 and F2.any() and not F2[:, :, -1].any()        # last bin zero (raft_fowt.py:2245)
    assert not np.array_equal(z["ref_run_case3_F2nd"][0], z["ref_run_case3_F2nd"][1])


# ---- packer.pack_general_qtf ------------------------------------------------------------------------------------------------
def _fowt_like(qtf, sec=2, n=150):
    from types import SimpleNamespace
    full = np.zeros(qtf["qtf"].shape[:3] + (n,), dtype=complex)
    full[..., :6] = qtf["qtf"]
    return SimpleNamespace(potSecOrder=sec, nDOF=n, w1_2nd=qtf["qtf_w"].copy(), w2_2nd=qtf["qtf_w"].copy(), heads_2nd=qtf["qtf_heads"].copy(),
                           qtf=full)


def test_pack_general_qtf_on_fixture_rows(tmp_path):
    from raft_b200 import packer
    qtf = marin_qtf(tmp_path)
    f = _fowt_like(qtf)
    Q = packer.pack_general_qtf(f)
    assert Q["qtf"].shape == (56, 56, 1, 6) and Q["qtf"].flags.c_contiguous
    assert np.array_equal(Q["qtf"], qtf["qtf"]) and np.array_equal(Q["qtf_w"], qtf["qtf_w"]) and np.array_equal(Q["qtf_heads"], qtf["qtf_heads"])
    f.qtf[3, 4, 0, 7] = 1e-30
    with pytest.raises(ValueError, match="DOFs 6 and up"):
        packer.pack_general_qtf(f)
    with pytest.raises(NotImplementedError, match="2015-2017"):
        packer.pack_general_qtf(_fowt_like(qtf, sec=1))
    assert packer.pack_general_qtf(_fowt_like(qtf, sec=0)) == {}
    g = _fowt_like(qtf)
    g.w2_2nd = g.w2_2nd * 1.01
    with pytest.raises(ValueError, match="same values"):
        packer.pack_general_qtf(g)


def test_pack_general_qtf_on_reference_fowt(tmp_path):
    from oracle import ref_harness as rh
    if not rh.reference_available():
        pytest.skip("the reference tree is not available")
    import sys
    sys.path.insert(0, GOLDEN)
    import make_golden_flexqtf
    from raft_b200 import packer
    _, fowt = make_golden_flexqtf.build(os.path.join(rh.REF_ROOT, "tests", "test_data", "VolturnUS-S-flexible.yaml"))
    Q = packer.pack_general_qtf(fowt)
    ref = marin_qtf(tmp_path)
    for k in ("qtf", "qtf_w", "qtf_heads"):
        assert np.array_equal(Q[k], ref[k]), k


# ---- C ABI: struct layout, workspace query, argument checks (host entry; nothing is launched) --------------------------------
def test_general_qtf_struct_layout(tmp_path):
    from raft_b200 import _lib
    prog = tmp_path / "layout.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "raftk.h"\nint main(){printf("%zu %zu %zu %zu %zu %zu\\n",'
                    'sizeof(raftk_general_qtf), offsetof(raftk_general_qtf, n_qtf_w), offsetof(raftk_general_qtf, n_qtf_head),'
                    'offsetof(raftk_general_qtf, qtf_w), offsetof(raftk_general_qtf, qtf_heads), offsetof(raftk_general_qtf, qtf));return 0;}\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    Q = _lib.RaftkGeneralQtf
    assert got == [C.sizeof(Q), Q.n_qtf_w.offset, Q.n_qtf_head.offset, Q.qtf_w.offset, Q.qtf_heads.offset, Q.qtf.offset]


def _structs(tmp_path, keep):
    from raft_b200 import solver
    P, M, B, Cm, fd, qtf, z = load_flexqtf(tmp_path)
    n, nw = int(P["gen_nDOF"]), len(P["w"])

    def ptr(name, a):
        keep[name] = a
        return a.ctypes.data
    g = solver._general_struct(P, M, B, Cm, ptr)
    f = solver._general_fd_struct(fd, n, nw, ptr)
    q = solver._general_qtf_struct(qtf, ptr)
    return g, f, q, qtf, n, nw


def test_qtf_workspace_query_without_device(tmp_path):
    """qtf = NULL gives the fd solve's size; a table adds the force and mean-drift buffers [n_cases,6,nw] and [n_cases,6]."""
    from raft_b200 import _lib
    keep = {}
    g, f, q, _, n, nw = _structs(tmp_path, keep)
    lib = _lib.lib
    for nC in (1, 4, 37):
        base = lib.raftk_general_fd_workspace_bytes(C.byref(g), C.byref(f), nC)
        assert base > 0 and lib.raftk_general_qtf_workspace_bytes(C.byref(g), C.byref(f), None, nC) == base
        extra = lib.raftk_general_qtf_workspace_bytes(C.byref(g), C.byref(f), C.byref(q), nC) - base
        assert extra == (nC * 6 * nw * 8 + 255) // 256 * 256 + (nC * 6 * 8 + 255) // 256 * 256
        assert lib.raftk_general_qtf_workspace_bytes(C.byref(g), None, C.byref(q), nC) - lib.raftk_general_workspace_bytes(C.byref(g), nC) == extra


def _rejects(tmp_path, msg, edit=None, cases_kw=None, g_edit=None, fd_none=False):
    from raft_b200 import _lib, solver
    keep = {}
    g, f, q, qtf, n, nw = _structs(tmp_path, keep)
    if edit:
        q = edit(q, keep)
    if g_edit:
        g_edit(g)
    arrays = dict(Hs=np.array([6.0]), Tp=np.array([12.0]), gamma=np.zeros(1), beta_deg=np.zeros(1), spec=np.zeros(1, dtype=np.int32))
    cs = solver.CaseTable(arrays)
    c = cs.struct(solver._host_ptr(cs.arrays))
    for k, v in (cases_kw or {}).items():
        keep["case_" + k] = v
        setattr(c, k, v.ctypes.data)
    o = _lib.RaftkSolveOpts(10, 0, 0.01, 0.0, 0, 0)
    Xi = np.zeros([1, n, nw], dtype=np.complex128)
    st = np.zeros([1, 4], dtype=np.int32)
    F2 = np.zeros([1, 6, nw])
    rc = _lib.lib.raftk_general_solve_dynamics_qtf_host(C.byref(g), None if fd_none else C.byref(f), C.byref(q), C.byref(c), C.byref(o),
                                                        Xi.ctypes.data, st.ctypes.data, None, F2.ctypes.data, None)
    assert rc == -1, rc
    err = _lib.lib.raftk_last_error().decode()
    assert msg in err, err
    assert solver.last_dispatch()["kernel"] == "none"
    assert not Xi.any() and not F2.any()


def _set(**kw):
    def edit(q, keep):
        for k, v in kw.items():
            if isinstance(v, np.ndarray):
                keep["edit_" + k] = v
                v = v.ctypes.data
            setattr(q, k, v)
        return q
    return edit


def test_qtf_rejects_counts_and_missing_tables(tmp_path):
    msg = "qtf needs n_qtf_w >= 2, n_qtf_head >= 1, qtf, qtf_w and qtf_heads"
    _rejects(tmp_path, msg, _set(n_qtf_w=1))
    _rejects(tmp_path, msg, _set(n_qtf_head=0))
    _rejects(tmp_path, msg, _set(qtf=None))
    _rejects(tmp_path, msg, _set(qtf_w=None))
    _rejects(tmp_path, msg, _set(qtf_heads=None))


def test_qtf_rejects_unsorted_frequencies_and_headings(tmp_path):
    qtf = marin_qtf(tmp_path)
    w = qtf["qtf_w"].copy()
    w[10], w[11] = w[11], w[10]
    _rejects(tmp_path, "qtf_w must be strictly increasing", _set(qtf_w=np.ascontiguousarray(w)))
    w = qtf["qtf_w"].copy()
    w[5] = w[4]
    _rejects(tmp_path, "qtf_w must be strictly increasing", _set(qtf_w=np.ascontiguousarray(w)))
    heads = np.array([0.0, 0.5, 0.5])
    big = np.zeros((56, 56, 3, 6), dtype=np.complex128)
    _rejects(tmp_path, "qtf_heads must be strictly increasing", _set(n_qtf_head=3, qtf_heads=heads, qtf=big))


def test_qtf_rejects_small_dof_count_and_large_grid(tmp_path):
    def few(g):
        g.n_dof = 5
    _rejects(tmp_path, "needs n_dof >= 6", g_edit=few, fd_none=True)

    def wide(g):
        g.nw = 227 * 1024 // 20 + 1
    _rejects(tmp_path, "nw too large", g_edit=wide, fd_none=True)


def test_qtf_keeps_rejecting_case_f2nd_and_xi_init(tmp_path):
    from raft_b200 import _lib
    keep = {}
    g, f, q, _, n, nw = _structs(tmp_path, keep)
    from raft_b200 import solver
    cs = solver.CaseTable(dict(Hs=np.array([6.0]), Tp=np.array([12.0]), gamma=np.zeros(1), beta_deg=np.zeros(1), spec=np.zeros(1, dtype=np.int32)))
    o = _lib.RaftkSolveOpts(10, 0, 0.01, 0.0, 0, 0)
    for field, arr in (("F_2nd", np.zeros([1, 6, nw])), ("Xi_init", np.zeros([1, 6, nw], dtype=np.complex128))):
        c = cs.struct(solver._host_ptr(cs.arrays))
        setattr(c, field, arr.ctypes.data)
        Xi = np.zeros([1, n, nw], dtype=np.complex128)
        st = np.zeros([1, 4], dtype=np.int32)
        ws = np.zeros(16, dtype=np.uint8)
        # the device entry refuses before it touches any pointer, the workspace included
        rc = _lib.lib.raftk_general_solve_dynamics_qtf_dev(C.byref(g), C.byref(f), C.byref(q), C.byref(c), C.byref(o), Xi.ctypes.data,
                                                           st.ctypes.data, None, None, None, ws.ctypes.data, ws.nbytes, None)
        assert rc == -1 and b"F_2nd / Xi_init are not supported" in _lib.lib.raftk_last_error(), field
