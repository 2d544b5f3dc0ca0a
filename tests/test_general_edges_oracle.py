"""CPU side of tests/test_general_edges.py: the synthetic inputs (tests/general_synth.py) are what they claim, every row of
the GPU matrix is sensitive to the mistakes its row is there to catch, the impedances are well enough conditioned for the
1e-10 response bound to mean something, and the output-channel entries refuse frequency powers other than 0, 1 and 2
(before any launch, so without a device)."""
import ctypes as C

import numpy as np
import pytest

import general_qtf_checker as gqc
import general_synth as gs
from conftest import relerr

SENS = 1e-6                                            # every mistake must move a result by this much (10^4 x the tolerance)


# ---- the builders -------------------------------------------------------------------------------------------------------
def test_support_crosses_panels_and_ends_on_last_dof():
    for n in (7, 9, 17):
        idx = gs.support(n)
        assert idx[-1] == n - 1 and np.all(np.diff(idx) > 0)
        if n > 8:                                      # DOFs on both sides of an 8-column panel boundary
            assert len({i // 8 for i in idx}) >= 2 and 7 in idx and 8 in idx
    r = gs.row("e", "stride")
    idx = r["fd"]["fd_idx"]
    assert 127 in idx and 128 in idx and 255 in idx
    assert min(gs.row("b")["fd"]["fd_idx"]) >= 6


@pytest.mark.parametrize("name,arg", [("a", 9), ("b", None), ("e", "stride"), ("d", "full")])
def test_fd_tables_antisymmetric_varying_and_scaled(name, arg):
    r = gs.row(name, arg)
    fd, M = r["fd"], r["M"]
    idx = fd["fd_idx"]
    for key in ("A_w", "B_w"):
        T = fd[key]
        d = np.abs(T[np.arange(len(idx)), np.arange(len(idx))])                 # units differ per DOF: scale to unit diagonal
        T = T / np.sqrt(d[:, None] * d[None, :])
        sym, asym = 0.5 * (T + T.transpose(1, 0, 2)), 0.5 * (T - T.transpose(1, 0, 2))
        frac = np.linalg.norm(asym, axis=(0, 1)) / np.linalg.norm(sym, axis=(0, 1))
        assert frac.min() >= 0.2, (key, frac.min())
        var = (fd[key].max(axis=-1) - fd[key].min(axis=-1)) / np.abs(fd[key]).max(axis=-1)
        assert var.min() >= 0.3, (key, var.min())
    dA = np.abs(fd["A_w"][np.arange(len(idx)), np.arange(len(idx))]).max(axis=-1) / np.diag(M)[idx]
    assert dA.min() >= 0.1 * 0.5 and dA.max() <= 0.3 * 1.5           # 0.1-0.3 of diag M, times the 1 +- 0.5 variation


def test_t0_dense_and_bem_tables():
    r = gs.row("a", 17)
    T0 = r["fd"]["T0"]
    assert T0.shape == (6, 17) and np.all(T0[:, 6:] != 0.0) and np.all(T0[:, :6] - np.eye(6) != 0.0)
    assert np.abs(T0[:, :6] - np.eye(6)).max() <= 0.05
    assert gs.row("c", 129)["fd"]["fd_idx"].size == 0 and len(gs.row("g", (40.0,))["fd"]["bem_headings"]) == 1
    assert "X_BEM" not in gs.row("b")["fd"]


def test_qtf_table_is_hermitian_and_leaves_bins_uncovered():
    for n, nw in ((6, 33), (64, 257)):
        r = gs.row("f", (n, nw))
        q, w = r["qtf"], r["P"]["w"]
        Q = q["qtf"]
        assert np.array_equal(Q, Q.transpose(1, 0, 2, 3).conj())
        assert (w < q["qtf_w"][0]).sum() >= 2 and (w > q["qtf_w"][-1]).sum() >= 2
        assert np.all(np.diff(q["qtf_w"]) > 0) and np.all(np.diff(q["qtf_heads"]) > 0)


def test_cases_mix_trains_with_headings_of_their_own():
    table, owner, first, trains = gs.cases((1, 3, 2))
    assert list(first) == [0, 1, 4] and table["primary"].tolist() == [0, 1, 1, 1, 4, 4]
    for tr in trains[1:]:
        assert np.all(np.abs(tr[1:, 2] - tr[0, 2]) >= 40.0)


# ---- sensitivity of every GPU row ---------------------------------------------------------------------------------------
def _run(orc, r, fd=None, qtf="same", trains=None):
    fd = r["fd"] if fd is None else fd
    qtf = r["qtf"] if qtf == "same" else qtf
    out = []
    for tr in (r["ct"][3] if trains is None else trains):
        X, st, Fb, F2, _ = gqc.solve_trains_qtf(orc, r["P"], r["M"], r["B"], r["Cm"], fd, qtf, tr, nIter=r["n_iter"])
        out.append((X, Fb, F2))
    return out


def _moved(a, b):
    """Largest relative change of Xi, F_BEM or F_2nd over the cases."""
    e = 0.0
    for (X, Fb, F2), (Y, Gb, G2) in zip(a, b):
        for u, v in ((X, Y), (Fb, Gb), (F2, G2)):
            if np.abs(v).max() > 0:
                e = max(e, relerr(u, v))
    return e


@pytest.mark.parametrize("name,arg", gs.ROWS)
def test_row_catches_its_mistakes(name, arg, oracle):
    r = gs.row(name, arg)
    fd, n = r["fd"], r["M"].shape[0]
    cap = gs.CaptureZ(oracle)
    base = _run(cap, r)
    assert gs.max_cond(cap.Z) < 1e8, gs.max_cond(cap.Z)
    mistakes = {"fd dropped": dict(fd=dict(fd_idx=np.zeros(0, dtype=np.int32)))}
    nf = len(fd["fd_idx"])
    if nf >= 2:
        mistakes["A_w, B_w transposed"] = dict(fd=dict(fd, A_w=fd["A_w"].transpose(1, 0, 2).copy(), B_w=fd["B_w"].transpose(1, 0, 2).copy()))
        # position t of the support read for DOF fd_idx[t - 1]: the tables rotated by one
        mistakes["support positions rotated"] = dict(fd=dict(fd, A_w=np.roll(fd["A_w"], 1, axis=(0, 1)), B_w=np.roll(fd["B_w"], 1, axis=(0, 1))))
    if nf == 1:
        mistakes["support shifted"] = dict(fd=dict(fd, fd_idx=np.array([fd["fd_idx"][0] - 1], dtype=np.int32)))
    if fd.get("X_BEM") is not None:
        mistakes["T0 = [I | 0]"] = dict(fd=dict(fd, T0=np.eye(6, n)))
    if r["qtf"] is not None:
        mistakes["F_2nd dropped"] = dict(qtf=None)
    trains = r["ct"][3]
    if any(len(t) > 1 for t in trains):
        same = [np.column_stack([t[:, :2], np.full(len(t), t[0, 2])]) for t in trains]
        mistakes["secondary with its primary's heading"] = dict(trains=same)
    for what, kw in mistakes.items():
        e = _moved(_run(oracle, r, **kw), base)
        assert e > SENS, (what, e)


# ---- wpow: refused before any launch ------------------------------------------------------------------------------------
def test_general_channel_stats_refuses_other_powers():
    from raft_b200 import _lib, solver
    w = np.linspace(0.1, 1.0, 8)
    Xi = np.ones((1, 6, 8), dtype=np.complex128)
    R = np.ones((2, 6))
    for bad in ([0, 3], [-1, 1], [2, 7]):
        with pytest.raises(ValueError, match="wpow must be 0, 1 or 2"):
            solver.general_channel_stats(R, np.array(bad), w, Xi, 0.1)
        p = np.array(bad, dtype=np.int32)
        sd = np.zeros(2)
        rc = _lib.lib.raftk_general_channel_stats_host(1, 6, 2, 8, C.c_double(0.1), w.ctypes.data, R.ctypes.data, p.ctypes.data,
                                                       Xi.ctypes.data, sd.ctypes.data, None, None)
        assert rc == -1 and b"wpow must be 0, 1 or 2" in _lib.lib.raftk_last_error()
        assert not sd.any()
