"""CPU checker for Model.solveDynamics of a FOWT with generalised degrees of freedom and frequency-dependent terms: the added
mass and damping of operating rotors and BEM coefficients (sum A_aero + A_BEM, sum B_aero + B_BEM; raft_model.py:1005-1010,
1045-1048) and the BEM wave excitation F_BEM = T^T F_BEM_fullDOF (raft_fowt.py:1796-1849, 1885-1887), with one or several
wave trains (raft_model.py:1200-1236).  Test infrastructure, independent of the CUDA path, built like
``general_trains_checker.py`` from the C checker's pinned routines:

* ``oracle.general_excitation`` / ``oracle.general_linearization``: inertial excitation, wave kinematics, drag linearisation;
* ``oracle.calc_hydro_excitation`` on the same node tables with the BEM table: the rigid checker's BEM excitation (heading
  bracket with wrap-around, interpolation, rotation, array phase) in full DOFs 0-5, mapped to reduced DOFs with ``T0``;
* ``oracle.system_response``: every train's response through the explicit inverse of the last impedance (raft_model.py:1191),
  in plain C, so the result does not move with the host's LAPACK build.

The impedance on the support of the frequency-dependent terms is grouped as the CUDA kernels group it: M + A_w and
(B + B_w) + B_drag (``fd`` = the dict of ``raft_b200.packer.pack_general_matrices``; every entry off the support is M, B)."""
import numpy as np

import general_trains_checker as gtc


def dense_fd(fd, n, nw):
    """A_w, B_w of ``fd`` scattered to [n, n, nw] (zero off the support)."""
    A, B = np.zeros([n, n, nw]), np.zeros([n, n, nw])
    idx = np.asarray(fd.get("fd_idx", np.zeros(0)), dtype=np.int64) if fd is not None else np.zeros(0, dtype=np.int64)
    if len(idx):
        A[np.ix_(idx, idx)] = fd["A_w"]
        B[np.ix_(idx, idx)] = fd["B_w"]
    return A, B


def bem_excitation(orc, P, fd, Hs, Tp, beta_deg):
    """F_BEM [nDOF, nw] of one JONSWAP train (gamma 0): the rigid checker's BEM force in full DOFs 0-5, T0^T applied."""
    n, nw = int(P["gen_nDOF"]), len(P["w"])
    if fd is None or fd.get("X_BEM") is None:
        return np.zeros([n, nw], dtype=complex)
    Q = dict(P, X_BEM=fd["X_BEM"], bem_headings=fd["bem_headings"], heading_adjust=fd.get("heading_adjust", 0.0),
             x_ref=fd.get("x_ref", 0.0), y_ref=fd.get("y_ref", 0.0))
    _, f6, _, _ = orc.calc_hydro_excitation(orc.OracleDesign(Q), 0, Hs, Tp, 0.0, beta_deg)
    return np.asarray(fd["T0"], dtype=float).T @ f6                   # T.T @ F_BEM_fullDOF (raft_fowt.py:1886)


def solve_trains_fd(orc, P, M, B, Cm, fd, trains, nIter=10, tol=0.01, XiStart=0.0):
    """``trains`` rows (Hs, Tp, heading_deg), JONSWAP with gamma 0; train 0 drives the linearisation
    -> Xi [nH, nDOF, nw], status (passes, converged, nan), F_BEM [nH, nDOF, nw]."""
    gd = orc.GeneralDesign(P)
    w = np.asarray(P["w"], dtype=float)
    tr = np.asarray(trains, dtype=float).reshape(-1, 3)
    n, nw = int(P["gen_nDOF"]), len(w)
    exc = [orc.general_excitation(gd, 0, t[0], t[1], 0.0, t[2]) for t in tr]
    Fb = np.array([bem_excitation(orc, P, fd, t[0], t[1], t[2]) for t in tr])
    Flin = [Fb[h] + exc[h][1] for h in range(len(tr))]              # F_BEM + F_hydro_iner (raft_model.py:1048, 1212)
    u0 = exc[0][2]
    A_w, B_w = dense_fd(fd, n, nw)
    Mw = M[:, :, None] + A_w
    Bw = B[:, :, None] + B_w
    XiLast = np.full([n, nw], XiStart, dtype=complex)
    passes, conv, nan = 0, 0, 0
    for _ in range(nIter + 1):
        Xlin = XiLast
        Bd, Fd = orc.general_linearization(gd, u0, Xlin)
        passes += 1
        Z = np.moveaxis(-w ** 2 * Mw + 1j * w * (Bw + Bd[:, :, None]) + Cm[:, :, None], 2, 0)   # [nw, n, n], raft_model.py:1086
        Xi = np.linalg.solve(Z, (Flin[0] + Fd).T[:, :, None])[:, :, 0].T
        if np.isnan(Xi).any():
            nan = 1
            break
        if np.all(np.abs(Xi - XiLast) / (np.abs(Xi) + tol) < tol):
            conv = 1
            break
        XiLast = 0.2 * XiLast + 0.8 * Xi
    Bmat = gtc.node_bmat(P, u0, Xlin)
    out = np.zeros([len(tr), n, nw], dtype=complex)
    for ih, (_, _, u) in enumerate(exc):
        Fdrag = Fd if ih == 0 else gtc.drag_excitation(P, Bmat, u)
        out[ih] = orc.system_response(Z, (Flin[ih] + Fdrag).T).T      # inv(Z) F, raft_model.py:1191, 1216
    return out, np.array([passes, conv, nan], dtype=np.int32), Fb
