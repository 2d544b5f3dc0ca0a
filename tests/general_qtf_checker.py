"""CPU checker for Model.solveDynamics of a FOWT with generalised degrees of freedom and second-order wave loads from an
external QTF (potSecOrder 2; raft_model.py:1035-1048, 1210-1212).  Test infrastructure, independent of the CUDA path, built on
``general_fd_checker.solve_trains_fd``'s steps and the C checker's pinned second-order force ``oracle.hydro_force_2nd``
(FOWT.calcHydroForce_2ndOrd, interpMode 'qtf'), which it uses unchanged:

* every train gets F_2nd of its own spectrum and heading on reduced DOFs 0-5 (the reference lumps it there, :1034);
* the primary's force joins the linear excitation before the drag loop: (F_BEM + F_hydro_iner) + F_2nd (:1048), then
  + F_drag in every pass (:1081);
* after the loop every train's response is solved again with the excitation summed in the reference's order,
  ((F_BEM + F_hydro_iner) + F_drag) + F_2nd (:1212), the primary's included.

``qtf`` is the dict of ``raft_b200.packer.pack_general_qtf`` (qtf [nw2,nw2,nheads,6], qtf_w, qtf_heads)."""
import numpy as np

import general_fd_checker as gfc
import general_trains_checker as gtc


D2R = 0.017453292519943295                                          # the kernels' pi / 180

# Response tolerances.  The slow-drift force loads the lowest bins, where the flexible FOWT's impedance is nearly singular
# (cond(Z) 3.2e10, 3.5e10, 7.9e9 in bins 0-2 of the flexqtf fixture; <= 7.5e9 above) and where the response now peaks.  There
# two correct solvers differ by cond * eps: against the reference's inv(Z) @ F (raft_model.py:1191, 1216) the checker's C
# inverse differs by up to 2.3e-9 of max|Xi| and an LU solve by 7.4e-10, while numpy's own inverse agrees to 4e-14 (measured).
# So the whole response is held to XI_RTOL_ALL and the bins from LOW_BINS up, where the measured difference is <= 4e-11, to
# XI_RTOL; the force itself changes the response by 100 % of max|Xi| (fixture ``qtf_effect_case0``).
LOW_BINS, XI_RTOL, XI_RTOL_ALL = 3, 1e-10, 1e-8


def xi_errors(X, ref):
    """-> (max|X - ref| / max|ref| over every bin, the same from bin LOW_BINS up), X and ref [.., nw]."""
    X, ref = np.asarray(X), np.asarray(ref)
    s = np.abs(ref).max()
    return np.abs(X - ref).max() / s, np.abs(X - ref)[..., LOW_BINS:].max() / s


def force_2nd(orc, P, qtf, Hs, Tp, beta_deg):
    """F_2nd [6, nw] and F_2nd_mean [6] of one JONSWAP train (gamma 0): oracle.hydro_force_2nd on the FOWT's table."""
    Q = dict(P, qtf=qtf["qtf"], qtf_w=qtf["qtf_w"], qtf_heads=qtf["qtf_heads"])
    od = orc.OracleDesign(Q)
    S = orc.jonswap(np.asarray(P["w"], dtype=float), Hs, Tp, 0.0)
    fm, f = orc.hydro_force_2nd(od, beta_deg * D2R, S)
    return f, fm


def solve_trains_qtf(orc, P, M, B, Cm, fd, qtf, trains, nIter=10, tol=0.01, XiStart=0.0):
    """``trains`` rows (Hs, Tp, heading_deg), JONSWAP with gamma 0; train 0 drives the linearisation
    -> Xi [nH, nDOF, nw], status (passes, converged, nan), F_BEM [nH, nDOF, nw], F_2nd [nH, 6, nw], F_2nd_mean [nH, 6]."""
    gd = orc.GeneralDesign(P)
    w = np.asarray(P["w"], dtype=float)
    tr = np.asarray(trains, dtype=float).reshape(-1, 3)
    n, nw = int(P["gen_nDOF"]), len(w)
    exc = [orc.general_excitation(gd, 0, t[0], t[1], 0.0, t[2]) for t in tr]
    Fb = np.array([gfc.bem_excitation(orc, P, fd, t[0], t[1], t[2]) for t in tr])
    F2, F2m = np.zeros([len(tr), 6, nw]), np.zeros([len(tr), 6])
    if qtf:
        for h, t in enumerate(tr):
            F2[h], F2m[h] = force_2nd(orc, P, qtf, t[0], t[1], t[2])
    F2n = np.zeros([len(tr), n, nw], dtype=complex)
    F2n[:, :6] = F2                                                 # fowt.Fhydro_2nd: zero from reduced DOF 6 up
    Flin = [(Fb[h] + exc[h][1]) for h in range(len(tr))]            # F_BEM + F_hydro_iner (raft_model.py:1048, 1212)
    F0 = Flin[0] + F2n[0]                                           # + Fhydro_2nd (:1048)
    u0 = exc[0][2]
    A_w, B_w = gfc.dense_fd(fd, n, nw)
    Mw = M[:, :, None] + A_w
    Bw = B[:, :, None] + B_w
    XiLast = np.full([n, nw], XiStart, dtype=complex)
    passes, conv, nan = 0, 0, 0
    for _ in range(nIter + 1):
        Xlin = XiLast
        Bd, Fd = orc.general_linearization(gd, u0, Xlin)
        passes += 1
        Z = np.moveaxis(-w ** 2 * Mw + 1j * w * (Bw + Bd[:, :, None]) + Cm[:, :, None], 2, 0)   # [nw, n, n], raft_model.py:1086
        Xi = np.linalg.solve(Z, (F0 + Fd).T[:, :, None])[:, :, 0].T
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
        Fwave = (Flin[ih] + Fdrag) + F2n[ih]                          # raft_model.py:1212
        out[ih] = orc.system_response(Z, Fwave.T).T                   # inv(Z) F, raft_model.py:1191, 1216
    return out, np.array([passes, conv, nan], dtype=np.int32), Fb, F2, F2m
