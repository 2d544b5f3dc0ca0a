"""CPU checker for Model.solveDynamics of a FOWT with generalised degrees of freedom and a case with several wave trains
(raft_model.py:994-1156, 1189-1236).  Test infrastructure, independent of the CUDA path: it drives the C checker's pinned
generalised-DOF routines (``oracle.general_excitation`` / ``oracle.general_linearization``) through the drag-linearisation loop
of train 0 (raft_fowt.py:1910) and restates in NumPy the one piece those routines do not return, the node drag matrices
``Bmat`` of the last pass (raft_member.py:2071-2116), which the drag excitation of the other trains uses
(``calcDragExcitation(ih)``, raft_fowt.py:1940-1957).  Every train's response is then inv(Z_last) (F_iner[ih] + F_drag[ih])
with the explicit inverse of raft_model.py:1191, like the reference, taken by the C checker (``oracle.system_response``): plain
C without BLAS, so the result does not move with the host's LAPACK build (on this cond ~1e6 impedance, NumPy's inverse differs
between hosts by ~1e-10)."""
import numpy as np


def node_bmat(P, u, Xi):
    """Bmat [Ns,3,3] of FOWT.calcHydroLinearization(Xi) (raft_member.py:2071-2116) for the packed generalised design ``P``
    (``packer.pack_general_dofs``), wave kinematics u [Ns,3,nw] and reduced response Xi [nDOF,nw]."""
    w, rho = np.asarray(P["w"], dtype=float), float(P["rho"])
    Tn, rr, mem = np.asarray(P["gen_Tn"]), np.asarray(P["gen_rr"]), np.asarray(P["node_mem"], dtype=np.int64)
    out = np.zeros([len(mem), 3, 3])
    c = np.sqrt(8.0 / np.pi)
    for il, m in enumerate(mem):
        q, p1, p2 = (np.asarray(P[k][m], dtype=float) for k in ("mem_q", "mem_p1", "mem_p2"))
        xn = Tn[il] @ Xi                                          # Xi_nodes = node.T @ Xi (raft_fowt.py:1921)
        th, r = xn[3:], rr[il]
        dr = xn[:3] + np.array([-th[2] * r[1] + th[1] * r[2], th[2] * r[0] - th[0] * r[2], -th[1] * r[0] + th[0] * r[1]])
        vrel = u[il] - 1j * w * dr
        vq = q[:, None] * (q @ vrel)
        vp = vrel - vq
        v1, v2 = p1[:, None] * (p1 @ vrel), p2[:, None] * (p2 @ vrel)
        rq = np.sqrt(0.5 * np.sum(np.abs(vq) ** 2))
        if int(P["mem_circ"][m]):
            r1 = r2 = np.sqrt(0.5 * np.sum(np.abs(vp) ** 2))
        else:
            r1, r2 = np.sqrt(0.5 * np.sum(np.abs(v1) ** 2)), np.sqrt(0.5 * np.sum(np.abs(v2) ** 2))
        Bq = c * rq * 0.5 * rho * P["node_a_q"][il] * P["node_Cd_q"][il]
        Bp1 = c * r1 * 0.5 * rho * P["node_a_p1"][il] * P["node_Cd_p1"][il]
        Bp2 = c * r2 * 0.5 * rho * P["node_a_p2"][il] * P["node_Cd_p2"][il]
        Be = c * rq * 0.5 * rho * P["node_a_End"][il] * P["node_Cd_End"][il]
        out[il] = Bq * np.outer(q, q) + Bp1 * np.outer(p1, p1) + Bp2 * np.outer(p2, p2) + Be * np.outer(q, q)
    return out


def drag_excitation(P, Bmat, u):
    """F_drag [nDOF,nw] = sum_j Tn_j^T [Bmat_j u_j ; rr_j x (Bmat_j u_j)]  (raft_member.py:2122-2152, raft_fowt.py:1940-1957)."""
    Tn, rr = np.asarray(P["gen_Tn"]), np.asarray(P["gen_rr"])
    F = np.zeros([Tn.shape[2], u.shape[2]], dtype=complex)
    for il in range(len(Bmat)):
        f = Bmat[il] @ u[il]
        f6 = np.concatenate([f, np.cross(rr[il][:, None], f, axis=0)])
        F += Tn[il].T @ f6
    return F


def solve_trains(orc, P, M, B, Cm, trains, nIter=10, tol=0.01, XiStart=0.0):
    """``trains`` rows (Hs, Tp, heading_deg), JONSWAP with gamma 0 -> Xi [nH,nDOF,nw] (Model.Xi[:nH]), status (passes,
    converged, nan), and the NumPy drag excitation of train 0 next to the C checker's (for a self-check)."""
    gd = orc.GeneralDesign(P)
    w = np.asarray(P["w"], dtype=float)
    tr = np.asarray(trains, dtype=float).reshape(-1, 3)
    exc = [orc.general_excitation(gd, 0, t[0], t[1], 0.0, t[2]) for t in tr]
    u0, F0 = exc[0][2], exc[0][1]
    n, nw = F0.shape
    XiLast = np.full([n, nw], XiStart, dtype=complex)
    passes, conv, nan = 0, 0, 0
    for _ in range(nIter + 1):
        Xlin = XiLast                                                # the iterate this pass linearises about
        Bd, Fd = orc.general_linearization(gd, u0, Xlin)
        passes += 1
        Z = np.moveaxis(-w ** 2 * M[:, :, None] + 1j * w * (B + Bd)[:, :, None] + Cm[:, :, None], 2, 0)   # [nw,n,n], raft_model.py:1086
        Xi = np.linalg.solve(Z, (F0 + Fd).T[:, :, None])[:, :, 0].T
        if np.isnan(Xi).any():
            nan = 1
            break
        if np.all(np.abs(Xi - XiLast) / (np.abs(Xi) + tol) < tol):
            conv = 1
            break
        XiLast = 0.2 * XiLast + 0.8 * Xi
    Bmat = node_bmat(P, u0, Xlin)
    Fd_np = drag_excitation(P, Bmat, u0)
    out = np.zeros([len(tr), n, nw], dtype=complex)
    for ih, (_, F, u) in enumerate(exc):
        Fdrag = Fd if ih == 0 else drag_excitation(P, Bmat, u)
        out[ih] = orc.system_response(Z, (F + Fdrag).T).T            # inv(Z) F, raft_model.py:1191, 1216
    return out, np.array([passes, conv, nan], dtype=np.int32), (Fd_np, Fd)
