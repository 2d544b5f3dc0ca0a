"""Packer: RAFT object graph (Model -> FOWT -> Member) -> flat SoA tables for the C-ABI.

This is the host half of the drop-in boundary (DESIGN.md section 2).  It is duck-typed: it reads the
attribute names the reference's objects carry (``fowt.memberList``, ``mem.r``, ``mem.q`` ...), so
the same function packs (a) live reference objects, when ``raft_b200`` is dropped into a RAFT
install (INTEGRATION.md), and (b) the objects built by ``raft_b200.member`` / ``raft_b200.fowt``.

Scope: rigid 6-DOF FOWTs (every member has one structural node that is rigidly tied to the FOWT's
reference node), with the inertial wave excitation of submerged rotors (``pack_rotor_excitation``) -- the BASELINE.json
configs plus MacCamy-Fuchs members and MHK turbines.
Anything else raises ``NotImplementedError`` (the caller falls back to the reference path; see
SURVEY.md section 8f row 4).

Reference formulas restated here (they live inside the reference's per-iteration loops, but are
iteration-invariant, so the packer hoists them):
  * drag areas               raft_member.py:2070-2072, 2105-2108
  * coefficient interpolation raft_member.py:2061-2064  (np.interp over stations)
  * linearisation prefactor   raft_member.py:2093-2095, 2110   sqrt(8/pi) * 1/2 rho a Cd
"""
import numpy as np

SQRT_8_OVER_PI = np.sqrt(8.0 / np.pi)


def _member_is_supported(mem):
    if getattr(mem, "type", "rigid") != "rigid":
        raise NotImplementedError("member %r: only rigid members are supported by the GPU path" % mem.name)


def _uses_mcf(mem):
    """MacCamy-Fuchs only alters Imat, which is computed for strip-theory (potMod False) members
    only (raft_member.py:1393, 1415); a potMod member with the MCF flag set is unaffected."""
    return bool(getattr(mem, "MCF", False)) and not bool(getattr(mem, "potMod", False))


def pack_members(fowt, rho=None, g=None, allow_flexible=False):
    """Flatten the submerged strip nodes of ``fowt.memberList`` into node + member tables.

    Only nodes with ``r_z < 0`` are kept (raft_member.py:1935, 1979, 2058, 2135); members with no
    submerged node are dropped.  Returns a dict of numpy arrays (float64 unless noted).
    """
    rho = float(fowt.rho_water if rho is None else rho)
    g = float(fowt.g if g is None else g)
    ref = getattr(fowt, "rigidBodyNode", None)
    prp = np.array(ref.r[:3] if ref is not None else fowt.r6[:3], dtype=float)

    mq, mp1, mp2, mrA, mcirc, mstart = [], [], [], [], [], [0]
    any_mcf = any(_uses_mcf(m) for m in fowt.memberList)
    nw = len(fowt.w) if any_mcf else 0
    in_p1_w, in_p2_w, Imat_w, mcf_flag = [], [], [], []
    cols = {k: [] for k in ("r", "mem", "ls", "cd_q", "cd_p1", "cd_p2", "in_q", "in_p1", "in_p2", "pa",
                            "Imat", "a_i", "a_q", "a_p1", "a_p2", "a_End", "Cd_q", "Cd_p1", "Cd_p2", "Cd_End")}
    for mem in fowt.memberList:
        if not allow_flexible:
            _member_is_supported(mem)
        sub = np.where(mem.r[:, 2] < 0)[0]
        if len(sub) == 0:
            continue
        circ = mem.shape == "circular"
        q, p1, p2 = (np.asarray(v, dtype=float) for v in (mem.q, mem.p1, mem.p2))
        im = len(mq)
        mq.append(q), mp1.append(p1), mp2.append(p2)
        mrA.append(np.array(mem.rA, dtype=float))
        mcirc.append(1 if circ else 0)
        for il in sub:
            ls = float(mem.ls[il])
            Cd_q = np.interp(ls, mem.stations, mem.Cd_q)
            Cd_p1 = np.interp(ls, mem.stations, mem.Cd_p1)
            Cd_p2 = np.interp(ls, mem.stations, mem.Cd_p2)
            Cd_End = np.interp(ls, mem.stations, mem.Cd_End)
            if circ:
                a_q = np.pi * mem.ds[il] * mem.dls[il]
                a_p1 = mem.ds[il] * mem.dls[il]
                a_p2 = mem.ds[il] * mem.dls[il]
                a_End = np.abs(np.pi * mem.ds[il] * mem.drs[il])
            else:
                # sic: ds[il,0] twice, as in raft_member.py:2070
                a_q = 2 * (mem.ds[il, 0] + mem.ds[il, 0]) * mem.dls[il]
                a_p1 = mem.ds[il, 0] * mem.dls[il]
                a_p2 = mem.ds[il, 1] * mem.dls[il]
                a_End = np.abs((mem.ds[il, 0] + mem.drs[il, 0]) * (mem.ds[il, 1] + mem.drs[il, 1])
                               - (mem.ds[il, 0] - mem.drs[il, 0]) * (mem.ds[il, 1] - mem.drs[il, 1]))
            pref = SQRT_8_OVER_PI * 0.5 * rho
            a_i = float(mem.a_i[il])
            if _uses_mcf(mem):
                # complex, frequency dependent transverse coefficient (raft_member.py:1415-1420, 1446);
                # the axial (end) term stays real.  Imat holds the k -> 0 values for reference only.
                Iw = np.array(mem.Imat_MCF[il], dtype=complex)            # [3,3,nw]
                Imat = np.real(Iw[:, :, 0])
                in_q = np.real(np.einsum("a,abw,b->w", q, Iw, q))[0]
                w1 = np.einsum("a,abw,b->w", p1, Iw, p1)
                w2 = np.einsum("a,abw,b->w", p2, Iw, p2)
                in_p1, in_p2 = np.real(w1[0]), np.real(w2[0])
                resid = Iw - (in_q * np.outer(q, q)[:, :, None] + np.outer(p1, p1)[:, :, None] * w1 + np.outer(p2, p2)[:, :, None] * w2)
                mcf_flag.append(1)
            else:
                Imat = np.array(mem.Imat[il], dtype=float)
                in_q, in_p1, in_p2 = q @ Imat @ q, p1 @ Imat @ p1, p2 @ Imat @ p2
                resid = Imat - (in_q * np.outer(q, q) + in_p1 * np.outer(p1, p1) + in_p2 * np.outer(p2, p2))
                if any_mcf:
                    w1, w2 = np.full(nw, in_p1, dtype=complex), np.full(nw, in_p2, dtype=complex)
                    Iw = np.repeat(Imat[:, :, None], nw, axis=2).astype(complex)
                mcf_flag.append(0)
            if np.abs(resid).max() > 1e-9 * max(1.0, np.abs(Imat).max()):
                raise NotImplementedError("member %r: Imat is not diagonal in the member frame" % mem.name)
            if any_mcf:
                in_p1_w.append(w1), in_p2_w.append(w2), Imat_w.append(Iw)
            cols["r"].append(np.array(mem.r[il], dtype=float))
            cols["mem"].append(im)
            cols["ls"].append(ls)
            cols["cd_q"].append(pref * (a_q * Cd_q + a_End * Cd_End))
            cols["cd_p1"].append(pref * a_p1 * Cd_p1)
            cols["cd_p2"].append(pref * a_p2 * Cd_p2)
            cols["in_q"].append(in_q), cols["in_p1"].append(in_p1), cols["in_p2"].append(in_p2)
            cols["pa"].append(rho * g * a_i)
            cols["Imat"].append(Imat), cols["a_i"].append(a_i)
            cols["a_q"].append(a_q), cols["a_p1"].append(a_p1), cols["a_p2"].append(a_p2), cols["a_End"].append(a_End)
            cols["Cd_q"].append(Cd_q), cols["Cd_p1"].append(Cd_p1), cols["Cd_p2"].append(Cd_p2), cols["Cd_End"].append(Cd_End)
        mstart.append(len(cols["ls"]))

    ns = len(cols["ls"])
    out = dict(
        prp=prp, rho=np.float64(rho), g=np.float64(g),
        mem_q=np.array(mq, dtype=float).reshape(-1, 3), mem_p1=np.array(mp1, dtype=float).reshape(-1, 3),
        mem_p2=np.array(mp2, dtype=float).reshape(-1, 3), mem_rA=np.array(mrA, dtype=float).reshape(-1, 3),
        mem_circ=np.array(mcirc, dtype=np.int32), mem_start=np.array(mstart, dtype=np.int32),
        node_r=np.array(cols["r"], dtype=float).reshape(ns, 3), node_mem=np.array(cols["mem"], dtype=np.int32),
        node_Imat=np.array(cols["Imat"], dtype=float).reshape(ns, 3, 3),
    )
    for k in ("ls", "cd_q", "cd_p1", "cd_p2", "in_q", "in_p1", "in_p2", "pa", "a_i",
              "a_q", "a_p1", "a_p2", "a_End", "Cd_q", "Cd_p1", "Cd_p2", "Cd_End"):
        out["node_" + k] = np.array(cols[k], dtype=float)
    if any_mcf:
        # MacCamy-Fuchs: per-node, per-frequency complex transverse inertia coefficients [Ns,nw]
        out["node_in_p1_w"] = np.array(in_p1_w, dtype=complex).reshape(ns, nw)
        out["node_in_p2_w"] = np.array(in_p2_w, dtype=complex).reshape(ns, nw)
        out["node_Imat_w"] = np.array(Imat_w, dtype=complex).reshape(ns, 3, 3, nw)   # oracle only
    return out


def pack_matrices(fowt, nw):
    """Iteration-invariant system matrices of one FOWT (raft_model.py:1045-1047).

    M0 = M_struc + A_hydro_morison (+ sum A_aero is frequency dependent -> A_w)
    B0 = B_struc + sum B_gyro
    C0 = C_struc + C_hydro + C_moor + C_elast
    A_w, B_w [6,6,nw]: frequency-dependent parts (A_BEM + sum A_aero, B_BEM + sum B_aero) or None.
    moorMod 2 (frequency-independent M/A/B_moor from MoorPy) is folded in by the caller if needed.
    """
    n = fowt.nDOF
    if n != 6:
        raise NotImplementedError("only 6-DOF rigid FOWTs are supported (nDOF=%d)" % n)
    M0 = np.array(fowt.M_struc, dtype=float) + np.array(fowt.A_hydro_morison, dtype=float)
    B0 = np.array(fowt.B_struc, dtype=float)
    B_gyro = getattr(fowt, "B_gyro", None)
    if B_gyro is not None and np.size(B_gyro):
        B0 = B0 + np.sum(B_gyro, axis=2)
    C0 = (np.array(fowt.C_struc, dtype=float) + np.array(fowt.C_hydro, dtype=float)
          + np.array(fowt.C_moor, dtype=float) + np.array(fowt.C_elast, dtype=float))
    A_w = np.zeros([n, n, nw])
    B_w = np.zeros([n, n, nw])
    have = False
    if getattr(fowt, "nrotors", 0) > 0:
        A_w += np.sum(fowt.A_aero, axis=3)
        B_w += np.sum(fowt.B_aero, axis=3)
        have = True
    A_BEM = getattr(fowt, "A_BEM", None)
    if A_BEM is not None and np.any(A_BEM):
        A_w += A_BEM
        have = True
    B_BEM = getattr(fowt, "B_BEM", None)
    if B_BEM is not None and np.any(B_BEM):
        B_w += B_BEM
        have = True
    out = dict(M0=M0, B0=B0, C0=C0)
    if have:
        # the reference's own layout [6,6,nw] (frequency fastest) -> coalesced per-frequency reads
        out["A_w"] = np.ascontiguousarray(A_w)
        out["B_w"] = np.ascontiguousarray(B_w)
    return out


def pack_operating_points(states):
    """Per-case aero-servo added mass and damping of FOWTs (raftk_cases.op, ``solver.CaseTable(ops=)``).

    ``states[d][c]``: FOWT d right after the reference's ``calcTurbineConstants(case c)`` (raft_fowt.py:1514-1586) -- the live
    FOWT or a dict with A_aero [6,6,nw,nrot], B_aero [6,6,nw,nrot] and B_gyro [6,6,nrot].  Its operating point is
    A(w) = sum_r A_aero[:,:,w,r] and B(w) = sum_r B_aero[:,:,w,r] + sum_r B_gyro[:,:,r]: what that case adds to the FOWT's
    mass and damping (raft_model.py:1045-1047).  Cases whose tables are bit-identical over every design share one point.
    -> dict(op [nC] int32, A_w, B_w [nD, n_op, 6, 6, nw], n_op).  The design's own matrices (``pack_matrices``) must then
    not carry these terms."""
    get = lambda s, k: s[k] if isinstance(s, dict) else getattr(s, k)       # noqa: E731
    nD = len(states)
    nC = len(states[0]) if nD else 0
    if nD < 1 or nC < 1 or any(len(row) != nC for row in states):
        raise ValueError("states must hold one snapshot per case (the same count) for every design")
    nw = None
    tabs = []                                                       # [nC][nD] (A, B)
    for c in range(nC):
        row = []
        for d in range(nD):
            s = states[d][c]
            n = get(s, "nDOF") if not isinstance(s, dict) and hasattr(s, "nDOF") else np.shape(get(s, "A_aero"))[0]
            if n != 6:
                raise NotImplementedError("operating points: only rigid 6-DOF FOWTs here (the follow-up for flexible FOWTs, "
                                          "raftk_general_*, is pack_general_operating_points)")
            A, B, G = (np.asarray(get(s, k), dtype=float) for k in ("A_aero", "B_aero", "B_gyro"))
            nw = A.shape[2] if nw is None and A.ndim == 4 else nw
            if A.ndim != 4 or A.shape[:2] != (6, 6) or B.shape != A.shape or A.shape[2] != nw or G.shape != (6, 6, A.shape[3]):
                raise ValueError("operating point of design %d, case %d: A_aero / B_aero must be [6,6,%s,nrot] and B_gyro [6,6,nrot]"
                                 % (d, c, nw))
            row.append((np.sum(A, axis=3), np.sum(B, axis=3) + np.sum(G, axis=2)[:, :, None]))
        tabs.append(row)
    op = np.zeros(nC, dtype=np.int32)
    seen, first = {}, []
    for c, row in enumerate(tabs):
        key = b"".join(np.ascontiguousarray(t).tobytes() for pair in row for t in pair)
        if key not in seen:
            seen[key] = len(first)
            first.append(c)
        op[c] = seen[key]
    A_w = np.ascontiguousarray([[tabs[c][d][0] for c in first] for d in range(nD)])
    B_w = np.ascontiguousarray([[tabs[c][d][1] for c in first] for d in range(nD)])
    return dict(op=op, A_w=A_w, B_w=B_w, n_op=len(first))


def pack_bem_excitation(fowt):
    """BEM excitation coefficient table for heading interpolation (raft_fowt.py:1796-1849).

    Returns ``None`` when the FOWT has no potential-flow excitation, else a dict with
    X_BEM [nhead, 6, nw] complex128 (the reference's layout), headings [nhead] (deg), heading_adjust.
    """
    if not (getattr(fowt, "potMod", False) or getattr(fowt, "potModMaster", 0) in (2, 3)):
        return None
    X = getattr(fowt, "X_BEM", None)
    if X is None:
        return None
    X = np.asarray(X)
    return dict(X_BEM=np.ascontiguousarray(X[:, :6, :]).astype(np.complex128),
                bem_headings=np.array(fowt.BEM_headings, dtype=float),
                heading_adjust=np.float64(fowt.heading_adjust))


def _skew(r):
    """H(r) with H(r) f = r x f (the moment rows of translateForce3to6DOF, helpers.py:468-483)."""
    return np.array([[0.0, -r[2], r[1]], [r[2], 0.0, -r[0]], [-r[1], r[0], 0.0]])


def _submerged_rotors(fowt):
    return [rot for rot in (getattr(fowt, "rotorList", None) or []) if np.asarray(rot.r3, dtype=float)[2] < 0]


def pack_rotor_excitation(fowt):
    """Inertial wave excitation of the FOWT's submerged rotors (MHK turbines; raft_fowt.py:1859-1888), duck-typed on a live
    FOWT: ``rotorList`` (``r3``, ``I_hydro``, ``R_q``, ``nodeList[0].id``), ``T`` and ``r6``.

    Per rotor with r3[2] < 0 the reference adds f6 = [f3; (r3 - r6) x f3 + I[3:,:3] ud] with f3 = I[:3,:3] ud,
    I = rotateMatrix6(I_hydro, R_q), to the hub node's rows of F_hydro_iner_fullDOF, and projects it through fowt.T.  So the
    reduced force is G ud with the real G = T_node^T ([I3; H(r3 - r6)] I[:3,:3] + [0; I[3:,:3]]) [6,3], T_node the hub node's
    6 rows of T; ud = i w u is the wave acceleration of getWaveKin at r3 (the kernels evaluate it per bin and wave train).
    The force is taken about the PRP and then through T_node, which for a hub node tied rigidly to the PRP adds the lever arm
    a second time -- the reference's arithmetic, kept.  The rotor's added mass is not packed here: the reference already
    has it in A_hydro_morison (raft_fowt.py:1616-1625), which ``pack_matrices`` puts into M0.
    -> dict(rot_r3 [nR,3], rot_G [nR,6,3]), empty without submerged rotors.  ValueError when a submerged rotor has no
    I_hydro (calcHydroConstants has not run)."""
    rotors = _submerged_rotors(fowt)
    if not rotors:
        return {}
    T = np.asarray(fowt.T, dtype=float)
    r6 = np.asarray(fowt.r6, dtype=float)
    r3s, Gs = [], []
    for rot in rotors:
        if getattr(rot, "I_hydro", None) is None:
            raise ValueError("submerged rotor at r3 = %s has no I_hydro: run calcHydroConstants first" % list(np.asarray(rot.r3)))
        R = np.asarray(rot.R_q, dtype=float)
        I6 = np.asarray(rot.I_hydro, dtype=float)
        I = np.zeros([6, 6])                     # rotateMatrix6 (helpers.py:604-640): the lower-left block is the upper-right's transpose
        I[:3, :3] = np.matmul(np.matmul(R, I6[:3, :3]), R.T)
        I[:3, 3:] = np.matmul(np.matmul(R, I6[:3, 3:]), R.T)
        I[3:, :3] = I[:3, 3:].T
        r3 = np.asarray(rot.r3, dtype=float)
        L = np.vstack([I[:3, :3], _skew(r3 - r6[:3]) @ I[:3, :3] + I[3:, :3]])
        nid = int(rot.nodeList[0].id)
        Gs.append(T[6 * nid:6 * nid + 6, :].T @ L)
        r3s.append(r3)
    if Gs[0].shape[0] != 6:
        raise NotImplementedError("rotor excitation: only rigid 6-DOF FOWTs (fowt.T must be [nFullDOF, 6])")
    return dict(rot_r3=np.array(r3s), rot_G=np.array(Gs))


def pack_fowt(fowt, w=None, k=None):
    """Everything the kernels need for one FOWT design: node/member tables, matrices, grid, and the excitation table of its
    submerged rotors (``pack_rotor_excitation``, or the ``rotor_excitation`` dict(r3, G) injected into a FOWT that builds no
    rotors: r3 relative to the FOWT's (x_ref, y_ref), G as pack_rotor_excitation gives it)."""
    w = np.array(fowt.w if w is None else w, dtype=float)
    k = np.array(fowt.k if k is None else k, dtype=float)
    out = pack_members(fowt)
    out.update(pack_matrices(fowt, len(w)))
    bem = pack_bem_excitation(fowt)
    if bem is not None:
        out.update(bem)
    out.update(w=w, k=k, depth=np.float64(fowt.depth), dw=np.float64(w[1] - w[0]),
               x_ref=np.float64(getattr(fowt, "x_ref", 0.0)), y_ref=np.float64(getattr(fowt, "y_ref", 0.0)))
    out.update(pack_qtf(fowt))
    inj = getattr(fowt, "rotor_excitation", None)
    if inj is None:
        out.update(pack_rotor_excitation(fowt))
    elif len(inj["r3"]):
        # injected hubs are relative to the FOWT's reference point (x_ref, y_ref), so that one table serves every FOWT of an
        # array; G is a global-frame matrix and does not turn with heading_adjust
        if float(getattr(fowt, "heading_adjust", 0.0)) != 0.0:
            raise NotImplementedError("an injected rotor_excitation table on a FOWT with heading_adjust != 0: G would have to "
                                      "turn with the FOWT; pack the rotated rotor with pack_rotor_excitation instead")
        off = np.array([float(getattr(fowt, "x_ref", 0.0)), float(getattr(fowt, "y_ref", 0.0)), 0.0])
        out.update(rot_r3=np.asarray(inj["r3"], dtype=float).reshape(-1, 3) + off, rot_G=np.asarray(inj["G"], dtype=float).reshape(-1, 6, 3))
    return out


def pack_eigen(fowt):
    """Mass and stiffness of FOWT.solveEigen (raft_fowt.py:1646-1660), duck-typed on a live FOWT, with the reference's own
    summation order: M = M_struc + A_hydro_morison + A_BEM[:, :, 0] (the BEM added mass at the grid's first bin) and
    C = fowt.getStiffness() when the object has it (which includes a MoorPy body's stiffness), else the same sum from the
    attributes: C_moor, yawstiff on DOF 5, body.getStiffness() of an attached body, then C_struc + C_hydro + C_elast
    (raft_fowt.py:1628-1644).  -> dict(M, C [nDOF,nDOF])."""
    n = int(fowt.nDOF)
    A_BEM = getattr(fowt, "A_BEM", None)
    A0 = np.asarray(A_BEM)[:, :, 0] if A_BEM is not None and np.size(A_BEM) else np.zeros([n, n])
    M = fowt.M_struc + fowt.A_hydro_morison + A0
    if hasattr(fowt, "getStiffness"):
        C = fowt.getStiffness()
    else:
        C = np.zeros([n, n])
        C += fowt.C_moor
        C[5, 5] += getattr(fowt, "yawstiff", 0.0)
        if getattr(fowt, "body", None):
            C += fowt.body.getStiffness()
        C += fowt.C_struc + fowt.C_hydro + fowt.C_elast
    return dict(M=np.array(M, dtype=float), C=np.array(C, dtype=float))


def pack_general_dofs(fowt):
    """Node tables + the per-strip-node blocks of ``fowt.T`` for FOWTs with generalised degrees of freedom (flexible
    members, nDOF > 6; raft_fowt.py:1854-1857, 1913-1929).  GROUNDWORK for the next row: so far only the CPU checker
    of the tests consumes these tables -- the CUDA path is rigid 6-DOF and ``pack_fowt`` keeps rejecting flexible members.
    Adds ``gen_nDOF``, ``gen_Tn`` [Ns,6,nDOF] (T rows of each strip node's structural node) and ``gen_rr`` [Ns,3]
    (offset from that node; zero on flexible members, whose strip nodes are their structural nodes).
    The nodes of potential-flow members (potMod) carry no strip-theory inertial excitation (raft_member.py:1980): their
    ``node_a_i`` is zero, like their Imat, and their wave force comes from the BEM table (``pack_general_matrices``).
    NotImplementedError for a FOWT with a submerged rotor: its inertial wave excitation (raft_fowt.py:1859-1888) is not part
    of the generalised-DOF solve."""
    _no_submerged_rotor(fowt)
    out = pack_members(fowt, allow_flexible=True)
    T = np.asarray(fowt.T, dtype=float)
    Tn, rr, pot = [], [], []
    for mem in fowt.memberList:
        sub = np.where(mem.r[:, 2] < 0)[0]
        for il in sub:
            node = mem.nodeList[0] if getattr(mem, "type", "rigid") == "rigid" else mem.nodeList[il]
            Tn.append(T[node.id * 6:(node.id + 1) * 6, :])
            rr.append(np.asarray(mem.r[il], dtype=float) - np.asarray(node.r[:3], dtype=float))
            pot.append(bool(getattr(mem, "potMod", False)))
    ns = len(out["node_ls"])
    if any(pot):
        out["node_a_i"] = np.where(np.array(pot), 0.0, out["node_a_i"])
    out.update(gen_nDOF=np.int32(T.shape[1]), gen_Tn=np.array(Tn, dtype=float).reshape(ns, 6, T.shape[1]),
               gen_rr=np.array(rr, dtype=float).reshape(ns, 3), w=np.array(fowt.w, dtype=float), k=np.array(fowt.k, dtype=float),
               depth=np.float64(fowt.depth), dw=np.float64(fowt.w[1] - fowt.w[0]),
               M0=np.zeros([6, 6]), B0=np.zeros([6, 6]), C0=np.zeros([6, 6]))
    return out


def pack_general_matrices(fowt, states=None):
    """System matrices of a FOWT with generalised degrees of freedom (raft_model.py:1045-1047), split into the constant part
    and the frequency-dependent part the solver adds on its support (C ABI ``raftk_general_fd``).  Duck-typed on a live FOWT.

    Returns dict(M, B, C [nDOF,nDOF], fd):
      M = M_struc + A_hydro_morison;  B = B_struc + sum B_gyro;  C = C_struc + C_hydro + C_moor + C_elast
      fd: ``fd_idx`` [n_fd] int32, the reduced DOFs whose rows or columns of sum A_aero + A_BEM or sum B_aero + B_BEM are
      nonzero (the rotor nodes' DOFs and DOFs 0-5, where readHydro lumps the BEM coefficients; raft_fowt.py:1479-1480,
      1557-1562); ``A_w``, ``B_w`` [n_fd,n_fd,nw] those sums restricted to it (every entry outside it is exactly zero);
      ``pack_bem_excitation``'s table (``X_BEM`` [nhead,6,nw] in full DOFs 0-5, ``bem_headings``, ``heading_adjust``) or
      none; ``T0`` [6,nDOF] = rows 0-5 of ``fowt.T`` (F_BEM = T^T F_BEM_fullDOF, raft_fowt.py:1885-1887); ``x_ref``, ``y_ref``.
    A FOWT without operating rotors and without BEM coefficients gets n_fd = 0.

    ``states``: one turbine state per load case, as ``pack_general_operating_points`` takes them for one design (the live
    FOWT right after ``calcTurbineConstants(case)``, or a dict).  The FOWT's own A_aero, B_aero and B_gyro are then ignored:
    B = B_struc; ``fd_idx`` is the union of the BEM support and the support of every state; ``fd``'s A_w / B_w carry the BEM
    terms alone (zero on the DOFs only the operating points touch); and the result gains ``ops``, the
    ``pack_general_operating_points`` dict on that support, for ``solver.CaseTable(ops=)``.
    NotImplementedError for a FOWT with a submerged rotor (``pack_general_dofs``)."""
    _no_submerged_rotor(fowt)
    n, nw = int(fowt.nDOF), len(fowt.w)
    M = np.array(fowt.M_struc, dtype=float) + np.array(fowt.A_hydro_morison, dtype=float)
    B = np.array(fowt.B_struc, dtype=float)
    B_gyro = getattr(fowt, "B_gyro", None)
    if states is None and B_gyro is not None and np.size(B_gyro):
        B = B + np.sum(B_gyro, axis=2)
    C = (np.array(fowt.C_struc, dtype=float) + np.array(fowt.C_hydro, dtype=float)
         + np.array(fowt.C_moor, dtype=float) + np.array(fowt.C_elast, dtype=float))
    A_w, B_w = np.zeros([n, n, nw]), np.zeros([n, n, nw])
    if states is None and getattr(fowt, "nrotors", 0) > 0:
        A_w = A_w + np.sum(fowt.A_aero, axis=3)
        B_w = B_w + np.sum(fowt.B_aero, axis=3)
    for name, acc in (("A_BEM", A_w), ("B_BEM", B_w)):
        t = getattr(fowt, name, None)
        if t is not None and np.size(t):
            acc += np.asarray(t, dtype=float)
    nz = np.any(A_w != 0, axis=2) | np.any(B_w != 0, axis=2)
    sup = nz.any(axis=0) | nz.any(axis=1)
    if states is not None:
        for s in states:
            sup |= _general_state_support(s)
    idx = np.nonzero(sup)[0].astype(np.int32)
    fd = dict(fd_idx=idx, A_w=np.ascontiguousarray(A_w[np.ix_(idx, idx)]), B_w=np.ascontiguousarray(B_w[np.ix_(idx, idx)]),
              T0=np.ascontiguousarray(np.asarray(fowt.T, dtype=float)[:6]),
              x_ref=np.float64(getattr(fowt, "x_ref", 0.0)), y_ref=np.float64(getattr(fowt, "y_ref", 0.0)))
    bem = pack_bem_excitation(fowt)
    if bem is not None:
        fd.update(bem)
    out = dict(M=M, B=B, C=C, fd=fd)
    if states is not None:
        out["ops"] = pack_general_operating_points([states], idx)
    return out


def _no_submerged_rotor(fowt):
    if _submerged_rotors(fowt):
        raise NotImplementedError("generalised DOFs: the inertial wave excitation of submerged rotors (MHK, raft_fowt.py:1859-1888) "
                                  "is on the rigid 6-DOF path only")


def _general_state(s):
    """(A_aero [n,n,nw,nrot], B_aero, B_gyro [n,n,nrot]) of one turbine state (live FOWT or dict), float arrays."""
    get = (lambda k: s[k]) if isinstance(s, dict) else (lambda k: getattr(s, k))     # noqa: E731
    return tuple(np.asarray(get(k), dtype=float) for k in ("A_aero", "B_aero", "B_gyro"))


def _general_state_support(s):
    """Reduced DOFs whose rows or columns of a turbine state's A_aero, B_aero or B_gyro hold a nonzero entry -> bool [n]."""
    A, B, G = _general_state(s)
    nz = np.any(A != 0, axis=(2, 3)) | np.any(B != 0, axis=(2, 3)) | np.any(G != 0, axis=2)
    return nz.any(axis=0) | nz.any(axis=1)


def pack_general_operating_points(states, fd_idx):
    """Per-case aero-servo added mass and damping of FOWTs with generalised degrees of freedom (raftk_cases.op on the
    raftk_general_* solves, ``solver.CaseTable(ops=)``), on the support ``fd_idx`` of their frequency-dependent terms.

    ``states[d][c]``: design d right after the reference's ``calcTurbineConstants(case c)`` (raft_fowt.py:1514-1586) -- the
    live FOWT or a dict with A_aero [n,n,nw,nrot], B_aero [n,n,nw,nrot] and B_gyro [n,n,nrot] in reduced DOFs (the reference's
    own T^T a T of the rotor node).  Its operating point is A(w) = sum_r A_aero[:,:,w,r] and B(w) = sum_r B_aero[:,:,w,r] +
    sum_r B_gyro[:,:,r] (the gyroscopic term in every bin), restricted to ``fd_idx`` ([n_fd] for every design, or [nD, n_fd]).
    Cases whose tables are bit-identical over every design share one point.  -> dict(op [nC] int32, A_w, B_w
    [nD, n_op, n_fd, n_fd, nw], n_op).  ValueError when a state is nonzero off ``fd_idx`` or its shapes disagree; the
    design's own matrices (``pack_general_matrices(fowt, states=...)``) must then not carry these terms."""
    nD = len(states)
    nC = len(states[0]) if nD else 0
    if nD < 1 or nC < 1 or any(len(row) != nC for row in states):
        raise ValueError("states must hold one snapshot per case (the same count) for every design")
    idx = np.asarray(fd_idx, dtype=np.int64)
    idx = np.broadcast_to(idx, (nD,) + idx.shape[-1:]) if idx.ndim == 1 else idx
    if idx.ndim != 2 or idx.shape[0] != nD or idx.shape[1] < 1:
        raise ValueError("fd_idx must be [n_fd] or [nD, n_fd] with n_fd >= 1")
    shape = None
    tabs = []                                                       # [nC][nD] (A, B)
    for c in range(nC):
        row = []
        for d in range(nD):
            A, B, G = _general_state(states[d][c])
            shape = A.shape[:3] if shape is None else shape
            n = A.shape[0] if A.ndim == 4 else -1
            if A.ndim != 4 or A.shape[:3] != shape or A.shape[1] != n or B.shape != A.shape or G.shape != (n, n, A.shape[3]):
                raise ValueError("operating point of design %d, case %d: A_aero / B_aero must be [n,n,nw,nrot] (%s) and B_gyro "
                                 "[n,n,nrot]" % (d, c, list(shape)))
            if np.any(idx[d] < 0) or np.any(idx[d] >= n):
                raise ValueError("fd_idx of design %d: entries outside [0, %d)" % (d, n))
            off = np.ones(n, dtype=bool)
            off[idx[d]] = False
            Ad, Bd = np.sum(A, axis=3), np.sum(B, axis=3) + np.sum(G, axis=2)[:, :, None]
            if np.any(Ad[off]) or np.any(Ad[:, off]) or np.any(Bd[off]) or np.any(Bd[:, off]) or np.any(G[off]) or np.any(G[:, off]):
                raise ValueError("operating point of design %d, case %d is nonzero off fd_idx (pack_general_matrices(fowt, "
                                 "states=...) takes the union of the supports)" % (d, c))
            sub = np.ix_(idx[d], idx[d])
            row.append((np.ascontiguousarray(Ad[sub]), np.ascontiguousarray(Bd[sub])))
        tabs.append(row)
    op = np.zeros(nC, dtype=np.int32)
    seen, first = {}, []
    for c, row in enumerate(tabs):
        key = b"".join(t.tobytes() for pair in row for t in pair)
        if key not in seen:
            seen[key] = len(first)
            first.append(c)
        op[c] = seen[key]
    A_w = np.ascontiguousarray([[tabs[c][d][0] for c in first] for d in range(nD)])
    B_w = np.ascontiguousarray([[tabs[c][d][1] for c in first] for d in range(nD)])
    return dict(op=op, A_w=A_w, B_w=B_w, n_op=len(first))


def pack_qtf(fowt):
    """External difference-frequency QTF of a FOWT (state left by FOWT.readQTF, raft_fowt.py:2081-2128):
    ``qtf`` complex [nw1, nw2, nheads, 6] (dimensional, Hermitian-filled), ``qtf_w`` [nw1] rad/s, ``qtf_heads``
    [nheads] rad.  Empty dict for potSecOrder 0; for potSecOrder 1 the member tables of the slender-body QTF
    (``pack_qtf_members``, keys ``qs_*``)."""
    sec = int(getattr(fowt, "potSecOrder", 0) or 0)
    if sec == 0:
        return {}
    if sec == 1:                                   # slender-body QTF, computed on the GPU from the member tables
        if int(getattr(fowt, "nDOF", 6)) != 6:
            raise NotImplementedError("slender-body QTF: rigid 6-DOF FOWTs only (the reference returns null QTFs otherwise, raft_fowt.py:2014)")
        return pack_qtf_members(fowt)
    w1, w2 = np.asarray(fowt.w1_2nd, dtype=float), np.asarray(fowt.w2_2nd, dtype=float)
    if w1.shape != w2.shape or not (w1 == w2).all():
        raise ValueError("Both frequency columns in the input QTF must contain the same values.")   # raft_fowt.py:2109
    return dict(qtf=np.ascontiguousarray(fowt.qtf, dtype=np.complex128), qtf_w=w1,
                qtf_heads=np.asarray(fowt.heads_2nd, dtype=float))


def pack_general_qtf(fowt):
    """External difference-frequency QTF of a FOWT with generalised degrees of freedom (nDOF > 6, potSecOrder 2) for the
    generalised-DOF solve (C ABI ``raftk_general_qtf``): ``qtf`` complex [nw1, nw1, nheads, 6], the reference's
    ``fowt.qtf`` [nw1, nw2, nheads, nDOF] cut to reduced DOFs 0-5 -- FOWT.readQTF fills only those from a .12d file and the
    force is lumped there (raft_fowt.py:2112-2123, raft_model.py:1034) -- with ``qtf_w`` [nw1] rad/s and ``qtf_heads``
    [nheads] rad.  Empty dict for potSecOrder 0.  ValueError if any DOF from 6 up carries a nonzero entry (the solve would drop
    it); NotImplementedError for potSecOrder 1, where the reference uses null QTFs for such FOWTs (raft_fowt.py:2015-2017)."""
    sec = int(getattr(fowt, "potSecOrder", 0) or 0)
    if sec == 0:
        return {}
    if sec == 1:
        raise NotImplementedError("slender-body QTF of a FOWT with generalised DOFs: the reference uses null QTFs there "
                                  "(raft_fowt.py:2015-2017)")
    w1, w2 = np.asarray(fowt.w1_2nd, dtype=float), np.asarray(fowt.w2_2nd, dtype=float)
    if w1.shape != w2.shape or not (w1 == w2).all():
        raise ValueError("Both frequency columns in the input QTF must contain the same values.")   # raft_fowt.py:2109
    q = np.asarray(fowt.qtf, dtype=np.complex128)
    if q.ndim != 4 or q.shape[3] < 6:
        raise ValueError("fowt.qtf must be [nw1, nw2, nheads, nDOF] with nDOF >= 6")
    if np.any(q[..., 6:] != 0):
        raise ValueError("fowt.qtf has nonzero entries on reduced DOFs 6 and up; the generalised-DOF solve loads DOFs 0-5 only")
    return dict(qtf=np.ascontiguousarray(q[..., :6]), qtf_w=w1, qtf_heads=np.asarray(fowt.heads_2nd, dtype=float))


def pack_qtf_members(fowt):
    """Tables of the slender-body QTF (potSecOrder 1; C ABI ``raftk_slender``), duck-typed on the reference's FOWT / Member
    objects.  Hoists what Member.calcQTF_slenderBody / correction_KAY evaluate inside their frequency-pair loops
    (raft_member.py:1560-1571 strip volume and coefficients, :1620-1625 end volume, :1528 waterline intersection,
    :1660-1674 waterline area, :1721-1760 Kim & Yue waterline point and integration segments).  Keys ``qs_*``; the
    submerged nodes and their order are those of ``pack_members``."""
    rho, g = float(fowt.rho_water), float(fowt.g)
    mq, mp1, mp2, mmcf, mwl, mrint, mawl, mrwl, mRwl = [], [], [], [], [], [], [], [], []
    cols = {k: [] for k in ("mem", "r", "v_side", "Ca_p1", "Ca_p2", "Ca_End", "v_end", "a_i")}
    seg = {k: [] for k in ("mem", "z1", "z2", "R", "rmid")}
    for mem in fowt.memberList:
        sub = np.where(mem.r[:, 2] < 0)[0]
        if len(sub) == 0:
            continue
        im = len(mq)
        circ = mem.shape == "circular"
        mq.append(np.array(mem.q, dtype=float)), mp1.append(np.array(mem.p1, dtype=float)), mp2.append(np.array(mem.p2, dtype=float))
        for il in sub:
            ls = float(mem.ls[il])
            if circ:
                v_i = 0.25 * np.pi * mem.ds[il] ** 2 * mem.dls[il]
            else:
                v_i = mem.ds[il, 0] * mem.ds[il, 1] * mem.dls[il]
            if mem.r[il, 2] + 0.5 * mem.dls[il] > 0:
                v_i = v_i * (0.5 * mem.dls[il] - mem.r[il, 2]) / mem.dls[il]
            if circ:
                v_e = np.pi / 12.0 * abs((mem.ds[il] + mem.drs[il]) ** 3 - (mem.ds[il] - mem.drs[il]) ** 3)
            else:
                v_e = np.pi / 12.0 * ((np.mean(mem.ds[il] + mem.drs[il])) ** 3 - (np.mean(mem.ds[il] - mem.drs[il])) ** 3)
            cols["mem"].append(im), cols["r"].append(np.array(mem.r[il], dtype=float))
            cols["v_side"].append(v_i), cols["v_end"].append(v_e), cols["a_i"].append(float(mem.a_i[il]))
            cols["Ca_p1"].append(np.interp(ls, mem.stations, mem.Ca_p1)), cols["Ca_p2"].append(np.interp(ls, mem.stations, mem.Ca_p2))
            cols["Ca_End"].append(np.interp(ls, mem.stations, mem.Ca_End))
        wl = bool(mem.r[-1, 2] * mem.r[0, 2] < 0)
        r_int, a_wl = np.zeros(3), 0.0
        if wl:
            r_int = mem.r[0, :] + (mem.r[-1, :] - mem.r[0, :]) * (0. - mem.r[0, 2]) / (mem.r[-1, 2] - mem.r[0, 2])
            i_wl = np.where(mem.r[:, 2] < 0)[0][-1]
            if circ:
                d_wl = 0.5 * (mem.ds[i_wl] + mem.ds[i_wl + 1]) if i_wl != len(mem.ds) - 1 else mem.ds[i_wl]
                a_wl = 0.25 * np.pi * d_wl ** 2
            else:
                if i_wl != len(mem.ds) - 1:
                    d1, d2 = 0.5 * (mem.ds[i_wl, 0] + mem.ds[i_wl + 1, 0]), 0.5 * (mem.ds[i_wl, 1] + mem.ds[i_wl + 1, 1])
                else:
                    d1, d2 = mem.ds[i_wl, 0], mem.ds[i_wl, 1]
                a_wl = d1 * d2
        kay = bool(getattr(mem, "MCF", False)) and bool(mem.rA[2] * mem.rB[2] < 0)
        rwl, Rwl = np.zeros(3), 1.0
        if kay:
            rwl = mem.rA + (mem.rB - mem.rA) * (0 - mem.rA[2]) / (mem.rB[2] - mem.rA[2])
            Rwl = float(np.interp(0, mem.r[:, 2], 0.5 * np.array(mem.ds)))
            for il, r1 in enumerate(mem.r[:-1]):
                z1 = r1[2]
                if z1 > 0:
                    continue
                r2 = mem.r[il + 1]
                z2 = 0 if r2[2] > 0 else r2[2]
                R1 = mem.ds[il] / 2
                if mem.dls[il] == 0:
                    R1 = mem.ds[il]
                R2 = mem.ds[il + 1] / 2
                if mem.dls[il + 1] == 0:
                    R2 = mem.ds[il]
                seg["mem"].append(im), seg["z1"].append(z1), seg["z2"].append(z2), seg["R"].append(0.5 * (R1 + R2)), seg["rmid"].append(0.5 * (r1 + r2))
        mmcf.append(1 if kay else 0), mwl.append(1 if wl else 0), mrint.append(r_int), mawl.append(a_wl), mrwl.append(rwl), mRwl.append(Rwl)
    ns, nm, nsg = len(cols["mem"]), len(mq), len(seg["mem"])
    out = dict(qs_mem_q=np.array(mq).reshape(nm, 3), qs_mem_p1=np.array(mp1).reshape(nm, 3), qs_mem_p2=np.array(mp2).reshape(nm, 3),
               qs_mem_mcf=np.array(mmcf, dtype=np.int32), qs_mem_wl=np.array(mwl, dtype=np.int32),
               qs_mem_r_int=np.array(mrint, dtype=float).reshape(nm, 3), qs_mem_a_wl=np.array(mawl, dtype=float),
               qs_mem_rwl=np.array(mrwl, dtype=float).reshape(nm, 3), qs_mem_R_wl=np.array(mRwl, dtype=float),
               qs_node_mem=np.array(cols["mem"], dtype=np.int32), qs_node_r=np.array(cols["r"], dtype=float).reshape(ns, 3),
               qs_seg_mem=np.array(seg["mem"], dtype=np.int32), qs_seg_z1=np.array(seg["z1"], dtype=float), qs_seg_z2=np.array(seg["z2"], dtype=float),
               qs_seg_R=np.array(seg["R"], dtype=float), qs_seg_rmid=np.array(seg["rmid"], dtype=float).reshape(nsg, 3),
               qs_M_struc=np.array(fowt.M_struc, dtype=float), qs_w=np.array(fowt.w1_2nd, dtype=float), qs_k=np.array(fowt.k1_2nd, dtype=float),
               qs_depth=np.float64(fowt.depth), qs_rho=np.float64(rho), qs_g=np.float64(g))
    for k in ("v_side", "Ca_p1", "Ca_p2", "Ca_End", "v_end", "a_i"):
        out["qs_node_" + k] = np.array(cols[k], dtype=float)
    return out


def pack_turbine_channels(fowt):
    """Turbine output channels of ``FOWT.saveTurbineOutputs`` as linear functionals of the 6-DOF response, for
    ``solver.channel_stats`` (C ABI ``raftk_channel_stats_*``).  Duck-typed on a live FOWT with rotors and RIGID towers:

      AxRNA, AyRNA, AzRNA  hub acceleration  w^2 (T_hub Xi)[0..2]                       raft_fowt.py:2422-2444
      Mbase                tower-base fore-aft bending moment  M_I + M_w + M_X_aero       raft_fowt.py:2504-2538

    Returns dict(names [(name, rotor index)], coef complex [nch,6,nw], avg [nch]) or None without rotors.
    ``avg`` follows the reference's mean values (:2428, :2435, :2442, :2533; the Mbase mean needs the statics results
    ``fowt.Xi0`` / ``fowt.f_aero0`` and is 0 when they are absent)."""
    from .bem import translate_matrix_6to6
    rotors = list(getattr(fowt, "rotorList", []) or [])
    if not rotors:
        return None
    w = np.asarray(fowt.w, dtype=float)
    nw, g = len(w), float(fowt.g)
    T_full = np.asarray(fowt.T, dtype=float)
    if T_full.shape[1] != 6:
        raise NotImplementedError("turbine channels: only rigid 6-DOF FOWTs (fowt.T must be [nFullDOF, 6])")
    names, coef, avg = [], [], []
    for ir, rotor in enumerate(rotors):
        node = rotor.nodeList[0]
        T = T_full[node.id * 6:(node.id + 1) * 6, :]                     # hub motion = T Xi (raft_model.py:1255)
        means = (abs(np.sin(node.r[4]) * g), abs(np.sin(node.r[3]) * g), abs(g))
        for ax, nm in enumerate(("AxRNA", "AyRNA", "AzRNA")):
            names.append((nm, ir))
            coef.append(T[ax][:, None] * (w ** 2)[None, :] + 0j)
            avg.append(means[ax])
        mem_tower = fowt.memberList[fowt.nplatmems + ir]
        if getattr(mem_tower, "type", "rigid") != "rigid":
            raise NotImplementedError("turbine channels: flexible towers (finite-element internal loads, raft_fowt.py:2541) are outside the GPU path")
        mRNA, IrRNA, zRNA = float(rotor.mRNA), float(rotor.IrRNA), float(rotor.r_rel[2])
        mtow = float(fowt.mtower[ir])
        m_turb = mtow + mRNA                                              # :2509
        zCG = (float(fowt.rCG_tow[ir][2]) * mtow + zRNA * mRNA) / m_turb  # :2510
        zBase = float(mem_tower.rA[2])
        hArm = zCG - zBase
        r_shift = np.asarray(mem_tower.nodeList[0].r0[:3], dtype=float) - np.array([0.0, 0.0, zCG])
        ICG = translate_matrix_6to6(np.asarray(mem_tower.M_struc, dtype=float), r_shift)[4, 4] + mRNA * (zRNA - zCG) ** 2 + IrRNA   # :2518
        A00 = np.asarray(fowt.A_aero, dtype=float)[0, 0, :, ir] if np.ndim(getattr(fowt, "A_aero", 0)) == 4 else np.zeros(nw)
        B00 = np.asarray(fowt.B_aero, dtype=float)[0, 0, :, ir] if np.ndim(getattr(fowt, "B_aero", 0)) == 4 else np.zeros(nw)
        c = np.zeros([6, nw], dtype=complex)
        c[0] = m_turb * hArm * w ** 2                                     # -m aCG hArm, aCG = -w^2 (Xi_0 + zCG Xi_4)  (:2515, :2521)
        c[4] = (m_turb * hArm * zCG * w ** 2 + ICG * w ** 2               # ... and -ICG (-w^2 Xi_4)
                + m_turb * g * hArm                                       # weight moment (:2522)
                - (-w ** 2 * A00 + 1j * w * B00) * (zRNA - zBase) ** 2)   # aero reaction moment (:2526)
        names.append(("Mbase", ir))
        coef.append(c)
        mean = 0.0
        if hasattr(fowt, "Xi0") and hasattr(fowt, "f_aero0"):
            F6 = np.asarray(rotors[0].nodeList[0].T, dtype=float) @ np.asarray(fowt.f_aero0, dtype=float)[:, ir]
            mean = m_turb * g * hArm * np.sin(fowt.Xi0[4]) + (F6[4] - hArm * F6[0])     # transformForce(.., offset=[0,0,-hArm])[4]  (:2533)
        avg.append(float(mean))
    return dict(names=names, coef=np.array(coef), avg=np.array(avg, dtype=float))


def pack_general_channels(fowt, tensions=None):
    """Output channels of ``FOWT.saveTurbineOutputs`` for a FOWT with generalised degrees of freedom, as real linear
    functionals of the reduced response: Y_ch(w) = w^wpow[ch] sum_b R[ch,b] Xi[b,w]  (``solver.general_channel_stats``,
    C ABI ``raftk_general_channel_stats_*``).  Duck-typed on a live FOWT:

      surge, sway, heave, roll, pitch, yaw   PRP motions from the rigidBodyNode rows of fowt.T    raft_fowt.py:2299-2353
                                             (x + SmallRotate(-r0, theta); rotations in degrees)
      AxRNA, AyRNA, AzRNA  per rotor         hub acceleration w^2 (T_hub Xi)[0..2]                  :2401-2444
      FbaseX .. MbaseZ     per flexible tower  internal loads at the tower base -Kf[base] T_tower Xi  :2541-2597

    Like the reference (:2302), the rigidBodyNode rows are taken at ``rigidBodyNode.id``, not ``6 * id``.
    Returns dict(names [(name, rotor index or None)], R [nch, nDOF], wpow [nch] int32 (0, 1 or 2; the channels here use 0
    and 2), avg [nch]).  ``avg`` holds the
    reference's mean values (Xi0_PRP from r6, the hub node's r, the tower nodes' Xi0); 0 where those inputs are absent.
    A rigid tower's Mbase (:2508-2538) mixes w^0 and w^2 terms with the aero matrices and is not a channel of this form:
    NotImplementedError.
    ``tensions``: the FOWT's mooring (``pack_mooring_tensions`` result, a MoorPy system or {J, T0}, J [2L, 6] on the PRP
    motions) adds rows ("Tmoor", line end k) = J[k] @ R_PRP with R_PRP in radians (:2355-2399), and
    ``tension`` = dict(row0, T0, w0) so that ``solver.general_case_metrics`` reports them as the reference's Tmoor_* arrays."""
    T = np.asarray(fowt.T, dtype=float)
    g = float(fowt.g)
    names, R, wpow, avg = [], [], [], []

    def add(name, ir, row, p, mean):
        names.append((name, ir)), R.append(np.asarray(row, dtype=float)), wpow.append(p), avg.append(float(mean))
    rb = fowt.rigidBodyNode
    Trb = T[rb.id:rb.id + 6, :]
    r = -np.asarray(rb.r0, dtype=float)[:3]
    S = np.array([[0.0, r[2], -r[1]], [-r[2], 0.0, r[0]], [r[1], -r[0], 0.0]])      # SmallRotate(r, th) = S th (helpers.py:396)
    r6 = np.asarray(getattr(fowt, "r6", np.zeros(6)), dtype=float)
    Xi0 = r6 - np.array([float(getattr(fowt, "x_ref", 0.0)), float(getattr(fowt, "y_ref", 0.0)), 0, 0, 0, 0])
    for a, nm in enumerate(("surge", "sway", "heave")):
        add(nm, None, Trb[a] + S[a] @ Trb[3:], 0, Xi0[a])
    for a, nm in enumerate(("roll", "pitch", "yaw")):
        add(nm, None, np.rad2deg(Trb[3 + a]), 0, np.rad2deg(Xi0[3 + a]))
    rotors = list(getattr(fowt, "rotorList", []) or [])
    for ir, rotor in enumerate(rotors):
        node = rotor.nodeList[0]
        Th = T[node.id * 6:(node.id + 1) * 6, :]
        means = (abs(np.sin(node.r[4]) * g), abs(np.sin(node.r[3]) * g), abs(g))
        for ax, nm in enumerate(("AxRNA", "AyRNA", "AzRNA")):
            add(nm, ir, Th[ax], 2, means[ax])
    for ir, rotor in enumerate(rotors):
        tow = fowt.memberList[fowt.nplatmems + ir]
        if getattr(tow, "type", "rigid") == "rigid":
            raise NotImplementedError("generalised channels: the tower-base moment of a rigid tower (raft_fowt.py:2508-2538) mixes "
                                      "frequency powers and aero terms; only flexible towers are supported")
        i0, i1 = tow.nodeList[0].id, tow.nodeList[-1].id
        Kf = np.asarray(tow.Kf, dtype=float)
        base = slice(0, 6) if tow.nodeList[0].r0[2] <= tow.nodeList[-1].r0[2] else slice(Kf.shape[0] - 6, Kf.shape[0])   # :2555-2560
        Rb = -Kf[base] @ T[i0 * 6:(i1 + 1) * 6, :]
        X0 = np.concatenate([np.asarray(getattr(n, "Xi0", np.zeros(6)), dtype=float) for n in tow.nodeList])
        F0 = (-Kf @ X0)[base]
        for a, nm in enumerate(("FbaseX", "FbaseY", "FbaseZ", "MbaseX", "MbaseY", "MbaseZ")):
            add(nm, ir, Rb[a], 0, F0[a])
    out = dict(names=names, R=np.array(R).reshape(len(names), T.shape[1]), wpow=np.array(wpow, dtype=np.int32),
               avg=np.array(avg, dtype=float))
    if tensions is not None:
        # mooring line-end tensions J @ Xi_PRP (:2355-2399, moorMod 0): PRP motions in metres and RADIANS -- the roll / pitch /
        # yaw rows above carry rad2deg and cannot be reused
        ten = tensions if isinstance(tensions, dict) and "n_lines" in tensions else pack_mooring_tensions(tensions)
        if ten["J"].shape[1] != 6:
            raise ValueError("the tension Jacobian of a FOWT must be [2L, 6] (its PRP motions)")
        R_prp = np.vstack([Trb[:3] + S @ Trb[3:], Trb[3:]])
        row0 = len(names)
        for k in range(len(ten["T0"])):
            add("Tmoor", k, ten["J"][k] @ R_prp, 0, ten["T0"][k])
        out.update(R=np.array(R).reshape(len(names), T.shape[1]), wpow=np.array(wpow, dtype=np.int32), avg=np.array(avg, dtype=float),
                   tension=dict(row0=row0, T0=ten["T0"].copy(), w0=float(np.asarray(fowt.w, dtype=float)[0])))
    return out


ROTOR_KEYS = ("omega_avg", "omega_std", "omega_max", "omega_min", "omega_PSD", "torque_avg", "torque_std", "torque_PSD",
              "power_avg", "bPitch_avg", "bPitch_std", "bPitch_PSD")


def pack_rotor_outputs(fowt, rotor_states, cases):
    """Inputs of the rotor channels of ``FOWT.saveTurbineOutputs`` (raft_fowt.py:2610-2679) for ``solver.rotor_stats`` /
    ``raftk_rotor_stats_*``.  Duck-typed on a live FOWT (``rotorList``, ``T``, the hub nodes' ``id``); ``rotor_states[c][ir]``
    is rotor ir after the reference's ``Rotor.calcAero`` for case c (CCBlade is out of scope), or a dict with the same
    attribute names: C, V_w (complex [nw]), kp_tau, ki_tau, kp_beta, ki_beta, Omega_case, aero_torque, Ng, aero_power,
    pitch_case, aeroServoMod, r3.  ``cases``: the case dicts, for the inflow speed.

    Rotor ir's hub row is column ir of the reference's stacked hub array XiHub[ih, ir, :] (:2402, :2423, :2644), that is
    DOF ir % 6 of rotor ir // 6's hub node: row 6 * rotorList[ir // 6].nodeList[0].id + ir % 6 of fowt.T.  With one rotor
    that is the hub surge, with two rotors the second one reads the first hub's sway -- the reference's indexing, kept.
    A (case, rotor) is active when aeroServoMod > 1 and the inflow speed (current_speed, default 1.0, below the waterline
    r3[2] < 0; wind_speed, default 10.0, otherwise) is above 0 (:2633-2640); an inactive one gets C = V_w = 0 and zero
    means, which is what the reference reports for it.  kp_tau / ki_tau are the rotor's raw attributes (-VS_KP, -VS_KI,
    raft_rotor.py:800-801), as :2650 uses them, not the gated locals of calcAero (:909-910).
    -> dict(R [nrot, nDOF], C, V_w complex [nC, nrot, nw], gains [nC, nrot, 4] (kp_tau, ki_tau, kp_beta, ki_beta),
    omega_avg, torque_avg (aero_torque / Ng), power_avg, bPitch_avg [nC, nrot], active [nC, nrot] bool, wind [nC] (the V_w
    of the case's last active rotor, the source of wind_PSD, or None)).  aeroServoMod 2 without C: NotImplementedError."""
    rotors = list(getattr(fowt, "rotorList", []) or [])
    T = np.asarray(fowt.T, dtype=float)
    nrot, nC = len(rotors), len(cases)
    if nrot == 0:
        raise ValueError("pack_rotor_outputs: the FOWT has no rotors")
    if len(rotor_states) != nC or any(len(s) != nrot for s in rotor_states):
        raise ValueError("rotor_states: one entry per case (%d), each with one state per rotor (%d)" % (nC, nrot))
    R = np.array([T[6 * rotors[ir // 6].nodeList[0].id + ir % 6] for ir in range(nrot)])
    out = dict(R=R, active=np.zeros([nC, nrot], dtype=bool), gains=np.zeros([nC, nrot, 4]), wind=[None] * nC)
    for k in ("omega_avg", "torque_avg", "power_avg", "bPitch_avg"):
        out[k] = np.zeros([nC, nrot])
    C_, V = [], []
    for c, case in enumerate(cases):
        Cc, Vc = [], []
        for ir in range(nrot):
            s = rotor_states[c][ir]
            get = (lambda k, d=None: s.get(k, d)) if isinstance(s, dict) else (lambda k, d=None: getattr(s, k, d))
            r3 = np.asarray(get("r3", getattr(rotors[ir], "r3", np.zeros(3))), dtype=float)
            mod = int(get("aeroServoMod", getattr(rotors[ir], "aeroServoMod", 0)))
            speed = float(case.get("current_speed", 1.0) if r3[2] < 0 else case.get("wind_speed", 10.0))
            if mod > 1 and speed > 0.0:
                if get("C") is None:
                    raise NotImplementedError("rotor outputs need the control transfer function C of Rotor.calcAero "
                                              "(aeroServoMod %d)" % mod)
                Cc.append(np.asarray(get("C"), dtype=complex))
                Vc.append(np.asarray(get("V_w"), dtype=complex))
                out["active"][c, ir] = True
                out["gains"][c, ir] = [float(get(k)) for k in ("kp_tau", "ki_tau", "kp_beta", "ki_beta")]
                out["omega_avg"][c, ir] = float(get("Omega_case"))
                out["torque_avg"][c, ir] = float(get("aero_torque")) / float(get("Ng"))
                out["power_avg"][c, ir] = float(get("aero_power"))
                out["bPitch_avg"][c, ir] = float(get("pitch_case"))
                out["wind"][c] = Vc[-1]                                       # the last active rotor's (:2679)
            else:
                Cc.append(None), Vc.append(None)
        C_.append(Cc), V.append(Vc)
    shapes = {np.shape(a) for row in C_ + V for a in row if a is not None}
    if len(shapes) > 1:
        raise ValueError("pack_rotor_outputs: C and V_w must all be [nw]")
    nw = shapes.pop()[0] if shapes else len(np.asarray(getattr(fowt, "w", [])))
    out["C"] = np.array([[np.zeros(nw, dtype=complex) if a is None else a for a in row] for row in C_]).reshape(nC, nrot, nw)
    out["V_w"] = np.array([[np.zeros(nw, dtype=complex) if a is None else a for a in row] for row in V]).reshape(nC, nrot, nw)
    return out


def pack_mooring_tensions(ms, moorMod=0):
    """Line-end tensions of a mooring system as linear functionals of the motions of its coupled bodies (moorMod 0,
    raft_fowt.py:2362-2367, raft_model.py:379-386): T_amp = J @ Xi.  Duck-typed on a MoorPy system as the reference holds it
    after lines2ss: J = ms.getCoupledStiffness(lines_only=True, tensions=True)[1] [2L, 6 * bodies], the mean tensions
    T0 = ms.getTensions() [2L], L = len(ms.lineList) (line ends A then B).  A plain dict {J, T0} stands in for the system.
    moorMod 1 / 2 take the tensions from MoorPy's dynamicSolve of every line (:2373-2386): NotImplementedError.
    -> dict(J [2L, nDOF], T0 [2L], n_lines L)."""
    if int(moorMod) != 0:
        raise NotImplementedError("mooring tensions for moorMod %d (MoorPy dynamicSolve per line) are not provided; moorMod 0 only"
                                  % int(moorMod))
    if isinstance(ms, dict):
        J, T0 = ms["J"], ms["T0"]
        n_lines = None
    else:
        J = ms.getCoupledStiffness(lines_only=True, tensions=True)[1]
        T0 = ms.getTensions()
        n_lines = len(ms.lineList)
    J, T0 = np.array(J, dtype=float), np.array(T0, dtype=float).reshape(-1)
    if J.ndim != 2 or J.shape[0] % 2 or T0.shape != (J.shape[0],):
        raise ValueError("the tension Jacobian must be [2L, nDOF] and the mean tensions [2L]")
    if n_lines is not None and 2 * n_lines != J.shape[0]:
        raise ValueError("the tension Jacobian has %d rows for %d lines" % (J.shape[0], n_lines))
    return dict(J=J, T0=T0, n_lines=J.shape[0] // 2)


SPECTRUM_IDS = {"JONSWAP": 0, "unit": 1, "constant": 2, "none": 3, "still": 3}


def pack_cases(cases):
    """Load cases -> SoA case table (first wave train of each case; raft_fowt.py:1742-1774).

    ``cases`` is a list of dicts with keys wave_spectrum, wave_period, wave_height, wave_heading,
    wave_gamma (scalars, or length-nWaves lists of which train 0 drives the linearisation).
    Returns dict(Hs, Tp, gamma, beta_deg [nC] float64, spec [nC] int32).
    Unknown spectrum -> ValueError, as raft_fowt.py:1774.
    """
    def first(v):
        return v if np.isscalar(v) else v[0]
    nC = len(cases)
    Hs, Tp, gam, beta = (np.zeros(nC) for _ in range(4))
    spec = np.zeros(nC, dtype=np.int32)
    for i, c in enumerate(cases):
        s = str(first(c.get("wave_spectrum", "JONSWAP")))
        if s not in SPECTRUM_IDS:
            raise ValueError(f"Wave spectrum input '{s}' not recognized.")
        spec[i] = SPECTRUM_IDS[s]
        Hs[i] = float(first(c["wave_height"]))
        Tp[i] = float(first(c["wave_period"]))
        gam[i] = float(first(c.get("wave_gamma", 0.0)))
        beta[i] = float(first(c.get("wave_heading", 0.0)))
    return dict(Hs=Hs, Tp=Tp, gamma=gam, beta_deg=beta, spec=spec)


def pack_case_trains(cases):
    """Load cases with one or several wave trains each (lists in the case dict, raft_fowt.py:1742-1752) ->
    flattened train table with the ``primary`` map of the C ABI: train 0 of every case drives the drag
    linearisation (raft_fowt.py:1910), its other trains reuse it (raft_model.py:1200-1236).

    Returns (table dict incl. ``primary`` [nT] int32, ``owner`` [nT] case index of every train,
    ``first`` [nC] index of every case's train 0)."""
    rows, owner, primary, first = [], [], [], []
    for ic, c in enumerate(cases):
        nH = 1 if np.isscalar(c.get("wave_heading", 0.0)) else len(c["wave_heading"])
        first.append(len(rows))
        for ih in range(nH):
            pick = lambda key, dflt=None: (c.get(key, dflt) if np.isscalar(c.get(key, dflt)) or isinstance(c.get(key, dflt), str)
                                           else c.get(key, dflt)[ih])
            rows.append(dict(wave_spectrum=pick("wave_spectrum", "JONSWAP"), wave_period=pick("wave_period"),
                             wave_height=pick("wave_height"), wave_heading=pick("wave_heading", 0.0), wave_gamma=pick("wave_gamma", 0.0)))
            owner.append(ic)
            primary.append(first[-1])
    table = pack_cases(rows)
    if len(rows) > len(cases):
        table["primary"] = np.array(primary, dtype=np.int32)
    return table, np.array(owner, dtype=np.int64), np.array(first, dtype=np.int64)
