"""Batched node-table builder: one pass of vectorised NumPy over the DESIGN axis (SURVEY.md 8f row 1).

A design sweep (the reference's parametersweep.py:29-95) varies member geometry -- end points, diameters, side lengths --
on a fixed topology.  ``raft_b200.member.Member`` / ``packer.pack_members`` build one design at a time (Python loops over
members and strip nodes, ~10 ms per VolturnUS-S variant); here every step runs once for ALL designs of a family:

  strip discretisation      raft_member.py:190-271     node counts differ per design: padded [nD, slots] + validity mask
  heading copies, frame     raft_member.py:69-79, 325-357; helpers.py:439-466, 587-602
  node positions            raft_member.py:359-362
  Ca/Cd station interp      raft_member.py:1315-1318, 2061-2064 (np.interp restated for per-design station arrays)
  volumes, end areas, a_i   raft_member.py:1324-1348
  drag areas + prefactor    raft_member.py:2070-2072, 2093-2095, 2105-2110
  A_hydro_morison           raft_member.py:1361, raft_fowt.py:1625

and the padded tables are compacted into the CSR arrays of ``solver.DesignBatch`` (include/raftk.h raftk_designs) with
boolean masks -- no per-design Python.  The formulas are the per-design builder's, evaluated element-wise in the same
order, so the tables agree with ``Member`` + ``pack_members`` to rounding (tests/test_builder_and_sweep.py: <= 1e-13).
Scope: rigid circular / rectangular members without MacCamy-Fuchs tables (those need per-node Hankel functions per
frequency: use the per-design path), every design of the family with the same stations / coefficients / topology.
"""
import numpy as np

from . import packer
from .member import _tile, rotation_matrix


class DesignFamily:
    """A template design plus per-design member geometry: ``geom[member_name]`` holds any of ``rA`` [nD,3], ``rB`` [nD,3],
    ``d`` ([nD] / [nD,n] circular, [nD,2] / [nD,n,2] rectangular); members not listed keep the template's values."""

    def __init__(self, base_design, geom, n_designs):
        self.base, self.geom, self.n = base_design, geom, int(n_designs)


def _interp_stations(x, xp, fp):
    """np.interp(x, xp, fp) with per-design abscissae: x [nD,S], xp [nD,n], fp [n] -> [nD,S] (same slope formula)."""
    if np.all(fp == fp[0]):
        return np.full(x.shape, float(fp[0]))
    n = xp.shape[1]
    j = np.clip((x[:, :, None] >= xp[:, None, :]).sum(axis=2) - 1, 0, n - 2)
    x0 = np.take_along_axis(xp, j, axis=1)
    x1 = np.take_along_axis(xp, j + 1, axis=1)
    f0, f1 = fp[j], fp[j + 1]
    with np.errstate(divide="ignore", invalid="ignore"):
        slope = (f1 - f0) / (x1 - x0)
        out = slope * (x - x0) + f0
    out = np.where(x1 == x0, f0, out)                      # repeated station (flat step): left value, like np.interp
    out = np.where(x <= xp[:, :1], fp[0], out)
    return np.where(x >= xp[:, -1:], fp[-1], out)


def _member_tables(mi, heading, geom, nD, dlsMax, rho, g, Rp, r0, nw_unused=0):
    """All designs' strips of one member copy.  -> dict of padded arrays [nD, S] (+ member-level [nD, ...]) and the mask."""
    if str(mi.get("type", "rigid")) != "rigid":
        raise NotImplementedError("member %r: only rigid members are supported by the GPU path" % mi["name"])
    rA0 = np.broadcast_to(np.asarray(geom.get("rA", mi["rA"]), dtype=float), (nD, 3)).copy()
    rB0 = np.broadcast_to(np.asarray(geom.get("rB", mi["rB"]), dtype=float), (nD, 3)).copy()
    if np.any(rA0[:, 2] == 0) or np.any(rB0[:, 2] == 0):
        raise ValueError("RAFT Members cannot start or end on the waterplane")
    rAB0 = rB0 - rA0
    L = np.sqrt(rAB0[:, 0] * rAB0[:, 0] + rAB0[:, 1] * rAB0[:, 1] + rAB0[:, 2] * rAB0[:, 2])
    potMod = bool(mi.get("potMod", False))
    gamma = float(mi.get("gamma", 0.0))
    if heading != 0.0:
        c, s = np.cos(np.deg2rad(heading)), np.sin(np.deg2rad(heading))
        rot = lambda r: np.stack([c * r[:, 0] + (-s) * r[:, 1], s * r[:, 0] + c * r[:, 1], r[:, 2]], axis=1)
        vertical = (rAB0[:, 0] == 0.0) & (rAB0[:, 1] == 0)
        if np.any(vertical) and not np.all(vertical):
            raise NotImplementedError("member %r is vertical in some designs of the family only" % mi["name"])
        rA0, rB0 = rot(rA0), rot(rB0)
        if np.all(vertical):
            gamma += heading
    st = np.array(mi["stations"], dtype=float)
    n = len(st)
    if n < 2:
        raise ValueError("At least two stations entries must be provided")
    if np.any(np.diff(st) < 0):
        raise ValueError("Member %s: the station list is not in ascending order." % mi["name"])
    s = ((st - st[0]) / (st[-1] - st[0]))[None, :] * L[:, None]                       # [nD,n]
    shape = str(mi["shape"])[0].lower()
    circ = shape == "c"
    if circ:
        gamma = 0.0
        if "d" in geom:
            dg = np.asarray(geom["d"], dtype=float)
            d = np.repeat(dg[:, None], n, axis=1) if dg.ndim == 1 else dg
        else:
            d = np.broadcast_to(_tile(mi, "d", n, None), (nD, n))
        d = d[:, :, None]                                                                  # [nD,n,1]
        if bool(mi.get("MCF", False)) and not potMod:
            raise NotImplementedError("MacCamy-Fuchs members need the per-design builder (frequency tables per node)")
    elif shape == "r":
        if "d" in geom:
            dg = np.asarray(geom["d"], dtype=float)
            d = np.repeat(dg[:, None, :], n, axis=1) if dg.ndim == 2 else dg
        else:
            v = np.array(mi["d"], dtype=float)
            v = v if v.shape == (n, 2) else np.tile(v, (n, 1))
            d = np.broadcast_to(v, (nD, n, 2))
    else:
        raise ValueError("The only allowable shape strings are circular and rectangular")
    nc = d.shape[2]

    # ---- strip discretisation (raft_member.py:190-271), padded over designs -----------------------------------------
    ls, dls, ds, drs, ok = [np.zeros([nD, 1])], [np.zeros([nD, 1])], [0.5 * d[:, :1, :]], [0.5 * d[:, :1, :]], [np.ones([nD, 1], bool)]
    for i in range(1, n):
        lstrip = s[:, i] - s[:, i - 1]
        pos = lstrip > 0.0
        if np.all(pos):
            ns = np.ceil(lstrip / dlsMax).astype(np.int64)
            dl = lstrip / ns
            m = 0.5 * (d[:, i, :] - d[:, i - 1, :]) / lstrip[:, None]
            jj = 0.5 + np.arange(int(ns.max()))
            ls.append(s[:, i - 1, None] + dl[:, None] * jj[None, :])
            dls.append(np.repeat(dl[:, None], len(jj), axis=1))
            ds.append(d[:, i - 1, None, :] + ((dl[:, None] * 2) * m)[:, None, :] * jj[None, :, None])
            drs.append(np.repeat((dl[:, None] * m)[:, None, :], len(jj), axis=1))
            ok.append(np.arange(len(jj))[None, :] < ns[:, None])
        elif not np.any(pos) and np.all(lstrip == 0.0):
            ls.append(s[:, i - 1, None]); dls.append(np.zeros([nD, 1]))
            ds.append(0.5 * (d[:, i - 1, None, :] + d[:, i, None, :])); drs.append(0.5 * (d[:, i, None, :] - d[:, i - 1, None, :]))
            ok.append(np.ones([nD, 1], bool))
        else:
            raise NotImplementedError("member %r: a station interval has zero length in some designs of the family only" % mi["name"])
    ls.append(s[:, -1:]); dls.append(np.zeros([nD, 1])); ds.append(0.5 * d[:, -1:, :]); drs.append(-0.5 * d[:, -1:, :]); ok.append(np.ones([nD, 1], bool))
    ls, dls, ok = np.concatenate(ls, axis=1), np.concatenate(dls, axis=1), np.concatenate(ok, axis=1)
    ds, drs = np.concatenate(ds, axis=1), np.concatenate(drs, axis=1)                    # [nD,S,nc]

    # ---- frame and node positions (raft_member.py:325-362) -----------------------------------------------------------
    rAB = rB0 - rA0
    q = rAB / np.sqrt(rAB[:, 0] * rAB[:, 0] + rAB[:, 1] * rAB[:, 1] + rAB[:, 2] * rAB[:, 2])[:, None]
    beta = np.arctan2(q[:, 1], q[:, 0])
    phi = np.arctan2(np.sqrt(q[:, 0] ** 2 + q[:, 1] ** 2), q[:, 2])
    s1, c1, s2, c2 = np.sin(beta), np.cos(beta), np.sin(phi), np.cos(phi)
    s3, c3 = np.sin(np.deg2rad(gamma)), np.cos(np.deg2rad(gamma))
    p1 = np.stack([c1 * c2 * c3 - s1 * s3, c1 * s3 + c2 * c3 * s1, -c3 * s2], axis=1)
    p2 = np.cross(q, p1)
    mv = lambda v: v @ Rp.T
    rA = r0[None, :] + mv(rA0)
    q, p1, p2 = mv(q), mv(p1), mv(p2)
    rB = rA + L[:, None] * q
    r = rA[:, None, :] + (ls / L[:, None])[:, :, None] * (rB - rA)[:, None, :]          # [nD,S,3]
    sub = ok & (r[:, :, 2] < 0)

    # ---- per-node coefficients (raft_member.py:1295-1357, 1387-1448; packer.pack_members) ---------------------------
    z = lambda x: np.where(sub, x, 0.0)
    out = dict(q=q, p1=p1, p2=p2, rA=rA, circ=circ, sub=sub, ls=ls, r=r)
    if circ:
        D, DR = ds[:, :, 0], drs[:, :, 0]
        v = 0.25 * np.pi * D ** 2 * dls
        v_end = np.pi / 12.0 * np.abs((D + DR) ** 3 - (D - DR) ** 3)
        a_i = np.pi * D * DR
        a_q, a_p1, a_p2 = np.pi * D * dls, D * dls, D * dls
        a_End = np.abs(np.pi * D * DR)
    else:
        v = ds[:, :, 0] * ds[:, :, 1] * dls
        v_end = np.pi / 12.0 * (np.mean(ds + drs, axis=2) ** 3 - np.mean(ds - drs, axis=2) ** 3)
        a_i = ((ds[:, :, 0] + drs[:, :, 0]) * (ds[:, :, 1] + drs[:, :, 1]) - (ds[:, :, 0] - drs[:, :, 0]) * (ds[:, :, 1] - drs[:, :, 1]))
        a_q = 2 * (ds[:, :, 0] + ds[:, :, 0]) * dls                                        # sic, raft_member.py:2070
        a_p1, a_p2 = ds[:, :, 0] * dls, ds[:, :, 1] * dls
        a_End = np.abs(a_i)
    cf = {}
    for name, key, dflt, idx in (("Cd_q", "Cd_q", 0.0, None), ("Cd_p1", "Cd", 0.6, 0), ("Cd_p2", "Cd", 0.6, 1), ("Cd_End", "CdEnd", 0.6, None),
                                 ("Ca_p1", "Ca", 0.97, 0), ("Ca_p2", "Ca", 0.97, 1), ("Ca_End", "CaEnd", 0.6, None)):
        cf[name] = _interp_stations(ls, s, _tile(mi, key, n, dflt, index=idx))
    pref = packer.SQRT_8_OVER_PI * 0.5 * rho
    out["cd_q"] = pref * (a_q * cf["Cd_q"] + a_End * cf["Cd_End"])
    out["cd_p1"] = pref * a_p1 * cf["Cd_p1"]
    out["cd_p2"] = pref * a_p2 * cf["Cd_p2"]
    if potMod:
        zero = np.zeros_like(ls)
        out.update(in_q=zero, in_p1=zero, in_p2=zero, pa=zero, ad_q=zero, ad_p1=zero, ad_p2=zero)
    else:
        pierce = sub & (r[:, :, 2] + 0.5 * dls > 0)
        with np.errstate(divide="ignore", invalid="ignore"):
            v = np.where(pierce, v * (0.5 * dls - r[:, :, 2]) / dls, v)
        out["ad_p1"], out["ad_p2"], out["ad_q"] = z(rho * v * cf["Ca_p1"]), z(rho * v * cf["Ca_p2"]), z(rho * v_end * cf["Ca_End"])
        out["in_p1"], out["in_p2"], out["in_q"] = z(rho * v * (1.0 + cf["Ca_p1"])), z(rho * v * (1.0 + cf["Ca_p2"])), z(rho * v_end * cf["Ca_End"])
        out["pa"] = rho * g * z(a_i)
    return out


def _added_mass(T, r_ref):
    """sum over submerged nodes of translateMatrix3to6DOF(Amat, r - r_ref) (raft_member.py:1361) for every design.

    Amat_j = a1_j p1 p1^T + a2_j p2 p2^T + aq_j q q^T with the member's (per-design) unit vectors, and H(r) v = v x r, so with
    c_j = d x (r_j - r_ref) for each direction d: sum Amat = (sum a_j) d d^T, sum Amat H = -d (sum a_j c_j)^T, sum H Amat H^T =
    sum a_j c_j c_j^T -- weighted sums over the node axis instead of [nD, S] batched 3 x 3 products (5 ms -> 0.6 ms per member)."""
    nD = T["q"].shape[0]
    A = np.zeros([nD, 6, 6])
    if not (np.any(T["ad_q"]) or np.any(T["ad_p1"]) or np.any(T["ad_p2"])):
        return A
    rr = T["r"] - r_ref[None, None, :]                                                     # [nD,S,3]
    ones = np.ones((1, rr.shape[1]))
    for d, a in ((T["p1"], T["ad_p1"]), (T["p2"], T["ad_p2"]), (T["q"], T["ad_q"])):
        a = np.where(T["sub"], a, 0.0)                                                     # [nD,S]
        c = np.cross(d[:, None, :], rr)                                                    # [nD,S,3]  = H(rr) d
        ac = a[:, :, None] * c
        s0 = a.sum(axis=1)                                                                 # [nD]
        s1 = (ones @ ac)[:, 0, :]                                                          # [nD,3]  (batched matmul: 6x faster than .sum(axis=1))
        A[:, :3, :3] += s0[:, None, None] * (d[:, :, None] * d[:, None, :])
        off = -d[:, :, None] * s1[:, None, :]                                              # sum_j Amat_j H_j
        A[:, :3, 3:] += off
        A[:, 3:, :3] += np.swapaxes(off, 1, 2)
        A[:, 3:, 3:] += np.swapaxes(ac, 1, 2) @ c                                          # sum_j a_j c_j c_j^T
    return A


def _count_classes(keys, valid, tol):
    """Per design: the number of step classes by the fused kernels' rule (raftk_fused.cuh step_classes_warp), greedy in key
    order: a key joins the first class whose key is within ``tol`` of it in every component, else opens one.
    keys [nD,P,c], valid [nD,P], tol [nD,P] (each key's own tolerance)."""
    nD = keys.shape[0]
    if keys.shape[1] == 0:
        return np.zeros(nD, dtype=np.int64)
    nc = keys.shape[2]
    # a key equal to the valid key before it has the same tolerance and the same first match, so it opens no class: only
    # the others are walked (the interior of a uniformly divided section repeats its step)
    rep = np.zeros(valid.shape, bool)
    rep[:, 1:] = valid[:, :-1] & np.all(keys[:, 1:] == keys[:, :-1], axis=2)
    valid = valid & ~rep
    pmax = int(valid.sum(axis=1).max())
    order = np.argsort(~valid, axis=1, kind="stable")[:, :pmax]
    keys = np.take_along_axis(keys, order[:, :, None], axis=1)
    valid = np.take_along_axis(valid, order, axis=1)
    tol = np.take_along_axis(tol, order, axis=1)
    cls = np.zeros((nD, pmax, nc))                                        # class keys so far
    n = np.zeros(nD, dtype=np.int64)
    rows = np.arange(nD)
    for p in range(pmax):
        r = int(n.max())
        hit = np.arange(r)[None, :] < n[:, None]
        for i in range(nc):
            hit &= np.abs(cls[:, :r, i] - keys[:, p, None, i]) <= tol[:, p, None]
        new = valid[:, p] & ~hit.any(axis=1)
        cls[rows[new], n[new]] = keys[new, p]
        n += new
    return n


def _base_rotors(matrices, A_mor, arrays, nD):
    """The base design's submerged rotors (``matrices['rotor_excitation']``, ``['A_hydro_rotor']``, as ``fowt.FOWT`` takes
    them) for every design of a family: the hubs do not move with the platform members a family varies, so every design
    gets the base table, and the rotor's added mass joins A_hydro_morison (in place) as in FOWT.calcHydroConstants."""
    if "A_hydro_rotor" in matrices:
        A_mor += np.asarray(matrices["A_hydro_rotor"], dtype=float)[None]
    rot = matrices.get("rotor_excitation")
    if rot is not None and len(rot["r3"]):
        r3, G = np.asarray(rot["r3"], dtype=float).reshape(-1, 3), np.asarray(rot["G"], dtype=float).reshape(-1, 6, 3)
        arrays["rot_count"] = np.full(nD, len(r3), dtype=np.int32)
        arrays["rot_r3"] = np.ascontiguousarray(np.broadcast_to(r3, (nD,) + r3.shape))
        arrays["rot_G"] = np.ascontiguousarray(np.broadcast_to(G, (nD,) + G.shape))


def build_family(family, w, k, depth, matrices, r6=None):
    """-> ``solver.DesignBatch`` of every design of ``family`` on the grid (w, k): the CSR node / member tables and the
    system matrices M0 = M_struc + A_hydro_morison, B0, C0 (statics stay at ``matrices``, as in sweep.build_variants)."""
    from . import solver
    base, nD = family.base, family.n
    w, k = np.ascontiguousarray(w, dtype=float), np.ascontiguousarray(k, dtype=float)
    site = base.get("site", {})
    rho, g = float(site.get("rho_water", 1025.0)), float(site.get("g", 9.81))
    plat = base["platform"]
    master = int(plat.get("potModMaster", 0))
    dls_default = float(plat.get("dlsMax", 5.0))
    r6 = np.zeros(6) if r6 is None else np.asarray(r6, dtype=float)
    Rp, r0 = rotation_matrix(*r6[3:]), r6[:3]
    names = [m["name"] for m in plat["members"]]
    if len(names) != len(set(names)):
        raise Exception("Member names must be unique. Please check the input data.")
    tabs = []
    for mi in plat["members"]:
        mi = dict(mi)
        if master == 1:
            mi["potMod"] = False
        elif master in (2, 3):
            mi["potMod"] = True
        heads = mi.get("heading", 0.0)
        for h in (np.atleast_1d(heads) if not np.isscalar(heads) else [heads]):
            tabs.append(_member_tables(mi, float(h), family.geom.get(mi["name"], {}), nD, float(mi.get("dlsMax", dls_default)), rho, g, Rp, r0))
    A_mor = np.zeros([nD, 6, 6])
    for T in tabs:
        A_mor += _added_mass(T, r0)

    # ---- compaction: padded [nD, member, slot] -> CSR (members without a submerged node are dropped per design) ------
    Nm = len(tabs)
    S = max(T["ls"].shape[1] for T in tabs)
    pad = lambda a: np.concatenate([a, np.zeros((nD, S - a.shape[1]) + a.shape[2:], dtype=a.dtype)], axis=1)
    keep = np.stack([pad(T["sub"]) for T in tabs], axis=1)                                 # [nD,Nm,S]
    cnt = keep.sum(axis=2)                                                                 # nodes per (design, member)
    has = cnt > 0
    arrays = {}
    for col in ("ls", "cd_q", "cd_p1", "cd_p2", "in_q", "in_p1", "in_p2", "pa"):
        arrays["node_" + col] = np.ascontiguousarray(np.stack([pad(T[col]) for T in tabs], axis=1)[keep])
    frame = np.stack([np.concatenate([T["q"], T["p1"], T["p2"]], axis=1) for T in tabs], axis=1)      # [nD,Nm,9]
    rA = np.stack([T["rA"] for T in tabs], axis=1)
    arrays["mem_frame"] = np.ascontiguousarray(frame[has])
    arrays["mem_rA"] = np.ascontiguousarray(rA[has])
    arrays["mem_arm"] = np.ascontiguousarray(rA[has] - r0[None, :])
    arrays["mem_circ"] = np.ascontiguousarray(np.broadcast_to(np.array([1 if T["circ"] else 0 for T in tabs], dtype=np.int32), (nD, Nm))[has])
    arrays["member_offset"] = np.concatenate([[0], np.cumsum(has.sum(axis=1))]).astype(np.int32)
    arrays["mem_node_start"] = np.concatenate([[0], np.cumsum(cnt[has])]).astype(np.int32)
    _base_rotors(matrices, A_mor, arrays, nD)
    M_struc = np.asarray(matrices.get("M_struc", np.zeros([6, 6])), dtype=float)
    arrays["M0"] = np.ascontiguousarray((M_struc[None] + A_mor).reshape(nD, 36))
    B0 = np.asarray(matrices.get("B_struc", np.zeros([6, 6])), dtype=float)
    C0 = sum(np.asarray(matrices.get(nm, np.zeros([6, 6])), dtype=float) for nm in ("C_struc", "C_hydro", "C_moor", "C_elast"))
    arrays["B0"] = np.ascontiguousarray(np.broadcast_to(B0.reshape(1, 36), (nD, 36)))
    arrays["C0"] = np.ascontiguousarray(np.broadcast_to(C0.reshape(1, 36), (nD, 36)))
    arrays["w"], arrays["k"] = w, k

    # ---- step-class hints of the fused solver (solver.DesignBatch._step_classes), all designs at once ----------------
    lsP = np.stack([pad(T["ls"]) for T in tabs], axis=1)
    qv = np.stack([T["q"] for T in tabs], axis=1)                                          # [nD,Nm,3]
    # kept strips first within every (design, member) row, so that consecutive slots are consecutive submerged nodes
    # (padding of a short section sits between its last strip and the next section otherwise)
    front = np.argsort(~keep, axis=2, kind="stable")
    lsP, keepF = np.take_along_axis(lsP, front, axis=2), np.take_along_axis(keep, front, axis=2)
    pair = keepF[:, :, 1:] & keepF[:, :, :-1]
    step = lsP[:, :, 1:] - lsP[:, :, :-1]
    kx, ky, kz = qv[:, :, None, 0] * step, qv[:, :, None, 1] * step, qv[:, :, None, 2] * step
    P = Nm * (S - 1)
    wk = np.stack([kx, ky], axis=3).reshape(nD, P, 2)
    wv = (pair & ((np.abs(kx) > solver.STEP_ZERO) | (np.abs(ky) > solver.STEP_ZERO))).reshape(nD, P)
    hv = (pair & (np.abs(kz) > solver.STEP_ZERO)).reshape(nD, P)
    z0 = rA[:, :, 2] + lsP[:, :, 0] * qv[:, :, 2]                                          # first submerged node of each member
    counts = (_count_classes(wk, wv, solver.STEP_RTOL * (np.abs(wk[..., 0]) + np.abs(wk[..., 1]))),
              _count_classes(kz.reshape(nD, P, 1), hv, solver.STEP_RTOL * np.abs(kz.reshape(nD, P))),
              _count_classes(z0[:, :, None], has, solver.Z0_RTOL * np.maximum(1.0, np.abs(z0))))
    batch = solver.DesignBatch.from_tables(
        arrays, n_designs=nD, depth=float(depth), rho=rho, g=g, dw=float(w[1] - w[0]),
        max_nodes=int(max(1, cnt.sum(axis=1).max())), max_members=int(max(1, has.sum(axis=1).max())),
        classes=tuple(int(max(1, c.max())) for c in counts))
    batch.A_hydro_morison = A_mor
    return batch



def build_family_native(family, w, k, depth, matrices, r6=None):
    """``build_family`` through the library's native builder (``raftk_build_family_host``, csrc/raftk_builder.h: the same
    formulas in plain C++ loops, ~2 ms instead of ~80 ms per 1250 VolturnUS-S variants).  Same scope and the same result
    (tables to rounding, identical counts and step-class hints: tests/test_builder_and_sweep.py)."""
    import ctypes as C
    from . import solver
    from ._lib import RaftkFamily, RaftkFamilyMember, RaftkFamilyTables, check, lib
    base, nD = family.base, family.n
    w, k = np.ascontiguousarray(w, dtype=float), np.ascontiguousarray(k, dtype=float)
    site = base.get("site", {})
    rho, g = float(site.get("rho_water", 1025.0)), float(site.get("g", 9.81))
    plat = base["platform"]
    master = int(plat.get("potModMaster", 0))
    dls_default = float(plat.get("dlsMax", 5.0))
    r6 = np.zeros(6) if r6 is None else np.asarray(r6, dtype=float)
    names = [m["name"] for m in plat["members"]]
    if len(names) != len(set(names)):
        raise Exception("Member names must be unique. Please check the input data.")
    keep, copies = [], []                       # arrays referenced by the C structs stay alive in ``keep``
    f64 = lambda a: np.ascontiguousarray(a, dtype=np.float64)
    for mi in plat["members"]:
        mi = dict(mi)
        if str(mi.get("type", "rigid")) != "rigid":
            raise NotImplementedError("member %r: only rigid members are supported by the GPU path" % mi["name"])
        if master == 1:
            mi["potMod"] = False
        elif master in (2, 3):
            mi["potMod"] = True
        geom = family.geom.get(mi["name"], {})
        st = np.array(mi["stations"], dtype=float)
        n = len(st)
        if n < 2:
            raise ValueError("At least two stations entries must be provided")
        if np.any(np.diff(st) < 0):
            raise ValueError("Member %s: the station list is not in ascending order." % mi["name"])
        shape = str(mi["shape"])[0].lower()
        potMod = bool(mi.get("potMod", False))
        if shape == "c":
            if "d" in geom:
                dg = np.asarray(geom["d"], dtype=float)
                d = np.repeat(dg[:, None], n, axis=1) if dg.ndim == 1 else dg
            else:
                d = np.broadcast_to(_tile(mi, "d", n, None), (nD, n))
            d = f64(d).reshape(nD, n, 1)
            if bool(mi.get("MCF", False)) and not potMod:
                raise NotImplementedError("MacCamy-Fuchs members need the per-design builder (frequency tables per node)")
        elif shape == "r":
            if "d" in geom:
                dg = np.asarray(geom["d"], dtype=float)
                d = np.repeat(dg[:, None, :], n, axis=1) if dg.ndim == 2 else dg
            else:
                v = np.array(mi["d"], dtype=float)
                v = v if v.shape == (n, 2) else np.tile(v, (n, 1))
                d = np.broadcast_to(v, (nD, n, 2))
            d = f64(d).reshape(nD, n, 2)
        else:
            raise ValueError("The only allowable shape strings are circular and rectangular")
        rA = f64(np.broadcast_to(np.asarray(geom.get("rA", mi["rA"]), dtype=float), (nD, 3)))
        rB = f64(np.broadcast_to(np.asarray(geom.get("rB", mi["rB"]), dtype=float), (nD, 3)))
        coef = [f64(_tile(mi, key, n, dflt, index=idx)) for key, dflt, idx in
                (("Cd_q", 0.0, None), ("Cd", 0.6, 0), ("Cd", 0.6, 1), ("CdEnd", 0.6, None), ("Ca", 0.97, 0), ("Ca", 0.97, 1), ("CaEnd", 0.6, None))]
        st = f64(st)
        keep += [st, rA, rB, d] + coef
        heads = mi.get("heading", 0.0)
        for h in (np.atleast_1d(heads) if not np.isscalar(heads) else [heads]):
            m = RaftkFamilyMember()
            m.n_stations, m.circular, m.pot_mod = n, 1 if shape == "c" else 0, 1 if potMod else 0
            m.gamma_deg, m.heading_deg, m.dls_max = float(mi.get("gamma", 0.0)), float(h), float(mi.get("dlsMax", dls_default))
            m.stations, m.rA, m.rB, m.d = st.ctypes.data, rA.ctypes.data, rB.ctypes.data, d.ctypes.data
            (m.Cd_q, m.Cd_p1, m.Cd_p2, m.Cd_End, m.Ca_p1, m.Ca_p2, m.Ca_End) = [c.ctypes.data for c in coef]
            copies.append(m)
    marr = (RaftkFamilyMember * len(copies))(*copies)
    fam = RaftkFamily()
    fam.n_designs, fam.n_members, fam.rho, fam.g = nD, len(copies), rho, g
    fam.Rp = (C.c_double * 9)(*rotation_matrix(*r6[3:]).reshape(9))
    fam.r0 = (C.c_double * 3)(*r6[:3])
    fam.members = marr
    nm, nn = C.c_int32(0), C.c_int32(0)
    check(lib.raftk_family_sizes(C.byref(fam), C.byref(nm), C.byref(nn)))
    nm, nn = nm.value, nn.value
    arrays = dict(member_offset=np.zeros(nD + 1, dtype=np.int32), mem_node_start=np.zeros(nm + 1, dtype=np.int32),
                  mem_circ=np.zeros(nm, dtype=np.int32), mem_frame=np.zeros([nm, 9]), mem_rA=np.zeros([nm, 3]), mem_arm=np.zeros([nm, 3]))
    for col in ("ls", "cd_q", "cd_p1", "cd_p2", "in_q", "in_p1", "in_p2", "pa"):
        arrays["node_" + col] = np.zeros(nn)
    A_mor = np.zeros([nD, 6, 6])
    t = RaftkFamilyTables()
    for name, a in arrays.items():
        setattr(t, name, a.ctypes.data)
    t.A_morison = A_mor.ctypes.data
    check(lib.raftk_build_family_host(C.byref(fam), C.byref(t)))
    _base_rotors(matrices, A_mor, arrays, nD)
    M_struc = np.asarray(matrices.get("M_struc", np.zeros([6, 6])), dtype=float)
    arrays["M0"] = np.ascontiguousarray((M_struc[None] + A_mor).reshape(nD, 36))
    B0 = np.asarray(matrices.get("B_struc", np.zeros([6, 6])), dtype=float)
    C0 = sum(np.asarray(matrices.get(nm_, np.zeros([6, 6])), dtype=float) for nm_ in ("C_struc", "C_hydro", "C_moor", "C_elast"))
    arrays["B0"] = np.ascontiguousarray(np.broadcast_to(B0.reshape(1, 36), (nD, 36)))
    arrays["C0"] = np.ascontiguousarray(np.broadcast_to(C0.reshape(1, 36), (nD, 36)))
    arrays["w"], arrays["k"] = w, k
    batch = solver.DesignBatch.from_tables(arrays, n_designs=nD, depth=float(depth), rho=rho, g=g, dw=float(w[1] - w[0]),
                                           max_nodes=int(t.max_nodes), max_members=int(t.max_members),
                                           classes=(int(t.max_w_classes), int(t.max_h_classes), int(t.max_z_classes)))
    batch.A_hydro_morison = A_mor
    del keep
    return batch
