"""Host-side driver of the C ABI: packed designs + case table -> libraftk.so -> NumPy / torch results.

Two routes, both straight through the C ABI (no CPU fallback anywhere):

* ``solve_dynamics`` / ``hydro_excitation`` / ``hydro_linearization``: HOST buffers in and out
  (``raftk_*_host``).  This is the reference-facing call: what ``Model.solveDynamics`` would invoke
  when ``raft_b200`` is dropped into RAFT (INTEGRATION.md), and what ``bench.py`` times as ``e2e``.
* ``DeviceSession``: tables, workspace and outputs resident in HBM as torch tensors
  (``raftk_*_dev`` on torch's current stream).  ``bench.py`` times this as ``value``; the sweep
  driver (``raft_b200.sweep``) all-gathers its output tensor over NCCL.
"""
import copy
import ctypes as C

import numpy as np

from . import _lib
from ._lib import (RaftkCases, RaftkDesigns, RaftkFarm, RaftkFarmBatch, RaftkFarmRagged, RaftkGeneral, RaftkGeneralBatch, RaftkGeneralFd, RaftkGeneralQtf, RaftkOutputs, RaftkSlender, RaftkSlenderBatch,
                   RaftkSlenderOutputs, RaftkSolveOpts, check, lib)

_F8 = np.float64
_C16 = np.complex128
_I4 = np.int32


class _Tables(dict):
    """The named host arrays of a DesignBatch / CaseTable.  Every mutation bumps ``version``, which keys the cached C struct
    of the host-buffer calls (building the ~30-pointer ctypes struct costs ~25 us of Python per call otherwise).  In-place edits of an array keep its address, so they need no invalidation."""
    version = 0

    def _bump(self):
        self.version += 1

    def __setitem__(self, k, v):
        dict.__setitem__(self, k, v); self._bump()

    def __delitem__(self, k):
        dict.__delitem__(self, k); self._bump()

    def update(self, *a, **kw):
        dict.update(self, *a, **kw); self._bump()

    def pop(self, *a):
        r = dict.pop(self, *a); self._bump(); return r

    def popitem(self):
        r = dict.popitem(self); self._bump(); return r

    def setdefault(self, k, d=None):
        r = dict.setdefault(self, k, d); self._bump(); return r

    def clear(self):
        dict.clear(self); self._bump()


def _host_struct(obj):
    """``obj.struct`` over the host arrays, cached until ``obj.arrays`` is mutated (a COPY is returned when the caller edits it)."""
    ver = obj.arrays.version if isinstance(obj.arrays, _Tables) else None
    c = getattr(obj, "_host_struct_cache", None)
    if ver is None or c is None or c[0] != ver:
        c = (ver, obj.struct(_host_ptr(obj.arrays)))
        obj._host_struct_cache = c
    return c[1]


class DesignBatch:
    """CSR concatenation of packed designs (``packer.pack_fowt`` dicts) sharing one frequency grid."""

    NODE_COLS = ("ls", "cd_q", "cd_p1", "cd_p2", "in_q", "in_p1", "in_p2", "pa")

    def __init__(self, packed):
        if isinstance(packed, dict):
            packed = [packed]
        if len(packed) == 0:
            raise ValueError("DesignBatch needs at least one design")
        P0 = packed[0]
        self.n_designs = len(packed)
        self.w = np.ascontiguousarray(P0["w"], dtype=_F8)
        self.k = np.ascontiguousarray(P0["k"], dtype=_F8)
        self.nw = len(self.w)
        self.depth, self.rho, self.g = float(P0["depth"]), float(P0["rho"]), float(P0["g"])
        self.dw = float(P0["dw"]) if "dw" in P0 else float(self.w[1] - self.w[0])
        a = self.arrays = _Tables()
        member_offset, mem_node_start = [0], [0]
        frames, rAs, arms, circs = [], [], [], []
        cols = {c: [] for c in self.NODE_COLS}
        max_nodes = max_members = 0
        for P in packed:
            if len(P["w"]) != self.nw or float(P["depth"]) != self.depth:
                raise ValueError("all designs of a batch must share the frequency grid and water depth")
            if P is not P0 and (not np.array_equal(np.asarray(P["w"], dtype=_F8), self.w) or float(P["rho"]) != self.rho
                                or float(P["g"]) != self.g):
                raise ValueError("all designs of a batch must share the frequency values, water density and g")
            nm = len(P["mem_circ"])
            frames.append(np.concatenate([P["mem_q"], P["mem_p1"], P["mem_p2"]], axis=1).reshape(nm, 9))
            rAs.append(np.asarray(P["mem_rA"], dtype=_F8).reshape(nm, 3))
            arms.append(np.asarray(P["mem_rA"], dtype=_F8).reshape(nm, 3) - np.asarray(P["prp"], dtype=_F8)[None, :])
            circs.append(np.asarray(P["mem_circ"], dtype=_I4))
            base = mem_node_start[-1]
            ms = np.asarray(P["mem_start"], dtype=np.int64)
            mem_node_start.extend((base + ms[1:]).tolist())
            member_offset.append(member_offset[-1] + nm)
            for c in self.NODE_COLS:
                cols[c].append(np.asarray(P["node_" + c], dtype=_F8))
            max_nodes = max(max_nodes, int(ms[-1]))
            max_members = max(max_members, nm)
        a["member_offset"] = np.array(member_offset, dtype=_I4)
        a["mem_frame"] = np.ascontiguousarray(np.concatenate(frames, axis=0), dtype=_F8)
        a["mem_rA"] = np.ascontiguousarray(np.concatenate(rAs, axis=0), dtype=_F8)
        a["mem_arm"] = np.ascontiguousarray(np.concatenate(arms, axis=0), dtype=_F8)
        a["mem_node_start"] = np.array(mem_node_start, dtype=_I4)
        a["mem_circ"] = np.ascontiguousarray(np.concatenate(circs), dtype=_I4)
        for c in self.NODE_COLS:
            a["node_" + c] = np.ascontiguousarray(np.concatenate(cols[c]), dtype=_F8)
        have_mcf = ["node_in_p1_w" in P and P["node_in_p1_w"] is not None for P in packed]
        if any(have_mcf):
            for c in ("in_p1", "in_p2"):
                a["node_%s_w" % c] = np.ascontiguousarray(np.concatenate([
                    np.asarray(P["node_%s_w" % c], dtype=np.complex128) if h
                    else np.repeat(np.asarray(P["node_" + c], dtype=np.complex128)[:, None], self.nw, axis=1)
                    for P, h in zip(packed, have_mcf)], axis=0))
        for mname in ("M0", "B0", "C0"):
            a[mname] = np.ascontiguousarray(np.stack([np.asarray(P[mname], dtype=_F8).reshape(36) for P in packed]))
        have_w = ["A_w" in P and P["A_w"] is not None for P in packed]
        if any(have_w):
            z = np.zeros([36, self.nw])
            a["A_w"] = np.ascontiguousarray(np.stack([np.asarray(P["A_w"], dtype=_F8).reshape(36, self.nw) if h else z
                                                      for P, h in zip(packed, have_w)]))
            a["B_w"] = np.ascontiguousarray(np.stack([np.asarray(P["B_w"], dtype=_F8).reshape(36, self.nw) if h else z
                                                      for P, h in zip(packed, have_w)]))
        self.n_bem_head = 0
        have_x = [P.get("X_BEM") is not None for P in packed]
        if any(have_x):
            # designs without BEM excitation in a mixed batch (strip-theory platform next to potMod ones) get zero tables
            Px = packed[have_x.index(True)]
            heads = np.ascontiguousarray(Px["bem_headings"], dtype=_F8)
            self.n_bem_head = len(heads)
            for P, h in zip(packed, have_x):
                if h and not np.array_equal(np.asarray(P["bem_headings"], dtype=_F8), heads):
                    raise ValueError("all designs of a batch must share the BEM heading list")
            zx = np.zeros([self.n_bem_head, 6, self.nw], dtype=np.complex128)
            a["bem_headings"] = heads
            a["X_BEM"] = np.ascontiguousarray(np.stack([np.asarray(P["X_BEM"], dtype=np.complex128) if h else zx
                                                        for P, h in zip(packed, have_x)]))
            a["bem_xyh"] = np.ascontiguousarray(np.array(
                [[float(P.get("x_ref", 0.0)), float(P.get("y_ref", 0.0)), float(P.get("heading_adjust", 0.0))] for P in packed],
                dtype=_F8))
        # external QTF (potSecOrder 2): packed [nw1,nw2,nheads,6] per design; one shared table when all designs
        # carry the same one (a geometry-preserving sweep), else stacked on a design axis
        self.n_qtf_w = self.n_qtf_head = 0
        self.qtf_shared = 0
        have_q = [P.get("qtf") is not None for P in packed]
        if any(have_q):
            if not all(have_q):
                raise ValueError("either all or none of the designs of a batch carry a QTF table")
            qw, qh = np.ascontiguousarray(P0["qtf_w"], dtype=_F8), np.ascontiguousarray(P0["qtf_heads"], dtype=_F8)
            for P in packed:
                if not (np.array_equal(P["qtf_w"], qw) and np.array_equal(P["qtf_heads"], qh)):
                    raise ValueError("all designs of a batch must share the QTF frequency and heading axes")
            self.n_qtf_w, self.n_qtf_head = len(qw), len(qh)
            a["qtf_w"], a["qtf_heads"] = qw, qh
            if all(P["qtf"] is P0["qtf"] for P in packed):
                self.qtf_shared = 1
                a["qtf"] = np.ascontiguousarray(P0["qtf"], dtype=np.complex128)
            else:
                a["qtf"] = np.ascontiguousarray(np.stack([np.asarray(P["qtf"], dtype=np.complex128) for P in packed]))
            if a["qtf"].shape[-4:] != (self.n_qtf_w, self.n_qtf_w, self.n_qtf_head, 6):
                raise ValueError("qtf must be [nw1, nw2, nheads, 6] with nw1 == nw2 == len(qtf_w)")
        # submerged rotors (packer.pack_rotor_excitation): padded per design, designs without rotors get rot_count = 0
        self.max_rotors = max(len(P.get("rot_r3", ())) for P in packed)
        if self.max_rotors:
            R = self.max_rotors
            a["rot_count"] = np.array([len(P.get("rot_r3", ())) for P in packed], dtype=_I4)
            a["rot_r3"], a["rot_G"] = np.zeros([self.n_designs, R, 3]), np.zeros([self.n_designs, R, 6, 3])
            for i, P in enumerate(packed):
                n = int(a["rot_count"][i])
                if n:
                    a["rot_r3"][i, :n] = np.asarray(P["rot_r3"], dtype=_F8).reshape(n, 3)
                    a["rot_G"][i, :n] = np.asarray(P["rot_G"], dtype=_F8).reshape(n, 6, 3)
        a["w"], a["k"] = self.w, self.k
        self.n_members_total = int(member_offset[-1])
        self.n_nodes_total = int(mem_node_start[-1])
        self.max_nodes = max(1, max_nodes)
        self.max_members = max(1, max_members)
        self.max_w_classes, self.max_h_classes, self.max_z_classes = self._step_classes(packed)
        self.walk_exact = fused_walk_exact(a, self.k, self.depth)

    @classmethod
    def from_tables(cls, arrays, n_designs, depth, rho, g, dw, max_nodes, max_members, classes):
        """DesignBatch straight from CSR tables (``raft_b200.batch_builder``): ``arrays`` holds the raftk_designs columns
        (member_offset, mem_*, node_*, M0/B0/C0, w, k); ``classes`` = (max_w, max_h, max_z) step-class hints."""
        self = cls.__new__(cls)
        self.arrays = a = _Tables(arrays)
        self.n_designs = int(n_designs)
        self.w, self.k = a["w"], a["k"]
        self.nw = len(self.w)
        self.depth, self.rho, self.g, self.dw = float(depth), float(rho), float(g), float(dw)
        self.n_bem_head = self.n_qtf_w = self.n_qtf_head = self.qtf_shared = 0
        self.max_rotors = int(a["rot_r3"].shape[1]) if "rot_r3" in a else 0
        self.n_members_total = int(a["member_offset"][-1])
        self.n_nodes_total = int(a["mem_node_start"][-1])
        self.max_nodes, self.max_members = int(max_nodes), int(max_members)
        self.max_w_classes, self.max_h_classes, self.max_z_classes = (int(c) for c in classes)
        self.walk_exact = fused_walk_exact(a, self.k, self.depth)
        return self

    PER_DESIGN = ("M0", "B0", "C0", "A_w", "B_w", "X_BEM", "bem_xyh", "rot_count", "rot_r3", "rot_G")
    PER_MEMBER = ("mem_frame", "mem_rA", "mem_arm", "mem_circ")

    def take(self, lo, hi):
        """Designs [lo, hi) as a batch of their own (a shard of ``sweep.ShardedFarmSolve``).  The size and step-class hints and the
        choice of node walk stay this batch's, so every design is planned, and solved, as it is here."""
        lo, hi = int(lo), int(hi)
        if not 0 <= lo < hi <= self.n_designs:
            raise ValueError("take(%d, %d): a non-empty range of the batch's %d designs" % (lo, hi, self.n_designs))
        a = self.arrays
        mo, ns = np.asarray(a["member_offset"]), np.asarray(a["mem_node_start"])
        m0, m1 = int(mo[lo]), int(mo[hi])
        n0, n1 = int(ns[m0]), int(ns[m1])
        b = copy.copy(self)
        b.__dict__.pop("_host_struct_cache", None)
        b.arrays = t = _Tables()
        for k, v in a.items():
            if k in self.PER_DESIGN or (k == "qtf" and not self.qtf_shared):
                t[k] = np.ascontiguousarray(v[lo:hi])
            elif k in self.PER_MEMBER:
                t[k] = np.ascontiguousarray(v[m0:m1])
            elif k.startswith("node_"):
                t[k] = np.ascontiguousarray(v[n0:n1])
            else:
                t[k] = v
        t["member_offset"] = np.ascontiguousarray(mo[lo:hi + 1] - m0, dtype=_I4)
        t["mem_node_start"] = np.ascontiguousarray(ns[m0:m1 + 1] - n0, dtype=_I4)
        b.n_designs, b.n_members_total, b.n_nodes_total = hi - lo, m1 - m0, n1 - n0
        return b

    @staticmethod
    def _step_classes(packed):
        """Step-class hints of the fused solvers: the largest number of classes of any design, counted by the kernels' rule
        (raftk_fused.cuh step_classes_warp, DESIGN.md section 5): greedy in node order, a key joins the first class whose key
        is within the tolerance of its own, else opens one.  Phase classes are keyed by (q_x,q_y)*step, depth classes by
        q_z*step, z classes by the members' first-node depths."""
        mw = mh = mz = 0
        for P in packed:
            wk, hk, zk = [], [], []
            ms = np.asarray(P["mem_start"], dtype=np.int64)
            for m in range(len(ms) - 1):
                q = np.asarray(P["mem_q"][m], dtype=float)
                ls = np.asarray(P["node_ls"][ms[m]:ms[m + 1]], dtype=float)
                if len(ls):
                    z0 = float(P["mem_rA"][m][2]) + ls[0] * q[2]
                    if not any(abs(a - z0) <= Z0_RTOL * max(1.0, abs(z0)) for a in zk):
                        zk.append(z0)
                for step in np.diff(ls):
                    kx, ky, kz = q[0] * step, q[1] * step, q[2] * step
                    if abs(kx) > STEP_ZERO or abs(ky) > STEP_ZERO:
                        tol = STEP_RTOL * (abs(kx) + abs(ky))
                        if not any(abs(a - kx) <= tol and abs(b - ky) <= tol for a, b in wk):
                            wk.append((kx, ky))
                    if abs(kz) > STEP_ZERO:
                        if not any(abs(a - kz) <= STEP_RTOL * abs(kz) for a in hk):
                            hk.append(kz)
            mw, mh, mz = max(mw, len(wk)), max(mh, len(hk)), max(mz, len(zk))
        return max(1, mw), max(1, mh), max(1, mz)

    def input_bytes(self):
        return int(sum(v.nbytes for v in self.arrays.values()))

    def struct(self, ptr):
        """Build the C struct; ``ptr(name)`` returns the address (host or device) of array ``name`` or None."""
        s = RaftkDesigns()
        s.n_designs, s.nw = self.n_designs, self.nw
        s.n_members_total, s.n_nodes_total = self.n_members_total, self.n_nodes_total
        s.max_nodes, s.max_members = self.max_nodes, self.max_members
        s.max_w_classes, s.max_h_classes, s.max_z_classes = self.max_w_classes, self.max_h_classes, self.max_z_classes
        s.walk_exact = int(self.walk_exact)
        s.depth, s.rho, s.g, s.dw = self.depth, self.rho, self.g, self.dw
        for name in ("w", "k", "member_offset", "mem_frame", "mem_rA", "mem_arm", "mem_node_start", "mem_circ",
                     "node_ls", "node_cd_q", "node_cd_p1", "node_cd_p2", "node_in_q", "node_in_p1", "node_in_p2",
                     "node_pa", "node_in_p1_w", "node_in_p2_w", "M0", "B0", "C0", "A_w", "B_w",
                     "bem_headings", "X_BEM", "bem_xyh", "qtf_w", "qtf_heads", "qtf", "rot_count", "rot_r3", "rot_G"):
            setattr(s, name, ptr(name) if name in self.arrays else None)
        s.n_bem_head = self.n_bem_head
        s.max_rotors = self.max_rotors
        s.n_qtf_w, s.n_qtf_head, s.qtf_shared = self.n_qtf_w, self.n_qtf_head, self.qtf_shared
        return s


class CaseTable:
    """SoA case table (``packer.pack_cases`` dict, or keyword arrays)."""

    def __init__(self, cases, zeta=None, F_2nd=None, Xi_init=None, ops=None):
        """``F_2nd``: optional real [nD,nC,6,nw] second-order force amplitudes added to the linear excitation.
        ``Xi_init``: optional complex [nD,nC,6,nw] starting iterate of the fixed-point loop (instead of xi_start).
        ``ops``: optional operating points (``packer.pack_operating_points``): dict(op [nC] int, A_w, B_w) with tables
        [nD, n_op, 6, 6, nw] per design or [n_op, 6, 6, nw] for one set every design shares -- the aero-servo added mass and
        damping (B_gyro folded into B_w) that the reference's calcTurbineConstants(case) adds to case c's system matrices:
        unit (d, c) solves with M0 + (A_w + ops.A_w[op[c]]) and B0 + B_drag + (B_w + ops.B_w[op[c]]) (raftk_cases.op).
        The generalised-DOF solves take square tables [.., n_fd, n_fd, nw] on the support of their ``fd``
        (``packer.pack_general_operating_points``); each solve checks the table size against its designs (``check_ops``,
        ``check_general_ops``)."""
        self.arrays = a = _Tables()
        for kname in ("Hs", "Tp", "gamma", "beta_deg"):
            a[kname] = np.ascontiguousarray(cases[kname], dtype=_F8)
        a["spec"] = np.ascontiguousarray(cases["spec"], dtype=_I4)
        if np.any((a["spec"] < 0) | (a["spec"] > 3)):
            raise ValueError("Wave spectrum input not recognized.")       # raft_fowt.py:1774
        self.n_cases = len(a["Hs"])
        if zeta is not None:
            a["zeta"] = np.ascontiguousarray(zeta, dtype=_F8)
        if cases.get("primary") is not None:
            pr = np.ascontiguousarray(cases["primary"], dtype=_I4)
            if len(pr) != self.n_cases or np.any(pr < 0) or np.any(pr >= self.n_cases) or np.any(pr[pr] != pr):
                raise ValueError("primary must map every case to a primary case (primary[primary[c]] == primary[c])")
            a["primary"] = pr
        if F_2nd is not None:
            a["F_2nd"] = np.ascontiguousarray(F_2nd, dtype=_F8)
        if Xi_init is not None:
            a["Xi_init"] = np.ascontiguousarray(Xi_init, dtype=np.complex128)
        self.ops, self.n_op, self.op_shared = None, 0, 0
        if ops is not None:
            op = np.ascontiguousarray(ops["op"], dtype=_I4)
            A, B = (np.ascontiguousarray(ops[k], dtype=_F8) for k in ("A_w", "B_w"))
            if op.shape != (self.n_cases,):
                raise ValueError("ops['op'] must name one operating point per case (%d)" % self.n_cases)
            if A.shape != B.shape or A.ndim not in (4, 5) or A.shape[-3] != A.shape[-2] or A.shape[-3] < 1:
                raise ValueError("ops A_w / B_w must both be [nD, n_op, m, m, nw] or [n_op, m, m, nw] (m = 6, or n_fd for "
                                 "generalised DOFs)")
            self.n_op, self.op_shared = int(A.shape[-4]), int(A.ndim == 4)
            if np.any(op < 0) or np.any(op >= self.n_op):
                raise ValueError("ops['op'] must lie in [0, %d)" % self.n_op)
            if "primary" in a and np.any(op[a["primary"]] != op):
                raise ValueError("a secondary wave train must share its primary's operating point")
            a["op"], a["op_A_w"], a["op_B_w"] = op, A, B
            self.ops = dict(op=op, A_w=A, B_w=B)

    def check_ops(self, batch):
        """Refuse operating-point tables whose design count or frequency grid is not ``batch``'s."""
        if self.ops is None:
            return
        A = self.ops["A_w"]
        if A.shape[-3:-1] != (6, 6):
            raise ValueError("operating-point tables %s: the rigid-body solves take 6 x 6 tables" % list(A.shape))
        if A.shape[-1] != batch.nw or (not self.op_shared and A.shape[0] != batch.n_designs):
            raise ValueError("operating-point tables %s do not match %d designs x %d bins" % (list(A.shape), batch.n_designs, batch.nw))

    def check_general_ops(self, n_fd, n_designs, nw):
        """Refuse operating points on a generalised-DOF solve whose ``fd`` has no support (n_fd = 0 or no fd), and tables that
        are not [n_designs, n_op, n_fd, n_fd, nw] or [n_op, n_fd, n_fd, nw]."""
        if self.ops is None:
            return
        if not n_fd:
            raise ValueError("per-case operating points without frequency-dependent terms (fd with n_fd >= 1) are not supported "
                             "for generalised-DOF FOWTs: pack them with packer.pack_general_matrices(fowt, states=...)")
        A = self.ops["A_w"]
        if A.shape[-3:-1] != (n_fd, n_fd) or A.shape[-1] != nw or (not self.op_shared and A.shape[0] != n_designs):
            raise ValueError("operating-point tables %s do not match %d designs x [%d, %d] support x %d bins"
                             % (list(A.shape), n_designs, n_fd, n_fd, nw))

    def input_bytes(self):
        return int(sum(v.nbytes for v in self.arrays.values()))

    def struct(self, ptr):
        s = RaftkCases()
        s.n_cases = self.n_cases
        for name in ("Hs", "Tp", "gamma", "beta_deg", "spec", "zeta", "primary", "F_2nd", "Xi_init", "op", "op_A_w", "op_B_w"):
            setattr(s, name, ptr(name) if name in self.arrays else None)
        s.n_op, s.op_shared = self.n_op, self.op_shared
        return s


def _host_ptr(arrays):
    return lambda name: arrays[name].ctypes.data


def _output_table(nD, nC, nw, nw2=0):
    """name -> (shape, numpy dtype) of every output of the rigid-FOWT solves; qtf and Xi_rao are on the second-order grid."""
    u = [nD, nC]
    return dict(Xi=(u + [6, nw], _C16), status=(u + [4], _I4), B_drag=(u + [6, 6], _F8), F_drag=(u + [6, nw], _C16),
                F_iner=(u + [6, nw], _C16), F_BEM=(u + [6, nw], _C16), zeta=([nC, nw], _F8), F_2nd=(u + [6, nw], _F8),
                F_2nd_mean=(u + [6], _F8), Xi_last=(u + [6, nw], _C16), qtf=(u + [nw2, nw2, 6], _C16), Xi_rao=(u + [6, nw2], _C16))


_HOST_OUTPUTS = ("Xi", "status", "B_drag", "F_drag", "F_iner", "F_BEM", "zeta", "F_2nd", "F_2nd_mean", "Xi_last")
_SESSION_OUTPUTS = _HOST_OUTPUTS[:-1]
_SLENDER_OUTPUTS = _HOST_OUTPUTS + ("qtf", "Xi_rao")


def _check_outputs(want, known):
    bad = [k for k in want if k not in known]
    if bad:
        raise ValueError("unknown outputs %s (known: %s)" % (bad, ", ".join(known)))


def _alloc_outputs(nD, nC, nw, want, known=_HOST_OUTPUTS, nw2=0, zeros=np.zeros):
    """The outputs named in ``want``, each one of ``known``, as ``zeros(shape, dtype)`` of the output table."""
    _check_outputs(want, known)
    table = _output_table(nD, nC, nw, nw2)
    return {k: zeros(*table[k]) for k in want}


def _torch_dtype(dtype):
    import torch
    return torch.from_numpy(np.empty(0, dtype)).dtype


def _torch_zeros(device):
    """``np.zeros`` for torch tensors on ``device``."""
    import torch
    return lambda shape, dtype: torch.zeros(shape, dtype=_torch_dtype(dtype), device=device)


def _opts(n_iter, tol, xi_start, cluster_size=0, flags=0):
    return RaftkSolveOpts(int(n_iter), int(cluster_size), float(tol), float(xi_start), flags, 0)


def _out_struct(outs, ptr):
    o = RaftkOutputs()
    for k in ("Xi", "status", "B_drag", "F_drag", "F_iner", "F_BEM", "zeta", "F_2nd", "F_2nd_mean", "Xi_last"):
        setattr(o, k, ptr(outs[k]) if k in outs else None)
    return o


def solve_dynamics(batch, cases, n_iter=10, tol=0.01, xi_start=0.0, cluster_size=0,
                   want=("Xi", "status", "B_drag"), out=None):
    """Model.solveDynamics for every (design, case), host buffers in/out (raft_model.py:966-1302).

    Returns a dict of NumPy arrays: Xi [nD,nC,6,nw] complex128, status [nD,nC,4] int32
    (passes, converged, flags, 0), B_drag [nD,nC,6,6], and optionally F_drag / F_iner / F_BEM / zeta.
    Designs that carry a QTF table (potSecOrder 2) get the difference-frequency force added to the linear
    excitation (raft_model.py:1035-1048); ask for it with ``want`` F_2nd [nD,nC,6,nw] / F_2nd_mean [nD,nC,6].
    """
    want = tuple(dict.fromkeys(tuple(want) + ("Xi", "status")))
    outs = out if out is not None else _alloc_outputs(batch.n_designs, cases.n_cases, batch.nw, want)
    cases.check_ops(batch)
    c = _host_struct(cases)
    o = _opts(n_iter, tol, xi_start, cluster_size)
    os_ = _out_struct(outs, lambda a: a.ctypes.data)

    def run(b):
        check(lib.raftk_solve_dynamics_host(C.byref(_host_struct(b)), C.byref(c), C.byref(o), C.byref(os_)))
        return outs
    return _retry_on_plan(batch, run)


def _plan_overflowed(status):
    """Whether a unit came back with RAFTK_FLAG_PLAN in ``status`` (numpy or torch): the batch's step-class hints were below
    the number of classes the kernels count (DesignBatch computes them by the kernels' rule, so only hints set by the
    caller can be), and those units ran no pass and hold zeros."""
    return bool((status[..., 2] & FLAG_PLAN).any())


def _retry_on_plan(batch, run):
    """``run(batch) -> outs``, run once more on ``worst_case_hints(batch)`` when a unit came back with RAFTK_FLAG_PLAN (a farm's
    Xi_sys was then assembled from those units' zero loads, so everything is solved again)."""
    outs = run(batch)
    if _plan_overflowed(outs["status"]):
        outs = run(worst_case_hints(batch))
        if _plan_overflowed(outs["status"]):
            raise _lib.RaftkError("step-class tables overflowed even with worst-case sizes")
    return outs


def worst_case_hints(batch):
    """A shallow copy of ``batch`` with the step-class hints at 0: the fused solvers then size their class tables for one
    class per node, which cannot overflow.  ``batch`` keeps its hints."""
    b = copy.copy(batch)
    b.max_w_classes = b.max_h_classes = b.max_z_classes = 0
    b.__dict__.pop("_host_struct_cache", None)
    return b


def solve_dynamics_farm(batch, cases, C_arr=None, M_arr=None, B_arr=None, n_iter=10, tol=0.01, xi_start=0.0, cluster_size=0,
                        want=("Xi", "status", "B_drag"), out=None):
    """Coupled farm response (raft_model.py:1164-1236), host buffers in/out, ONE call: the designs of ``batch`` are the N
    FOWTs of the array; every FOWT's drag linearisation runs as in ``solve_dynamics``, then the 6N x 6N system
    blockdiag(Z_i) + (-w^2 M_arr + i w B_arr + C_arr) is assembled and solved per (case, frequency) on the device.
    Array matrices: [6N,6N], or [1,6N,6N] as for a batch of one farm.
    -> the per-FOWT output dict plus ``Xi_sys`` complex [nC, 6N, nw] and ``info`` [nC, nw] (k+1 of a zero pivot).
    ``out``: caller-owned result arrays (e.g. page-locked ones from ``pinned_empty``: device-to-host copies then run at
    the link rate instead of through the driver's staging of pageable memory); missing ones are allocated."""
    cases.check_ops(batch)
    return _solve_farms(batch, cases, batch.n_designs, None, M_arr, B_arr, C_arr, _opts(n_iter, tol, xi_start, cluster_size), want, out)


def _farm_batch_matrices(n_farms, n, M_arr, B_arr, C_arr):
    """The array matrices of a farm batch as C-contiguous float64 -> (dict name -> array, arr_shared): every matrix given is
    [6N,6N] (one set for every farm) or every one is [F,6N,6N]."""
    mats = {nm: np.ascontiguousarray(v, dtype=_F8) for nm, v in (("M_arr", M_arr), ("B_arr", B_arr), ("C_arr", C_arr)) if v is not None}
    shapes = {a.shape for a in mats.values()}
    if len(shapes) > 1 or not shapes <= {(n, n), (n_farms, n, n)}:
        raise ValueError("M_arr, B_arr and C_arr must all be [%d, %d] or all be [%d, %d, %d]" % (n, n, n_farms, n, n))
    return mats, 0 if shapes == {(n_farms, n, n)} else 1


def _farm_setup(N, F, nC, nw, M_arr, B_arr, C_arr, out=None, device=None, outputs=True):
    """``F`` farms of ``N`` FOWTs as the farm-batch entries take them; ``F`` None is one farm, a batch of one whose outputs
    have no farm axis.  -> (RaftkFarmBatch, matrices, Xi_sys [F,nC,6N,nw], info [F,nC,nw]).  Host arrays, or with ``device``
    torch tensors there; ``out``: host Xi_sys / info the caller owns, checked and used in place; ``outputs=False``: none are
    allocated (Xi_sys, info None), the caller sets them on the struct."""
    n = 6 * N
    mats, shared = _farm_batch_matrices(F or 1, n, M_arr, B_arr, C_arr)
    lead = [] if F is None else [F]
    res = dict(Xi_sys=(lead + [nC, n, nw], _C16), info=(lead + [nC, nw], _I4))
    if device is None:
        ptr = lambda a: a.ctypes.data   # noqa: E731
        for k, (shape, dt) in res.items():
            a = (out or {}).get(k)
            if a is not None and (a.shape != tuple(shape) or a.dtype != dt or not a.flags.c_contiguous):
                raise ValueError("out[%r] must be a C-contiguous %s array %s" % (k, np.dtype(dt).name, shape))
            res[k] = np.zeros(shape, dt) if a is None else a
    else:
        import torch
        ptr = lambda t: t.data_ptr()    # noqa: E731
        mats = {nm: torch.from_numpy(a).to(device) for nm, a in mats.items()}
        res = {k: _torch_zeros(device)(*v) if outputs else None for k, v in res.items()}
    f = RaftkFarmBatch()
    f.n_farms, f.n_fowt, f.arr_shared = F or 1, N, shared
    for nm in ("M_arr", "B_arr", "C_arr"):
        setattr(f, nm, ptr(mats[nm]) if nm in mats else None)
    f.Xi_sys, f.info = (ptr(res["Xi_sys"]), ptr(res["info"])) if outputs else (None, None)
    return f, mats, res["Xi_sys"], res["info"]


def _solve_farms(batch, cases, N, F, M_arr, B_arr, C_arr, o, want, out):
    """``solve_dynamics_farm`` (``F`` None) and ``solve_dynamics_farm_batch`` through raftk_solve_dynamics_farm_batch_host."""
    f, mats, xi, info = _farm_setup(N, F, cases.n_cases, batch.nw, M_arr, B_arr, C_arr, out)
    want = tuple(dict.fromkeys(tuple(want) + ("Xi", "status")))
    outs = dict(out) if out is not None else {}
    outs.update(_alloc_outputs(batch.n_designs, cases.n_cases, batch.nw, tuple(k for k in want if k not in outs)))
    outs["Xi_sys"], outs["info"] = xi, info
    c = _host_struct(cases)
    os_ = _out_struct(outs, lambda a: a.ctypes.data)

    def run(b):
        check(lib.raftk_solve_dynamics_farm_batch_host(C.byref(_host_struct(b)), C.byref(c), C.byref(o), C.byref(os_), C.byref(f)))
        return outs
    return _retry_on_plan(batch, run)


def solve_dynamics_farm_batch(batch, cases, n_fowt, C_arr=None, M_arr=None, B_arr=None, n_iter=10, tol=0.01, xi_start=0.0, cluster_size=0,
                              want=("Xi", "status", "B_drag"), out=None):
    """``solve_dynamics_farm`` for F farms of ``n_fowt`` FOWTs each in ONE call (a layout or shared-mooring study): design
    ``f * n_fowt + i`` of ``batch`` is FOWT i of farm f, all farms over the same case table.  Array matrices: [6N,6N] used by
    every farm, or [F,6N,6N].  -> the per-FOWT output dict plus ``Xi_sys`` complex [F, nC, 6N, nw] and ``info`` [F, nC, nw];
    farm f's rows are what ``solve_dynamics_farm`` returns for that farm alone, bit for bit."""
    N = int(n_fowt)
    cases.check_ops(batch)
    if N < 1 or batch.n_designs % N:
        raise ValueError("n_fowt must divide the batch's %d designs" % batch.n_designs)
    return _solve_farms(batch, cases, N, batch.n_designs // N, M_arr, B_arr, C_arr, _opts(n_iter, tol, xi_start, cluster_size), want,
                        out)


def ragged_offsets(farm_sizes):
    """The CSR arrays of a ragged farm batch: -> (farm_fowt0 int32 [F+1], the first design of each farm and n_designs last;
    arr_offset int64 [F+1], the first double of each farm's [6N_f,6N_f] array matrix in the packed M_arr / B_arr / C_arr)."""
    N = np.asarray(farm_sizes, dtype=np.int64).reshape(-1)
    fowt0 = np.zeros(len(N) + 1, dtype=np.int32)
    fowt0[1:] = np.cumsum(N)
    arr = np.zeros(len(N) + 1, dtype=np.int64)
    arr[1:] = np.cumsum(36 * N * N)
    return fowt0, arr


def ragged_views(Xi_flat, farm_sizes, n_cases, nw):
    """Farm f's [nC, 6N_f, nw] block of a ragged batch's flat Xi_sys (numpy or torch), as views of ``Xi_flat``: farm f starts at
    6 nC nw farm_fowt0[f] complex values."""
    fowt0, _ = ragged_offsets(farm_sizes)
    per = 6 * n_cases * nw
    return [Xi_flat[per * int(a):per * int(b)].reshape(n_cases, 6 * (int(b) - int(a)), nw) for a, b in zip(fowt0[:-1], fowt0[1:])]


def _ragged_matrices(farm_sizes, M_arr, B_arr, C_arr):
    """The array matrices of a ragged batch -> (dict name -> C-contiguous float64 array, arr_shared): each given matrix is a
    list of F matrices [6N_f,6N_f], packed farm after farm; when every N_f is the same N it may also be one [6N,6N] set for
    every farm or a stacked [F,6N,6N] (one per farm), as the uniform batch takes them."""
    sizes = [int(n) for n in farm_sizes]
    mats, shared = {}, set()
    for nm, v in (("M_arr", M_arr), ("B_arr", B_arr), ("C_arr", C_arr)):
        if v is None:
            continue
        if not isinstance(v, (list, tuple)):
            a, n = np.asarray(v), 6 * sizes[0]
            equal = len(set(sizes)) == 1
            if equal and a.shape == (len(sizes), n, n):
                v = list(a)
            elif not (equal and a.shape == (n, n)):
                raise ValueError("%s: a list of %d matrices [6N_f, 6N_f] in farm order, or with every N_f = N one [6N, 6N] set "
                                 "or a stacked [F, 6N, 6N]; got shape %s for sizes %s" % (nm, len(sizes), a.shape, sizes))
        if isinstance(v, (list, tuple)):
            if len(v) != len(sizes) or any(np.shape(m) != (6 * n, 6 * n) for m, n in zip(v, sizes)):
                raise ValueError("%s: a list of %d matrices [6N_f, 6N_f] in farm order" % (nm, len(sizes)))
            mats[nm] = np.concatenate([np.ascontiguousarray(m, dtype=_F8).reshape(-1) for m in v])
            shared.add(0)
        else:
            mats[nm] = np.ascontiguousarray(v, dtype=_F8)
            shared.add(1)
    if len(shared) > 1:
        raise ValueError("M_arr, B_arr and C_arr must all be shared [6N,6N] sets or all be per-farm lists")
    return mats, (1 if shared == {1} else 0)


def _ragged_setup(farm_sizes, nC, nw, M_arr, B_arr, C_arr, out=None, device=None):
    """A ragged batch as raftk_farm_ragged takes it -> (RaftkFarmRagged, arrays to keep alive, Xi_sys flat, info [F,nC,nw]).
    Host arrays, or with ``device`` torch tensors there (the CSR arrays stay on the host either way)."""
    fowt0, arr = ragged_offsets(farm_sizes)
    mats, shared = _ragged_matrices(farm_sizes, M_arr, B_arr, C_arr)
    F, nD = len(fowt0) - 1, int(fowt0[-1])
    res = dict(Xi_sys=([6 * nD * nC * nw], _C16), info=([F, nC, nw], _I4))
    if device is None:
        ptr = lambda a: a.ctypes.data   # noqa: E731
        for k, (shape, dt) in res.items():
            a = (out or {}).get(k)
            if a is not None and (a.shape != tuple(shape) or a.dtype != dt or not a.flags.c_contiguous):
                raise ValueError("out[%r] must be a C-contiguous %s array %s" % (k, np.dtype(dt).name, shape))
            res[k] = np.zeros(shape, dt) if a is None else a
    else:
        import torch
        ptr = lambda t: t.data_ptr()    # noqa: E731
        mats = {nm: torch.from_numpy(a).to(device) for nm, a in mats.items()}
        res = {k: _torch_zeros(device)(*v) for k, v in res.items()}
    f = RaftkFarmRagged()
    f.n_farms, f.arr_shared = F, shared
    f.farm_fowt0, f.arr_offset = fowt0.ctypes.data, arr.ctypes.data
    for nm in ("M_arr", "B_arr", "C_arr"):
        setattr(f, nm, ptr(mats[nm]) if nm in mats else None)
    f.Xi_sys, f.info = ptr(res["Xi_sys"]), ptr(res["info"])
    return f, (fowt0, arr, mats), res["Xi_sys"], res["info"]


def solve_dynamics_farm_ragged(batch, cases, farm_sizes, C_arr=None, M_arr=None, B_arr=None, n_iter=10, tol=0.01, xi_start=0.0,
                               cluster_size=0, want=("Xi", "status", "B_drag"), out=None):
    """``solve_dynamics_farm`` for farms of different sizes in ONE call (array-size and layout studies): farm f has
    ``farm_sizes[f]`` FOWTs, the designs of ``batch`` are every farm's FOWTs in order, farm after farm, all farms over the same
    case table.  Array matrices: one [6N,6N] set for every farm (only when all sizes are equal), or lists of F matrices
    [6N_f,6N_f].  -> the per-FOWT output dict plus ``Xi_sys``, a list of per-farm complex [nC, 6N_f, nw] views of the flat
    buffer ``Xi_sys_flat``, and ``info`` [F, nC, nw]; farm f's arrays are what ``solve_dynamics_farm`` returns for that farm
    alone, bit for bit.  ``out``: caller-owned per-FOWT arrays, ``Xi_sys`` (flat) and ``info``."""
    cases.check_ops(batch)
    nC, nw = cases.n_cases, batch.nw
    f, keep, xi, info = _ragged_setup(farm_sizes, nC, nw, M_arr, B_arr, C_arr, out)
    want = tuple(dict.fromkeys(tuple(want) + ("Xi", "status")))
    outs = dict(out) if out is not None else {}
    outs.update(_alloc_outputs(batch.n_designs, nC, nw, tuple(k for k in want if k not in outs and k not in ("Xi_sys", "info"))))
    outs.pop("Xi_sys", None)
    c = _host_struct(cases)
    o = _opts(n_iter, tol, xi_start, cluster_size)
    os_ = _out_struct(outs, lambda a: a.ctypes.data)

    def run(b):
        check(lib.raftk_solve_dynamics_farm_ragged_host(C.byref(_host_struct(b)), C.byref(c), C.byref(o), C.byref(os_), C.byref(f)))
        return outs
    res = _retry_on_plan(batch, run)
    del keep
    res["Xi_sys_flat"], res["info"] = xi, info
    res["Xi_sys"] = ragged_views(xi, farm_sizes, nC, nw)
    return res


FLAG_NAN, FLAG_SINGULAR, FLAG_PLAN, FLAG_XCHG = 1, 2, 4, 8        # include/raftk.h RAFTK_FLAG_*
STEP_RTOL, STEP_ZERO, Z0_RTOL = 5e-14, 1e-14, 1e-12                # step-class tolerances (csrc/raftk_common.cuh)
DEEP_KH = 89.4                 # depth_funcs' deep-water branch (helpers.py:211)
WALK_SEED_EXP = 700.0          # deep-water seed exp(k z0) stays a normal double: e^-700 > DBL_MIN = e^-708.4
WALK_DOWN_EXP = 10.0           # a downward walk grows its seed's rounding by e^(k drop): e^10 * 2^-53 = 2.4e-12


def fused_walk_exact(a, k, depth):
    """Whether the fused solvers' node walk (DESIGN.md section 4) is exact for every member of the CSR tables ``a`` on the
    wave numbers ``k`` at water depth ``depth``.  The walk seeds a member's depth factors at its first submerged node z0,
    (C+S)/2 and (C-S)/2, and multiplies them by exp(+-k dz) per step.  It is inexact where
      - a deep-water bin (k h > 89.4) has k |z0| > WALK_SEED_EXP: the seed exp(k z0) is subnormal or zero, and so is every
        node of the member, the surface ones included;
      - a finite-depth bin has k (z0 - z_min) > WALK_DOWN_EXP on a member that walks down from z0: (C-S)/2 is the
        difference of two nearly equal numbers there, and its rounding grows by exp(k dz) at every step down.
    The planner sends inexact designs to the v1 solver, which evaluates depth_funcs at every node."""
    k = np.asarray(k, dtype=_F8)
    start = np.asarray(a["mem_node_start"], dtype=np.int64)
    cnt = np.diff(start)
    if not len(cnt) or not cnt.sum() or not np.any(k > 0):
        return True
    frame, rA, ls = (np.asarray(a[n], dtype=_F8) for n in ("mem_frame", "mem_rA", "node_ls"))
    mem = np.repeat(np.arange(len(cnt)), cnt)
    z = rA[mem, 2] + ls * frame[mem, 2]
    full = cnt > 0
    z0 = z[start[:-1][full]]
    drop = z0 - np.minimum.reduceat(z, start[:-1][full])
    deep = k * depth > DEEP_KH
    k_deep, k_fin = (float(k[m].max()) if np.any(m) else 0.0 for m in (deep, ~deep))
    return bool(k_deep * max(0.0, -float(z0.min())) <= WALK_SEED_EXP and k_fin * float(drop.max()) <= WALK_DOWN_EXP)


def raise_on_flags(status):
    """Translate the status flags of solved units into the reference's exceptions: NaN in the response ->
    ``Exception("Nan detected in response vector Xi.")`` (raft_model.py:1098-1099); a singular impedance ->
    ``numpy.linalg.LinAlgError`` (what ``np.linalg.solve`` raises at raft_model.py:1089)."""
    fl = np.asarray(status)[..., 2]
    if np.any(fl & FLAG_PLAN):
        raise _lib.RaftkError("fused solver: step-class tables overflowed the hint; outputs of those units are zero")
    if np.any(fl & FLAG_XCHG):
        raise _lib.RaftkError("fused solver: the exchange between a unit's CTAs timed out; outputs of those units are invalid")
    if np.any(fl & FLAG_SINGULAR) and not np.any(fl & FLAG_NAN):
        raise np.linalg.LinAlgError("Singular matrix")
    if np.any(fl & FLAG_NAN):
        raise Exception("Nan detected in response vector Xi.")


def hydro_excitation(batch, cases, want=("F_iner", "F_BEM", "zeta")):
    """FOWT.calcHydroExcitation for every (design, case) (raft_fowt.py:1732-1888), host buffers."""
    outs = _alloc_outputs(batch.n_designs, cases.n_cases, batch.nw, want)
    os_ = _out_struct(outs, lambda a: a.ctypes.data)
    check(lib.raftk_hydro_excitation_host(C.byref(_host_struct(batch)), C.byref(_host_struct(cases)), C.byref(os_)))
    return outs


def qtf_slender(P, beta_rad, Xi_rao):
    """FOWT.calcQTF_slenderBody on the GPU (raft_fowt.py:1988-2078) for one design and n (heading, motion RAO) pairs.
    ``P``: packed design with the ``qs_*`` tables (``packer.pack_qtf_members``); ``beta_rad`` [n]; ``Xi_rao`` complex
    [n,6,nw2] motion RAOs on the second-order grid (zeros = fixed body) -> qtf complex [n,nw2,nw2,6], Hermitian-filled."""
    beta = np.ascontiguousarray(np.atleast_1d(beta_rad), dtype=_F8)
    Xi = np.ascontiguousarray(Xi_rao, dtype=np.complex128)
    n, nw2 = len(beta), len(P["qs_w"])
    if Xi.shape != (n, 6, nw2):
        raise ValueError("Xi_rao must be [n,6,nw2] on the second-order grid")
    keep = {}

    def ptr_of(name, a):
        keep[name] = a
        return a.ctypes.data
    s = _slender_struct(P, ptr_of)
    out = np.zeros([n, nw2, nw2, 6], dtype=np.complex128)
    check(lib.raftk_qtf_slender_host(C.byref(s), n, beta.ctypes.data, Xi.ctypes.data, out.ctypes.data))
    return out


def _slender_struct(P, ptr_of):
    """raftk_slender for a design's ``qs_*`` tables; ``ptr_of(name, array)`` returns the address to store (host or device).
    The kernels find a node's member by scanning ``mem_node_start``, so the nodes of one member must be contiguous and in
    member order: an unsorted ``qs_node_mem`` would silently pair nodes with the wrong members."""
    start = _slender_node_start(P)
    s = RaftkSlender()
    s.n_nodes, s.n_members, s.n_seg, s.nw = int(start[-1]), len(start) - 1, len(P["qs_seg_mem"]), len(P["qs_w"])
    s.depth, s.rho, s.g = float(P["qs_depth"]), float(P["qs_rho"]), float(P["qs_g"])
    for name in _lib.SLENDER_ARRAYS:
        a = start if name == "mem_node_start" else np.asarray(P["qs_" + name])
        a = np.ascontiguousarray(a, dtype=_I4 if name in _SLENDER_I4 else _F8)
        setattr(s, name, ptr_of(name, a))
    return s


_SLENDER_I4 = ("mem_mcf", "mem_wl", "mem_node_start", "seg_mem")


def _slender_node_start(P):
    """Each member's first strip node in the design's ``qs_*`` tables ([n_members + 1])."""
    nm = len(P["qs_mem_mcf"])
    node_mem = np.asarray(P["qs_node_mem"], dtype=np.int64)
    if np.any(np.diff(node_mem) < 0) or (len(node_mem) and (node_mem[0] < 0 or node_mem[-1] >= nm)):
        raise ValueError("qs_node_mem must be non-decreasing member indices in [0, %d)" % nm)
    return np.concatenate([[0], np.cumsum(np.bincount(node_mem, minlength=nm))])


class SlenderBatch:
    """raftk_slender_batch: the ``qs_*`` tables (``packer.pack_qtf_members``) of several designs on ONE second-order grid,
    concatenated in design order with node / member / segment offsets; each design keeps its own member-local
    ``mem_node_start`` and ``seg_mem``."""

    def __init__(self, packed):
        if isinstance(packed, dict):
            packed = [packed]
        P0 = packed[0]
        qw = np.ascontiguousarray(P0["qs_w"], dtype=_F8)
        site = tuple(float(P0["qs_" + k]) for k in ("depth", "rho", "g"))
        cols = {n: [] for n in _lib.SLENDER_ARRAYS if n not in ("w", "k")}
        offs = dict(node=[0], member=[0], seg=[0])
        for P in packed:
            if not np.array_equal(np.asarray(P["qs_w"], dtype=_F8), qw):
                raise ValueError("all designs of a batch must share the second-order frequency grid")
            if tuple(float(P["qs_" + k]) for k in ("depth", "rho", "g")) != site:
                raise ValueError("all designs of a batch must share the water depth, density and g of their second-order tables")
            start = _slender_node_start(P)
            for name in cols:
                a = start if name == "mem_node_start" else P["qs_" + name]
                cols[name].append(np.asarray(a, dtype=_I4 if name in _SLENDER_I4 else _F8).reshape(-1))
            offs["node"].append(offs["node"][-1] + int(start[-1]))
            offs["member"].append(offs["member"][-1] + len(start) - 1)
            offs["seg"].append(offs["seg"][-1] + len(P["qs_seg_mem"]))
        self.arrays = {n: np.ascontiguousarray(np.concatenate(v)) for n, v in cols.items()}
        self.arrays["w"], self.arrays["k"] = qw, np.ascontiguousarray(P0["qs_k"], dtype=_F8)
        for n, v in offs.items():
            self.arrays[n + "_offset"] = np.array(v, dtype=_I4)
        self.n_designs, self.nw2 = len(packed), len(qw)
        self.depth, self.rho, self.g = site
        self.max_nodes, self.max_members, self.max_seg = (int(np.diff(offs[n]).max()) for n in ("node", "member", "seg"))

    def struct(self, ptr):
        """The C struct; ``ptr(name)`` returns the address (host or device) of array ``name``."""
        s = RaftkSlenderBatch()
        s.n_designs, s.max_nodes, s.max_members, s.max_seg = self.n_designs, self.max_nodes, self.max_members, self.max_seg
        s.node_offset, s.member_offset, s.seg_offset = ptr("node_offset"), ptr("member_offset"), ptr("seg_offset")
        c = s.cols
        c.n_nodes, c.n_members, c.n_seg = (int(self.arrays[n + "_offset"][-1]) for n in ("node", "member", "seg"))
        c.nw, c.depth, c.rho, c.g = self.nw2, self.depth, self.rho, self.g
        for name in _lib.SLENDER_ARRAYS:
            setattr(c, name, ptr(name))
        return s


def _slender_inputs(packed, cases):
    """The checks of ``solve_dynamics_slender`` -> (design batch without the second-order tables, slender tables, case table
    without F_2nd / Xi_init)."""
    if isinstance(packed, dict):
        packed = [packed]
    if "primary" in cases.arrays:
        raise NotImplementedError("potSecOrder 1 with several wave trains fails in the reference itself (raft_model.py:1229 rebinds Fhydro_2nd)")
    sb = SlenderBatch(packed)
    batch = DesignBatch([{k: v for k, v in P.items() if not k.startswith(("qtf", "qs_"))} for P in packed])
    base = {k: v for k, v in cases.arrays.items() if k not in ("F_2nd", "Xi_init")}
    return batch, sb, CaseTable(base, zeta=base.get("zeta"), ops=cases.ops)


def _check_slender_iters(n_iter):
    if n_iter < 1:
        raise ValueError("potSecOrder 1 needs nIter >= 1")


def slender_flow_host(packed, cases, n_iter=10, tol=0.01, xi_start=0.0, cluster_size=0, want=("Xi", "status", "B_drag"), qtf_chunk=0):
    """``solve_dynamics_slender`` in ONE library call (raftk_solve_dynamics_slender_host: the whole flow on the device, host
    buffers in and out) -> dict of NumPy arrays named as in ``want`` (``SlenderSession``'s names)."""
    batch, sb, ct = _slender_inputs(packed, cases)
    _check_slender_iters(n_iter)
    want = tuple(dict.fromkeys(("Xi", "status") + tuple(want)))
    outs = _alloc_outputs(batch.n_designs, ct.n_cases, batch.nw, want, _SLENDER_OUTPUTS, sb.nw2)
    so = RaftkSlenderOutputs(outs["qtf"].ctypes.data if "qtf" in outs else None, outs["Xi_rao"].ctypes.data if "Xi_rao" in outs else None,
                             int(qtf_chunk), 0)
    o = _opts(n_iter, tol, xi_start, cluster_size)
    check(lib.raftk_solve_dynamics_slender_host(C.byref(_host_struct(batch)), C.byref(sb.struct(_host_ptr(sb.arrays))), C.byref(_host_struct(ct)),
                                                C.byref(o), C.byref(_out_struct(outs, lambda a: a.ctypes.data)), C.byref(so)))
    return outs


class SlenderSession:
    """``solve_dynamics_slender`` (Model.solveDynamics with potSecOrder 1, raft_model.py:1052-1142) with tables, workspace and
    outputs resident in HBM (torch tensors): ``solve()`` enqueues raftk_solve_dynamics_slender_dev on torch's current stream --
    loop A, RAOs, slender-body QTF, second-order force, loop B and the merge, with no host synchronisation.  ``want``: the
    names of ``DeviceSession`` plus F_2nd, F_2nd_mean, Xi_last, qtf [nD,nC,nw2,nw2,6] and Xi_rao [nD,nC,6,nw2].
    ``qtf_chunk``: units whose QTF tables are built at once in the workspace (0: all); each unit's QTF alone takes
    96 nw2^2 bytes.  ``farm_response()`` couples the designs as the FOWTs of an array, second-order force included."""

    def __init__(self, packed, cases, device=None, want=("Xi", "status", "B_drag"), qtf_chunk=0):
        import torch
        self.torch = torch
        batch, sb, ct = _slender_inputs(packed, cases)
        self.want = want = tuple(dict.fromkeys(("Xi", "status") + tuple(want)))
        _check_outputs(want, _SLENDER_OUTPUTS)
        own = tuple(k for k in want if k in ("Xi_last", "qtf", "Xi_rao"))
        self.dev = DeviceSession(batch, ct, device=device, workspace_bytes=0, want=tuple(k for k in want if k not in own))
        self.device, self.batch, self.slender = self.dev.device, batch, sb
        self.d_struct, self.c_struct = self.dev.d_struct, self.dev.c_struct
        with torch.cuda.device(self.device):
            self.st = {k: torch.from_numpy(v).to(self.device) for k, v in sb.arrays.items()}
            self.s_struct = sb.struct(lambda name: self.st[name].data_ptr())
            self.out = dict(self.dev.out)
            self.out.update(_alloc_outputs(batch.n_designs, ct.n_cases, batch.nw, own, _SLENDER_OUTPUTS, sb.nw2, _torch_zeros(self.device)))
            self.o_struct = _out_struct(self.out, lambda t: t.data_ptr())
            ptr = lambda k: self.out[k].data_ptr() if k in self.out else None   # noqa: E731
            self.so = RaftkSlenderOutputs(ptr("qtf"), ptr("Xi_rao"), int(qtf_chunk), 0)
            self.workspace_bytes = int(lib.raftk_solve_dynamics_slender_workspace_bytes(C.byref(self.d_struct), C.byref(self.s_struct),
                                                                                         ct.n_cases, int(qtf_chunk)))
            self.workspace = torch.empty(self.workspace_bytes, dtype=torch.uint8, device=self.device)
        self.qtf_chunk = int(qtf_chunk)

    def solve(self, n_iter=10, tol=0.01, xi_start=0.0, cluster_size=0):
        """Enqueue the potSecOrder 1 solve of every unit on the current stream; returns the output dict (async)."""
        _check_slender_iters(n_iter)
        o = _opts(n_iter, tol, xi_start, cluster_size)
        with self.torch.cuda.device(self.device):
            check(lib.raftk_solve_dynamics_slender_dev(C.byref(self.d_struct), C.byref(self.s_struct), C.byref(self.c_struct), C.byref(o),
                                                       C.byref(self.o_struct), C.byref(self.so), self.workspace.data_ptr(),
                                                       self.workspace_bytes, self.dev._stream()))
        return self.out

    def farm_response(self, C_arr=None, M_arr=None, B_arr=None):
        """Enqueue the coupled 6N-DOF system response of the LAST ``solve`` (raft_model.py:1164-1216) with each FOWT's
        second-order force in its excitation (:1212) -> (Xi_sys [nC,6N,nw], info).  Needs want with B_drag, F_drag, F_iner,
        F_2nd (and F_BEM when the designs carry BEM excitation)."""
        need = ("B_drag", "F_drag", "F_iner", "F_2nd") + (("F_BEM",) if self.batch.n_bem_head else ())
        missing = [k for k in need if k not in self.out]
        if missing:
            raise ValueError("farm_response needs the outputs %s in want" % missing)
        cf = RaftkCases.from_buffer_copy(self.c_struct)
        cf.F_2nd = self.out["F_2nd"].data_ptr()
        self.dev.c_struct, self.dev.o_struct = cf, self.o_struct
        return self.dev.farm_response(C_arr=C_arr, M_arr=M_arr, B_arr=B_arr)


def get_rao(Xi, zeta):
    """helpers.getRAO (helpers.py:762-784): response per unit wave amplitude, zero where |zeta| <= 1e-6."""
    Xi, zeta = np.asarray(Xi), np.asarray(zeta)
    ok = np.abs(zeta) > 1e-6
    out = np.zeros_like(Xi, dtype=complex)
    out[..., ok] = Xi[..., ok] / zeta[ok]
    return out


def solve_dynamics_slender(packed, cases, n_iter=10, tol=0.01, xi_start=0.0, cluster_size=0, want=("Xi", "status", "B_drag")):
    """Model.solveDynamics with potSecOrder 1 (raft_model.py:1052-1142) for every (design, case): (A) the drag-linearisation
    loop without second-order forces; (B) where it converged: motion RAOs -> slender-body QTF on the second-order grid ->
    difference-frequency force -> the loop continues from the SAME iterate with the force added and its counter reset
    (the reference sets iiter = 0 and the loop header increments it to 1, raft_model.py:1106-1131, so loop (B) runs at
    most n_iter passes: it is launched with n_iter - 1, i.e. max_pass = n_iter).  Units whose loop (A) did not converge
    keep its result and get no QTF / second-order force (zeros), like the reference, which never computes them there.
    n_iter = 0 is rejected: the reference would still add F_2nd to the final system response (documented deviation).
    ``packed``: list of packed designs carrying ``qs_*`` tables on one second-order grid; ``cases``: CaseTable (single
    wave train per case).  Extra outputs: F_2nd, F_2nd_mean, qtf [nD,nC,nw2,nw2,6]."""
    if isinstance(packed, dict):
        packed = [packed]
    batch, sb, ct = _slender_inputs(packed, cases)
    _check_slender_iters(n_iter)
    nD, nC, nw = batch.n_designs, cases.n_cases, batch.nw
    base = ct.arrays
    wantA = tuple(dict.fromkeys(tuple(want) + ("Xi", "status", "zeta", "Xi_last")))
    A = solve_dynamics(batch, ct, n_iter=n_iter, tol=tol, xi_start=xi_start, cluster_size=cluster_size, want=wantA)
    qw = sb.arrays["w"]
    beta_rad = cases.arrays["beta_deg"] * 0.017453292519943295
    qtf = np.zeros([nD, nC, len(qw), len(qw), 6], dtype=np.complex128)
    for d, P in enumerate(packed):
        Xi2 = np.zeros([nC, 6, len(qw)], dtype=np.complex128)
        for c in range(nC):
            r = get_rao(A["Xi"][d, c], A["zeta"][c])
            for a in range(6):
                Xi2[c, a] = np.interp(qw, batch.w, r[a], left=0, right=0)          # raft_fowt.py:2021-2023
        qtf[d] = qtf_slender(P, beta_rad, Xi2)
    qb = copy.copy(batch)                                                           # the designs with these QTFs as their table
    qb.__dict__.pop("_host_struct_cache", None)
    qb.arrays = _Tables(batch.arrays, qtf_w=qw, qtf_heads=np.zeros(1), qtf=np.ascontiguousarray(qtf.reshape(nD, nC, len(qw), len(qw), 1, 6)))
    qb.n_qtf_w, qb.n_qtf_head, qb.qtf_shared = len(qw), 1, 2
    F2 = second_order_force(qb, CaseTable(base, zeta=base.get("zeta")))
    B = solve_dynamics(batch, CaseTable(base, zeta=base.get("zeta"), F_2nd=F2["F_2nd"], Xi_init=A["Xi_last"], ops=cases.ops), n_iter=n_iter - 1, tol=tol,
                       xi_start=xi_start, cluster_size=cluster_size, want=wantA)
    ok = A["status"][:, :, 1] == 1                                                   # units whose first loop converged
    out = {}
    for k in wantA:
        if k == "zeta":
            out[k] = A[k]
            continue
        sel = ok.reshape(ok.shape + (1,) * (A[k].ndim - 2))
        out[k] = np.where(sel, B[k], A[k])
    out["status"][:, :, 0] = A["status"][:, :, 0] + np.where(ok, B["status"][:, :, 0], 0)
    out["status"][:, :, 2] = A["status"][:, :, 2] | np.where(ok, B["status"][:, :, 2], 0)
    okf = ok[:, :, None, None]
    out["F_2nd"] = np.where(okf, F2["F_2nd"], 0.0)
    out["F_2nd_mean"] = np.where(ok[:, :, None], F2["F_2nd_mean"], 0.0)
    out["qtf"] = np.where(ok[:, :, None, None, None], qtf, 0.0)
    return out


def _general_struct(P, M, B, Cm, ptr_of):
    """raftk_general for a packed flexible design; ``ptr_of(name, array)`` returns the address to store (host or device)."""
    n, nw, Ns = int(P["gen_nDOF"]), len(P["w"]), len(P["node_ls"])
    g = RaftkGeneral()
    g.n_dof, g.nw, g.n_nodes = n, nw, Ns
    g.depth, g.rho, g.dw = float(P["depth"]), float(P["rho"]), float(P["dw"])
    mem = np.asarray(P["node_mem"], dtype=np.int64)
    frame = np.concatenate([np.asarray(P["mem_q"])[mem], np.asarray(P["mem_p1"])[mem], np.asarray(P["mem_p2"])[mem]], axis=1) if Ns else np.zeros([0, 9])
    cd = np.stack([np.asarray(P["node_a_q"]) * np.asarray(P["node_Cd_q"]), np.asarray(P["node_a_p1"]) * np.asarray(P["node_Cd_p1"]),
                   np.asarray(P["node_a_p2"]) * np.asarray(P["node_Cd_p2"]), np.asarray(P["node_a_End"]) * np.asarray(P["node_Cd_End"])], axis=1) if Ns else np.zeros([0, 4])
    arrays = dict(w=P["w"], k=P["k"], node_r=P["node_r"], node_frame=frame, node_circ=np.asarray(P["mem_circ"], dtype=_I4)[mem] if Ns else np.zeros(0, dtype=_I4),
                  node_Imat=P["node_Imat"], node_a_i=P["node_a_i"], node_cd=cd, Tn=P["gen_Tn"], rr=P["gen_rr"], M=M, B=B, C=Cm)
    if P.get("node_Imat_w") is not None:
        arrays["node_Imat_w"] = np.ascontiguousarray(P["node_Imat_w"], dtype=np.complex128)
    for name in _lib.GENERAL_ARRAYS:
        if name not in arrays:
            setattr(g, name, None)
            continue
        a = np.ascontiguousarray(arrays[name], dtype=_I4 if name == "node_circ" else (np.complex128 if name == "node_Imat_w" else _F8))
        setattr(g, name, ptr_of(name, a))
    return g


def _general_fd_struct(fd, n, nw, ptr_of):
    """raftk_general_fd for the ``fd`` dict of ``packer.pack_general_matrices`` (keys fd_idx, A_w, B_w [n_fd,n_fd,nw]; optional
    X_BEM [nhead,6,nw], bem_headings, heading_adjust, T0 [6,nDOF]; x_ref, y_ref), or None for fd=None."""
    if fd is None:
        return None
    f = RaftkGeneralFd()
    idx = np.ascontiguousarray(fd.get("fd_idx", np.zeros(0)), dtype=_I4)
    f.n_fd = nf = len(idx)
    if nf:
        A_w, B_w = (np.ascontiguousarray(fd[k], dtype=_F8) for k in ("A_w", "B_w"))
        if A_w.shape != (nf, nf, nw) or B_w.shape != (nf, nf, nw):
            raise ValueError("fd: A_w and B_w must be [n_fd, n_fd, nw] = [%d, %d, %d]" % (nf, nf, nw))
        f.fd_idx, f.A_w, f.B_w = ptr_of("fd_idx", idx), ptr_of("fd_A_w", A_w), ptr_of("fd_B_w", B_w)
    if fd.get("X_BEM") is not None:
        hd = np.ascontiguousarray(fd["bem_headings"], dtype=_F8)
        X = np.ascontiguousarray(fd["X_BEM"], dtype=np.complex128)
        T0 = np.ascontiguousarray(fd["T0"], dtype=_F8)
        if X.shape != (len(hd), 6, nw) or T0.shape != (6, n):
            raise ValueError("fd: X_BEM must be [n_bem_head, 6, nw] and T0 [6, nDOF]")
        f.n_bem_head = len(hd)
        f.bem_headings, f.X_BEM, f.T0 = ptr_of("fd_bem_headings", hd), ptr_of("fd_X_BEM", X), ptr_of("fd_T0", T0)
        f.heading_adjust = float(fd.get("heading_adjust", 0.0))
    f.x_ref, f.y_ref = float(fd.get("x_ref", 0.0)), float(fd.get("y_ref", 0.0))
    return f


def _general_qtf_struct(qtf, ptr_of):
    """raftk_general_qtf for the dict of ``packer.pack_general_qtf`` (qtf complex [nw2,nw2,nheads,6], qtf_w [nw2] rad/s,
    qtf_heads [nheads] rad), or None for qtf=None or {} (potSecOrder 0)."""
    if not qtf:
        return None
    qw = np.ascontiguousarray(qtf["qtf_w"], dtype=_F8)
    qh = np.ascontiguousarray(qtf["qtf_heads"], dtype=_F8)
    Q = np.ascontiguousarray(qtf["qtf"], dtype=np.complex128)
    if Q.shape != (len(qw), len(qw), len(qh), 6):
        raise ValueError("qtf must be [nw2, nw2, nheads, 6] with nw2 = len(qtf_w), nheads = len(qtf_heads)")
    q = RaftkGeneralQtf()
    q.n_qtf_w, q.n_qtf_head = len(qw), len(qh)
    q.qtf_w, q.qtf_heads, q.qtf = ptr_of("qtf_w", qw), ptr_of("qtf_heads", qh), ptr_of("qtf", Q)
    return q


class _GeneralResident:
    """What ``GeneralSession`` and ``GeneralBatchSession`` share: their tables uploaded into torch tensors on ``device``
    (``keep``), the workspace and output tensors over the leading unit axes (``[nT]`` or ``[nD, nT]``), the solve's
    enqueueing and the reductions of the last ``solve()`` on the resident Xi [..., nT, nDOF, nw]."""

    def _open(self, device):
        import torch
        self.torch = torch
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.keep = {}

    def _to_dev(self, name, a):
        t = self.torch.from_numpy(a.view(np.float64) if a.dtype == np.complex128 else a).to(self.device)
        self.keep[name] = t
        return t.data_ptr()

    def _upload_cases(self, cases):
        self.ct = {k: self.torch.from_numpy(v).to(self.device) for k, v in cases.arrays.items()}
        self.c_struct = cases.struct(lambda name: self.ct[name].data_ptr())

    def _outputs(self, lead, n, nw, F_BEM):
        """The workspace of ``workspace_bytes`` and the outputs: Xi, status, F_BEM with ``F_BEM``, F_2nd and F_2nd_mean with
        a QTF table."""
        torch, dev, qtf = self.torch, self.device, self.qtf is not None
        self.workspace = torch.empty(self.workspace_bytes, dtype=torch.uint8, device=dev)
        self.Xi = torch.zeros(lead + [n, nw], dtype=torch.complex128, device=dev)
        self.status = torch.zeros(lead + [4], dtype=torch.int32, device=dev)
        self.F_BEM = torch.zeros(lead + [n, nw], dtype=torch.complex128, device=dev) if F_BEM else None
        self.F_2nd = torch.zeros(lead + [6, nw], dtype=torch.float64, device=dev) if qtf else None
        self.F_2nd_mean = torch.zeros(lead + [6], dtype=torch.float64, device=dev) if qtf else None

    def _enqueue(self, entry, structs, n_iter, tol, xi_start, *max_chunk):
        """``entry`` (a raftk_general_*_dev solve) on the resident tables and outputs, on torch's current stream."""
        o = _opts(n_iter, tol, xi_start)
        ptr = lambda t: t.data_ptr() if t is not None else None   # noqa: E731
        with self.torch.cuda.device(self.device):
            stream = self.torch.cuda.current_stream(self.device).cuda_stream
            check(entry(*_refs(*structs), C.byref(self.c_struct), C.byref(o), self.Xi.data_ptr(), self.status.data_ptr(), ptr(self.F_BEM),
                        ptr(self.F_2nd), ptr(self.F_2nd_mean), self.workspace.data_ptr(), self.workspace_bytes, *max_chunk, stream))
        return (self.Xi, self.status) if self.F_BEM is None else (self.Xi, self.status, self.F_BEM)

    def stats(self, R, wpow, psd=True, amp=False):
        """Output-channel statistics of the last ``solve()`` on the device (raftk_general_channel_stats_dev, on each design's
        slice of Xi): R [nch,nDOF] (``packer.pack_general_channels``), or [nD,nch,nDOF] in a design batch, wpow [nch] ->
        (std [..., nT,nch], PSD [..., nT,nch,nw] or None, amplitudes complex [..., nT,nch,nw] or None), torch tensors."""
        return _general_channel_stats(_session_buffers(self), R, wpow, self.keep["w"], self.Xi, self.dw, psd, amp)

    def rotor_stats(self, R, C_, V_w, gains, case_row0=None, psd=True):
        """Rotor speed, generator torque and blade pitch statistics of the last ``solve()`` on the device
        (raftk_rotor_stats_dev, no host round trip, every design in one launch sequence): ``R`` [nrot, nDOF] or, in a design
        batch, [nD, nrot, nDOF] (each design's hub rows); ``C``, ``V_w``, ``gains`` ([nC, nrot, ...], or per design [nD, nC,
        nrot, ...]) and ``case_row0`` as ``rotor_stats`` (``packer.pack_rotor_outputs``; the first train of every case, e.g.
        ``pack_case_trains``' ``first`` + [nT]).  -> (std [..., nC, nrot, 3], PSD [..., nC, nrot, 3, nw] or None), torch tensors."""
        return _rotor_stats(_session_buffers(self), R, C_, V_w, gains, self.keep["w"], self.Xi, self.dw, case_row0, None, psd)

    def fatigue(self, m, R=None, wpow=None, coef=None, case_row0=None, f_eq=1.0, method="dirlik", weights=None, life=None,
                moments=True, tile_w=0):
        """Fatigue DELs of the last ``solve()`` on the device (raftk_fatigue_dev, no host round trip, every design in one
        launch sequence): ``R`` [nch, nDOF] or, in a design batch, [nD, nch, nDOF] with ``wpow`` (``packer.pack_general_channels``'
        rows) or ``coef``, and the other arguments as ``fatigue``; ``case_row0`` groups the trains into cases.  -> dict of
        torch tensors as ``fatigue`` (DEL [..., nC, nch], ...)."""
        return _fatigue(_session_buffers(self), self.Xi, self.keep["w"], m, R, wpow, coef, case_row0, f_eq, method, weights, life,
                        moments, tile_w)

    def stress_ring(self, fa, ss, angles=None, d=10.0, t=0.083, m=None, f_eq=1.0, method="dirlik", weights=None, case_row0=None,
                    col0=None, psd=False, mean=None, wpow=None, tile_w=0):
        """Tower-base axial stress around the circumference of the last ``solve()`` (raftk_stress_ring_dev on the resident Xi,
        one unit per design): ``fa`` / ``ss`` the fore-aft / side-side rows (MbaseY / MbaseX of ``packer.pack_general_channels``),
        [n_rings, nDOF] or, in a design batch, [nD, n_rings, nDOF]; the other arguments as ``stress_ring``.  -> dict of torch
        tensors as ``stress_ring`` (std [..., nC, n_rings, nA], ...)."""
        return _stress_ring(_session_buffers(self), self.Xi, self.keep["w"], fa, ss, angles, d, t, m, f_eq, method, weights, case_row0,
                            col0, psd, mean, wpow, self.dw, tile_w)


class GeneralSession(_GeneralResident):
    """Generalised-DOF solve with tables, workspace and outputs resident in HBM (torch tensors), kernels on torch's current
    stream: ``solve()`` enqueues raftk_general_solve_dynamics_dev -> (Xi [nT,nDOF,nw] complex, status [nT,4]); ``cases`` may
    carry wave trains (``packer.pack_case_trains``).  ``stats(R, wpow)`` reduces the device Xi to output-channel statistics
    on the device (raftk_general_channel_stats_dev), so the responses never leave HBM.  ``fd``: frequency-dependent added
    mass, damping and BEM excitation (``packer.pack_general_matrices``); with ``F_BEM=True`` ``solve()`` also returns the BEM
    excitation in reduced DOFs, complex [nT,nDOF,nw].  ``qtf``: second-order wave loads (``packer.pack_general_qtf``); every
    ``solve()`` then leaves the force of every case and train in the device tensors ``F_2nd`` [nT,6,nw] and ``F_2nd_mean``
    [nT,6] (reduced DOFs 0-5).  ``max_chunk_cases``: None runs the table in one launch sequence (at most 65535 cases, a
    workspace for every case at once); an integer K streams it in chunks of whole train groups of at most K cases (0: one
    chunk) through a workspace sized for one chunk (raftk_general_solve_dynamics_stream_dev, ``general_chunk_for_budget``),
    with the same results.  ``cases`` may carry per-case operating points, as for ``general_solve_dynamics``."""

    def __init__(self, P, M, B, Cm, cases, device=None, fd=None, F_BEM=False, qtf=None, max_chunk_cases=None):
        self._open(device)
        with self.torch.cuda.device(self.device):
            self.g = _general_struct(P, M, B, Cm, self._to_dev)
            self._upload_cases(cases)
            n, nw, nC = int(P["gen_nDOF"]), len(P["w"]), cases.n_cases
            cases.check_general_ops(int(len(fd.get("fd_idx", ()))) if fd is not None else 0, 1, nw)
            self.fd = _general_fd_struct(fd, n, nw, self._to_dev)
            self.qtf = _general_qtf_struct(qtf, self._to_dev)
            g, fdp, qp = _refs(self.g, self.fd, self.qtf)
            self.max_chunk_cases = None if max_chunk_cases is None else int(max_chunk_cases)
            if self.max_chunk_cases is None:
                self.workspace_bytes = int(lib.raftk_general_qtf_workspace_bytes(g, fdp, qp, nC))
            else:
                if self.max_chunk_cases < 0:
                    raise ValueError("max_chunk_cases must be >= 0 (0: all cases in one chunk)")
                self.workspace_bytes = int(lib.raftk_general_stream_workspace_bytes(g, fdp, qp, nC, self.max_chunk_cases))
            self._outputs([nC], n, nw, F_BEM)
        self.n, self.nw, self.n_cases, self.dw = n, nw, nC, float(P["dw"])

    def solve(self, n_iter=10, tol=0.01, xi_start=0.0):
        structs = (self.g, self.fd, self.qtf)
        if self.max_chunk_cases is None:
            return self._enqueue(lib.raftk_general_solve_dynamics_qtf_dev, structs, n_iter, tol, xi_start)
        return self._enqueue(lib.raftk_general_solve_dynamics_stream_dev, structs, n_iter, tol, xi_start, self.max_chunk_cases)


def general_solve_dynamics(P, M, B, Cm, cases, n_iter=10, tol=0.01, xi_start=0.0, fd=None, F_BEM=False, qtf=None, F_2nd=False,
                           max_chunk_cases=None):
    """Model.solveDynamics for one FOWT with generalised degrees of freedom (flexible members), host buffers:
    ``P`` from ``packer.pack_general_dofs`` (node tables + ``gen_Tn``, ``gen_rr``), constant system
    matrices ``M, B, Cm`` [nDOF,nDOF], ``cases`` a CaseTable, with wave trains when built from ``packer.pack_case_trains``
    (train 0 of a case drives the linearisation, raft_model.py:1200-1236) -> (Xi complex [nT,nDOF,nw], status [nT,4]).
    ``fd``: frequency-dependent added mass and damping (operating rotors, BEM coefficients) and BEM excitation, the ``fd``
    dict of ``packer.pack_general_matrices`` (whose M, B, C are then the constant matrices).  ``F_BEM=True`` appends the BEM
    excitation of every case and train in reduced DOFs, complex [nT,nDOF,nw], to the result.  ``qtf``: second-order wave
    loads (potSecOrder 2), the dict of ``packer.pack_general_qtf``; ``F_2nd=True`` (with ``qtf``) then appends the force of
    every case and train on reduced DOFs 0-5, F_2nd [nT,6,nw] and F_2nd_mean [nT,6].  ``max_chunk_cases``: None solves the
    table in one launch sequence; an integer K streams it through a device workspace for K cases (``GeneralSession``).
    ``cases`` may carry per-case operating points on the support of ``fd`` (``CaseTable(ops=)``, tables [1 or none, n_op,
    n_fd, n_fd, nw]; ``packer.pack_general_matrices(fowt, states=...)``); without fd they are refused."""
    n, nw = int(P["gen_nDOF"]), len(P["w"])
    keep = {}

    def ptr(name, a):
        keep[name] = a
        return a.ctypes.data
    g = _general_struct(P, M, B, Cm, ptr)
    f = _general_fd_struct(fd, n, nw, ptr)
    q = _general_qtf_struct(qtf, ptr)
    if F_2nd and q is None:
        raise ValueError("F_2nd=True needs a QTF table (qtf=, packer.pack_general_qtf)")
    cases.check_general_ops(f.n_fd if f is not None else 0, 1, nw)
    nC = cases.n_cases
    Xi = np.zeros([nC, n, nw], dtype=np.complex128)
    st = np.zeros([nC, 4], dtype=_I4)
    Fb = np.zeros([nC, n, nw], dtype=np.complex128) if F_BEM else None
    F2, F2m = (np.zeros([nC, 6, nw]), np.zeros([nC, 6])) if F_2nd else (None, None)
    c = cases.struct(_host_ptr(cases.arrays))
    o = _opts(n_iter, tol, xi_start)
    hp = lambda a: a.ctypes.data if a is not None else None   # noqa: E731
    fp, qp = (C.byref(f) if f is not None else None), (C.byref(q) if q is not None else None)
    if max_chunk_cases is None:
        check(lib.raftk_general_solve_dynamics_qtf_host(C.byref(g), fp, qp, C.byref(c), C.byref(o), Xi.ctypes.data, st.ctypes.data, hp(Fb),
                                                        hp(F2), hp(F2m)))
    else:
        check(lib.raftk_general_solve_dynamics_stream_host(C.byref(g), fp, qp, C.byref(c), C.byref(o), Xi.ctypes.data, st.ctypes.data,
                                                           hp(Fb), hp(F2), hp(F2m), int(max_chunk_cases)))
    return (Xi, st) + ((Fb,) if F_BEM else ()) + ((F2, F2m) if F_2nd else ())


def general_stream_workspace_bytes(P, fd, qtf, n_cases, max_chunk_cases):
    """raftk_general_stream_workspace_bytes: device workspace of the streamed generalised-DOF solve of ``n_cases`` cases in
    chunks of at most ``max_chunk_cases`` (0: all).  Depends on the counts only (DOFs, bins, nodes, BEM and QTF tables present)."""
    n, nw = int(P["gen_nDOF"]), len(P["w"])
    g = RaftkGeneral()
    g.n_dof, g.nw, g.n_nodes = n, nw, len(P["node_ls"])
    none = lambda name, a: None       # noqa: E731
    f, q = _general_fd_struct(fd, n, nw, none), _general_qtf_struct(qtf, none)
    return int(lib.raftk_general_stream_workspace_bytes(C.byref(g), C.byref(f) if f is not None else None,
                                                        C.byref(q) if q is not None else None, int(n_cases), int(max_chunk_cases)))


def general_chunk_plan(primary, n_cases, max_chunk_cases):
    """The chunks raftk_general_solve_dynamics_stream_* cut a case table into -> [c_0 = 0, c_1, ..., n_cases]: whole train
    groups (``sweep.general_groups``) packed greedily in table order into chunks of at most ``max_chunk_cases`` (0: all).
    ValueError where the library refuses the table: interleaved groups, a group larger than a chunk."""
    return _chunk_plan(primary, n_cases, 1, max_chunk_cases, "max_chunk_cases")


def _chunk_plan(primary, n_cases, n_designs, max_chunk, cap_name):
    """The chunk starts of ``n_designs`` designs' units over a case table, design-major, and n_designs * n_cases: every
    design's train groups in table order, packed greedily into chunks of at most ``max_chunk`` units (0: all); a chunk may
    cross design boundaries.  ``cap_name``: the chunk cap's argument name in the messages."""
    from .sweep import general_groups
    n, nD = int(n_cases), int(n_designs)
    nU = n * nD
    K = nU if (max_chunk <= 0 or max_chunk >= nU) else int(max_chunk)
    g = general_groups(primary, n)
    for a, b in zip(g[:-1], g[1:]):
        if b - a > K:
            raise ValueError("a train group has %d cases, more than %s = %d" % (b - a, cap_name, K))
    cuts = [0]
    for d in range(nD):
        for a, b in zip(g[:-1], g[1:]):
            if d * n + b - cuts[-1] > K:
                cuts.append(int(d * n + a))
    return cuts + [nU]


def general_chunk_for_budget(P, fd, qtf, n_cases, budget_bytes):
    """The largest ``max_chunk_cases`` whose streamed workspace fits ``budget_bytes`` (``n_cases`` when the whole table fits).
    The chunk must still hold the largest train group of the table; ValueError when not even one case fits."""
    n_cases, budget = int(n_cases), int(budget_bytes)
    ws = lambda k: general_stream_workspace_bytes(P, fd, qtf, n_cases, k)     # noqa: E731
    if ws(n_cases) <= budget:
        return n_cases
    if ws(1) > budget:
        raise ValueError("a workspace of %d bytes does not hold one case (%d bytes)" % (budget, ws(1)))
    return _largest_chunk(ws, 1, n_cases, budget)


def _largest_chunk(ws, lo, n_units, budget):
    """The largest chunk in [lo, n_units) whose workspace ``ws(chunk)`` fits ``budget``, given that ws(lo) fits and the
    whole, ws(n_units), does not: ws grows with the chunk below n_units."""
    hi = n_units - 1
    while lo < hi:
        mid = (lo + hi + 1) // 2
        if ws(mid) <= budget:
            lo = mid
        else:
            hi = mid - 1
    return lo


# ---- post-solve reductions (rotor, fatigue, channel statistics, eigen), written once for host and device buffers ------------
class _Host:
    """Host buffers (numpy) for a reduction: ``raftk_<name>_host`` stages them through the library's device arena and
    returns with the results in them."""

    @staticmethod
    def array(a, dtype):
        return np.ascontiguousarray(a, dtype=dtype)

    @staticmethod
    def empty(shape, dtype=_F8):
        return np.zeros(shape, dtype=dtype)

    @staticmethod
    def ptr(a):
        return None if a is None else a.ctypes.data

    @staticmethod
    def call(name, *args, ws=None):
        check(getattr(lib, "raftk_%s_host" % name)(*args))


_HOST = _Host()


class _Device:
    """Torch tensors on ``device`` for a reduction: ``raftk_<name>_dev`` is enqueued on torch's current stream, after a
    workspace sized by ``raftk_<name>_workspace_bytes(*ws)`` when the entry takes one.  ``reads`` holds the inputs this
    object converted and the workspace: the enqueued launches read them after ``call`` returns, so whoever enqueues keeps
    the object until they are done."""

    def __init__(self, device):
        import torch
        self.torch, self.device, self.reads = torch, torch.device(device), []
        self._dtype = {_F8: torch.float64, _C16: torch.complex128, _I4: torch.int32}

    def array(self, a, dtype):
        if isinstance(a, self.torch.Tensor):
            a = a.to(device=self.device, dtype=self._dtype[dtype]).contiguous()
        else:
            a = self.torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)).to(self.device)
        self.reads.append(a)
        return a

    def empty(self, shape, dtype=_F8):
        return self.torch.empty(shape, dtype=self._dtype[dtype], device=self.device)

    @staticmethod
    def ptr(a):
        return None if a is None else a.data_ptr()

    def call(self, name, *args, ws=None):
        torch = self.torch
        with torch.cuda.device(self.device):
            if ws is not None:
                wsb = int(getattr(lib, "raftk_%s_workspace_bytes" % name)(*ws))
                buf = torch.empty(max(wsb, 1), dtype=torch.uint8, device=self.device)
                self.reads.append(buf)
                args += (buf.data_ptr(), wsb)
            check(getattr(lib, "raftk_%s_dev" % name)(*args, torch.cuda.current_stream(self.device).cuda_stream))


def _buffers_for(Xi):
    """The buffers a module-level reduction runs on: ``_Device`` on Xi's device when Xi is a torch CUDA tensor (a resident
    response, e.g. the gathered ``Xi_sys`` of ``sweep.ShardedFarmSolve.step``), else host buffers.  The device form enqueues on
    torch's current stream and returns torch tensors; tensors it made from host inputs are freed in stream order."""
    import sys
    torch = sys.modules.get("torch")
    if torch is not None and isinstance(Xi, torch.Tensor) and Xi.is_cuda:
        return _Device(Xi.device)
    return _HOST


def _session_buffers(session):
    """Device buffers for one reduction of ``session``, held as its ``_reads`` until its next reduction."""
    session._reads = _Device(session.device)
    return session._reads


def combine_trains(std, psd, idx):
    """helpers.getRMS / getPSD of a case with several wave trains (helpers.py:678-700) from per-train reductions ``std``
    [nT,...] and ``psd`` [nT,...,nw]: the squares sum over the trains ``idx`` -> (sqrt(sum std^2), sum PSD)."""
    return np.sqrt((std[idx] ** 2).sum(axis=0)), psd[idx].sum(axis=0)


def _check_wpow(wpow):
    if wpow.size and (wpow.min() < 0 or wpow.max() > 2):
        raise ValueError("wpow must be 0, 1 or 2 (displacement, velocity, acceleration)")


def _unit_response(be, Xi, w):
    """The response of a per-unit reduction on ``be``'s buffers: Xi complex [n_units, n_rows, n_dof, nw] or [n_rows, n_dof,
    nw], w [nw] -> (Xi [n_units, n_rows, n_dof, nw], w, whether Xi had no unit axis)."""
    Xi = be.array(Xi, _C16)
    squeeze = Xi.ndim == 3
    if squeeze:
        Xi = Xi[None]
    if Xi.ndim != 4:
        raise ValueError("Xi must be [n_units, n_rows, n_dof, nw] or [n_rows, n_dof, nw]")
    w = be.array(w, _F8)
    if tuple(w.shape) != (Xi.shape[3],):
        raise ValueError("w must be [nw]")
    return Xi, w, squeeze


def _case_rows(case_row0, n_rows):
    """``case_row0`` [nC + 1], the first row of every case (None: one row per case), checked -> int32 host array."""
    case_row0 = np.arange(n_rows + 1, dtype=_I4) if case_row0 is None else np.ascontiguousarray(case_row0, dtype=_I4)
    if len(case_row0) < 2 or case_row0[0] != 0 or case_row0[-1] != n_rows or np.any(np.diff(case_row0) < 1):
        raise ValueError("case_row0 must start at 0, end at %d and give every case at least one row" % n_rows)
    return case_row0


def _case_weights(weights, n_cases):
    """Case probabilities ``weights`` [n_cases] of a lifetime sum, or None, checked -> float64 host array or None."""
    if weights is None:
        return None
    weights = np.ascontiguousarray(weights, dtype=_F8)
    if weights.shape != (n_cases,) or not np.all(np.isfinite(weights)) or np.any(weights < 0) or not weights.sum() > 0:
        raise ValueError("weights must be [nC], finite, >= 0 and not all 0")
    return weights


def general_channel_stats(R, wpow, w, Xi, dw, psd=True, amp=False):
    """Output channels of a FOWT with generalised DOFs, Y = w^wpow R Xi (``packer.pack_general_channels``), host buffers:
    R [nch,nDOF], wpow [nch] 0, 1 or 2, w [nw], Xi complex [nU,nDOF,nw] -> (std [nU,nch], PSD [nU,nch,nw] or None,
    amplitudes complex [nU,nch,nw] or None)."""
    return _general_channel_stats(_HOST, R, wpow, w, Xi, dw, psd, amp)


def _general_channel_stats(be, R, wpow, w, Xi, dw, psd, amp):
    """``general_channel_stats`` on ``be``'s buffers; also design by design, R [nD,nch,nDOF] on Xi [nD,nU,nDOF,nw] -> outputs
    [nD,nU,...] (one entry call per design).  wpow stays [nch]."""
    R, wpow, w, Xi = be.array(R, _F8), np.ascontiguousarray(wpow, dtype=_I4), be.array(w, _F8), be.array(Xi, _C16)
    squeeze = Xi.ndim == 3
    if squeeze:
        R, Xi = R[None], Xi[None]
    if (Xi.ndim != 4 or R.ndim != 3 or R.shape[0] != Xi.shape[0] or R.shape[2] != Xi.shape[2] or wpow.shape != (R.shape[1],)
            or tuple(w.shape) != (Xi.shape[3],)):
        raise ValueError("R must be [nch,nDOF], wpow [nch], w [nw] for Xi [nU,nDOF,nw]")
    nD, nU, n, nw = Xi.shape
    nch = R.shape[1]
    _check_wpow(wpow)
    wp = be.array(wpow, _I4)
    sd = be.empty([nD, nU, nch])
    P = be.empty([nD, nU, nch, nw]) if psd else None
    A = be.empty([nD, nU, nch, nw], _C16) if amp else None
    for d in range(nD):
        be.call("general_channel_stats", nU, n, nch, nw, float(dw), be.ptr(w), be.ptr(R[d]), be.ptr(wp), be.ptr(Xi[d]), be.ptr(sd[d]),
                be.ptr(P[d]) if psd else None, be.ptr(A[d]) if amp else None)
    if squeeze:
        sd, P, A = sd[0], (P[0] if psd else None), (A[0] if amp else None)
    return sd, P, A


def _farm_channels_struct(R, wpow, n_farms, n, dw, tile_w):
    """R [nch,n] (every farm) or [F,nch,n] and wpow -> (raftk_farm_channels without pointers to outputs, R, wpow) checked."""
    R = np.ascontiguousarray(R, dtype=_F8)
    if R.ndim == 2:
        R_shared = 1
    elif R.ndim == 3 and R.shape[0] == n_farms:
        R_shared = 0
    else:
        raise ValueError("R must be [nch, %d] or [%d, nch, %d]" % (n, n_farms, n))
    nch = R.shape[-2]
    if R.shape[-1] != n:
        raise ValueError("R must be [nch, %d] or [%d, nch, %d]" % (n, n_farms, n))
    wpow = np.zeros(nch, dtype=_I4) if wpow is None else np.ascontiguousarray(wpow, dtype=_I4)
    if wpow.shape != (nch,):
        raise ValueError("wpow must be [nch]")
    _check_wpow(wpow)
    if not dw > 0:
        raise ValueError("dw must be > 0")
    ch = _lib.RaftkFarmChannels()
    ch.n_ch, ch.R_shared, ch.wpow, ch.dw, ch.tile_w = nch, R_shared, wpow.ctypes.data, float(dw), int(tile_w)
    return ch, R, wpow


def farm_channel_stats(R, Xi_sys, dw, w=None, wpow=None, psd=True, amp=False, tile_w=0):
    """Channels of farm batches on the device (raftk_farm_channel_stats_host), host buffers: Y[f,r,ch] = w^wpow R_f Xi_sys[f,r]
    -- mooring tensions with R = the line-end tension Jacobian dT/dx (raft_model.py:371-433, raft_fowt.py:2355-2399).
    ``R`` [nch,6N] for every farm or [F,nch,6N]; ``Xi_sys`` complex [F,nR,6N,nw] (``solve_dynamics_farm_batch``; [nR,6N,nw]
    for one farm); ``dw`` the PSD divisor (the reference's Tmoor_PSD uses w[0]); ``w`` [nw], needed when a ``wpow`` is 1 or 2.
    -> (std [F,nR,nch], PSD [F,nR,nch,nw] or None, amplitudes complex [F,nR,nch,nw] or None), without the farm axis when
    ``Xi_sys`` had none.  Bit-identical to ``general_channel_stats`` on the same R and Xi.  Several wave trains of a case:
    ``combine_trains``.  ``tile_w``: bins per CTA (0 automatic; -1 reads Xi_sys from L2), the results do not depend on it.
    With ``Xi_sys`` a torch CUDA tensor (a resident response, e.g. ``sweep.ShardedFarmSolve.step``'s gathered ``Xi_sys``) it runs
    raftk_farm_channel_stats_dev on torch's current stream instead and returns torch tensors.
    A ragged batch (``solve_dynamics_farm_ragged``): ``Xi_sys`` the list of per-farm [nR,6N_f,nw] views and ``R`` a list of
    [nch_f,6N_f] -> lists of per-farm results, each farm's as this function returns for that farm alone."""
    if isinstance(Xi_sys, (list, tuple)):
        return _farm_ragged_channel_stats(_buffers_for(Xi_sys[0]), R, Xi_sys, dw, w, wpow, psd, amp, tile_w)
    return _farm_channel_stats(_buffers_for(Xi_sys), R, Xi_sys, dw, w, wpow, psd, amp, tile_w)


def _ptr_of(a):
    return a.data_ptr() if hasattr(a, "data_ptr") else a.__array_interface__["data"][0]


def _contiguous_run(views):
    """Whether complex128 ``views`` (numpy or torch) lie back to back, in order, in one buffer."""
    for k, v in enumerate(views):
        if hasattr(v, "data_ptr"):
            ok, nb = v.is_contiguous() and str(v.dtype) == "torch.complex128", v.numel() * 16
        else:
            ok, nb = v.flags.c_contiguous and v.dtype == _C16, v.nbytes
        if not ok or (k + 1 < len(views) and _ptr_of(views[k + 1]) != _ptr_of(v) + nb):
            return False
    return True


def _farm_ragged_channel_stats(be, R, views, dw, w, wpow, psd, amp, tile_w):
    """``farm_channel_stats`` of a ragged batch (raftk_farm_ragged_channel_stats_*): ``views`` the per-farm [nR,6N_f,nw] arrays
    (one flat buffer, as ``solve_dynamics_farm_ragged`` returns them, is read in place; otherwise they are packed), ``R`` a
    list of [nch_f,6N_f], ``wpow`` None or a list of [nch_f] -> lists of per-farm (std [nR,nch_f], PSD, amplitudes)."""
    F = len(views)
    if not isinstance(R, (list, tuple)) or len(R) != F:
        raise ValueError("a ragged Xi_sys (a list of per-farm views) takes a list of one R per farm")
    if any(v.ndim != 3 or v.shape[0] != views[0].shape[0] or v.shape[2] != views[0].shape[2] or v.shape[1] % 6 for v in views):
        raise ValueError("ragged Xi_sys: per-farm [nR, 6N_f, nw] arrays with one nR and nw")
    nR, nw = int(views[0].shape[0]), int(views[0].shape[2])
    sizes = [int(v.shape[1]) // 6 for v in views]
    Rs = [np.ascontiguousarray(r, dtype=_F8) for r in R]
    if any(r.ndim != 2 or r.shape[1] != 6 * n or r.shape[0] < 1 for r, n in zip(Rs, sizes)):
        raise ValueError("R: a list of [nch_f, 6N_f] matrices, one per farm")
    nch = [r.shape[0] for r in Rs]
    ch0 = np.zeros(F + 1, dtype=_I4)
    ch0[1:] = np.cumsum(nch)
    wp = np.zeros(int(ch0[-1]), dtype=_I4) if wpow is None else np.concatenate([np.asarray(p, dtype=_I4).reshape(-1) for p in wpow])
    if wp.shape != (int(ch0[-1]),):
        raise ValueError("wpow: a list of [nch_f], one per farm")
    _check_wpow(wp)
    if not dw > 0:
        raise ValueError("dw must be > 0")
    ch = _lib.RaftkFarmChannels()
    ch.n_ch, ch.R_shared, ch.wpow, ch.dw, ch.tile_w = int(ch0[-1]), 0, wp.ctypes.data, float(dw), int(tile_w)
    fowt0, _ = ragged_offsets(sizes)
    if _contiguous_run(views):
        xi = views[0]
    elif hasattr(views[0], "data_ptr"):
        import torch
        xi = torch.cat([v.reshape(-1).to(torch.complex128) for v in views])
        be.reads.append(xi)                     # read by the enqueued launch
    else:
        xi = np.concatenate([np.asarray(v, dtype=_C16).reshape(-1) for v in views])
    w = None if w is None else be.array(w, _F8)
    if w is not None and tuple(w.shape) != (nw,):
        raise ValueError("w must be [nw]")
    Rd = be.array(np.concatenate([r.reshape(-1) for r in Rs]), _F8)
    n_all = int(ch0[-1]) * nR
    sd = be.empty([n_all])
    P = be.empty([n_all * nw]) if psd else None
    A = be.empty([n_all * nw], _C16) if amp else None
    ch.R, ch.std, ch.psd, ch.amp = be.ptr(Rd), be.ptr(sd), be.ptr(P), be.ptr(A)
    be.call("farm_ragged_channel_stats", F, nR, nw, fowt0.ctypes.data, ch0.ctypes.data, be.ptr(w), _ptr_of(xi), C.byref(ch),
            ws=(F, nR, nw, fowt0.ctypes.data, ch0.ctypes.data, C.byref(ch)))
    cut = lambda a, per: [a[nR * int(ch0[k]) * per:nR * int(ch0[k + 1]) * per].reshape(  # noqa: E731
        (nR, nch[k]) + ((nw,) if per > 1 else ())) for k in range(F)]
    return cut(sd, 1), (cut(P, nw) if psd else None), (cut(A, nw) if amp else None)


def _farm_channel_stats(be, R, Xi_sys, dw, w, wpow, psd, amp, tile_w):
    """``farm_channel_stats`` on ``be``'s buffers (R and wpow: numpy)."""
    Xi_sys = be.array(Xi_sys, _C16)
    squeeze = Xi_sys.ndim == 3
    if squeeze:
        Xi_sys = Xi_sys[None]
    if Xi_sys.ndim != 4:
        raise ValueError("Xi_sys must be [F, nR, n, nw] or [nR, n, nw]")
    F, nR, n, nw = Xi_sys.shape
    ch, R, wpow = _farm_channels_struct(R, wpow, F, n, dw, tile_w)
    w = None if w is None else be.array(w, _F8)
    if w is not None and tuple(w.shape) != (nw,):
        raise ValueError("w must be [nw]")
    nch = ch.n_ch
    R = be.array(R, _F8)
    sd = be.empty([F, nR, nch])
    P = be.empty([F, nR, nch, nw]) if psd else None
    A = be.empty([F, nR, nch, nw], _C16) if amp else None
    ch.R, ch.std, ch.psd, ch.amp = be.ptr(R), be.ptr(sd), be.ptr(P), be.ptr(A)
    be.call("farm_channel_stats", F, nR, n, nw, be.ptr(w), be.ptr(Xi_sys), C.byref(ch), ws=(F, nR, nw, C.byref(ch)))
    if squeeze:
        sd, P, A = sd[0], (P[0] if psd else None), (A[0] if amp else None)
    return sd, P, A


def tension_metrics(T0, std, psd):
    """Model.analyzeCases' Tmoor entries (raft_fowt.py:2389-2399, raft_model.py:406-418) from the mean tensions T0 [2L] and one
    case's combined statistics std [2L], PSD [2L,nw]: avg, std, max / min = avg +- 3 std, PSD."""
    T0 = np.asarray(T0, dtype=float)
    return dict(Tmoor_avg=T0.copy(), Tmoor_std=np.array(std, dtype=float), Tmoor_max=T0 + 3 * std, Tmoor_min=T0 - 3 * std,
                Tmoor_PSD=np.array(psd, dtype=float))


def _rotor_struct(R, C_, V_w, gains, n_units, nw, dw, case_row0, col0):
    """Shapes of rotor_stats' inputs (numpy arrays or torch tensors) checked -> (raftk_rotor_outputs without data pointers,
    case_row0, col0 as int32 host arrays).  R [nrot, n_r] (every unit) or [n_units, nrot, n_r]; C, V_w [nC, nrot, nw] (every
    unit) or [n_units, nC, nrot, nw]; gains [..., 4] over the same leading axes."""
    if len(R.shape) not in (2, 3) or (len(R.shape) == 3 and R.shape[0] != n_units):
        raise ValueError("R must be [nrot, n_r] or [%d, nrot, n_r]" % n_units)
    nrot, n_r = R.shape[-2:]
    if len(C_.shape) not in (3, 4) or (len(C_.shape) == 4 and C_.shape[0] != n_units) or tuple(C_.shape[-2:]) != (nrot, nw):
        raise ValueError("C must be [nC, %d, %d] or [%d, nC, %d, %d]" % (nrot, nw, n_units, nrot, nw))
    if tuple(V_w.shape) != tuple(C_.shape) or tuple(gains.shape) != tuple(C_.shape[:-1]) + (4,):
        raise ValueError("V_w must have C's shape and gains C's leading axes + [4]")
    nC = C_.shape[-3]
    case_row0 = np.arange(nC + 1, dtype=_I4) if case_row0 is None else np.ascontiguousarray(case_row0, dtype=_I4)
    col0 = np.zeros(nrot, dtype=_I4) if col0 is None else np.ascontiguousarray(col0, dtype=_I4)
    if case_row0.shape != (nC + 1,) or col0.shape != (nrot,):
        raise ValueError("case_row0 must be [nC + 1] and col0 [nrot]")
    ro = _lib.RaftkRotorOutputs()
    ro.n_cases, ro.n_rot, ro.n_r = nC, nrot, n_r
    ro.R_shared, ro.tf_shared = int(len(R.shape) == 2), int(len(C_.shape) == 3)
    ro.col0, ro.case_row0, ro.dw = col0.ctypes.data, case_row0.ctypes.data, float(dw)
    return ro, case_row0, col0


def rotor_stats(R, C_, V_w, gains, w, Xi, dw, case_row0=None, col0=None, psd=True):
    """Rotor speed, generator torque and blade pitch statistics on the device (raftk_rotor_stats_host), host buffers
    (FOWT.saveTurbineOutputs raft_fowt.py:2610-2679): per unit, case and rotor, the hub row y = R[rot] . Xi[col0[rot]:...],
    phi = C y over the case's rows plus the wind row -C V_w / (j w), and omega = j w phi, torque = (j w kp_tau + ki_tau) phi,
    bPitch = (j w kp_beta + ki_beta) phi.  ``Xi`` complex [n_units, n_rows, n_dof, nw] or [n_rows, n_dof, nw]; ``R``, ``C``,
    ``V_w``, ``gains`` as ``packer.pack_rotor_outputs`` gives them for every unit, or with a leading unit axis;
    ``case_row0`` [nC + 1] the first row of every case (None: one row per case); ``col0`` [nrot] the first column of every
    rotor's hub row (None: 0).  -> (std [n_units, nC, nrot, 3] (omega rpm, torque N m, bPitch deg), PSD [n_units, nC, nrot,
    3, nw] or None), without the unit axis when ``Xi`` had none.
    With ``Xi`` a torch CUDA tensor (a resident response, e.g. ``sweep.ShardedFarmSolve.step``'s gathered ``Xi_sys``) it runs
    raftk_rotor_stats_dev on torch's current stream instead and returns torch tensors."""
    return _rotor_stats(_buffers_for(Xi), R, C_, V_w, gains, w, Xi, dw, case_row0, col0, psd)


def _rotor_stats(be, R, C_, V_w, gains, w, Xi, dw, case_row0, col0, psd):
    """``rotor_stats`` on ``be``'s buffers (case_row0 and col0: numpy)."""
    Xi, w, squeeze = _unit_response(be, Xi, w)
    nU, nR, n, nw = Xi.shape
    R, C_, V_w, gains = be.array(R, _F8), be.array(C_, _C16), be.array(V_w, _C16), be.array(gains, _F8)
    ro, rows, cols = _rotor_struct(R, C_, V_w, gains, nU, nw, dw, case_row0, col0)
    sd = be.empty([nU, ro.n_cases, ro.n_rot, 3])
    P = be.empty([nU, ro.n_cases, ro.n_rot, 3, nw]) if psd else None
    ro.R, ro.C, ro.V_w, ro.gains = be.ptr(R), be.ptr(C_), be.ptr(V_w), be.ptr(gains)
    ro.std, ro.psd = be.ptr(sd), be.ptr(P)
    be.call("rotor_stats", nU, nR, n, nw, be.ptr(w), be.ptr(Xi), C.byref(ro))
    if squeeze:
        sd, P = sd[0], (P[0] if psd else None)
    return sd, P


def rotor_metrics(rotors, ic, std, psd, dw):
    """The rotor entries FOWT.saveTurbineOutputs stores for case ``ic`` (raft_fowt.py:2617-2679) from ``rotors``
    (``packer.pack_rotor_outputs``) and the case's statistics std [nrot, 3], PSD [nrot, 3, nw]: *_avg / *_std [nrot],
    omega_max / min = avg +- 2 std, *_PSD [nw, nrot], power_avg, and wind_PSD = getPSD(V_w, dw) of the case's last active
    rotor (absent when none is active).  Inactive rotors report zeros, as in the reference."""
    std, psd = np.asarray(std, dtype=float), np.asarray(psd, dtype=float)
    m = {}
    for j, nm in enumerate(("omega", "torque", "bPitch")):
        m[nm + "_avg"] = np.array(rotors[nm + "_avg"][ic], dtype=float)
        m[nm + "_std"] = std[:, j].copy()
        m[nm + "_PSD"] = np.ascontiguousarray(psd[:, j].T)
    m["omega_max"] = m["omega_avg"] + 2 * m["omega_std"]
    m["omega_min"] = m["omega_avg"] - 2 * m["omega_std"]
    m["power_avg"] = np.array(rotors["power_avg"][ic], dtype=float)
    if rotors["wind"][ic] is not None:
        m["wind_PSD"] = 0.5 * np.abs(rotors["wind"][ic]) ** 2 / dw
    return m


FATIGUE_METHODS = {"dirlik": 0, "narrowband": 1}
FATIGUE_ZERO, FATIGUE_NARROWBAND = 1, 2          # info bits (include/raftk.h RAFTK_FATIGUE_ZERO / _NARROWBAND)


def _fatigue_law(m, f_eq, method, prefix=""):
    """The DEL closed form's Woehler exponent ``m`` (scalar, per channel, or None: no DEL), ``f_eq`` and ``method`` checked;
    ``prefix`` starts every refusal."""
    if m is not None and not (np.all(np.isfinite(m)) and np.all(np.asarray(m) > 0)):
        raise ValueError(prefix + ("every m" if np.ndim(m) else "m") + " must be finite and > 0")
    if not (np.isfinite(f_eq) and f_eq > 0):
        raise ValueError(prefix + "f_eq must be finite and > 0")
    if method not in FATIGUE_METHODS:
        raise ValueError(prefix + "method must be one of %s" % sorted(FATIGUE_METHODS))


def _fatigue_struct(n_units, n_rows, n, nw, m, R, wpow, coef, case_row0, f_eq, method, weights, tile_w):
    """Shapes and options of fatigue's inputs (R / coef numpy arrays or torch tensors) checked -> (raftk_fatigue without data
    pointers, the host arrays it points to).  R [nch, n] (every unit) or [n_units, nch, n]; coef [nch, n, nw] (every unit),
    [n_units, nch, n, nw] or [n_units, n_rows, nch, n, nw] (one set per row, e.g. per-case operating points)."""
    if (R is None) == (coef is None):
        raise ValueError("fatigue: give exactly one of R (real rows) and coef (complex coefficients)")
    fa = _lib.RaftkFatigue()
    if R is not None:
        if len(R.shape) not in (2, 3) or (len(R.shape) == 3 and R.shape[0] != n_units) or R.shape[-1] != n:
            raise ValueError("R must be [nch, %d] or [%d, nch, %d]" % (n, n_units, n))
        nch = R.shape[-2]
        fa.R_shared = int(len(R.shape) == 2)
        wpow = np.zeros(nch, dtype=_I4) if wpow is None else np.ascontiguousarray(wpow, dtype=_I4)
        if wpow.shape != (nch,):
            raise ValueError("wpow must be [nch]")
        _check_wpow(wpow)
    else:
        lead = {3: (), 4: (n_units,), 5: (n_units, n_rows)}.get(len(coef.shape))
        if lead is None or tuple(coef.shape[:len(lead)]) != lead or tuple(coef.shape[-2:]) != (n, nw):
            raise ValueError("coef must be [nch, %d, %d], [%d, nch, %d, %d] or [%d, %d, nch, %d, %d]" % (n, nw, n_units, n, nw, n_units, n_rows, n, nw))
        nch = coef.shape[-3]
        fa.coef_mode = len(coef.shape) - 3
        if wpow is not None:
            raise ValueError("wpow applies to real rows R only")
    m = np.ascontiguousarray(np.broadcast_to(np.asarray(m, dtype=_F8), (nch,)))
    _fatigue_law(m, f_eq, method)
    case_row0 = _case_rows(case_row0, n_rows)
    nC = len(case_row0) - 1
    weights = _case_weights(weights, nC)
    fa.n_cases, fa.n_ch, fa.method, fa.tile_w = nC, nch, FATIGUE_METHODS[method], int(tile_w)
    fa.case_row0, fa.m, fa.f_eq = case_row0.ctypes.data, m.ctypes.data, float(f_eq)
    fa.wpow = wpow.ctypes.data if R is not None else None
    fa.weights = weights.ctypes.data if weights is not None else None
    return fa, (case_row0, m, wpow, weights)


def fatigue(Xi, w, m, R=None, wpow=None, coef=None, case_row0=None, f_eq=1.0, method="dirlik", weights=None, life=None,
            moments=True, tile_w=0):
    """Spectral fatigue damage-equivalent loads on the device (raftk_fatigue_host), host buffers.  Per unit, case and channel
    the moments lambda_k = sum over the case's rows and bins of w^k |Y|^2 / 2 (k = 0, 1, 2, 4) of the channel Y = w^wpow R Xi
    (real rows) or Y = sum_b coef[b] Xi[b] (complex per-bin coefficients), then Dirlik's closed form (``method="dirlik"``,
    narrow band where the spectrum is too narrow for it) or the narrow-band form (``"narrowband"``) of the damage rate d,
    and DEL = (d / f_eq)^(1/m).  ``Xi`` complex [n_units, n_rows, n_dof, nw] or [n_rows, n_dof, nw]; ``w`` [nw] rad/s; ``m``
    the Woehler exponent, scalar or [nch]; ``R`` / ``coef`` as ``_fatigue_struct``; ``case_row0`` [nC + 1] the first row of
    every case (None: one row per case); ``weights`` [nC] case probabilities; ``life`` (default: weights given) adds DEL_life
    = (sum_c p_c d_c / (f_eq sum_c p_c))^(1/m).  -> dict(DEL [n_units, nC, nch], info int32 (FATIGUE_ZERO, FATIGUE_NARROWBAND
    bits), moments [n_units, nC, nch, 4] (l0, l1, l2, l4) or absent, DEL_life [n_units, nch] or absent), without the unit
    axis when ``Xi`` had none.  ``tile_w``: bins per CTA (0 automatic, -1 reads Xi from L2); the results do not depend on it.
    With ``Xi`` a torch CUDA tensor (a resident response, e.g. ``sweep.ShardedFarmSolve.step``'s gathered ``Xi_sys``) it runs
    raftk_fatigue_dev on torch's current stream instead and returns torch tensors."""
    return _fatigue(_buffers_for(Xi), Xi, w, m, R, wpow, coef, case_row0, f_eq, method, weights, life, moments, tile_w)


def _fatigue(be, Xi, w, m, R, wpow, coef, case_row0, f_eq, method, weights, life, moments, tile_w):
    """``fatigue`` on ``be``'s buffers (m, wpow, case_row0 and weights: numpy)."""
    Xi, w, squeeze = _unit_response(be, Xi, w)
    nU, nR, n, nw = Xi.shape
    R = None if R is None else be.array(R, _F8)
    coef = None if coef is None else be.array(coef, _C16)
    fa, keep = _fatigue_struct(nU, nR, n, nw, m, R, wpow, coef, case_row0, f_eq, method, weights, tile_w)
    life = weights is not None if life is None else bool(life)
    nC, nch = fa.n_cases, fa.n_ch
    out = dict(DEL=be.empty([nU, nC, nch]), info=be.empty([nU, nC, nch], _I4))
    if moments:
        out["moments"] = be.empty([nU, nC, nch, 4])
    if life:
        out["DEL_life"] = be.empty([nU, nch])
    fa.R, fa.coef, fa.DEL, fa.info = be.ptr(R), be.ptr(coef), be.ptr(out["DEL"]), be.ptr(out["info"])
    fa.moments, fa.DEL_life = be.ptr(out.get("moments")), be.ptr(out.get("DEL_life"))
    be.call("fatigue", nU, nR, n, nw, be.ptr(w), be.ptr(Xi), C.byref(fa), ws=(nU, nR, nw, C.byref(fa)))
    return {k: v[0] for k, v in out.items()} if squeeze else out


STRESS_ANGLES = np.linspace(0, 2 * np.pi, 50)       # helpers.getSigmaXPSD's default angles (helpers.py:1164)
STRESS_HOT = ("angle", "std", "angle_DEL", "DEL", "std_exact", "angle_exact")   # include/raftk.h raftk_stress_ring hot


def _stress_channels(be, fa, ss, n_units, n_rows, n, nw, wpow):
    """Fore-aft / side-side channels of stress_ring -> (stacked R or coef on ``be``, n_rings, n_r, n_ch, R_shared or coef_mode,
    wpow [n_rings, n_ch] int32 or None).  Real rows: fa [n_r], [n_rings, n_r] or [n_units, n_rings, n_r]; complex per-bin
    coefficients: fa [n_r, nw], [n_rings, n_r, nw], [n_units, n_rings, n_r, nw] or [n_units, n_rows, n_rings, n_r, nw];
    ss None (fore-aft only) or the same form and shape."""
    def cplx(a):
        return a.is_complex() if hasattr(a, "is_complex") else np.iscomplexobj(a)
    coef = cplx(fa)
    if ss is not None and (cplx(ss) != coef or tuple(ss.shape) != tuple(fa.shape)):
        raise ValueError("stress_ring: ss must have fa's form and shape")
    dt = _C16 if coef else _F8
    chans = [be.array(fa, dt)] + ([] if ss is None else [be.array(ss, dt)])
    nd = len(chans[0].shape)
    tail = 2 if coef else 1                               # (n_r, nw) or (n_r,)
    if coef:
        lead = {2: (), 3: (), 4: (n_units,), 5: (n_units, n_rows)}.get(nd)
        mode = {2: 0, 3: 0, 4: 1, 5: 2}.get(nd)
    else:
        lead = {1: (), 2: (), 3: (n_units,)}.get(nd)
        mode = {1: 1, 2: 1, 3: 0}.get(nd)
    if lead is None or tuple(chans[0].shape[:len(lead)]) != lead or (coef and chans[0].shape[-1] != nw):
        raise ValueError("stress_ring: fa must be real [n_r], [n_rings, n_r] or [%d, n_rings, n_r], or complex [n_r, %d], "
                         "[n_rings, n_r, %d], [%d, n_rings, n_r, %d] or [%d, %d, n_rings, n_r, %d]"
                         % (n_units, nw, nw, n_units, nw, n_units, n_rows, nw))
    if nd == len(lead) + tail:                            # one ring
        chans = [c.reshape(tuple(lead) + (1,) + tuple(c.shape[len(lead):])) for c in chans]
    n_rings, n_r = chans[0].shape[len(lead)], chans[0].shape[len(lead) + 1]
    if n_r > n:
        raise ValueError("stress_ring: the channels read %d columns of a response with %d" % (n_r, n))
    stk = np if isinstance(chans[0], np.ndarray) else be.torch
    X = stk.stack(chans, len(lead) + 1) if len(chans) == 2 else chans[0].reshape(tuple(lead) + (n_rings, 1) + tuple(chans[0].shape[len(lead) + 1:]))
    X = be.array(X, dt)
    if coef:
        if wpow is not None:
            raise ValueError("wpow applies to real rows only")
        return X, n_rings, n_r, len(chans), mode, None
    wp = np.ascontiguousarray(np.broadcast_to(np.zeros(1, dtype=_I4) if wpow is None else np.asarray(wpow, dtype=_I4), (n_rings, len(chans))))
    _check_wpow(wp)
    return X, n_rings, n_r, len(chans), mode, wp


def stress_ring(Xi, w, fa, ss, angles=None, d=10.0, t=0.083, m=None, f_eq=1.0, method="dirlik", weights=None, case_row0=None,
                col0=None, psd=False, mean=None, wpow=None, dw=None, tile_w=0):
    """Tower-base axial stress around the circumference on the device (raftk_stress_ring_host), host buffers: the reference's
    helpers.getSigmaXPSD (helpers.py:1164) for every unit, case, ring (tower base) and angle, and its statistics.  Thin-wall
    section, Izz = pi/8 t d^3, sigma(theta) = (a cos theta - b sin theta) (d/2) / Izz / 1e6 (MPa) of the fore-aft moment a
    (``fa``) and the side-side moment b (``ss``; None: fore-aft only, as a rigid tower's Mbase) over the case's rows.  The
    response is walked once for the cross-spectral moments of a and b; every angle follows in closed form.
    ``Xi`` complex [n_units, n_rows, n_dof, nw] or [n_rows, n_dof, nw]; ``fa`` / ``ss`` real rows (``packer.pack_general_
    channels``' MbaseY / MbaseX rows, ``wpow`` [n_rings, 2]) or complex per-bin coefficients (``pack_turbine_channels``'
    Mbase), as ``_stress_channels``; ``angles`` rad (None: 50 over [0, 2 pi]); ``d``, ``t`` diameter and wall thickness (m);
    ``col0`` [n_rings] the first response column of every ring's channels (FOWT i of a farm: 6 i); ``mean`` the channels'
    mean values, broadcast to [n_units, nC, n_rings, n_ch] (None: 0); ``m``: the Woehler exponent of the per-angle DELs
    (``fatigue``'s closed form, ``f_eq``, ``method``); ``weights`` [nC] with m: the per-angle lifetime DEL_life, as
    ``fatigue``'s, and its hot spot; ``psd``: per-bin stress PSD, divided by ``dw`` (default w[1] - w[0]).
    -> dict(std, avg, max, min [n_units, nC, n_rings, nA] (max / min = avg +- 3 std), hot [n_units, nC, n_rings, 6] (
    ``STRESS_HOT``: sampled argmax angle and std, argmax angle and DEL, exact largest std and its angle in [0, pi)), DEL and
    info (with m), DEL_life [n_units, n_rings, nA] and hot_life [n_units, n_rings, 2] (angle, DEL) with weights and m, psd [n_units,
    nC, n_rings, nA, nw] with psd), without the unit axis when ``Xi`` had none.  ``tile_w`` as ``fatigue``.
    With ``Xi`` a torch CUDA tensor (a resident response, e.g. ``sweep.ShardedFarmSolve.step``'s gathered ``Xi_sys``) it runs
    raftk_stress_ring_dev on torch's current stream instead and returns torch tensors."""
    return _stress_ring(_buffers_for(Xi), Xi, w, fa, ss, angles, d, t, m, f_eq, method, weights, case_row0, col0, psd, mean, wpow, dw,
                        tile_w)


def _stress_ring(be, Xi, w, fa, ss, angles, d, t, m, f_eq, method, weights, case_row0, col0, psd, mean, wpow, dw, tile_w):
    """``stress_ring`` on ``be``'s buffers (angles, case_row0, col0, wpow and weights: numpy)."""
    Xi, w, squeeze = _unit_response(be, Xi, w)
    nU, nR, n, nw = Xi.shape
    X, n_rings, n_r, n_ch, mode, wp = _stress_channels(be, fa, ss, nU, nR, n, nw, wpow)
    angles = np.ascontiguousarray(STRESS_ANGLES if angles is None else np.atleast_1d(np.asarray(angles, dtype=_F8)))
    if angles.ndim != 1 or not 1 <= len(angles) <= 256 or not np.all(np.isfinite(angles)):
        raise ValueError("angles must be 1 to 256 finite values (rad)")
    if not (np.isfinite(d) and d > 0 and np.isfinite(t) and t > 0):
        raise ValueError("d and t must be finite and > 0")
    _fatigue_law(m, f_eq, method)
    case_row0 = _case_rows(case_row0, nR)
    nC = len(case_row0) - 1
    if n_rings > 64:
        raise ValueError("at most 64 rings per call")
    col0 = np.zeros(n_rings, dtype=_I4) if col0 is None else np.ascontiguousarray(np.broadcast_to(np.asarray(col0, dtype=_I4), (n_rings,)))
    if np.any(col0 < 0) or np.any(col0 > n - n_r):
        raise ValueError("col0 must lie in [0, %d]" % (n - n_r))
    weights = _case_weights(weights, nC)
    life = weights is not None and m is not None
    dw = (float(w[1] - w[0]) if nw > 1 else 1.0) if dw is None else float(dw)
    if psd and not (np.isfinite(dw) and dw > 0):
        raise ValueError("dw must be finite and > 0")
    mu = None if mean is None else be.array(np.broadcast_to(np.asarray(mean, dtype=_F8), (nU, nC, n_rings, n_ch)), _F8)
    sr = _lib.RaftkStressRing()
    sr.n_cases, sr.n_rings, sr.n_ch, sr.n_r, sr.n_angles = nC, n_rings, n_ch, n_r, len(angles)
    sr.method, sr.tile_w = FATIGUE_METHODS[method], int(tile_w)
    if wp is None:
        sr.coef_mode = mode
    else:
        sr.R_shared = mode
    sr.case_row0, sr.col0, sr.wpow, sr.angles = case_row0.ctypes.data, col0.ctypes.data, None if wp is None else wp.ctypes.data, angles.ctypes.data
    sr.d, sr.t, sr.m, sr.f_eq, sr.dw = float(d), float(t), 0.0 if m is None else float(m), float(f_eq), dw
    sr.weights = None if weights is None else weights.ctypes.data
    shp = [nU, nC, n_rings, len(angles)]
    out = {k: be.empty(shp) for k in ("std", "avg", "max", "min")}
    out["hot"] = be.empty([nU, nC, n_rings, 6])
    if m is not None:
        out["DEL"], out["info"] = be.empty(shp), be.empty(shp, _I4)
    if life:
        out["DEL_life"], out["hot_life"] = be.empty([nU, n_rings, len(angles)]), be.empty([nU, n_rings, 2])
    if psd:
        out["psd"] = be.empty(shp + [nw])
    if wp is None:
        sr.coef = be.ptr(X)
    else:
        sr.R = be.ptr(X)
    sr.mean = be.ptr(mu)
    for k in ("std", "avg", "max", "min", "hot", "DEL", "info", "DEL_life", "hot_life", "psd"):
        setattr(sr, k, be.ptr(out.get(k)))
    be.call("stress_ring", nU, nR, n, nw, be.ptr(w), be.ptr(Xi), C.byref(sr), ws=(nU, nR, nw, C.byref(sr)))
    return {k: v[0] for k, v in out.items()} if squeeze else out


def stress_hot(r, ic=None):
    """``sigmaX_hot`` entries from a stress_ring result without the unit axis: case ``ic`` -> per ring dict(angle, std,
    angle_DEL, DEL (with m), std_exact, angle_exact) as arrays [n_rings]; ``ic`` None: the lifetime's dict(angle, DEL)."""
    if ic is None:
        h = np.asarray(r["hot_life"])
        return dict(angle=h[:, 0].copy(), DEL=h[:, 1].copy())
    h = np.asarray(r["hot"][ic])
    out = {k: h[:, j].copy() for j, k in enumerate(STRESS_HOT)}
    if "DEL" not in r:
        del out["angle_DEL"], out["DEL"]
    return out


def stress_entries(r, ic):
    """The ``sigmaX_*`` entries of case ``ic`` from a stress_ring result without the unit axis: _avg / _std / _max / _min
    [n_rings, nA], _PSD [n_rings, nA, nw] (with psd), _DEL [n_rings, nA] (with m) and _hot (``stress_hot``)."""
    m = {"sigmaX" + s: np.array(r[k][ic]) for s, k in (("_avg", "avg"), ("_std", "std"), ("_max", "max"), ("_min", "min"))}
    if "psd" in r:
        m["sigmaX_PSD"] = np.array(r["psd"][ic])
    if "DEL" in r:
        m["sigmaX_DEL"] = np.array(r["DEL"][ic])
    m["sigmaX_hot"] = stress_hot(r, ic)
    return m


def stress_options(stress):
    """The ``stress=`` option of ``Model``, ``general_analyze_cases`` and ``general_analyze_cases_batch``: dict(d=10.0,
    t=0.083, angles=None (50 over [0, 2 pi]), m=None, f_eq=1.0, method="dirlik", weights=None, psd=False) -> the same dict,
    checked and completed."""
    if not isinstance(stress, dict):
        raise ValueError("stress= must be a dict, e.g. dict(d=10.0, t=0.083, m=4.0)")
    bad = sorted(set(stress) - {"d", "t", "angles", "m", "f_eq", "method", "weights", "psd"})
    if bad:
        raise ValueError("stress=: unknown option(s) %s" % bad)
    o = dict(d=float(stress.get("d", 10.0)), t=float(stress.get("t", 0.083)),
             angles=np.array(STRESS_ANGLES if stress.get("angles") is None else stress["angles"], dtype=float),
             m=None if stress.get("m") is None else float(stress["m"]), f_eq=float(stress.get("f_eq", 1.0)),
             method=stress.get("method", "dirlik"), weights=stress.get("weights"), psd=bool(stress.get("psd", False)))
    if not (np.isfinite(o["d"]) and o["d"] > 0 and np.isfinite(o["t"]) and o["t"] > 0):
        raise ValueError("stress=: d and t must be finite and > 0")
    _fatigue_law(o["m"], o["f_eq"], o["method"], "stress=: ")
    if o["angles"].ndim != 1 or not 1 <= len(o["angles"]) <= 256 or not np.all(np.isfinite(o["angles"])):
        raise ValueError("stress=: angles must be 1 to 256 finite values (rad)")
    return o


def stress_rows(names):
    """Rows of the tower-base moments in channels ``names`` [(name, rotor index)]: -> (fore-aft rows, side-side rows or
    None, per rotor), a flexible tower's MbaseY / MbaseX, else a rigid tower's Mbase (fore-aft only).  ValueError when
    there is neither."""
    idx = {(nm, ir): k for k, (nm, ir) in enumerate(names)}
    rot = sorted({ir for nm, ir in names if nm in ("Mbase", "MbaseY") and ir is not None})
    if rot and all(("MbaseY", ir) in idx and ("MbaseX", ir) in idx for ir in rot):
        return [idx["MbaseY", ir] for ir in rot], [idx["MbaseX", ir] for ir in rot]
    if rot and all(("Mbase", ir) in idx for ir in rot):
        return [idx["Mbase", ir] for ir in rot], None
    raise ValueError("stress=: the channels have no tower-base moment (Mbase, or MbaseY and MbaseX)")


def fatigue_options(fatigue):
    """The ``fatigue=`` option of ``Model``, ``general_analyze_cases`` and ``general_analyze_cases_batch``:
    dict(m={channel name: Woehler exponent}, f_eq=1.0, method="dirlik", weights=None) -> the same dict, checked and completed.
    Channel names are those of the channels (``Mbase``, ``AxRNA``, ``FbaseX`` .. ``MbaseZ``, ``surge`` ...) and ``Tmoor`` for
    mooring line-end tensions; ``weights`` [nCases] adds the lifetime DELs (``results['fatigue']``)."""
    if not isinstance(fatigue, dict) or not isinstance(fatigue.get("m"), dict) or not fatigue["m"]:
        raise ValueError("fatigue= must be a dict with m = {channel name: Woehler exponent}, e.g. dict(m={'Mbase': 4.0})")
    bad = sorted(set(fatigue) - {"m", "f_eq", "method", "weights"})
    if bad:
        raise ValueError("fatigue=: unknown option(s) %s" % bad)
    for nm, e in fatigue["m"].items():
        if not (np.isfinite(e) and e > 0):
            raise ValueError("fatigue=: the exponent of %r must be finite and > 0" % nm)
    return dict(m=dict(fatigue["m"]), f_eq=float(fatigue.get("f_eq", 1.0)), method=fatigue.get("method", "dirlik"),
                weights=fatigue.get("weights"))


def fatigue_selection(names, m):
    """The DEL outputs of channels ``names`` [(name, index or None)] under exponents ``m`` -> [(output name, row, index,
    exponent)].  A flexible tower's ``Mbase`` is the alias of its ``MbaseY`` (raft_fowt.py:2599-2604), so m['Mbase'] also
    selects the MbaseY rows when no channel is called Mbase."""
    plain = {nm for nm, _ in names}
    sel = []
    for k, (nm, ir) in enumerate(names):
        if nm in m:
            sel.append((nm, k, ir, float(m[nm])))
        if nm == "MbaseY" and "Mbase" in m and "Mbase" not in plain:
            sel.append(("Mbase", k, ir, float(m["Mbase"])))
    return sel


def fatigue_entries(sel, DEL):
    """``<name>_DEL`` entries of one case (or of the lifetime) from the DELs [len(sel)] of ``fatigue_selection``'s outputs:
    a scalar for a channel without index, else an array over the index (rotors [nrot], line ends [2L])."""
    size = {}
    for nm, _, ir, _ in sel:
        if ir is not None:
            size[nm] = max(size.get(nm, 0), ir + 1)
    out = {}
    for j, (nm, _, ir, _) in enumerate(sel):
        if ir is None:
            out[nm + "_DEL"] = float(DEL[j])
        else:
            out.setdefault(nm + "_DEL", np.zeros(size[nm]))[ir] = DEL[j]
    return out


def _general_fatigue(opts, channels, P, Xi, owner, first, n_cases, metrics, out):
    """general_analyze_cases' fatigue= on one design: the DELs of the named channels into every case's metrics, the lifetime
    DELs into out['fatigue'] when weights are given."""
    if channels is None:
        raise ValueError("fatigue= needs channels (packer.pack_general_channels)")
    sel = fatigue_selection(channels["names"], opts["m"])
    missing = sorted(set(opts["m"]) - {s[0] for s in sel})
    if missing:
        raise ValueError("fatigue=: no channel named %s" % missing)
    rows = [s[1] for s in sel]
    r = fatigue(Xi, P["w"], [s[3] for s in sel], R=np.asarray(channels["R"])[rows], wpow=np.asarray(channels["wpow"])[rows],
                case_row0=np.append(first, len(owner)), f_eq=opts["f_eq"], method=opts["method"], weights=opts["weights"],
                moments=False)
    for ic in range(n_cases):
        metrics.setdefault(ic, {}).update(fatigue_entries(sel, r["DEL"][ic]))
    if "DEL_life" in r:
        out["fatigue"] = fatigue_entries(sel, r["DEL_life"])


def general_case_metrics(channels, std, psd, amp, idx, dw=None):
    """The entries FOWT.saveTurbineOutputs stores for one case (raft_fowt.py:2299-2604) from per-train channel statistics
    (std [nT,nch], PSD [nT,nch,nw], amplitudes [nT,nch,nw]) of the case's trains ``idx``: ``*_avg/_std/_max/_min/_PSD`` of every
    channel, ``*_RA`` of the six PRP motions (all trains plus the zero row of Model.Xi), per-rotor channels as arrays
    [nrotors] / PSD [nw, nrotors], and the ``Mbase`` alias of a flexible tower's MbaseY (:2599-2604).  Mooring tension rows
    (``channels['tension']``) give Tmoor_avg/std/max/min [2L] and Tmoor_PSD [2L,nw], whose PSD divides by w[0] like the
    reference's (:2370, :2399): ``dw``, the divisor of ``psd``, is then required."""
    sd, ps = combine_trains(std, psd, idx)
    names, avg = channels["names"], channels["avg"]
    nw = psd.shape[-1]
    ten = channels.get("tension")
    nrot = 1 + max([ir for nm, ir in names if ir is not None and nm != "Tmoor"], default=-1)
    m = {}
    if ten is not None:
        if dw is None:
            raise ValueError("general_case_metrics: tension rows need dw, the PSD divisor of psd")
        rows = slice(ten["row0"], ten["row0"] + len(ten["T0"]))
        m.update(tension_metrics(ten["T0"], sd[rows], ps[rows] * (float(dw) / ten["w0"])))
    for k, (nm, ir) in enumerate(names):
        if nm == "Tmoor":
            continue
        if ir is None:
            m[nm + "_avg"], m[nm + "_std"] = avg[k], sd[k]
            m[nm + "_max"], m[nm + "_min"] = avg[k] + 3 * sd[k], avg[k] - 3 * sd[k]
            m[nm + "_PSD"] = ps[k]
            ra = np.zeros([len(idx) + 1, nw], dtype=complex)
            ra[:-1] = amp[idx, k]
            m[nm + "_RA"] = ra
            continue
        rotor_channel_entries(m, nm, ir, nrot, avg[k], sd[k], ps[k])
    if "MbaseY_std" in m:
        for suffix in ("_avg", "_std", "_max", "_min", "_PSD"):
            m["Mbase" + suffix] = m["MbaseY" + suffix].copy()
    return m


def rotor_channel_entries(m, nm, ir, nrot, avg, std, psd):
    """Rotor ``ir``'s value of the per-rotor channel ``nm`` into one case's entries ``m`` (raft_fowt.py:2401-2444, 2504-2538):
    ``nm``_avg / _std / _max / _min [nrot] with max / min = avg +- 3 std, and ``nm``_PSD [nw, nrot] from the PSD [nw]."""
    for suffix in ("_avg", "_std", "_max", "_min"):
        m.setdefault(nm + suffix, np.zeros(nrot))
    m.setdefault(nm + "_PSD", np.zeros([len(psd), nrot]))
    m[nm + "_avg"][ir], m[nm + "_std"][ir] = avg, std
    m[nm + "_max"][ir], m[nm + "_min"][ir] = avg + 3 * std, avg - 3 * std
    m[nm + "_PSD"][:, ir] = psd


def general_analyze_cases(P, M, B, Cm, cases, channels=None, n_iter=10, tol=0.01, xi_start=0.0, fd=None, qtf=None, rotors=None,
                          turbine_constants=None, ops=None, fatigue=None, stress=None):
    """Model.analyzeCases (dynamics and output statistics) for one FOWT with generalised degrees of freedom: ``cases`` a list
    of case dicts, scalar or list-valued wave keys (several wave trains); ``channels`` from ``packer.pack_general_channels``.
    -> dict(Xi_trains [per case: nTrains,nDOF,nw], status [nC,4] of train 0, case_metrics {case: saveTurbineOutputs entries},
    empty without channels; with ``pack_general_channels(fowt, tensions=...)`` they include Tmoor_*).  ``fd``: frequency-dependent terms, as for ``general_solve_dynamics``.  ``qtf``: second-order
    wave loads (``packer.pack_general_qtf``); the result then also holds, per case, the reference FOWT's ``Fhydro_2nd``
    (complex [nTrains,nDOF,nw]) and ``Fhydro_2nd_mean`` ([nTrains,nDOF]), zero from reduced DOF 6 up (raft_model.py:1034-1036).
    ``rotors``: ``packer.pack_rotor_outputs`` of the FOWT for these cases; every case's metrics then hold the rotor entries
    (omega / torque / bPitch / power, wind_PSD; ``rotor_metrics``).  ``ops``: per-case operating points, one per case of
    ``cases`` (op [nC]; ``packer.pack_general_matrices(fowt, states=...)['ops']``, whose M, B and fd then go with it): every
    wave train of a case is solved at its case's point.  ``turbine_constants`` (raw per-case snapshots, as
    ``Model(turbine_constants=)``): NotImplementedError, since M, B and fd come here already packed.
    ``fatigue``: dict(m={channel name: Woehler exponent}, f_eq=1.0, method="dirlik", weights=None) (``fatigue_options``)
    adds every case's ``<name>_DEL`` of the named channels (per-rotor channels [nrot], ``Tmoor_DEL`` [2L], ``Mbase_DEL`` the
    alias of ``MbaseY_DEL``) and, with weights, the lifetime DELs in the result's ``fatigue``.  Without it nothing changes.
    ``stress``: dict(d=10.0, t=0.083, angles=None, m=None, f_eq=1.0, method="dirlik", weights=None, psd=False)
    (``stress_options``) adds every case's tower-base axial stress around the circumference from MbaseY (fore-aft) and MbaseX
    (side-side) (``stress_ring``, helpers.getSigmaXPSD): ``sigmaX_avg/_std/_max/_min`` [nrot, nA], ``sigmaX_PSD``
    [nrot, nA, nw] with psd, ``sigmaX_DEL`` [nrot, nA] with m, and ``sigmaX_hot`` (``stress_hot``); with weights (and m) the
    lifetime ``sigmaX_DEL`` and ``sigmaX_hot`` in the result's ``fatigue``.  Without it nothing changes."""
    from .packer import pack_case_trains
    _no_general_ops(turbine_constants)
    opts = None if fatigue is None else fatigue_options(fatigue)
    sopts = stress_options_for(stress, [channels])
    table, owner, first = pack_case_trains(cases)
    q = bool(qtf)
    res = general_solve_dynamics(P, M, B, Cm, CaseTable(table, ops=_train_ops(ops, owner, len(cases))), n_iter=n_iter, tol=tol,
                                 xi_start=xi_start, fd=fd, qtf=qtf, F_2nd=q)
    return _general_case_results(P, res[0], res[1], owner, first, len(cases), channels, res[2:4] if q else None, rotors, opts, sopts)


def stress_options_for(stress, channels):
    """``stress=`` (``stress_options``) checked against the channels of every FOWT or design it applies to, before anything
    is solved: each must have a tower-base moment (``stress_rows``); None (no channels) is refused.  None when ``stress`` is."""
    if stress is None:
        return None
    o = stress_options(stress)
    for ch in channels:
        if ch is None:
            raise ValueError("stress= needs channels (packer.pack_general_channels)")
        stress_rows(ch["names"])
    return o


def _general_stress(opts, channels, P, Xi, owner, first, n_cases, metrics, out):
    """general_analyze_cases' stress= on one design: the tower-base stress ring of every rotor's tower into every case's
    metrics, the lifetime DELs and their hot spot into out['fatigue'] when weights and m are given."""
    fa, ss = stress_rows(channels["names"])
    R, wp, avg = np.asarray(channels["R"]), np.asarray(channels["wpow"]), np.asarray(channels["avg"])
    rows = fa if ss is None else np.stack([fa, ss], axis=1)
    r = stress_ring(Xi, P["w"], R[fa], None if ss is None else R[ss], opts["angles"], opts["d"], opts["t"], m=opts["m"],
                    f_eq=opts["f_eq"], method=opts["method"], weights=opts["weights"], case_row0=np.append(first, len(owner)),
                    psd=opts["psd"], mean=avg[rows].reshape(len(fa), -1), wpow=wp[rows].reshape(len(fa), -1), dw=float(P["dw"]))
    for ic in range(n_cases):
        metrics.setdefault(ic, {}).update(stress_entries(r, ic))
    if "DEL_life" in r:
        out.setdefault("fatigue", {}).update(sigmaX_DEL=np.array(r["DEL_life"]), sigmaX_hot=stress_hot(r))


def _general_case_results(P, Xi, st, owner, first, n_cases, channels, F2nd, rotors=None, fatigue=None, stress=None):
    """general_analyze_cases' result for one design from its train table's Xi [nT,nDOF,nw], status [nT,4] and, with a QTF
    table, (F_2nd [nT,6,nw], F_2nd_mean [nT,6])."""
    raise_on_flags(st[first])                                           # raft_model.py:1089, :1098-1099
    metrics = {}
    if channels is not None:
        sd, ps, amp = general_channel_stats(channels["R"], channels["wpow"], P["w"], Xi, float(P["dw"]), psd=True, amp=True)
        for ic in range(n_cases):
            metrics[ic] = general_case_metrics(channels, sd, ps, amp, np.nonzero(owner == ic)[0], dw=float(P["dw"]))
    if rotors is not None:
        if rotors["C"].shape[0] != n_cases:
            raise ValueError("rotors: packed for %d cases, %d given" % (rotors["C"].shape[0], n_cases))
        rsd, rps = rotor_stats(rotors["R"], rotors["C"], rotors["V_w"], rotors["gains"], P["w"], Xi, float(P["dw"]),
                               case_row0=np.append(first, len(owner)))
        for ic in range(n_cases):
            metrics.setdefault(ic, {}).update(rotor_metrics(rotors, ic, rsd[ic], rps[ic], float(P["dw"])))
    out = dict(Xi_trains=[Xi[owner == ic] for ic in range(n_cases)], status=st[first], case_metrics=metrics)
    if F2nd is not None:
        n, nw = Xi.shape[1], Xi.shape[2]
        F2, F2m = np.zeros([len(Xi), n, nw], dtype=np.complex128), np.zeros([len(Xi), n])
        F2[:, :6], F2m[:, :6] = F2nd[0], F2nd[1]
        out["Fhydro_2nd"] = [F2[owner == ic] for ic in range(n_cases)]
        out["Fhydro_2nd_mean"] = [F2m[owner == ic] for ic in range(n_cases)]
    if fatigue is not None:
        _general_fatigue(fatigue, channels, P, Xi, owner, first, n_cases, metrics, out)
    if stress is not None:
        _general_stress(stress, channels, P, Xi, owner, first, n_cases, metrics, out)
    return out


# ---- design batches of flexible FOWTs (raftk_general_batch_*) ------------------------------------------------------------
def _capture():
    got = {}

    def ptr(name, a):
        got[name] = a
    return got, ptr


class GeneralBatch:
    """The tables of a design batch of FOWTs with generalised DOFs (include/raftk.h raftk_general_batch): ``designs`` a list of
    per-design inputs, each a dict with keys P, M, B, Cm and optional fd, qtf, or a tuple (P, M, B, Cm[, fd[, qtf]]) in the
    layouts of ``general_solve_dynamics`` (``packer.pack_general_dofs`` / ``pack_general_matrices`` / ``pack_general_qtf``).
    The node tables are concatenated (CSR ``node_offset``), the matrices and frequency-dependent tables stacked on a leading
    design axis.  ``qtf``: one second-order table shared by every design (then no design may carry its own).  The designs must
    share n_dof, the frequency grid, depth and rho, the count of fd DOFs and BEM headings, and the QTF grid: a ValueError names
    the first design that differs from design 0."""

    def __init__(self, designs, qtf=None):
        designs = [self._entry(e) for e in designs]
        if not designs:
            raise ValueError("a design batch needs at least one design")
        if qtf and any(e.get("qtf") for e in designs):
            raise ValueError("qtf=: a shared QTF table, but design %d carries its own" % next(d for d, e in enumerate(designs) if e.get("qtf")))
        per = []
        for e in designs:
            ga, gp = _capture()
            g = _general_struct(e["P"], e["M"], e["B"], e["Cm"], gp)
            fa, fp = _capture()
            f = _general_fd_struct(e.get("fd"), g.n_dof, g.nw, fp)
            qa, qp = _capture()
            q = _general_qtf_struct(qtf if qtf else e.get("qtf"), qp)
            per.append((g, ga, f, fa, q, qa))
        g0, ga0, f0, _, q0, qa0 = per[0]
        for d, (g, ga, f, _, q, qa) in enumerate(per[1:], 1):
            why = None
            if g.n_dof != g0.n_dof:
                why = "n_dof (%d against %d)" % (g.n_dof, g0.n_dof)
            elif g.nw != g0.nw or g.dw != g0.dw or not (np.array_equal(ga["w"], ga0["w"]) and np.array_equal(ga["k"], ga0["k"])):
                why = "the frequency grid"
            elif g.depth != g0.depth:
                why = "depth"
            elif g.rho != g0.rho:
                why = "rho"
            elif (f is None) != (f0 is None):
                why = "fd (frequency-dependent tables given for one design and not the other)"
            elif f is not None and f.n_fd != f0.n_fd:
                why = "n_fd (%d against %d)" % (f.n_fd, f0.n_fd)
            elif f is not None and f.n_bem_head != f0.n_bem_head:
                why = "n_bem_head (%d against %d)" % (f.n_bem_head, f0.n_bem_head)
            elif (q is None) != (q0 is None):
                why = "qtf (a QTF table given for one design and not the other)"
            elif q is not None and not (np.array_equal(qa["qtf_w"], qa0["qtf_w"]) and np.array_equal(qa["qtf_heads"], qa0["qtf_heads"])):
                why = "the QTF grid"
            elif ("node_Imat_w" in ga) != ("node_Imat_w" in ga0):
                why = "node_Imat_w (MacCamy-Fuchs tables given for one design and not the other)"
            if why:
                raise ValueError("design %d: %s differs from design 0" % (d, why))
        self.n_designs, self.n, self.nw = len(per), int(g0.n_dof), int(g0.nw)
        self.depth, self.rho, self.dw = g0.depth, g0.rho, g0.dw
        self.node_counts = np.array([g.n_nodes for g, *_ in per], dtype=_I4)
        self.node_offset = np.concatenate([[0], np.cumsum(self.node_counts)]).astype(_I4)
        self.max_nodes = int(self.node_counts.max())
        A = {}
        for name in _lib.GENERAL_ARRAYS:
            if name in ("w", "k"):
                A[name] = ga0[name]
            elif name in ("M", "B", "C"):
                A[name] = np.ascontiguousarray(np.stack([p[1][name] for p in per]))
            elif name in ga0:                          # node tables, flattened and concatenated in design order
                A[name] = np.ascontiguousarray(np.concatenate([p[1][name].ravel() for p in per]))
        self.arrays = A
        self.fd = None
        if f0 is not None:
            F = dict(fd_idx=np.ascontiguousarray(np.stack([p[3].get("fd_idx", np.zeros(0, dtype=_I4)) for p in per]), dtype=_I4))
            for name in ("fd_A_w", "fd_B_w", "fd_bem_headings", "fd_X_BEM", "fd_T0"):
                if name in per[0][3]:
                    F[name] = np.ascontiguousarray(np.stack([p[3][name] for p in per]))
            F["x_ref"] = np.array([p[2].x_ref for p in per])
            F["y_ref"] = np.array([p[2].y_ref for p in per])
            F["heading_adjust"] = np.array([p[2].heading_adjust for p in per])
            self.fd = F
            self.n_fd, self.n_bem_head = int(f0.n_fd), int(f0.n_bem_head)
        self.qtf, self.qtf_shared = None, 1 if qtf else 0
        if q0 is not None:
            self.qtf = dict(qtf_w=qa0["qtf_w"], qtf_heads=qa0["qtf_heads"],
                            qtf=qa0["qtf"] if qtf else np.ascontiguousarray(np.stack([p[5]["qtf"] for p in per])))
            self.n_qtf_w, self.n_qtf_head = int(q0.n_qtf_w), int(q0.n_qtf_head)

    @staticmethod
    def _entry(e):
        if isinstance(e, dict):
            return e
        return dict(zip(("P", "M", "B", "Cm", "fd", "qtf"), e))

    def structs(self, ptr_of):
        """(raftk_general, raftk_general_batch, raftk_general_fd or None, raftk_general_qtf or None); ``ptr_of(name, array)``
        returns the address to store (host or device, None for the size queries)."""
        g = RaftkGeneral()
        g.n_dof, g.nw, g.n_nodes = self.n, self.nw, int(self.node_offset[-1])
        g.depth, g.rho, g.dw = self.depth, self.rho, self.dw
        for name in _lib.GENERAL_ARRAYS:
            setattr(g, name, ptr_of(name, self.arrays[name]) if name in self.arrays else None)
        b = RaftkGeneralBatch()
        b.n_designs, b.max_nodes, b.qtf_shared = self.n_designs, self.max_nodes, self.qtf_shared
        b.node_offset = ptr_of("node_offset", self.node_offset)
        f = None
        if self.fd is not None:
            F = self.fd
            f = RaftkGeneralFd()
            f.n_fd, f.n_bem_head = self.n_fd, self.n_bem_head
            if self.n_fd:
                f.fd_idx, f.A_w, f.B_w = ptr_of("fd_idx", F["fd_idx"]), ptr_of("fd_A_w", F["fd_A_w"]), ptr_of("fd_B_w", F["fd_B_w"])
            if self.n_bem_head:
                f.bem_headings, f.X_BEM, f.T0 = (ptr_of(k, F[k]) for k in ("fd_bem_headings", "fd_X_BEM", "fd_T0"))
            b.x_ref, b.y_ref, b.heading_adjust = (ptr_of(k, F[k]) for k in ("x_ref", "y_ref", "heading_adjust"))
        q = None
        if self.qtf is not None:
            q = RaftkGeneralQtf()
            q.n_qtf_w, q.n_qtf_head = self.n_qtf_w, self.n_qtf_head
            q.qtf_w, q.qtf_heads, q.qtf = (ptr_of(k, self.qtf[k]) for k in ("qtf_w", "qtf_heads", "qtf"))
        return g, b, f, q


def _as_batch(designs, qtf=None):
    if isinstance(designs, GeneralBatch):
        if qtf:
            raise ValueError("qtf= applies when the batch is built here; give it to GeneralBatch")
        return designs
    return GeneralBatch(designs, qtf=qtf)


def _refs(*structs):
    return [C.byref(s) if s is not None else None for s in structs]


def general_batch_workspace_bytes(batch, n_cases, max_chunk_units=0):
    """raftk_general_batch_workspace_bytes: device workspace of a design batch (``GeneralBatch``) over ``n_cases`` cases in
    chunks of at most ``max_chunk_units`` (design, case) units (0: all).  Depends on the counts only."""
    g, b, f, q = batch.structs(lambda name, a: None)
    return int(lib.raftk_general_batch_workspace_bytes(*_refs(g, b, f, q), int(n_cases), int(max_chunk_units)))


def general_batch_chunk_plan(primary, n_cases, n_designs, max_chunk_units):
    """The chunks raftk_general_batch_solve_dynamics_* cut the units (design, case), design-major, into -> [u_0 = 0, ...,
    n_designs * n_cases]: every design's train groups in table order, packed greedily into chunks of at most
    ``max_chunk_units`` (0: all); a chunk may cross design boundaries.  ValueError where the library refuses the plan."""
    return _chunk_plan(primary, n_cases, n_designs, max_chunk_units, "max_chunk_units")


def general_batch_chunk_for_budget(batch, n_cases, budget_bytes, primary=None):
    """The largest ``max_chunk_units`` whose workspace fits ``budget_bytes`` (all units when everything fits).  With the
    table's ``primary`` map the chunk must also hold its largest train group; ValueError when it cannot."""
    nU, budget = int(n_cases) * batch.n_designs, int(budget_bytes)
    ws = lambda k: general_batch_workspace_bytes(batch, n_cases, k)       # noqa: E731
    big = 1
    if primary is not None:
        from .sweep import general_groups
        big = int(np.diff(general_groups(primary, int(n_cases))).max())
    if ws(nU) <= budget:
        return nU
    if ws(big) > budget:
        raise ValueError("a workspace of %d bytes does not hold %d units (%d bytes)" % (budget, big, ws(big)))
    return _largest_chunk(ws, big, nU, budget)


def general_solve_dynamics_batch(designs, cases, n_iter=10, tol=0.01, xi_start=0.0, F_BEM=False, F_2nd=False, max_chunk_units=0, qtf=None):
    """``general_solve_dynamics`` for a design batch in one call, host buffers: ``designs`` a ``GeneralBatch`` or its list of
    per-design inputs (``qtf``: a table shared by all), ``cases`` a CaseTable run by every design -> (Xi complex
    [nD,nT,nDOF,nw], status [nD,nT,4]) + (F_BEM [nD,nT,nDOF,nw],) with ``F_BEM`` + (F_2nd [nD,nT,6,nw], F_2nd_mean [nD,nT,6])
    with ``F_2nd``.  ``Xi[d]`` is what ``general_solve_dynamics`` returns for design d alone.  ``max_chunk_units``: the most
    (design, case) units per chunk of the device workspace (0: all)."""
    bt = _as_batch(designs, qtf)
    keep = {}

    def ptr(name, a):
        keep[name] = a
        return a.ctypes.data
    g, b, f, q = bt.structs(ptr)
    if F_2nd and q is None:
        raise ValueError("F_2nd=True needs a QTF table")
    cases.check_general_ops(f.n_fd if f is not None else 0, bt.n_designs, bt.nw)
    nD, nC, n, nw = bt.n_designs, cases.n_cases, bt.n, bt.nw
    Xi = np.zeros([nD, nC, n, nw], dtype=np.complex128)
    st = np.zeros([nD, nC, 4], dtype=_I4)
    Fb = np.zeros([nD, nC, n, nw], dtype=np.complex128) if F_BEM else None
    F2, F2m = (np.zeros([nD, nC, 6, nw]), np.zeros([nD, nC, 6])) if F_2nd else (None, None)
    c = cases.struct(_host_ptr(cases.arrays))
    o = _opts(n_iter, tol, xi_start)
    hp = lambda a: a.ctypes.data if a is not None else None   # noqa: E731
    check(lib.raftk_general_batch_solve_dynamics_host(*_refs(g, b, f, q), C.byref(c), C.byref(o), Xi.ctypes.data, st.ctypes.data, hp(Fb),
                                                      hp(F2), hp(F2m), int(max_chunk_units)))
    return (Xi, st) + ((Fb,) if F_BEM else ()) + ((F2, F2m) if F_2nd else ())


class GeneralBatchSession(_GeneralResident):
    """A design batch (``GeneralBatch`` or its list of per-design inputs) with tables, workspace and outputs resident in HBM,
    kernels on torch's current stream, the contract of ``GeneralSession``: ``solve()`` enqueues
    raftk_general_batch_solve_dynamics_dev -> (Xi [nD,nT,nDOF,nw] complex, status [nD,nT,4]) (+ F_BEM [nD,nT,nDOF,nw] with
    ``F_BEM=True``); with a QTF table every ``solve()`` leaves ``F_2nd`` [nD,nT,6,nw] and ``F_2nd_mean`` [nD,nT,6] on the
    device.  ``max_chunk_units``: the most (design, case) units per chunk of the workspace (0: all; ``general_batch_chunk_for_budget``).
    ``stats(R, wpow)`` takes channel rows per design, R [nD,nch,nDOF] (``packer.pack_general_channels`` of each design)."""

    def __init__(self, designs, cases, device=None, F_BEM=False, qtf=None, max_chunk_units=0):
        self._open(device)
        self.batch = bt = _as_batch(designs, qtf)
        if int(max_chunk_units) < 0:
            raise ValueError("max_chunk_units must be >= 0 (0: all units in one chunk)")
        self.max_chunk_units = int(max_chunk_units)
        nD, nC, n, nw = bt.n_designs, cases.n_cases, bt.n, bt.nw
        cases.check_general_ops(bt.n_fd if bt.fd is not None else 0, nD, nw)
        with self.torch.cuda.device(self.device):
            self.g, self.b, self.fd, self.qtf = bt.structs(self._to_dev)
            self._upload_cases(cases)
            self.workspace_bytes = general_batch_workspace_bytes(bt, nC, self.max_chunk_units)
            self._outputs([nD, nC], n, nw, F_BEM)
        self.n_designs, self.n, self.nw, self.n_cases, self.dw = nD, n, nw, nC, bt.dw

    def solve(self, n_iter=10, tol=0.01, xi_start=0.0):
        return self._enqueue(lib.raftk_general_batch_solve_dynamics_dev, (self.g, self.b, self.fd, self.qtf), n_iter, tol, xi_start,
                             self.max_chunk_units)

    def eigen(self, A0=None, yawstiff=0.0, sort="ascending", modes=True):
        """Natural frequencies and mode shapes of every design on the device, on torch's current stream (async):
        raftk_eigen_dev on M + A0 and Cm + yawstiff e5 e5^T from the resident tables.  ``A0`` [6,6] or [nD,6,6]: the BEM added
        mass at the grid's first bin (A_BEM[:6, :6, 0]; readHydro lumps it on the reduced DOFs 0-5), None for none;
        ``yawstiff`` scalar or [nD].  -> dict(lam [nD,n], fns [nD,n] = sqrt(lam) / 2 pi, modes [nD,n,n] or None) complex,
        info [nD] int32 (RAFTK_EIG_* flags), torch tensors; ``sort`` as ``solve_eigen``."""
        nD, n = self.n_designs, self.n
        return _session_eigen(self, self.keep["M"].view(nD, n, n), self.keep["C"].view(nD, n, n), A0, yawstiff, sort, modes)


def _no_general_ops(turbine_constants):
    if turbine_constants is not None:
        raise NotImplementedError("turbine_constants= (raw per-case snapshots) is not taken by the generalised-DOF analysis, whose "
                                  "M, B and fd come packed and would count the snapshots' terms twice: pack them with "
                                  "packer.pack_general_matrices(fowt, states=...) and pass its M, B, fd and ops=")


def _train_ops(ops, owner, n_cases):
    """Per-case operating points (op [n_cases]) expanded to the rows of a train table (``pack_case_trains``' owner)."""
    if ops is None:
        return None
    op = np.asarray(ops["op"])
    if op.shape != (n_cases,):
        raise ValueError("ops['op'] must name one operating point per case (%d), got shape %s" % (n_cases, list(op.shape)))
    return dict(op=op[owner], A_w=ops["A_w"], B_w=ops["B_w"])


def general_analyze_cases_batch(designs, cases, channels=None, n_iter=10, tol=0.01, xi_start=0.0, qtf=None, rotors=None,
                                turbine_constants=None, ops=None, fatigue=None, stress=None):
    """``general_analyze_cases`` for every design of a batch in one solve: ``designs`` a list of per-design inputs (or a
    ``GeneralBatch`` built from them), ``cases`` a list of case dicts run by every design, ``channels`` None or one
    ``packer.pack_general_channels`` dict per design, ``rotors`` None or one ``packer.pack_rotor_outputs`` dict per design
    -> a list with, for each design, what ``general_analyze_cases`` returns for that design alone.  ``ops``: one operating
    point per case, tables per design [nD, n_op, n_fd, n_fd, nw] or shared [n_op, n_fd, n_fd, nw]
    (``packer.pack_general_operating_points``).  ``turbine_constants``: NotImplementedError, as for ``general_analyze_cases``.
    ``fatigue``, ``stress``: as for ``general_analyze_cases``, every design with the same options."""
    from .packer import pack_case_trains
    _no_general_ops(turbine_constants)
    opts = None if fatigue is None else fatigue_options(fatigue)
    bt = _as_batch(designs, qtf)
    if channels is not None and len(channels) != bt.n_designs:
        raise ValueError("channels: one entry per design (%d), got %d" % (bt.n_designs, len(channels)))
    if rotors is not None and len(rotors) != bt.n_designs:
        raise ValueError("rotors: one entry per design (%d), got %d" % (bt.n_designs, len(rotors)))
    sopts = None if stress is None else stress_options_for(stress, [None] * bt.n_designs if channels is None else channels)
    table, owner, first = pack_case_trains(cases)
    q = bt.qtf is not None
    res = general_solve_dynamics_batch(bt, CaseTable(table, ops=_train_ops(ops, owner, len(cases))), n_iter=n_iter, tol=tol,
                                       xi_start=xi_start, F_2nd=q)
    P = dict(w=bt.arrays["w"], dw=bt.dw)
    return [_general_case_results(P, res[0][d], res[1][d], owner, first, len(cases), None if channels is None else channels[d],
                                  (res[2][d], res[3][d]) if q else None, None if rotors is None else rotors[d], opts, sopts)
            for d in range(bt.n_designs)]


def second_order_force(batch, cases):
    """FOWT.calcHydroForce_2ndOrd (raft_fowt.py:2158-2253) for every (design, case) from the designs' QTF table,
    host buffers -> dict(F_2nd [nD,nC,6,nw] real amplitudes, F_2nd_mean [nD,nC,6])."""
    if batch.n_qtf_w == 0:
        raise ValueError("the designs carry no QTF table (potSecOrder 2 / packer.pack_qtf)")
    outs = _alloc_outputs(batch.n_designs, cases.n_cases, batch.nw, ("F_2nd", "F_2nd_mean"))
    os_ = _out_struct(outs, lambda a: a.ctypes.data)
    check(lib.raftk_second_order_force_host(C.byref(_host_struct(batch)), C.byref(_host_struct(cases)), C.byref(os_)))
    return outs


def hydro_linearization(batch, cases, Xi, want=("B_drag", "F_drag")):
    """FOWT.calcHydroLinearization(Xi) + calcDragExcitation(0) (raft_fowt.py:1891-1957), host buffers.

    ``Xi`` complex [nD,nC,6,nw] (or [6,nw], broadcast to every unit)."""
    nD, nC, nw = batch.n_designs, cases.n_cases, batch.nw
    Xi = np.asarray(Xi, dtype=np.complex128)
    if Xi.shape == (6, nw):
        Xi = np.broadcast_to(Xi, (nD, nC, 6, nw))
    Xi = np.ascontiguousarray(Xi)
    if Xi.shape != (nD, nC, 6, nw):
        raise ValueError("Xi must have shape [nD,nC,6,nw] or [6,nw]")
    outs = _alloc_outputs(nD, nC, nw, want)
    os_ = _out_struct(outs, lambda a: a.ctypes.data)
    check(lib.raftk_hydro_linearization_host(C.byref(_host_struct(batch)), C.byref(_host_struct(cases)), Xi.ctypes.data, C.byref(os_)))
    return outs


def farm_workspace_bytes(n_fowt, n_cases, nw):
    """Device workspace the farm system response needs: 0 while the [6N][6N+1] system fits in shared memory, else one slab
    per resident CTA of the global-memory kernel.  Answers for an H100 without a device."""
    return farm_batch_workspace_bytes(1, n_fowt, n_cases, nw)


def farm_batch_workspace_bytes(n_farms, n_fowt, n_cases, nw):
    """``farm_workspace_bytes`` for a batch of ``n_farms`` farms (raftk_farm_batch_workspace_bytes): the slabs are capped at the
    n_farms * n_cases * nw systems of the call."""
    d, c, f = RaftkDesigns(), RaftkCases(), RaftkFarmBatch()
    d.n_designs, d.nw, c.n_cases, f.n_farms, f.n_fowt, f.arr_shared = int(n_farms) * int(n_fowt), int(nw), int(n_cases), int(n_farms), int(n_fowt), 1
    return int(lib.raftk_farm_batch_workspace_bytes(C.byref(d), C.byref(c), C.byref(f)))


def system_solve(Z, F):
    """Farm system response (raft_model.py:1164-1216): Z [nw,n,n], F [nw,n] or [nw,n,nrhs] -> Xi, info."""
    Z = np.array(Z, dtype=np.complex128, order="C")
    F = np.array(F, dtype=np.complex128, order="C")
    squeeze = F.ndim == 2
    if squeeze:
        F = np.ascontiguousarray(F[:, :, None])
    nw, n, nrhs = F.shape
    if Z.shape != (nw, n, n):
        raise ValueError("Z must be [nw,n,n] matching F")
    info = np.zeros(nw, dtype=_I4)
    check(lib.raftk_system_solve_host(n, nw, nrhs, Z.ctypes.data, F.ctypes.data, info.ctypes.data))
    return (F[:, :, 0] if squeeze else F), info


EIG_SMALL_DIAG, EIG_NONPOSITIVE, EIG_COMPLEX, EIG_SINGULAR, EIG_NOCONV = 1, 2, 4, 8, 16    # include/raftk.h RAFTK_EIG_*
_EIG_SORT = {"dof": 0, "ascending": 1}


def _eigen_struct(n_systems, n, sort, M=None, C_=None, lam=None, modes=None, info=None):
    if sort not in _EIG_SORT:
        raise ValueError("sort must be 'dof' or 'ascending', not %r" % (sort,))
    e = _lib.RaftkEigen()
    e.n_systems, e.n, e.sort = int(n_systems), int(n), _EIG_SORT[sort]
    e.M, e.C, e.lam, e.modes, e.info = M, C_, lam, modes, info
    return e


def eigen_workspace_bytes(n_systems, n):
    """Device workspace of the eigen analysis (raftk_eigen_workspace_bytes): 0 for n <= 12, else whole per-CTA slabs.
    Answers for an H100 without a device."""
    return int(lib.raftk_eigen_workspace_bytes(C.byref(_eigen_struct(n_systems, n, "dof"))))


def eigen_outputs(lam, modes, info):
    """numpy's conventions for the raw outputs: lam -> real dtype when every eigenvalue is real (NaN slots of systems without a
    spectrum do not count), likewise modes; fns = sqrt(lam) / 2 pi as the reference writes it (NaN for a negative real)."""
    real = bool(np.all((lam.imag == 0.0) | np.isnan(lam.imag)))
    if real:
        lam = np.ascontiguousarray(lam.real)
        modes = None if modes is None else np.ascontiguousarray(modes.real)
    with np.errstate(invalid="ignore"):
        fns = np.sqrt(lam) / 2.0 / np.pi
    return dict(lam=lam, fns=fns, modes=modes, info=info)


def solve_eigen(M, C_, sort="dof", modes=True):
    """Natural frequencies and mode shapes of systems M x'' + C x = 0 on the GPU (raftk_eigen_host): the eigenvalues and unit
    2-norm right eigenvectors of M^-1 C, as np.linalg.eig(np.linalg.solve(M, C)) returns them, in the reference's order
    (``sort='dof'``: raft_model.py:490-516; ``'ascending'``: np.argsort).  M, C [n,n] or [nS,n,n] ->
    dict(lam [nS,n], fns [nS,n] Hz, modes [nS,n,n] (column j = mode j) or None, info [nS] RAFTK_EIG_* flags); real dtypes
    when every eigenvalue is real.  ``eigen_raise`` turns the flags into the reference's exceptions."""
    M = np.ascontiguousarray(M, dtype=_F8)
    K = np.ascontiguousarray(C_, dtype=_F8)
    squeeze = M.ndim == 2
    if squeeze:
        M, K = M[None], K[None]
    r = _eigen(_HOST, M, K, sort, modes)
    out = eigen_outputs(r["lam"], r["modes"], r["info"])
    if squeeze:
        out = {k: (None if v is None else v[0]) for k, v in out.items()}
    return out


def _eigen(be, M, K, sort, modes):
    """The eigen analysis of M, K [nS,n,n] on ``be``'s buffers -> dict(lam, modes, info), raw (complex)."""
    M, K = be.array(M, _F8), be.array(K, _F8)
    if M.ndim != 3 or M.shape != K.shape or M.shape[1] != M.shape[2]:
        raise ValueError("M and C must both be [n,n] or [n_systems,n,n]")
    nS, n = M.shape[:2]
    lam = be.empty([nS, n], _C16)
    V = be.empty([nS, n, n], _C16) if modes else None
    info = be.empty([nS], _I4)
    e = _eigen_struct(nS, n, sort, be.ptr(M), be.ptr(K), be.ptr(lam), be.ptr(V), be.ptr(info))
    be.call("eigen", C.byref(e), ws=(C.byref(e),))
    return dict(lam=lam, modes=V, info=info)


def eigen_raise(M, C_, info, sort="dof"):
    """The reference's exceptions for one system's flags, in its order (raft_model.py:478-500, raft_fowt.py:1667-1683):
    RuntimeError naming the diagonals of M and C below 1; np.linalg.LinAlgError for a singular M (np.linalg.solve) or a QR
    iteration that did not converge (np.linalg.eig); with ``sort='dof'`` RuntimeError on an eigenvalue <= 0."""
    info = int(info)
    if info & EIG_SMALL_DIAG:
        msg = ""
        for i in range(len(M)):
            if M[i, i] < 1.0:
                msg += f'Diagonal entry {i} of system mass matrix is less than 1 ({M[i, i]}). '
            if C_[i, i] < 1.0:
                msg += f'Diagonal entry {i} of system stiffness matrix is less than 1 ({C_[i, i]}). '
        raise RuntimeError('System matrices computed by RAFT have one or more small or negative diagonals: ' + msg)
    if info & EIG_SINGULAR:
        raise np.linalg.LinAlgError("Singular matrix")
    if info & EIG_NOCONV:
        raise np.linalg.LinAlgError("Eigenvalues did not converge")
    if sort == "dof" and info & EIG_NONPOSITIVE:
        raise RuntimeError("Error: zero or negative system eigenvalues detected.")


def eigen_fns_modes(M, C_, sort):
    """One system as Model.solveEigen / FOWT.solveEigen return it: (fns, modes) or the reference's exception.  A DOF claim
    that leaves rows unclaimed returns fewer modes, as the reference does."""
    r = solve_eigen(M, C_, sort=sort)
    eigen_raise(M, C_, r["info"], sort)
    fns, modes = r["fns"], r["modes"]
    keep = ~np.isnan(r["lam"].real)
    return fns[keep], modes[:, keep]


def _session_eigen(session, M, K, A0, yawstiff, sort, modes):
    """A session's eigen(): the eigen analysis of ``_eigen_inputs`` on its resident M, K [nD,n,n], plus fns = sqrt(lam) / 2 pi."""
    nD, n = M.shape[:2]
    be = _session_buffers(session)
    r = _eigen(be, *_eigen_inputs(M, K, A0, yawstiff, nD, n, session.device), sort, modes)
    return dict(lam=r["lam"], fns=be.torch.sqrt(r["lam"]) / (2.0 * np.pi), modes=r["modes"], info=r["info"])


def _eigen_inputs(M, K, A0, yawstiff, nD, n, device):
    """M + A0 on DOFs 0-5 (A0 [6,6] shared or [nD,6,6]) and K + yawstiff on DOF 5 (scalar or [nD]), as new tensors."""
    import torch
    M = M.clone()
    K = K.clone()
    if A0 is not None:
        A = torch.as_tensor(np.asarray(A0, dtype=_F8), device=device)
        if tuple(A.shape) not in ((6, 6), (nD, 6, 6)):
            raise ValueError("A0 must be [6,6] or [%d,6,6]" % nD)
        M[:, :6, :6] += A
    y = torch.as_tensor(np.asarray(yawstiff, dtype=_F8), device=device)
    if y.ndim not in (0, 1) or (y.ndim == 1 and y.shape[0] != nD):
        raise ValueError("yawstiff must be a scalar or [%d]" % nD)
    K[:, 5, 5] += y
    return M, K


_PINNED = []


def response_stats(Xi, dw, psd=True, rot_deg=True):
    """std / PSD per DOF of responses Xi [...,6,nw] (FOWT.saveTurbineOutputs, raft_fowt.py:2299-2353):
    std = sqrt(1/2 sum |Xi|^2), PSD = 1/2 |Xi|^2 / dw, rotations in degrees.  -> (std [...,6], PSD [...,6,nw] or None)."""
    Xi = np.ascontiguousarray(Xi, dtype=np.complex128)
    lead, nw = Xi.shape[:-2], Xi.shape[-1]
    if Xi.shape[-2] != 6:
        raise ValueError("Xi must be [..., 6, nw]")
    n = int(np.prod(lead)) if lead else 1
    sd = np.zeros(lead + (6,))
    P = np.zeros(lead + (6, nw)) if psd else None
    check(lib.raftk_response_stats_host(n, nw, float(dw), 1 if rot_deg else 0, Xi.ctypes.data, sd.ctypes.data,
                                        P.ctypes.data if psd else None))
    return sd, P


def channel_stats(coef, Xi, dw, psd=True, amp=False):
    """Statistics of linear output channels Y = sum_dof coef * Xi (nacelle accelerations, tower-base moment;
    raft_fowt.py:2401-2444, 2504-2538; coefficients from ``packer.pack_turbine_channels``).
    ``coef`` complex [nD,nch,6,nw] (or [nch,6,nw]); ``Xi`` complex [nD,nC,6,nw] (or [nC,6,nw])
    -> (std [nD,nC,nch], PSD [nD,nC,nch,nw] or None, amplitudes complex [nD,nC,nch,nw] or None)."""
    coef = np.ascontiguousarray(coef, dtype=np.complex128)
    Xi = np.ascontiguousarray(Xi, dtype=np.complex128)
    squeeze = coef.ndim == 3
    if squeeze:
        coef, Xi = coef[None], Xi[None]
    nD, nch, _, nw = coef.shape
    if Xi.ndim != 4 or Xi.shape[0] != nD or Xi.shape[2:] != (6, nw) or coef.shape[2] != 6:
        raise ValueError("coef must be [nD,nch,6,nw] and Xi [nD,nC,6,nw]")
    nC = Xi.shape[1]
    sd = np.zeros([nD, nC, nch])
    P = np.zeros([nD, nC, nch, nw]) if psd else None
    A = np.zeros([nD, nC, nch, nw], dtype=np.complex128) if amp else None
    check(lib.raftk_channel_stats_host(nD, nC, nch, nw, float(dw), coef.ctypes.data, Xi.ctypes.data, sd.ctypes.data,
                                       P.ctypes.data if psd else None, A.ctypes.data if amp else None))
    if squeeze:
        sd, P, A = sd[0], (P[0] if psd else None), (A[0] if amp else None)
    return sd, P, A


def pinned_empty(shape, dtype):
    """NumPy array backed by page-locked host memory (cudaHostAlloc) for the e2e path."""
    dtype = np.dtype(dtype)
    n = int(np.prod(shape)) * dtype.itemsize
    p = lib.raftk_host_alloc(max(n, 1))
    if not p:
        raise MemoryError("cudaHostAlloc failed")
    buf = (C.c_char * max(n, 1)).from_address(p)
    arr = np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)
    _PINNED.append((buf, p))        # keep alive; page-locked blocks live until process exit
    return arr


class DeviceSession:
    """Tables, workspace and outputs resident in HBM (torch tensors); kernels on torch's current stream."""

    def __init__(self, batch, cases, device=None, want=("Xi", "status", "B_drag"), workspace_bytes=None, tables=False, out_tensors=None):
        """``tables=True`` sizes the workspace for ``excitation()`` / ``linearization()`` (global wave tables);
        the default covers ``solve()`` only (the fused solver keeps its tables on chip).  ``out_tensors``: outputs the
        caller already owns (name -> tensor of the documented shape), e.g. this rank's block of a peer-shared array."""
        want = tuple(dict.fromkeys(tuple(want) + ("Xi", "status") + (("F_2nd", "F_2nd_mean") if batch.n_qtf_w else ())))
        _check_outputs(want, _SESSION_OUTPUTS)
        import torch
        self.torch = torch
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.batch, self.cases = batch, cases
        cases.check_ops(batch)
        with torch.cuda.device(self.device):
            # every input table (design + case columns) lives in ONE device block, 256-byte aligned slots: a caller that
            # refreshes the tables from the host (sweep.ShardedSolve.step_host) sends them with a single copy
            items, total = [], 0
            for grp, arrs in (("d", batch.arrays), ("c", cases.arrays)):
                for k, v in arrs.items():
                    v = np.ascontiguousarray(v)
                    v = v.view(np.float64) if v.dtype == np.complex128 else v
                    items.append((grp, k, v, total))
                    total += (v.nbytes + 255) // 256 * 256
            host_block = np.zeros(max(total, 256), dtype=np.uint8)
            for _, _, v, off in items:
                host_block[off:off + v.nbytes] = v.reshape(-1).view(np.uint8)
            self.tables = torch.from_numpy(host_block).to(self.device)
            self.table_bytes = int(total)
            self.dt, self.ct = {}, {}
            for grp, k, v, off in items:
                tdt = torch.from_numpy(np.empty(0, dtype=v.dtype)).dtype
                t = self.tables[off:off + v.nbytes].view(tdt).view(v.shape) if v.nbytes else torch.from_numpy(v).to(self.device)
                (self.dt if grp == "d" else self.ct)[k] = t
            self.d_struct = batch.struct(lambda name: self.dt[name].data_ptr())
            self.c_struct = cases.struct(lambda name: self.ct[name].data_ptr())
            need = (lib.raftk_workspace_bytes if tables else lib.raftk_solve_workspace_bytes)(C.byref(self.d_struct), cases.n_cases)
            self.workspace_bytes = int(need if workspace_bytes is None else workspace_bytes)
            self.workspace = torch.empty(self.workspace_bytes, dtype=torch.uint8, device=self.device)
            shapes = _output_table(batch.n_designs, cases.n_cases, batch.nw)
            given = dict(out_tensors or {})
            for k, t in given.items():
                shape, dt = shapes[k][0], _torch_dtype(shapes[k][1])
                if tuple(t.shape) != tuple(shape) or t.dtype != dt or not t.is_contiguous():
                    raise ValueError("out_tensors[%r] must be a contiguous %s tensor of shape %s" % (k, dt, shape))
            zeros = _torch_zeros(self.device)
            self.out = {k: (given[k] if k in given else zeros(*shapes[k])) for k in want}
            self.o_struct = _out_struct(self.out, lambda t: t.data_ptr())

    def _stream(self):
        return self.torch.cuda.current_stream(self.device).cuda_stream

    def _opts(self, n_iter, tol, xi_start, cluster_size):
        """Solve options; from the second call with the same cluster size on, the per-design plan blobs that the first call
        left in the session's workspace are reused (the session owns tables and workspace, so they cannot have changed)."""
        key = int(cluster_size)
        o = _opts(n_iter, tol, xi_start, key, 1 if getattr(self, "_plan_key", None) == key else 0)
        self._plan_key = key
        return o

    def solve(self, n_iter=10, tol=0.01, xi_start=0.0, cluster_size=0):
        """Enqueue Model.solveDynamics for all units on the current stream; returns the output dict (async)."""
        o = self._opts(n_iter, tol, xi_start, cluster_size)
        with self.torch.cuda.device(self.device):
            check(lib.raftk_solve_dynamics_dev(C.byref(self.d_struct), C.byref(self.c_struct), C.byref(o),
                                               C.byref(self.o_struct), self.workspace.data_ptr(), self.workspace_bytes,
                                               self._stream()))
        return self.out

    def solve_gather(self, peers, o_struct=None, n_iter=10, tol=0.01, xi_start=0.0, cluster_size=0, timeout_flag=None):
        """``solve`` with the multi-GPU exchange fused into the kernel (``raft_b200.sweep.PeerExchange``): every finished
        unit is stored into all ranks' gathered arrays over NVLink, then the stream waits for the peers' arrival flags."""
        o = self._opts(n_iter, tol, xi_start, cluster_size)
        os_ = self.o_struct if o_struct is None else o_struct
        with self.torch.cuda.device(self.device):
            check(lib.raftk_solve_dynamics_gather_dev(C.byref(self.d_struct), C.byref(self.c_struct), C.byref(o), C.byref(os_),
                                                      C.byref(peers), self.workspace.data_ptr(), self.workspace_bytes, self._stream()))
            check(lib.raftk_peer_barrier_dev(C.byref(peers), timeout_flag, self._stream()))

    def farm_response(self, C_arr=None, M_arr=None, B_arr=None, n_fowt=None, farm_sizes=None):
        """Enqueue the coupled 6N-DOF system response of the LAST ``solve`` (the session's designs are the FOWTs of the
        array; it must have been created with want including B_drag, F_drag, F_iner [+ F_BEM]).  -> (Xi_sys [nC,6N,nw], info).
        Any N: farms whose system does not fit in shared memory are solved in a device workspace sized once
        (raftk_farm_workspace_bytes) and kept with the session.
        ``n_fowt``: the session's designs are n_designs / n_fowt farms of n_fowt FOWTs each (design f * n_fowt + i is FOWT i
        of farm f), array matrices [6N,6N] for every farm or [F,6N,6N] -> (Xi_sys [F,nC,6N,nw], info [F,nC,nw]).  The
        matrices, outputs and workspace of either form are set up on its first call and kept with the session.
        ``farm_sizes``: the session's designs are farms of farm_sizes[f] FOWTs each, farm after farm (a ragged batch,
        raftk_farm_ragged_response_ws_dev), array matrices as ``solve_dynamics_farm_ragged`` -> (Xi_sys, a list of per-farm
        [nC,6N_f,nw] views of one flat tensor, info [F,nC,nw]); set up again when the sizes change."""
        torch = self.torch
        if farm_sizes is not None:
            if n_fowt is not None:
                raise ValueError("farm_response: give n_fowt or farm_sizes, not both")
            return self._farm_ragged(farm_sizes, M_arr, B_arr, C_arr)
        N = self.batch.n_designs if n_fowt is None else int(n_fowt)
        if N < 1 or self.batch.n_designs % N:
            raise ValueError("n_fowt must divide the session's %d designs" % self.batch.n_designs)
        f, _, xi, info, ws, wsb = self._farm_setup(N, n_fowt, M_arr, B_arr, C_arr)
        launch = lib.raftk_farm_response_ws_dev if n_fowt is None else lib.raftk_farm_batch_response_ws_dev
        with torch.cuda.device(self.device):
            check(launch(C.byref(self.d_struct), C.byref(self.c_struct), C.byref(self.o_struct), C.byref(f), ws.data_ptr(), wsb, self._stream()))
        return xi, info

    def _farm_ragged(self, farm_sizes, M_arr, B_arr, C_arr):
        sizes = tuple(int(n) for n in farm_sizes)
        if getattr(self, "_farm_rag", (None,))[0] != sizes:
            with self.torch.cuda.device(self.device):
                f, keep, xi, info = _ragged_setup(sizes, self.cases.n_cases, self.batch.nw, M_arr, B_arr, C_arr, device=self.device)
                wsb = int(lib.raftk_farm_ragged_workspace_bytes(C.byref(self.d_struct), C.byref(self.c_struct), C.byref(f)))
                if wsb == 0:                # a shape raftk_farm_ragged refuses: its reason
                    raise _lib.RaftkError("raftk error: %s" % lib.raftk_last_error().decode("utf-8", "replace"))
                ws = self.torch.empty(wsb, dtype=self.torch.uint8, device=self.device)
            self._farm_rag = (sizes, f, keep, xi, info, ws, wsb, ragged_views(xi, sizes, self.cases.n_cases, self.batch.nw))
        _, f, _, _, info, ws, wsb, views = self._farm_rag
        with self.torch.cuda.device(self.device):
            check(lib.raftk_farm_ragged_response_ws_dev(C.byref(self.d_struct), C.byref(self.c_struct), C.byref(self.o_struct), C.byref(f),
                                                        ws.data_ptr(), wsb, self._stream()))
        return views, info

    def farm_response_ragged_gather(self, peers, farm_row0, fowt_row0, n_farms_total, Xi_sys, info, farm_sizes, C_arr=None, M_arr=None,
                                    B_arr=None):
        """``farm_response(farm_sizes=...)`` of this rank's farms stored at their global offsets of every rank's copy
        (raftk_farm_ragged_response_gather_dev; ``sweep.ShardedFarmSolve(farm_sizes=...)``): the session's designs are
        designs [fowt_row0, ...) of the whole batch, farms [farm_row0, farm_row0 + len(farm_sizes)) of ``n_farms_total``;
        ``Xi_sys`` (flat) and ``info`` [F_r,nC,nw] are their rows of this rank's own copy.  Follow with raftk_peer_barrier_dev."""
        sizes = tuple(int(n) for n in farm_sizes)
        if getattr(self, "_farm_rag_gather", (None,))[0] != sizes:
            with self.torch.cuda.device(self.device):
                f, keep, _, _ = _ragged_setup(sizes, self.cases.n_cases, self.batch.nw, M_arr, B_arr, C_arr, device=self.device)
                wsb = int(lib.raftk_farm_ragged_workspace_bytes(C.byref(self.d_struct), C.byref(self.c_struct), C.byref(f)))
                if wsb == 0:
                    raise _lib.RaftkError("raftk error: %s" % lib.raftk_last_error().decode("utf-8", "replace"))
                ws = self.torch.empty(wsb, dtype=self.torch.uint8, device=self.device)
            self._farm_rag_gather = (sizes, f, keep, ws, wsb)
        _, f, _, ws, wsb = self._farm_rag_gather
        g = RaftkFarmRagged.from_buffer_copy(f)
        g.Xi_sys, g.info = Xi_sys.data_ptr(), info.data_ptr()
        with self.torch.cuda.device(self.device):
            check(lib.raftk_farm_ragged_response_gather_dev(C.byref(self.d_struct), C.byref(self.c_struct), C.byref(self.o_struct),
                                                            C.byref(g), C.byref(peers), int(farm_row0), int(fowt_row0),
                                                            int(n_farms_total), ws.data_ptr(), wsb, self._stream()))

    def _farm_setup(self, N, n_fowt, M_arr, B_arr, C_arr, gather=False):
        """The farm struct, matrices, outputs and workspace of ``farm_response``'s form ``n_fowt``, set up on first use;
        ``gather``: those of ``farm_response_gather``, kept apart and without outputs (they live in the gathered copies)."""
        torch = self.torch
        # one farm is kept as the single-farm struct (raftk_farm), which callers hand to the single-farm entries, and launches
        # through them; its matrices and outputs are set up as a batch of one
        key, query = ("_farm", lib.raftk_farm_workspace_bytes) if n_fowt is None else ("_farm_batch", lib.raftk_farm_batch_workspace_bytes)
        if gather:
            key = "_farm_gather"
        if not hasattr(self, key) or getattr(self, key)[0].n_fowt != N:
            with torch.cuda.device(self.device):
                f, mats, xi, info = _farm_setup(N, None if n_fowt is None else self.batch.n_designs // N, self.cases.n_cases,
                                                self.batch.nw, M_arr, B_arr, C_arr, device=self.device, outputs=not gather)
                if n_fowt is None:
                    f = RaftkFarm(n_fowt=N, M_arr=f.M_arr, B_arr=f.B_arr, C_arr=f.C_arr, Xi_sys=f.Xi_sys, info=f.info)
                wsb = int(query(C.byref(self.d_struct), C.byref(self.c_struct), C.byref(f)))
                ws = torch.empty(max(wsb, 1), dtype=torch.uint8, device=self.device)
            setattr(self, key, (f, mats, xi, info, ws, wsb))
        return getattr(self, key)

    def farm_response_gather(self, peers, farm_row0, Xi_sys, info, n_fowt, C_arr=None, M_arr=None, B_arr=None):
        """``farm_response(n_fowt=...)`` of this rank's farms with the results stored into every rank's gathered copy
        (raftk_farm_batch_response_gather_dev; ``sweep.ShardedFarmSolve``): ``Xi_sys`` [F,nC,6N,nw] and ``info`` [F,nC,nw] are
        farms [farm_row0, farm_row0 + F) of this rank's own copy, and the per-FOWT status of the last ``solve`` goes to every
        copy too.  Matrices and workspace as ``farm_response``; follow with raftk_peer_barrier_dev."""
        N = int(n_fowt)
        if N < 1 or self.batch.n_designs % N:
            raise ValueError("n_fowt must divide the session's %d designs" % self.batch.n_designs)
        f, _, _, _, ws, wsb = self._farm_setup(N, N, M_arr, B_arr, C_arr, gather=True)
        g = RaftkFarmBatch.from_buffer_copy(f)
        g.Xi_sys, g.info = Xi_sys.data_ptr(), info.data_ptr()
        with self.torch.cuda.device(self.device):
            check(lib.raftk_farm_batch_response_gather_dev(C.byref(self.d_struct), C.byref(self.c_struct), C.byref(self.o_struct),
                                                           C.byref(g), C.byref(peers), int(farm_row0), ws.data_ptr(), wsb, self._stream()))

    def _response(self, what, farm, n_fowt):
        """The resident response reduction ``what`` runs on: the last ``solve``'s Xi [nD,nC,6,nw], or with ``farm`` the Xi_sys of
        the last ``farm_response`` of the form ``n_fowt`` names ([nC,6N,nw] for one farm, which the reductions return without
        the unit axis, [F,nC,6N,nw] for a batch)."""
        if not farm:
            return self.out["Xi"]
        key = "_farm" if n_fowt is None else "_farm_batch"
        if not hasattr(self, key):
            raise RuntimeError("%s: call farm_response(n_fowt=%r) first" % (what, n_fowt))
        return getattr(self, key)[2]

    def farm_channel_stats(self, R, dw, wpow=None, psd=True, amp=False, n_fowt=None, tile_w=0):
        """Enqueue channel statistics of the LAST ``farm_response`` on the resident Xi_sys (raftk_farm_channel_stats_dev; no
        host round trip): mooring tensions with R the tension Jacobian.  ``n_fowt`` names the form of ``farm_response`` that
        ran (None: one farm).  ``R``, ``dw``, ``wpow``, ``tile_w`` as ``farm_channel_stats``.  -> torch tensors (std [F,nC,nch],
        PSD [F,nC,nch,nw] or None, amplitudes complex [F,nC,nch,nw] or None), without the farm axis for ``n_fowt=None``."""
        xi = self._response("farm_channel_stats", True, n_fowt)
        return _farm_channel_stats(_session_buffers(self), R, xi, dw, self.dt["w"], wpow, psd, amp, tile_w)

    def rotor_stats(self, R, C_, V_w, gains, dw, case_row0=None, col0=None, psd=True, farm=False, n_fowt=None):
        """Enqueue rotor speed, generator torque and blade pitch statistics on a resident response (raftk_rotor_stats_dev; no
        host round trip).  ``farm=False``: the last ``solve``'s Xi [nD, nC, 6, nw], one unit per design; ``farm=True``: the
        Xi_sys of the LAST ``farm_response`` of the form ``n_fowt`` names (as ``farm_channel_stats``), one unit per farm, FOWT
        i's hub rows at ``col0`` = 6 i.  ``R``, ``C``, ``V_w``, ``gains``, ``case_row0``, ``col0`` as ``rotor_stats`` (numpy or
        torch).  -> (std [nU, nCases, nrot, 3], PSD [nU, nCases, nrot, 3, nw] or None) torch tensors, without the unit axis
        for one farm (``farm=True``, ``n_fowt=None``)."""
        xi = self._response("rotor_stats", farm, n_fowt)
        return _rotor_stats(_session_buffers(self), R, C_, V_w, gains, self.dt["w"], xi, dw, case_row0, col0, psd)

    def fatigue(self, m, R=None, wpow=None, coef=None, case_row0=None, f_eq=1.0, method="dirlik", weights=None, life=None,
                moments=True, tile_w=0, farm=False, n_fowt=None):
        """Enqueue fatigue DELs on a resident response (raftk_fatigue_dev; no host round trip).  ``farm=False``: the last
        ``solve``'s Xi [nD, nC, 6, nw], one unit per design (e.g. ``coef`` [nch, 6, nw] of ``packer.pack_turbine_channels``
        for Mbase); ``farm=True``: the Xi_sys of the LAST ``farm_response`` of the form ``n_fowt`` names (as
        ``farm_channel_stats``), one unit per farm (e.g. the tension Jacobian as ``R``).  The other arguments as ``fatigue``.
        -> dict of torch tensors as ``fatigue``, without the unit axis for one farm (``farm=True``, ``n_fowt=None``)."""
        xi = self._response("fatigue", farm, n_fowt)
        return _fatigue(_session_buffers(self), xi, self.dt["w"], m, R, wpow, coef, case_row0, f_eq, method, weights, life, moments,
                        tile_w)

    def stress_ring(self, fa, ss, angles=None, d=10.0, t=0.083, m=None, f_eq=1.0, method="dirlik", weights=None, case_row0=None,
                    col0=None, psd=False, mean=None, wpow=None, tile_w=0, farm=False, n_fowt=None):
        """Enqueue the tower-base axial stress around the circumference on a resident response (raftk_stress_ring_dev; no host
        round trip).  ``farm=False``: the last ``solve``'s Xi [nD, nC, 6, nw], one unit per design (e.g. ``fa`` the Mbase
        coefficients of ``packer.pack_turbine_channels``, ``ss`` None); ``farm=True``: the Xi_sys of the LAST ``farm_response``
        of the form ``n_fowt`` names, one unit per farm, FOWT i's tower at ``col0`` = 6 i.  The other arguments as
        ``stress_ring``.  -> dict of torch tensors as ``stress_ring``, without the unit axis for one farm."""
        xi = self._response("stress_ring", farm, n_fowt)
        return _stress_ring(_session_buffers(self), xi, self.dt["w"], fa, ss, angles, d, t, m, f_eq, method, weights, case_row0, col0,
                            psd, mean, wpow, self.batch.dw, tile_w)

    def eigen(self, A0=None, yawstiff=0.0, sort="dof", modes=True):
        """Natural frequencies and mode shapes of every design on the device, on torch's current stream (async):
        raftk_eigen_dev on M0 + A0 and C0 + yawstiff e5 e5^T from the resident tables (FOWT.solveEigen, raft_fowt.py:1646-1729).
        ``A0`` [6,6] or [nD,6,6]: the BEM added mass at the grid's first bin (A_BEM[:, :, 0]), None for none -- the resident
        A_w cannot stand in for it, it also holds the aero added mass; ``yawstiff`` scalar or [nD].  -> dict(lam [nD,6],
        fns [nD,6] = sqrt(lam) / 2 pi, modes [nD,6,6] or None) complex, info [nD] int32 (RAFTK_EIG_* flags), torch tensors;
        ``sort`` as ``solve_eigen``."""
        nD = self.batch.n_designs
        return _session_eigen(self, self.dt["M0"].view(nD, 6, 6), self.dt["C0"].view(nD, 6, 6), A0, yawstiff, sort, modes)

    def second_order_force(self):
        """Enqueue FOWT.calcHydroForce_2ndOrd for all units -> out['F_2nd'], out['F_2nd_mean'] (async)."""
        with self.torch.cuda.device(self.device):
            check(lib.raftk_second_order_force_dev(C.byref(self.d_struct), C.byref(self.c_struct), C.byref(self.o_struct),
                                                   self._stream()))
        return self.out

    def excitation(self):
        with self.torch.cuda.device(self.device):
            check(lib.raftk_hydro_excitation_dev(C.byref(self.d_struct), C.byref(self.c_struct), C.byref(self.o_struct),
                                                 self.workspace.data_ptr(), self.workspace_bytes, self._stream()))
        return self.out

    def linearization(self, Xi):
        """Xi: complex128 torch tensor [nD,nC,6,nw] on the session's device (after ``excitation``)."""
        with self.torch.cuda.device(self.device):
            check(lib.raftk_hydro_linearization_dev(C.byref(self.d_struct), C.byref(self.c_struct), Xi.data_ptr(),
                                                    C.byref(self.o_struct), self.workspace.data_ptr(),
                                                    self.workspace_bytes, self._stream()))
        return self.out


def launch_count():
    return int(lib.raftk_launch_count())


DISPATCH_FAMILIES = ("none", "solve", "qtf", "general", "farm", "system", "eigen")          # include/raftk.h RAFTK_FAMILY_*
DISPATCH_KERNELS = ("none", "v1", "fused128", "fused256", "fused2-cluster", "fused2-grid", "qtf-tiles", "qtf-diag", "qtf-diag-mix",
                    "gen-blocked", "gen-unblocked", "farm-rows12", "farm-warp", "farm-block", "sys-unblocked", "sys-blocked",
                    "farm-global", "sys-global", "eig-small", "eig-cta-smem", "eig-cta-slab")   # RAFTK_KERNEL_*


def last_dispatch():
    """The kernel variant the last library call on this thread launched (raftk_last_dispatch) -> dict(family, kernel,
    cluster_size, bins_per_cta, threads_per_cta, f0_global, direct_d2h, trains, chunks); family / kernel as names."""
    r = _lib.RaftkDispatch()
    check(lib.raftk_last_dispatch(C.byref(r)))
    d = {n: int(getattr(r, n)) for n, _ in r._fields_ if not n.startswith("_")}
    d["family"], d["kernel"] = DISPATCH_FAMILIES[d["family"]], DISPATCH_KERNELS[d["kernel"]]
    d["farm_classes"] = tuple(DISPATCH_KERNELS[k] for k in range(len(DISPATCH_KERNELS)) if d["farm_classes"] >> k & 1)
    for n in ("f0_global", "direct_d2h", "trains"):
        d[n] = bool(d[n])
    return d


def fp64_peak_gflops(iters=20000):
    return float(lib.raftk_fp64_peak_gflops(int(iters)))


def profile_enable(on=True):
    lib.raftk_profile_enable(1 if on else 0)


def profile_read():
    """-> (ms[3], launches[3]) device time of the depth-table, excitation and drag-solve kernels of the last call."""
    ms = (C.c_double * 3)()
    n = (C.c_int * 3)()
    check(lib.raftk_profile_read(ms, n))
    return list(ms), list(n)
