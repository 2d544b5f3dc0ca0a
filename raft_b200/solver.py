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
from ._lib import (RaftkCases, RaftkDesigns, RaftkFarm, RaftkGeneral, RaftkGeneralFd, RaftkGeneralQtf, RaftkOutputs, RaftkSlender, RaftkSlenderBatch,
                   RaftkSlenderOutputs, RaftkSolveOpts, check, lib)

_F8 = np.float64
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
        a["w"], a["k"] = self.w, self.k
        self.n_members_total = int(member_offset[-1])
        self.n_nodes_total = int(mem_node_start[-1])
        self.max_nodes = max(1, max_nodes)
        self.max_members = max(1, max_members)
        self.max_w_classes, self.max_h_classes, self.max_z_classes = self._step_classes(packed)

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
        self.n_members_total = int(a["member_offset"][-1])
        self.n_nodes_total = int(a["mem_node_start"][-1])
        self.max_nodes, self.max_members = int(max_nodes), int(max_members)
        self.max_w_classes, self.max_h_classes, self.max_z_classes = (int(c) for c in classes)
        return self

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
        s.depth, s.rho, s.g, s.dw = self.depth, self.rho, self.g, self.dw
        for name in ("w", "k", "member_offset", "mem_frame", "mem_rA", "mem_arm", "mem_node_start", "mem_circ",
                     "node_ls", "node_cd_q", "node_cd_p1", "node_cd_p2", "node_in_q", "node_in_p1", "node_in_p2",
                     "node_pa", "node_in_p1_w", "node_in_p2_w", "M0", "B0", "C0", "A_w", "B_w",
                     "bem_headings", "X_BEM", "bem_xyh", "qtf_w", "qtf_heads", "qtf"):
            setattr(s, name, ptr(name) if name in self.arrays else None)
        s.n_bem_head = self.n_bem_head
        s.n_qtf_w, s.n_qtf_head, s.qtf_shared = self.n_qtf_w, self.n_qtf_head, self.qtf_shared
        return s


class CaseTable:
    """SoA case table (``packer.pack_cases`` dict, or keyword arrays)."""

    def __init__(self, cases, zeta=None, F_2nd=None, Xi_init=None):
        """``F_2nd``: optional real [nD,nC,6,nw] second-order force amplitudes added to the linear excitation.
        ``Xi_init``: optional complex [nD,nC,6,nw] starting iterate of the fixed-point loop (instead of xi_start)."""
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

    def input_bytes(self):
        return int(sum(v.nbytes for v in self.arrays.values()))

    def struct(self, ptr):
        s = RaftkCases()
        s.n_cases = self.n_cases
        for name in ("Hs", "Tp", "gamma", "beta_deg", "spec", "zeta", "primary", "F_2nd", "Xi_init"):
            setattr(s, name, ptr(name) if name in self.arrays else None)
        return s


def _host_ptr(arrays):
    return lambda name: arrays[name].ctypes.data


def _alloc_outputs(nD, nC, nw, want, alloc=np.zeros):
    shapes = dict(Xi=([nD, nC, 6, nw], np.complex128), status=([nD, nC, 4], _I4), B_drag=([nD, nC, 6, 6], _F8),
                  F_drag=([nD, nC, 6, nw], np.complex128), F_iner=([nD, nC, 6, nw], np.complex128),
                  F_BEM=([nD, nC, 6, nw], np.complex128), zeta=([nC, nw], _F8),
                  F_2nd=([nD, nC, 6, nw], _F8), F_2nd_mean=([nD, nC, 6], _F8), Xi_last=([nD, nC, 6, nw], np.complex128))
    return {k: alloc(shapes[k][0], dtype=shapes[k][1]) for k in want}


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
    d = _host_struct(batch)
    c = _host_struct(cases)
    o = RaftkSolveOpts(int(n_iter), int(cluster_size), float(tol), float(xi_start), 0, 0)
    os_ = _out_struct(outs, lambda a: a.ctypes.data)
    check(lib.raftk_solve_dynamics_host(C.byref(d), C.byref(c), C.byref(o), C.byref(os_)))
    if _plan_overflowed(outs):
        check(lib.raftk_solve_dynamics_host(C.byref(_host_struct(worst_case_hints(batch))), C.byref(c), C.byref(o), C.byref(os_)))
        _raise_on_plan(outs)
    return outs


def _plan_overflowed(outs):
    """Whether a unit came back with RAFTK_FLAG_PLAN: the batch's step-class hints were below the number of classes the
    kernels count (DesignBatch computes them by the kernels' rule, so only hints set by the caller can be), and those
    units ran no pass and hold zeros."""
    return bool(np.any(np.asarray(outs["status"])[..., 2] & FLAG_PLAN))


def worst_case_hints(batch):
    """A shallow copy of ``batch`` with the step-class hints at 0: the fused solvers then size their class tables for one
    class per node, which cannot overflow.  ``batch`` keeps its hints."""
    b = copy.copy(batch)
    b.max_w_classes = b.max_h_classes = b.max_z_classes = 0
    b.__dict__.pop("_host_struct_cache", None)
    return b


def _raise_on_plan(outs):
    if _plan_overflowed(outs):
        raise _lib.RaftkError("step-class tables overflowed even with worst-case sizes")


def solve_dynamics_farm(batch, cases, C_arr=None, M_arr=None, B_arr=None, n_iter=10, tol=0.01, xi_start=0.0, cluster_size=0,
                        want=("Xi", "status", "B_drag"), out=None):
    """Coupled farm response (raft_model.py:1164-1236), host buffers in/out, ONE call: the designs of ``batch`` are the N
    FOWTs of the array; every FOWT's drag linearisation runs as in ``solve_dynamics``, then the 6N x 6N system
    blockdiag(Z_i) + (-w^2 M_arr + i w B_arr + C_arr) is assembled and solved per (case, frequency) on the device.
    -> the per-FOWT output dict plus ``Xi_sys`` complex [nC, 6N, nw] and ``info`` [nC, nw] (k+1 of a zero pivot).
    ``out``: caller-owned result arrays (e.g. page-locked ones from ``pinned_empty``: device-to-host copies then run at
    the link rate instead of through the driver's staging of pageable memory); missing ones are allocated."""
    N, nC, nw = batch.n_designs, cases.n_cases, batch.nw
    n = 6 * N
    want = tuple(dict.fromkeys(tuple(want) + ("Xi", "status")))
    outs = dict(out) if out is not None else {}
    for k_, v in _alloc_outputs(N, nC, nw, tuple(k for k in want if k not in outs)).items():
        outs[k_] = v
    mats = {}
    for nm, v in (("M_arr", M_arr), ("B_arr", B_arr), ("C_arr", C_arr)):
        if v is not None:
            a = np.ascontiguousarray(v, dtype=_F8)
            if a.shape != (n, n):
                raise ValueError("%s must be [%d, %d]" % (nm, n, n))
            mats[nm] = a
    if "Xi_sys" not in outs:
        outs["Xi_sys"] = np.zeros([nC, n, nw], dtype=np.complex128)
    if "info" not in outs:
        outs["info"] = np.zeros([nC, nw], dtype=_I4)
    if outs["Xi_sys"].shape != (nC, n, nw) or outs["Xi_sys"].dtype != np.complex128 or not outs["Xi_sys"].flags.c_contiguous:
        raise ValueError("out['Xi_sys'] must be a C-contiguous complex128 array [%d, %d, %d]" % (nC, n, nw))
    f = RaftkFarm()
    f.n_fowt = N
    for nm in ("M_arr", "B_arr", "C_arr"):
        setattr(f, nm, mats[nm].ctypes.data if nm in mats else None)
    f.Xi_sys, f.info = outs["Xi_sys"].ctypes.data, outs["info"].ctypes.data
    d = _host_struct(batch)
    c = _host_struct(cases)
    o = RaftkSolveOpts(int(n_iter), int(cluster_size), float(tol), float(xi_start), 0, 0)
    os_ = _out_struct(outs, lambda a: a.ctypes.data)
    check(lib.raftk_solve_dynamics_farm_host(C.byref(d), C.byref(c), C.byref(o), C.byref(os_), C.byref(f)))
    if _plan_overflowed(outs):                      # Xi_sys was assembled from those units' zero loads: solve it all again
        check(lib.raftk_solve_dynamics_farm_host(C.byref(_host_struct(worst_case_hints(batch))), C.byref(c), C.byref(o), C.byref(os_), C.byref(f)))
        _raise_on_plan(outs)
    return outs


FLAG_NAN, FLAG_SINGULAR, FLAG_PLAN, FLAG_XCHG = 1, 2, 4, 8        # include/raftk.h RAFTK_FLAG_*
STEP_RTOL, STEP_ZERO, Z0_RTOL = 5e-14, 1e-14, 1e-12                # step-class tolerances (csrc/raftk_common.cuh)


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
    d = batch.struct(_host_ptr(batch.arrays))
    c = cases.struct(_host_ptr(cases.arrays))
    os_ = _out_struct(outs, lambda a: a.ctypes.data)
    check(lib.raftk_hydro_excitation_host(C.byref(d), C.byref(c), C.byref(os_)))
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
    return batch, sb, CaseTable(base, zeta=base.get("zeta"))


def _slender_shapes(nD, nC, nw, nw2):
    return dict(Xi=([nD, nC, 6, nw], "c"), status=([nD, nC, 4], "i"), B_drag=([nD, nC, 6, 6], "f"), F_drag=([nD, nC, 6, nw], "c"),
                F_iner=([nD, nC, 6, nw], "c"), F_BEM=([nD, nC, 6, nw], "c"), zeta=([nC, nw], "f"), F_2nd=([nD, nC, 6, nw], "f"),
                F_2nd_mean=([nD, nC, 6], "f"), Xi_last=([nD, nC, 6, nw], "c"), qtf=([nD, nC, nw2, nw2, 6], "c"), Xi_rao=([nD, nC, 6, nw2], "c"))


def _slender_want(want, shapes):
    want = tuple(dict.fromkeys(("Xi", "status") + tuple(want)))
    bad = [k for k in want if k not in shapes]
    if bad:
        raise ValueError("unknown outputs %s (known: %s)" % (bad, ", ".join(shapes)))
    return want


def slender_flow_host(packed, cases, n_iter=10, tol=0.01, xi_start=0.0, cluster_size=0, want=("Xi", "status", "B_drag"), qtf_chunk=0):
    """``solve_dynamics_slender`` in ONE library call (raftk_solve_dynamics_slender_host: the whole flow on the device, host
    buffers in and out) -> dict of NumPy arrays named as in ``want`` (``SlenderSession``'s names)."""
    batch, sb, ct = _slender_inputs(packed, cases)
    if n_iter < 1:
        raise ValueError("potSecOrder 1 needs nIter >= 1")
    shapes = _slender_shapes(batch.n_designs, ct.n_cases, batch.nw, sb.nw2)
    want = _slender_want(want, shapes)
    dt = dict(c=np.complex128, i=_I4, f=_F8)
    outs = {k: np.zeros(shapes[k][0], dtype=dt[shapes[k][1]]) for k in want}
    so = RaftkSlenderOutputs(outs["qtf"].ctypes.data if "qtf" in outs else None, outs["Xi_rao"].ctypes.data if "Xi_rao" in outs else None,
                             int(qtf_chunk), 0)
    o = RaftkSolveOpts(int(n_iter), int(cluster_size), float(tol), float(xi_start), 0, 0)
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
        shapes = _slender_shapes(batch.n_designs, ct.n_cases, batch.nw, sb.nw2)
        self.want = want = _slender_want(want, shapes)
        self.dev = DeviceSession(batch, ct, device=device, workspace_bytes=0,
                                 want=tuple(k for k in want if k not in ("Xi_last", "qtf", "Xi_rao")))
        self.device, self.batch, self.slender = self.dev.device, batch, sb
        self.d_struct, self.c_struct = self.dev.d_struct, self.dev.c_struct
        dt = dict(c=torch.complex128, i=torch.int32, f=torch.float64)
        with torch.cuda.device(self.device):
            self.st = {k: torch.from_numpy(v).to(self.device) for k, v in sb.arrays.items()}
            self.s_struct = sb.struct(lambda name: self.st[name].data_ptr())
            self.out = dict(self.dev.out)
            for k in ("Xi_last", "qtf", "Xi_rao"):
                if k in want:
                    self.out[k] = torch.zeros(shapes[k][0], dtype=dt[shapes[k][1]], device=self.device)
            self.o_struct = _out_struct(self.out, lambda t: t.data_ptr())
            ptr = lambda k: self.out[k].data_ptr() if k in self.out else None   # noqa: E731
            self.so = RaftkSlenderOutputs(ptr("qtf"), ptr("Xi_rao"), int(qtf_chunk), 0)
            self.workspace_bytes = int(lib.raftk_solve_dynamics_slender_workspace_bytes(C.byref(self.d_struct), C.byref(self.s_struct),
                                                                                         ct.n_cases, int(qtf_chunk)))
            self.workspace = torch.empty(self.workspace_bytes, dtype=torch.uint8, device=self.device)
        self.qtf_chunk = int(qtf_chunk)

    def solve(self, n_iter=10, tol=0.01, xi_start=0.0, cluster_size=0):
        """Enqueue the potSecOrder 1 solve of every unit on the current stream; returns the output dict (async)."""
        if n_iter < 1:
            raise ValueError("potSecOrder 1 needs nIter >= 1")
        o = RaftkSolveOpts(int(n_iter), int(cluster_size), float(tol), float(xi_start), 0, 0)
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
    if "primary" in cases.arrays:
        raise NotImplementedError("potSecOrder 1 with several wave trains fails in the reference itself (raft_model.py:1229 rebinds Fhydro_2nd)")
    if n_iter < 1:
        raise ValueError("potSecOrder 1 needs nIter >= 1")
    plain = [{k: v for k, v in P.items() if not k.startswith(("qtf", "qs_"))} for P in packed]
    batch = DesignBatch(plain)
    nD, nC, nw = batch.n_designs, cases.n_cases, batch.nw
    base = {k: v for k, v in cases.arrays.items() if k not in ("F_2nd", "Xi_init")}
    wantA = tuple(dict.fromkeys(tuple(want) + ("Xi", "status", "zeta", "Xi_last")))
    A = solve_dynamics(batch, CaseTable(base, zeta=base.get("zeta")), n_iter=n_iter, tol=tol, xi_start=xi_start, cluster_size=cluster_size, want=wantA)
    qw = np.ascontiguousarray(packed[0]["qs_w"], dtype=_F8)
    beta_rad = cases.arrays["beta_deg"] * 0.017453292519943295
    qtf = np.zeros([nD, nC, len(qw), len(qw), 6], dtype=np.complex128)
    for d, P in enumerate(packed):
        if not np.array_equal(P["qs_w"], qw):
            raise ValueError("all designs of a batch must share the second-order frequency grid")
        Xi2 = np.zeros([nC, 6, len(qw)], dtype=np.complex128)
        for c in range(nC):
            r = get_rao(A["Xi"][d, c], A["zeta"][c])
            for a in range(6):
                Xi2[c, a] = np.interp(qw, batch.w, r[a], left=0, right=0)          # raft_fowt.py:2021-2023
        qtf[d] = qtf_slender(P, beta_rad, Xi2)
    qb = DesignBatch(plain)
    qb.arrays["qtf_w"], qb.arrays["qtf_heads"] = qw, np.zeros(1)
    qb.arrays["qtf"] = np.ascontiguousarray(qtf.reshape(nD, nC, len(qw), len(qw), 1, 6))
    qb.n_qtf_w, qb.n_qtf_head, qb.qtf_shared = len(qw), 1, 2
    F2 = second_order_force(qb, CaseTable(base, zeta=base.get("zeta")))
    B = solve_dynamics(batch, CaseTable(base, zeta=base.get("zeta"), F_2nd=F2["F_2nd"], Xi_init=A["Xi_last"]), n_iter=n_iter - 1, tol=tol,
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


class GeneralSession:
    """Generalised-DOF solve with tables, workspace and outputs resident in HBM (torch tensors), kernels on torch's current
    stream: ``solve()`` enqueues raftk_general_solve_dynamics_dev -> (Xi [nT,nDOF,nw] complex, status [nT,4]); ``cases`` may
    carry wave trains (``packer.pack_case_trains``).  ``stats(R, wpow)`` reduces the device Xi to output-channel statistics
    on the device (raftk_general_channel_stats_dev), so the responses never leave HBM.  ``fd``: frequency-dependent added
    mass, damping and BEM excitation (``packer.pack_general_matrices``); with ``F_BEM=True`` ``solve()`` also returns the BEM
    excitation in reduced DOFs, complex [nT,nDOF,nw].  ``qtf``: second-order wave loads (``packer.pack_general_qtf``); every
    ``solve()`` then leaves the force of every case and train in the device tensors ``F_2nd`` [nT,6,nw] and ``F_2nd_mean``
    [nT,6] (reduced DOFs 0-5)."""

    def __init__(self, P, M, B, Cm, cases, device=None, fd=None, F_BEM=False, qtf=None):
        import torch
        self.torch = torch
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.keep = {}

        def to_dev(name, a):
            t = torch.from_numpy(a.view(np.float64) if a.dtype == np.complex128 else a).to(self.device)
            self.keep[name] = t
            return t.data_ptr()
        with torch.cuda.device(self.device):
            self.g = _general_struct(P, M, B, Cm, to_dev)
            self.ct = {k: torch.from_numpy(v).to(self.device) for k, v in cases.arrays.items()}
            self.c_struct = cases.struct(lambda name: self.ct[name].data_ptr())
            n, nw, nC = int(P["gen_nDOF"]), len(P["w"]), cases.n_cases
            self.fd = _general_fd_struct(fd, n, nw, to_dev)
            self.qtf = _general_qtf_struct(qtf, to_dev)
            fdp = C.byref(self.fd) if self.fd is not None else None
            qp = C.byref(self.qtf) if self.qtf is not None else None
            self.workspace_bytes = int(lib.raftk_general_qtf_workspace_bytes(C.byref(self.g), fdp, qp, nC))
            self.workspace = torch.empty(self.workspace_bytes, dtype=torch.uint8, device=self.device)
            self.Xi = torch.zeros([nC, n, nw], dtype=torch.complex128, device=self.device)
            self.status = torch.zeros([nC, 4], dtype=torch.int32, device=self.device)
            self.F_BEM = torch.zeros([nC, n, nw], dtype=torch.complex128, device=self.device) if F_BEM else None
            self.F_2nd = torch.zeros([nC, 6, nw], dtype=torch.float64, device=self.device) if self.qtf is not None else None
            self.F_2nd_mean = torch.zeros([nC, 6], dtype=torch.float64, device=self.device) if self.qtf is not None else None
        self.n, self.nw, self.n_cases, self.dw = n, nw, nC, float(P["dw"])
        self._ch = None

    def solve(self, n_iter=10, tol=0.01, xi_start=0.0):
        o = RaftkSolveOpts(int(n_iter), 0, float(tol), float(xi_start), 0, 0)
        ptr = lambda t: t.data_ptr() if t is not None else None   # noqa: E731
        with self.torch.cuda.device(self.device):
            check(lib.raftk_general_solve_dynamics_qtf_dev(C.byref(self.g), C.byref(self.fd) if self.fd is not None else None,
                                                           C.byref(self.qtf) if self.qtf is not None else None, C.byref(self.c_struct),
                                                           C.byref(o), self.Xi.data_ptr(), self.status.data_ptr(), ptr(self.F_BEM),
                                                           ptr(self.F_2nd), ptr(self.F_2nd_mean), self.workspace.data_ptr(),
                                                           self.workspace_bytes, self.torch.cuda.current_stream(self.device).cuda_stream))
        return (self.Xi, self.status) if self.F_BEM is None else (self.Xi, self.status, self.F_BEM)

    def stats(self, R, wpow, psd=True, amp=False):
        """Output-channel statistics of the last ``solve()`` (``packer.pack_general_channels``: R [nch,nDOF], wpow [nch]) on
        the device -> (std [nT,nch], PSD [nT,nch,nw] or None, amplitudes complex [nT,nch,nw] or None), torch tensors."""
        torch = self.torch
        R = np.ascontiguousarray(R, dtype=_F8)
        wpow = np.ascontiguousarray(wpow, dtype=_I4)
        if R.ndim != 2 or R.shape[1] != self.n or wpow.shape != (R.shape[0],):
            raise ValueError("R must be [nch, %d] and wpow [nch]" % self.n)
        _check_wpow(wpow)
        nch = R.shape[0]
        with torch.cuda.device(self.device):
            if self._ch is None or not (np.array_equal(self._ch[0], R) and np.array_equal(self._ch[1], wpow)):
                self._ch = (R, wpow, torch.from_numpy(R).to(self.device), torch.from_numpy(wpow).to(self.device))
            dR, dp = self._ch[2], self._ch[3]
            sd = torch.empty([self.n_cases, nch], dtype=torch.float64, device=self.device)
            P = torch.empty([self.n_cases, nch, self.nw], dtype=torch.float64, device=self.device) if psd else None
            A = torch.empty([self.n_cases, nch, self.nw], dtype=torch.complex128, device=self.device) if amp else None
            check(lib.raftk_general_channel_stats_dev(self.n_cases, self.n, nch, self.nw, self.dw, self.keep["w"].data_ptr(), dR.data_ptr(),
                                                      dp.data_ptr(), self.Xi.data_ptr(), sd.data_ptr(), P.data_ptr() if psd else None,
                                                      A.data_ptr() if amp else None, torch.cuda.current_stream(self.device).cuda_stream))
        return sd, P, A


def general_solve_dynamics(P, M, B, Cm, cases, n_iter=10, tol=0.01, xi_start=0.0, fd=None, F_BEM=False, qtf=None, F_2nd=False):
    """Model.solveDynamics for one FOWT with generalised degrees of freedom (flexible members), host buffers:
    ``P`` from ``packer.pack_general_dofs`` (node tables + ``gen_Tn``, ``gen_rr``), constant system
    matrices ``M, B, Cm`` [nDOF,nDOF], ``cases`` a CaseTable, with wave trains when built from ``packer.pack_case_trains``
    (train 0 of a case drives the linearisation, raft_model.py:1200-1236) -> (Xi complex [nT,nDOF,nw], status [nT,4]).
    ``fd``: frequency-dependent added mass and damping (operating rotors, BEM coefficients) and BEM excitation, the ``fd``
    dict of ``packer.pack_general_matrices`` (whose M, B, C are then the constant matrices).  ``F_BEM=True`` appends the BEM
    excitation of every case and train in reduced DOFs, complex [nT,nDOF,nw], to the result.  ``qtf``: second-order wave
    loads (potSecOrder 2), the dict of ``packer.pack_general_qtf``; ``F_2nd=True`` (with ``qtf``) then appends the force of
    every case and train on reduced DOFs 0-5, F_2nd [nT,6,nw] and F_2nd_mean [nT,6]."""
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
    nC = cases.n_cases
    Xi = np.zeros([nC, n, nw], dtype=np.complex128)
    st = np.zeros([nC, 4], dtype=_I4)
    Fb = np.zeros([nC, n, nw], dtype=np.complex128) if F_BEM else None
    F2, F2m = (np.zeros([nC, 6, nw]), np.zeros([nC, 6])) if F_2nd else (None, None)
    c = cases.struct(_host_ptr(cases.arrays))
    o = RaftkSolveOpts(int(n_iter), 0, float(tol), float(xi_start), 0, 0)
    hp = lambda a: a.ctypes.data if a is not None else None   # noqa: E731
    check(lib.raftk_general_solve_dynamics_qtf_host(C.byref(g), C.byref(f) if f is not None else None, C.byref(q) if q is not None else None,
                                                    C.byref(c), C.byref(o), Xi.ctypes.data, st.ctypes.data, hp(Fb), hp(F2), hp(F2m)))
    return (Xi, st) + ((Fb,) if F_BEM else ()) + ((F2, F2m) if F_2nd else ())


def combine_trains(std, psd, idx):
    """helpers.getRMS / getPSD of a case with several wave trains (helpers.py:678-700) from per-train reductions ``std``
    [nT,...] and ``psd`` [nT,...,nw]: the squares sum over the trains ``idx`` -> (sqrt(sum std^2), sum PSD)."""
    return np.sqrt((std[idx] ** 2).sum(axis=0)), psd[idx].sum(axis=0)


def _check_wpow(wpow):
    if wpow.size and (wpow.min() < 0 or wpow.max() > 2):
        raise ValueError("wpow must be 0, 1 or 2 (displacement, velocity, acceleration)")


def general_channel_stats(R, wpow, w, Xi, dw, psd=True, amp=False):
    """Output channels of a FOWT with generalised DOFs, Y = w^wpow R Xi (``packer.pack_general_channels``), host buffers:
    R [nch,nDOF], wpow [nch] 0, 1 or 2, w [nw], Xi complex [nU,nDOF,nw] -> (std [nU,nch], PSD [nU,nch,nw] or None,
    amplitudes complex [nU,nch,nw] or None)."""
    R = np.ascontiguousarray(R, dtype=_F8)
    wpow = np.ascontiguousarray(wpow, dtype=_I4)
    w = np.ascontiguousarray(w, dtype=_F8)
    Xi = np.ascontiguousarray(Xi, dtype=np.complex128)
    nU, n, nw = Xi.shape
    nch = R.shape[0]
    if R.shape != (nch, n) or wpow.shape != (nch,) or w.shape != (nw,):
        raise ValueError("R must be [nch,nDOF], wpow [nch], w [nw] for Xi [nU,nDOF,nw]")
    _check_wpow(wpow)
    sd = np.zeros([nU, nch])
    P = np.zeros([nU, nch, nw]) if psd else None
    A = np.zeros([nU, nch, nw], dtype=np.complex128) if amp else None
    check(lib.raftk_general_channel_stats_host(nU, n, nch, nw, float(dw), w.ctypes.data, R.ctypes.data, wpow.ctypes.data, Xi.ctypes.data,
                                               sd.ctypes.data, P.ctypes.data if psd else None, A.ctypes.data if amp else None))
    return sd, P, A


def general_case_metrics(channels, std, psd, amp, idx):
    """The entries FOWT.saveTurbineOutputs stores for one case (raft_fowt.py:2299-2604) from per-train channel statistics
    (std [nT,nch], PSD [nT,nch,nw], amplitudes [nT,nch,nw]) of the case's trains ``idx``: ``*_avg/_std/_max/_min/_PSD`` of every
    channel, ``*_RA`` of the six PRP motions (all trains plus the zero row of Model.Xi), per-rotor channels as arrays
    [nrotors] / PSD [nw, nrotors], and the ``Mbase`` alias of a flexible tower's MbaseY (:2599-2604)."""
    sd, ps = combine_trains(std, psd, idx)
    names, avg = channels["names"], channels["avg"]
    nw = psd.shape[-1]
    nrot = 1 + max([ir for _, ir in names if ir is not None], default=-1)
    m = {}
    for k, (nm, ir) in enumerate(names):
        if ir is None:
            m[nm + "_avg"], m[nm + "_std"] = avg[k], sd[k]
            m[nm + "_max"], m[nm + "_min"] = avg[k] + 3 * sd[k], avg[k] - 3 * sd[k]
            m[nm + "_PSD"] = ps[k]
            ra = np.zeros([len(idx) + 1, nw], dtype=complex)
            ra[:-1] = amp[idx, k]
            m[nm + "_RA"] = ra
            continue
        for suffix in ("_avg", "_std", "_max", "_min"):
            m.setdefault(nm + suffix, np.zeros(nrot))
        m.setdefault(nm + "_PSD", np.zeros([nw, nrot]))
        m[nm + "_avg"][ir], m[nm + "_std"][ir] = avg[k], sd[k]
        m[nm + "_max"][ir], m[nm + "_min"][ir] = avg[k] + 3 * sd[k], avg[k] - 3 * sd[k]
        m[nm + "_PSD"][:, ir] = ps[k]
    if "MbaseY_std" in m:
        for suffix in ("_avg", "_std", "_max", "_min", "_PSD"):
            m["Mbase" + suffix] = m["MbaseY" + suffix].copy()
    return m


def general_analyze_cases(P, M, B, Cm, cases, channels=None, n_iter=10, tol=0.01, xi_start=0.0, fd=None, qtf=None):
    """Model.analyzeCases (dynamics and output statistics) for one FOWT with generalised degrees of freedom: ``cases`` a list
    of case dicts, scalar or list-valued wave keys (several wave trains); ``channels`` from ``packer.pack_general_channels``.
    -> dict(Xi_trains [per case: nTrains,nDOF,nw], status [nC,4] of train 0, case_metrics {case: saveTurbineOutputs entries},
    empty without channels).  ``fd``: frequency-dependent terms, as for ``general_solve_dynamics``.  ``qtf``: second-order
    wave loads (``packer.pack_general_qtf``); the result then also holds, per case, the reference FOWT's ``Fhydro_2nd``
    (complex [nTrains,nDOF,nw]) and ``Fhydro_2nd_mean`` ([nTrains,nDOF]), zero from reduced DOF 6 up (raft_model.py:1034-1036)."""
    from .packer import pack_case_trains
    table, owner, first = pack_case_trains(cases)
    q = bool(qtf)
    res = general_solve_dynamics(P, M, B, Cm, CaseTable(table), n_iter=n_iter, tol=tol, xi_start=xi_start, fd=fd, qtf=qtf, F_2nd=q)
    Xi, st = res[0], res[1]
    raise_on_flags(st[first])                                           # raft_model.py:1089, :1098-1099
    metrics = {}
    if channels is not None:
        sd, ps, amp = general_channel_stats(channels["R"], channels["wpow"], P["w"], Xi, float(P["dw"]), psd=True, amp=True)
        for ic in range(len(cases)):
            metrics[ic] = general_case_metrics(channels, sd, ps, amp, np.nonzero(owner == ic)[0])
    out = dict(Xi_trains=[Xi[owner == ic] for ic in range(len(cases))], status=st[first], case_metrics=metrics)
    if q:
        n, nw = Xi.shape[1], Xi.shape[2]
        F2, F2m = np.zeros([len(Xi), n, nw], dtype=np.complex128), np.zeros([len(Xi), n])
        F2[:, :6], F2m[:, :6] = res[2], res[3]
        out["Fhydro_2nd"] = [F2[owner == ic] for ic in range(len(cases))]
        out["Fhydro_2nd_mean"] = [F2m[owner == ic] for ic in range(len(cases))]
    return out


def second_order_force(batch, cases):
    """FOWT.calcHydroForce_2ndOrd (raft_fowt.py:2158-2253) for every (design, case) from the designs' QTF table,
    host buffers -> dict(F_2nd [nD,nC,6,nw] real amplitudes, F_2nd_mean [nD,nC,6])."""
    if batch.n_qtf_w == 0:
        raise ValueError("the designs carry no QTF table (potSecOrder 2 / packer.pack_qtf)")
    outs = _alloc_outputs(batch.n_designs, cases.n_cases, batch.nw, ("F_2nd", "F_2nd_mean"))
    d = batch.struct(_host_ptr(batch.arrays))
    c = cases.struct(_host_ptr(cases.arrays))
    os_ = _out_struct(outs, lambda a: a.ctypes.data)
    check(lib.raftk_second_order_force_host(C.byref(d), C.byref(c), C.byref(os_)))
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
    d = batch.struct(_host_ptr(batch.arrays))
    c = cases.struct(_host_ptr(cases.arrays))
    os_ = _out_struct(outs, lambda a: a.ctypes.data)
    check(lib.raftk_hydro_linearization_host(C.byref(d), C.byref(c), Xi.ctypes.data, C.byref(os_)))
    return outs


def farm_workspace_bytes(n_fowt, n_cases, nw):
    """Device workspace the farm system response needs (raftk_farm_workspace_bytes): 0 while the [6N][6N+1] system fits in
    shared memory, else one slab per resident CTA of the global-memory kernel.  Answers for an H100 without a device."""
    d, c, f = RaftkDesigns(), RaftkCases(), RaftkFarm()
    d.n_designs, d.nw, c.n_cases, f.n_fowt = int(n_fowt), int(nw), int(n_cases), int(n_fowt)
    return int(lib.raftk_farm_workspace_bytes(C.byref(d), C.byref(c), C.byref(f)))


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
        import torch
        self.torch = torch
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.batch, self.cases = batch, cases
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
            nD, nC, nw = batch.n_designs, cases.n_cases, batch.nw
            want = tuple(dict.fromkeys(tuple(want) + ("Xi", "status") + (("F_2nd", "F_2nd_mean") if batch.n_qtf_w else ())))
            shapes = dict(Xi=([nD, nC, 6, nw], torch.complex128), status=([nD, nC, 4], torch.int32),
                          F_2nd=([nD, nC, 6, nw], torch.float64), F_2nd_mean=([nD, nC, 6], torch.float64),
                          B_drag=([nD, nC, 6, 6], torch.float64), F_drag=([nD, nC, 6, nw], torch.complex128),
                          F_iner=([nD, nC, 6, nw], torch.complex128), F_BEM=([nD, nC, 6, nw], torch.complex128),
                          zeta=([nC, nw], torch.float64))
            given = dict(out_tensors or {})
            for k, t in given.items():
                if tuple(t.shape) != tuple(shapes[k][0]) or t.dtype != shapes[k][1] or not t.is_contiguous():
                    raise ValueError("out_tensors[%r] must be a contiguous %s tensor of shape %s" % (k, shapes[k][1], shapes[k][0]))
            self.out = {k: (given[k] if k in given else torch.zeros(shapes[k][0], dtype=shapes[k][1], device=self.device)) for k in want}
            self.o_struct = _out_struct(self.out, lambda t: t.data_ptr())

    def _stream(self):
        return self.torch.cuda.current_stream(self.device).cuda_stream

    def _opts(self, n_iter, tol, xi_start, cluster_size):
        """Solve options; from the second call with the same cluster size on, the per-design plan blobs that the first call
        left in the session's workspace are reused (the session owns tables and workspace, so they cannot have changed)."""
        key = int(cluster_size)
        o = RaftkSolveOpts(int(n_iter), key, float(tol), float(xi_start), 1 if getattr(self, "_plan_key", None) == key else 0, 0)
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

    def farm_response(self, C_arr=None, M_arr=None, B_arr=None):
        """Enqueue the coupled 6N-DOF system response of the LAST ``solve`` (the session's designs are the FOWTs of the
        array; it must have been created with want including B_drag, F_drag, F_iner [+ F_BEM]).  -> (Xi_sys [nC,6N,nw], info).
        Any N: farms whose system does not fit in shared memory are solved in a device workspace sized once
        (raftk_farm_workspace_bytes) and kept with the session."""
        torch = self.torch
        N, nC, nw = self.batch.n_designs, self.cases.n_cases, self.batch.nw
        n = 6 * N
        if not hasattr(self, "_farm"):
            with torch.cuda.device(self.device):
                mats = {nm: (torch.from_numpy(np.ascontiguousarray(v, dtype=_F8)).to(self.device) if v is not None else None)
                        for nm, v in (("M_arr", M_arr), ("B_arr", B_arr), ("C_arr", C_arr))}
                xi = torch.zeros([nC, n, nw], dtype=torch.complex128, device=self.device)
                info = torch.zeros([nC, nw], dtype=torch.int32, device=self.device)
            f = RaftkFarm()
            f.n_fowt = N
            for nm, t in mats.items():
                setattr(f, nm, t.data_ptr() if t is not None else None)
            f.Xi_sys, f.info = xi.data_ptr(), info.data_ptr()
            wsb = int(lib.raftk_farm_workspace_bytes(C.byref(self.d_struct), C.byref(self.c_struct), C.byref(f)))
            with torch.cuda.device(self.device):
                ws = torch.empty(max(wsb, 1), dtype=torch.uint8, device=self.device)
            self._farm = (f, mats, xi, info, ws, wsb)
        f, _, xi, info, ws, wsb = self._farm
        with torch.cuda.device(self.device):
            check(lib.raftk_farm_response_ws_dev(C.byref(self.d_struct), C.byref(self.c_struct), C.byref(self.o_struct), C.byref(f),
                                                 ws.data_ptr(), wsb, self._stream()))
        return xi, info

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


DISPATCH_FAMILIES = ("none", "solve", "qtf", "general", "farm", "system")          # include/raftk.h RAFTK_FAMILY_*
DISPATCH_KERNELS = ("none", "v1", "fused128", "fused256", "fused2-cluster", "fused2-grid", "qtf-tiles", "qtf-diag", "qtf-diag-mix",
                    "gen-blocked", "gen-unblocked", "farm-rows12", "farm-warp", "farm-block", "sys-unblocked", "sys-blocked",
                    "farm-global", "sys-global")   # RAFTK_KERNEL_*


def last_dispatch():
    """The kernel variant the last library call on this thread launched (raftk_last_dispatch) -> dict(family, kernel,
    cluster_size, bins_per_cta, threads_per_cta, f0_global, direct_d2h, trains, chunks); family / kernel as names."""
    r = _lib.RaftkDispatch()
    check(lib.raftk_last_dispatch(C.byref(r)))
    d = {n: int(getattr(r, n)) for n, _ in r._fields_ if not n.startswith("_")}
    d["family"], d["kernel"] = DISPATCH_FAMILIES[d["family"]], DISPATCH_KERNELS[d["kernel"]]
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
