"""The rigid solvers' statistical drag linearisation and fixed-point loop (calcHydroLinearization + calcDragExcitation,
raft_fowt.py:1891-1957, raft_member.py:2071-2117, and the loop of raft_model.py:1081-1133) against a high-precision
reference, entry by entry and bin by bin, in every rigid kernel.

The reference restates the linearisation per node and per direction from the packed design's own tables (node_ls,
node_cd_*, mem_q/p1/p2, mem_rA, prp, mem_circ, w, k, depth), the case and the planted iterate, in double-double
arithmetic (error-free transforms, vectorised): the node arm r = (rA - prp) + ls q and V_d = [d; r x d] exactly, the body
velocity -i w V_d . Xi, the squared relative velocities summed over every bin, vRMS = sqrt(sum / 2) (circular members:
the total transverse RMS for both transverse directions), b_d = cd_d vRMS_d, B_drag = sum_nodes,d b_d V_d V_d^T and
F_drag(w) = sum_nodes,d b_d u_d(w) V_d.  The wave velocity u_d = zeta w E (C h_d + i S d_z) is the double-precision value
of the kernels' formula (the kinematics are pinned by test_wave_kinematics_edges.py); zeta is the solver's output.
Alongside every entry the reference carries a magnitude taken over the kernels' algorithm: the magnitude RMS
b~_d = cd_d sqrt(sum_w (|u_d| + w sum_a |V_d,a| |Xi_a|)^2 / 2) (what rounding inside the relative velocity can leave
behind where it cancels) in the factored member sums sum b~, sum b~ |ls|, sum b~ ls^2 (raftk_tables.cuh:437-464), so a
cancellation that the factored form itself causes is charged to the bound, not to the kernel.  Bounds:
  |B_kernel - B_ref|_ab <= C_B u M_ab entry by entry, and per bin and DOF group (0-2, 3-5)
  max_a |F_kernel - F_ref|_a <= C_F u max_a M_F,a, with u = 2^-53;
the fused kernels walk member nodes with step-factor recurrences, so with waves on they are held to C_B_WALK (1 + L) u M
and C_F_WALK (1 + L) u M instead, L the longest member walk in nodes; v1 evaluates every node's kinematics directly and
meets C_B, C_F with no walk term.

Planted inputs (cfg2 regridded per kernel, its tables edited; the reference needs no physical consistency):
  * direction masks by (chunk + slot) mod 4: axial only, transverse only, both, none, at slot jj = 0 and 9 of chunks
    and across chunk boundaries, on members longer than a chunk, Ns = 53 (not a multiple of CHUNK_NODES);
  * circular members next to rectangular ones, Cd_p2 = 1.7 Cd_p1 on the rectangular ones;
  * pontoon 5 re-based 2000 m from the reference point, its nodes shifted along it to within 21 m of the point (the
    same spacings, so the same step classes): the factored member sums of its yaw entry cancel by more than 1e3;
  * Xi_init in the null space of four (node, direction) velocity projections: the relative velocity of nodes 7 (both
    transverse, circular), 25 (axial, rectangular) and 48 (transverse 2, rectangular) cancels at every bin, so the
    reference vRMS there is ~1e-16 of the magnitude RMS;
  * bin amplitudes spanning 10 decades, the RMS dominated by a few bins in the last CTA's slice.
Family A: spec NONE (zero wave velocity: F_drag must be exactly 0).  Family B: JONSWAP and unit spectra at headings 0,
180, -180 and 37 deg.  Each fused kernel runs one pass from Xi_init (n_iter = 0); v1, which takes no Xi_init, runs
hydro_linearization (k_drag_solve mode 1).  Wave trains: a train table solved to convergence on every fused kernel that
takes trains; each primary against the reference linearised about its Xi_last, each secondary train's F_drag bin by bin
against the reference at its own zeta and heading with its primary's coefficients.

Scaling: Xi_init times 2^s at s = +-300 with spec NONE gives B_drag times 2^s bit for bit (exact while every nonzero
relative-velocity component keeps 2^-511 <= |v| < 2^512, so that its square stays normal: DESIGN.md section 6).

Fixed-point loop, spec NONE: the load is zero, so Xi is exactly 0 on every pass, the test |d| / (|x| + tol) < tol reads
|XiLast| < tol^2 and the next iterate is RN(0.2 XiLast).  Each case plants |Xi_init| <= tol^2 (1 - 1e-6) everywhere but
one (bin, DOF) at tol^2 5^k (1 -+ 1e-6): the unit must report k + 1 (k + 2) passes, capped at n_iter + 1, converged
accordingly, and Xi_last must be Xi_init relaxed passes - 1 times, bit for bit.  The planted entry sits at every DOF, at
the first and last bin of every CTA and at the ragged tail.  tol = 0.5, 0.01, 1e-6 and 1e-70 (RAFTK_TOL_MIN, the smallest
positive tol the entries accept); v1 takes the constant xi_start instead.  With a zero iterate (d = x = 0 at every bin)
every kernel converges on the first pass at tol = 1e-70 and never at tol = 0, as the reference does; a tol in
(0, 1e-70), negative or NaN is refused before any launch.

Heterogeneous batch: cfg2, the planted cfg2, cfg1 and a random design (7 / 7 / 1 / 3 members, 53 / 53 / 26 / 29 nodes,
different circular/rectangular mixes, drag masks and step classes) on one site and grid: every unit's outputs bit-identical to the
design launched alone on the same kernel and cluster size.

Without a GPU: the reference against 40-digit mpmath, the planted edges reached on each kernel's layout (the direction
masks, accumulator slots and reduction rounds of k_fused_plan's rule restated on the packed design), and three faults
modelled on the CPU (a dropped node, a swapped circular flag, the translational block off by 1e-9) that break the bounds
by more than 100x.

Measured on an H100 80GB HBM3 (700 W limit), over every test of this file: worst |dB| / (u M) = 1.88 and worst
|dF| / (u M) = 0.48 without the walk term (v1, and every kernel without waves), 0.16 (B) and 0.038 (F) against (1 + L) u M
in the fused kernels with waves; the bounds keep about 10x of margin.  The GPU part of the file runs in about 30 s.

Tiny tol exposed a defect, now fixed at the entries: k_rao_fused2 tested d.d < (tol (|x| + tol))^2, which underflows to
0 < 0 at d = x = 0 once tol^4 underflows (tol below about 1e-81), so a still-water unit never converged; k_rao_fused's
|d| < tol |x| + tol^2 did the same below about 1e-162; and every kernel's d.d (v1's and the generalised-DOF solve's
sqrt(d.d) too) underflows for |d| < 1e-154, where a tiny tol makes the decision differ from the reference's.  With
tol >= 1e-70 every square the decision depends on stays normal, so the solve entries refuse 0 < tol < 1e-70."""
import math

import numpy as np
import pytest

from test_dispatch_solve import CLUSTER, FORCE, GRID, SHAPES, _check_record, _design, _train_table
from test_farm_edges import _two_prod

gpu = pytest.mark.gpu
U = 2.0 ** -53
C_B = 20.0                   # |dB| <= C_B u M_B
C_F = 5.0                    # |dF| <= C_F u M_F (per bin and DOF group)
C_B_WALK = 2.0               # with waves on, the fused kernels: |dB| <= C_B_WALK (1 + L) u M_B
C_F_WALK = 0.4               # and |dF| <= C_F_WALK (1 + L) u M_F
TOLS = (0.5, 0.01, 1e-6, 1e-70)                       # 1e-70: RAFTK_TOL_MIN, the smallest positive tol the entries accept
CHUNK = 10                   # CHUNK_NODES (raftk_common.cuh)
SPEC_JONSWAP, SPEC_UNIT, SPEC_NONE = 0, 1, 3
FAR_MEMBER, FAR_ARM = 5, 2000.0
CANCEL = [(7, 1), (7, 2), (25, 0), (48, 2)]          # (node, direction 0 = q, 1 = p1, 2 = p2) whose velocity cancels
NEED_MASK = {7: 2, 25: 1, 48: 2}                       # mask bits those nodes need: 1 = axial, 2 = transverse

# (design, nw, cluster_size, environment, kernel, f0_global): the first cfg2 shape of test_dispatch_solve.SHAPES for each
# variant, and its forced-v1 shapes at 333 bins
KID = ["fused128", "fused256", "fused256-f0g", "fused2-cluster", "fused2-grid", "v1"]
_VARIANTS = [("fused128", False, {}), ("fused256", False, {}), ("fused256", True, {}), ("fused2-cluster", False, CLUSTER),
             ("fused2-grid", False, GRID), ("v1", False, {})]
KERNELS = [next(s for s in SHAPES if s[0] == "cfg2" and s[4] == k and s[5] == f and s[3] == env) for k, f, env in _VARIANTS]
V1_FORCED = [s for s in SHAPES if s[0] == "cfg2" and s[3] == FORCE and s[1] == 333]
assert [s[2] for s in V1_FORCED] == [1, 2, 4, 8]
LOOP = KERNELS + V1_FORCED
LID = KID + ["v1-forced-cs%d" % cs for cs in (1, 2, 4, 8)]

SEA = dict(Hs=np.array([0.0, 6.0, 0.0, 3.0, 9.0]), Tp=np.array([10.0, 12.0, 10.0, 8.0, 15.0]), gamma=np.zeros(5),
           beta_deg=np.array([0.0, 0.0, 180.0, -180.0, 37.0]),
           spec=np.array([SPEC_NONE, SPEC_JONSWAP, SPEC_UNIT, SPEC_JONSWAP, SPEC_JONSWAP], dtype=np.int32))


# ---- double-double arithmetic (pairs (hi, lo) of arrays) -----------------------------------------------------------
def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _norm(s, e):
    hi = s + e
    return hi, e - (hi - s)


def _dd(a):
    a = np.asarray(a, dtype=float)
    return a, np.zeros_like(a)


def _add(x, y):
    s, e = _two_sum(x[0], y[0])
    return _norm(s, e + (x[1] + y[1]))


def _mul(x, y):
    p, e = _two_prod(x[0], y[0])
    return _norm(p, e + (x[0] * y[1] + x[1] * y[0]))


def _neg(x):
    return -x[0], -x[1]


def _sum(x, axis):
    """Sequential double-double sum along ``axis``."""
    hi, lo = np.moveaxis(x[0], axis, 0), np.moveaxis(x[1], axis, 0)
    acc = (np.zeros_like(hi[0]), np.zeros_like(hi[0]))
    for t in range(hi.shape[0]):
        acc = _add(acc, (hi[t], lo[t]))
    return acc


def _sqrt(x):
    h = np.sqrt(x[0])
    p, e = _two_prod(h, h)
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.where(h > 0, (((x[0] - p) - e) + x[1]) / (2.0 * np.where(h > 0, h, 1.0)), 0.0)
    return _norm(h, r)


def _cross(a, b):
    """a x b, a double-double [.., 3], b double [.., 3]."""
    out = []
    for i, j in ((1, 2), (2, 0), (0, 1)):
        out.append(_add(_mul((a[0][..., i], a[1][..., i]), _dd(b[..., j])), _neg(_mul((a[0][..., j], a[1][..., j]), _dd(b[..., i])))))
    return np.stack([o[0] for o in out], -1), np.stack([o[1] for o in out], -1)


# ---- the reference --------------------------------------------------------------------------------------------------
def _nodes(P):
    """Per node: member index, ls, frame rows (q, p1, p2) [Ns, 3, 3], arm rA - prp (double-double), circ flag."""
    ms = np.asarray(P["mem_start"])
    mem = np.repeat(np.arange(len(ms) - 1), np.diff(ms))
    fr = np.stack([np.asarray(P[k], dtype=float) for k in ("mem_q", "mem_p1", "mem_p2")], 1)[mem]
    rA = np.asarray(P["mem_rA"], dtype=float)[mem]
    arm = _two_sum(rA, -np.asarray(P["prp"], dtype=float)[None, :])
    return mem, np.asarray(P["node_ls"], dtype=float), fr, arm, np.asarray(P["mem_circ"])[mem] != 0


def _depth(k, h, z):
    """depth_funcs (raftk_common.cuh) -> S, C."""
    k = np.asarray(k, dtype=float)
    with np.errstate(over="ignore", invalid="ignore"):
        deep = k * h > 89.4
        sh = np.sinh(np.where(deep, 1.0, k * h))
        S = np.where(deep, np.exp(k * z), np.sinh(k * (z + h)) / sh)
        C = np.where(deep, np.exp(k * z), np.cosh(k * (z + h)) / sh)
    return S, C


def _wave(P, zeta, beta_deg):
    """Wave velocity along q, p1, p2 at every node and bin, the kernels' formula in double: [3, Ns, nw] complex."""
    _, ls, fr, _, _ = _nodes(P)
    mem = _nodes(P)[0]
    rA = np.asarray(P["mem_rA"], dtype=float)[mem]
    w, k = np.asarray(P["w"], dtype=float), np.asarray(P["k"], dtype=float)
    b = beta_deg * (np.pi / 180.0)
    sb, cb = np.sin(b), np.cos(b)
    x, y, z = (rA[:, i] + ls * fr[:, 0, i] for i in range(3))
    ph = -(k[None, :] * (cb * x[:, None] + sb * y[:, None]))
    E = (zeta * w)[None, :] * (np.cos(ph) + 1j * np.sin(ph))
    S, C = _depth(k[None, :], float(P["depth"]), z[:, None])
    out = []
    for d in range(3):
        h = fr[:, d, 0] * cb + fr[:, d, 1] * sb
        out.append(E * (C * h[:, None] + 1j * S * fr[:, d, 2][:, None]))
    return np.array(out)


def _V(P):
    """V_d = [d; r x d], r = arm + ls q, double-double: [3][6] pairs of [Ns] arrays; and the kernels' magnitudes
    [d; |a x d|] and [0; |q x d|] (the ls term) as double [3, Ns, 6]."""
    _, ls, fr, arm, _ = _nodes(P)
    q = fr[:, 0]
    r = _add(arm, _mul(_dd(ls[:, None] * np.ones(3)), _dd(q)))
    V, Vm, Um = [], np.zeros((3, len(ls), 6)), np.zeros((3, len(ls), 6))
    am = np.abs(arm[0])
    for d in range(3):
        dv = fr[:, d]
        rxd = _cross(r, dv)
        V.append([_dd(dv[:, a]) for a in range(3)] + [(rxd[0][:, a], rxd[1][:, a]) for a in range(3)])
        Vm[d, :, :3] = np.abs(dv)
        Vm[d, :, 3:] = [[am[j, 1] * abs(dv[j, 2]) + am[j, 2] * abs(dv[j, 1]), am[j, 2] * abs(dv[j, 0]) + am[j, 0] * abs(dv[j, 2]),
                         am[j, 0] * abs(dv[j, 1]) + am[j, 1] * abs(dv[j, 0])] for j in range(len(ls))]
        Um[d, :, 3:] = np.abs(np.cross(q, dv))
    return V, Vm, Um


def reference(P, Xi, zeta, beta_deg, nodes=None, coef=None):
    """B_drag [6, 6], F_drag [6, nw] (complex) of one unit, as double-double pairs collapsed to double; the per-node
    coefficients b [3, Ns] (double-double), their magnitudes b~ [3, Ns], and the bound magnitudes M_B [6, 6], M_F [6, nw].
    ``nodes``: restrict every sum to these nodes (mpmath check).  ``coef``: (b, b~) of another unit instead of the
    linearisation about Xi (a secondary wave train's load with its primary's coefficients; Xi is then unused)."""
    mem, ls, fr, _, circ = _nodes(P)
    Ns = len(ls)
    keep = np.zeros(Ns, bool)
    keep[np.arange(Ns) if nodes is None else nodes] = True
    w = np.asarray(P["w"], dtype=float)
    u = _wave(P, zeta, beta_deg)
    # |u| with the phase argument's conditioning: x, y and k (x cos b + y sin b) are rounded (a relative error of
    # ~k (|x| + |y|) u in E, the kinematics' own, not the linearisation's)
    rA = np.asarray(P["mem_rA"], dtype=float)[mem]
    ph = 1.0 + np.asarray(P["k"], dtype=float)[None, :] * (np.abs(rA[:, 0]) + np.abs(rA[:, 1])
                                                        + np.abs(ls) * (np.abs(fr[:, 0, 0]) + np.abs(fr[:, 0, 1])))[:, None]
    ua = np.abs(u) * ph[None]
    V, Vm, Um = _V(P)
    cd = np.stack([np.asarray(P[k], dtype=float) for k in ("node_cd_q", "node_cd_p1", "node_cd_p2")])
    if coef is not None:
        b, bm = coef
        ss = smag = None
    else:
        b, bm, ss, smag = _coefficients(P, Xi, u, ua, V, Vm, Um, cd, ls, circ, w)
    return _sums(P, b, bm, u, ua, V, Vm, Um, mem, ls, keep, w, ss, smag)


def _coefficients(P, Xi, u, ua, V, Vm, Um, cd, ls, circ, w):
    """Per node and direction: b (double-double), b~, and the sums of squares (double-double) and of magnitudes."""
    Ns = len(ls)
    xr, xi = np.asarray(Xi.real, dtype=float), np.asarray(Xi.imag, dtype=float)
    ss, smag = [], []
    for d in range(3):
        sr = si = (np.zeros((Ns, len(w))), np.zeros((Ns, len(w))))
        for a in range(6):
            va = (V[d][a][0][:, None] * np.ones(len(w)), V[d][a][1][:, None] * np.ones(len(w)))
            sr = _add(sr, _mul(va, _dd(np.broadcast_to(xr[a], (Ns, len(w))))))
            si = _add(si, _mul(va, _dd(np.broadcast_to(xi[a], (Ns, len(w))))))
        W = _dd(np.broadcast_to(w, (Ns, len(w))))
        ar = _add(_dd(u[d].real), _mul(W, si))                 # u + (-i w s)
        ai = _add(_dd(u[d].imag), _neg(_mul(W, sr)))
        ss.append(_sum(_add(_mul(ar, ar), _mul(ai, ai)), 1))
        mag = ua[d] + w[None, :] * ((Vm[d] + np.abs(ls)[:, None] * Um[d]) @ np.abs(Xi))
        smag.append(np.sum(mag * mag, axis=1))
    b, bm = [], np.zeros((3, Ns))
    half = _dd(np.full(Ns, 0.5))
    tr = _add(ss[1], ss[2])
    for d in range(3):
        s = (np.where(circ, tr[0], ss[d][0]), np.where(circ, tr[1], ss[d][1])) if d else ss[0]
        sm = np.where(circ, smag[1] + smag[2], smag[d]) if d else smag[0]
        b.append(_mul(_dd(cd[d]), _sqrt(_mul(half, s))))
        bm[d] = np.abs(cd[d]) * np.sqrt(0.5 * sm) * (1 + 4 * U)
    return b, bm, ss, smag


def _sums(P, b, bm, u, ua, V, Vm, Um, mem, ls, keep, w, ss, smag):
    """B_drag and F_drag from the coefficients (double-double), and the bound magnitudes over the factored member sums."""
    B = [[(np.zeros(1), np.zeros(1)) for _ in range(6)] for _ in range(6)]
    Fr = [(np.zeros(len(w)), np.zeros(len(w))) for _ in range(6)]
    Fi = [(np.zeros(len(w)), np.zeros(len(w))) for _ in range(6)]
    for j in np.nonzero(keep)[0]:
        for d in range(3):
            bj = (b[d][0][j:j + 1], b[d][1][j:j + 1])
            Vj = [(V[d][a][0][j:j + 1], V[d][a][1][j:j + 1]) for a in range(6)]
            for a in range(6):
                bv = _mul(bj, Vj[a])
                for c in range(6):
                    B[a][c] = _add(B[a][c], _mul(bv, Vj[c]))
                bvw = (np.broadcast_to(bv[0], len(w)), np.broadcast_to(bv[1], len(w)))
                Fr[a] = _add(Fr[a], _mul(bvw, _dd(u[d, j].real)))
                Fi[a] = _add(Fi[a], _mul(bvw, _dd(u[d, j].imag)))
    Bref = np.array([[B[a][c][0][0] + B[a][c][1][0] for c in range(6)] for a in range(6)])
    Fref = np.array([Fr[a][0] + Fr[a][1] + 1j * (Fi[a][0] + Fi[a][1]) for a in range(6)])
    # magnitudes over the kernels' factored member sums
    MB, MF = np.zeros((6, 6)), np.zeros((6, len(w)))
    for m in np.unique(mem[keep]):
        jm = np.nonzero((mem == m) & keep)[0]
        for d in range(3):
            Vd, Ud = Vm[d, jm[0]], Um[d, jm[0]]
            s0, s1, s2 = bm[d, jm].sum(), (bm[d, jm] * np.abs(ls[jm])).sum(), (bm[d, jm] * ls[jm] ** 2).sum()
            MB += s0 * np.outer(Vd, Vd) + s1 * (np.outer(Vd, Ud) + np.outer(Ud, Vd)) + s2 * np.outer(Ud, Ud)
            au = ua[d, jm]
            MF += Vd[:, None] * (bm[d, jm] @ au)[None, :] + Ud[:, None] * ((bm[d, jm] * np.abs(ls[jm])) @ au)[None, :]
    return dict(B=Bref, F=Fref, b=b, bm=bm, MB=MB * (1 + 8 * U), MF=MF * (1 + 8 * U), ss=ss, smag=smag)


def _ratios(Bk, Fk, ref):
    """(worst |dB| / (u M_B), worst per-bin, per-group |dF| / (u M_F)); entries with a zero magnitude must be exact."""
    dB = np.abs(Bk - ref["B"])
    assert np.all(dB[ref["MB"] == 0] == 0)
    rb = float((dB / np.where(ref["MB"] > 0, U * ref["MB"], 1.0)).max())
    dF = np.abs(Fk - ref["F"])
    rf = 0.0
    for g in (slice(0, 3), slice(3, 6)):
        e, m = dF[g].max(0), ref["MF"][g].max(0)
        assert np.all(e[m == 0] == 0)
        rf = max(rf, float((e / np.where(m > 0, U * m, 1.0)).max()))
    return rb, rf


# ---- planted inputs -------------------------------------------------------------------------------------------------
def _combo(j):
    """Direction mask of node j: 0 none, 1 axial, 2 transverse, 3 both; (chunk + slot) mod 4."""
    return (j // CHUNK + j % CHUNK) % 4


def _plant(nw):
    """cfg2 on the nw-bin grid with the edited drag tables and the far member (module docstring)."""
    P = dict(_design("cfg2", nw))
    ms = np.asarray(P["mem_start"])
    cq, c1, c2 = (np.array(P[k], dtype=float) for k in ("node_cd_q", "node_cd_p1", "node_cd_p2"))
    circ = np.asarray(P["mem_circ"])
    mem = np.repeat(np.arange(len(ms) - 1), np.diff(ms))
    q0, p0 = cq[cq > 0].mean(), c1[c1 > 0].mean()
    for j in range(len(cq)):
        mk = _combo(j) | NEED_MASK.get(j, 0)
        cq[j] = (cq[j] or q0 * (1 + 0.01 * j)) if mk & 1 else 0.0
        if mk & 2:
            c1[j] = c1[j] or p0 * (1 + 0.013 * j)
            c2[j] = c1[j] if circ[mem[j]] else 1.7 * c1[j]
        else:
            c1[j] = c2[j] = 0.0
    P["node_cd_q"], P["node_cd_p1"], P["node_cd_p2"] = cq, c1, c2
    rA = np.array(P["mem_rA"], dtype=float)
    ls = np.array(P["node_ls"], dtype=float)
    j0, j1 = ms[FAR_MEMBER], ms[FAR_MEMBER + 1]
    q = np.asarray(P["mem_q"], dtype=float)[FAR_MEMBER]
    rA[FAR_MEMBER] = np.asarray(P["prp"], dtype=float) - FAR_ARM * q + np.array([0.0, 0.0, rA[FAR_MEMBER][2]])
    ls[j0:j1] += FAR_ARM - 0.5 * ls[j1 - 1]                  # the same spacings: the same step classes and layout
    P["mem_rA"], P["node_ls"] = rA, ls
    return P


def _slices(shape):
    """Bins per CTA and the number of CTAs of the kernel's layout."""
    nw, cs = shape[1], shape[2]
    return -(-nw // cs), cs


def _planted_xi(P, shape):
    """Xi_init [6, nw]: per bin a complex combination of the null space of the CANCEL projections, amplitudes spanning 10
    decades, the largest ones in the last CTA's slice."""
    nw = len(P["w"])
    V, _, _ = _V(P)
    G = np.array([[V[d][a][0][j] for a in range(6)] for j, d in CANCEL])
    N = np.linalg.svd(G)[2][len(CANCEL):]                                  # [2, 6]
    rng = np.random.default_rng(11)
    amp = 10.0 ** rng.uniform(-10, -2, size=(len(N), nw))
    nwl, cs = _slices(shape)
    last = np.arange(nw) >= (cs - 1) * nwl
    amp[:, last & (np.arange(nw) % 7 == 3)] = 1.0
    c = amp * np.exp(2j * np.pi * rng.uniform(size=(len(N), nw)))
    return (N.T @ c).astype(complex)


# ---- without a GPU --------------------------------------------------------------------------------------------------
def test_reference_against_mpmath():
    """The double-double per-node sums, coefficients, B_drag and F_drag equal a 40-digit mpmath evaluation of the same
    formula to 1e-28 on six nodes (a cancelling one among them) and eight bins, with waves on."""
    import mpmath as mp
    mp.mp.dps = 40
    shape = KERNELS[0]
    P = _plant(shape[1])
    nw = shape[1]
    Xi = _planted_xi(P, shape)
    sub = np.array([0, 7, 13, 25, 37, 48])
    bins = np.array([0, 1, 50, 99, 100, 150, 199, 200])
    Xs = np.zeros_like(Xi)
    Xs[:, bins] = Xi[:, bins]
    zeta = np.zeros(nw)
    zeta[bins] = np.linspace(0.3, 1.7, len(bins))
    ref = reference(P, Xs, zeta, 37.0, nodes=sub)
    mem, ls, fr, _, circ = _nodes(P)
    u = _wave(P, zeta, 37.0)
    w = np.asarray(P["w"], dtype=float)
    cd = [np.asarray(P[k], dtype=float) for k in ("node_cd_q", "node_cd_p1", "node_cd_p2")]
    rA, prp = np.asarray(P["mem_rA"], dtype=float), np.asarray(P["prp"], dtype=float)
    Bm = [[mp.mpf(0)] * 6 for _ in range(6)]
    Fm = [[mp.mpc(0)] * nw for _ in range(6)]
    for j in sub:
        r = [mp.mpf(rA[mem[j], t]) - mp.mpf(prp[t]) + mp.mpf(ls[j]) * mp.mpf(fr[j, 0, t]) for t in range(3)]
        Vs, ssm = [], []
        for d in range(3):
            dv = [mp.mpf(fr[j, d, t]) for t in range(3)]
            V = dv + [r[1] * dv[2] - r[2] * dv[1], r[2] * dv[0] - r[0] * dv[2], r[0] * dv[1] - r[1] * dv[0]]
            s = mp.mpf(0)
            for i in range(nw):
                v = mp.mpc(u[d, j, i]) - 1j * mp.mpf(w[i]) * mp.fsum(V[a] * mp.mpc(Xs[a, i]) for a in range(6))
                s += abs(v) ** 2
            Vs.append(V)
            ssm.append(s)
            hi, lo = ref["ss"][d][0][j], ref["ss"][d][1][j]
            assert abs(mp.mpf(hi) + mp.mpf(lo) - s) <= 1e-28 * ref["smag"][d][j], (j, d)
        for d in range(3):
            s = (ssm[1] + ssm[2]) if (d and circ[j]) else ssm[d]
            b = mp.mpf(cd[d][j]) * mp.sqrt(s / 2)
            assert abs(mp.mpf(ref["b"][d][0][j]) + mp.mpf(ref["b"][d][1][j]) - b) <= 1e-28 * ref["bm"][d][j], (j, d)
            for a in range(6):
                for c in range(6):
                    Bm[a][c] += b * Vs[d][a] * Vs[d][c]
                for i in bins:
                    Fm[a][i] += b * mp.mpc(u[d, j, i]) * Vs[d][a]
    for a in range(6):
        for c in range(6):
            assert abs(mp.mpf(ref["B"][a, c]) - Bm[a][c]) <= U * abs(Bm[a][c]) + 1e-28 * ref["MB"][a, c], (a, c)
        for i in bins:
            assert abs(mp.mpc(ref["F"][a, i]) - Fm[a][i]) <= 2 * U * abs(Fm[a][i]) + 1e-28 * ref["MF"][a, i], (a, i)


@pytest.mark.parametrize("shape", KERNELS, ids=KID)
def test_planted_inputs_reach_their_edges(shape):
    """On each kernel's layout: every mask combination at slots 0 and 9 and on both sides of a chunk boundary, members
    longer than a chunk, Ns not a multiple of CHUNK_NODES; circular next to rectangular members with Cd_p1 != Cd_p2; the
    CANCEL nodes' reference vRMS below 1e-13 of their magnitude RMS; the far member's factored sums cancelling by more
    than 1e3; the RMS of most nodes dominated by bins of the last CTA's slice."""
    P = _plant(shape[1])
    ms = np.asarray(P["mem_start"])
    Ns = int(ms[-1])
    cq, c1, c2 = (np.asarray(P[k]) for k in ("node_cd_q", "node_cd_p1", "node_cd_p2"))
    plan = _plan_chunks(P)
    mk = np.array([(cm >> (3 * (j % CHUNK))) & 3 for j in range(Ns) for cm in [plan[j // CHUNK][0]]])
    for jj in (0, CHUNK - 1):
        assert {int(mk[j]) for j in range(jj, Ns, CHUNK)} == {0, 1, 2, 3}, jj
    used = 0
    for ch, (cm, slots, rm) in enumerate(plan):
        written, read = _walk_slots(cm, min(CHUNK, Ns - ch * CHUNK))
        assert written == slots and read <= written, ch                      # the coefficients read what the walk wrote
        assert all(rm >> (sl // 8) & 1 for sl in range(32) if slots >> sl & 1), ch   # every written slot is reduced
        used |= slots
    for sl in (0, CHUNK - 1, CHUNK, 2 * CHUNK - 1, 2 * CHUNK, 3 * CHUNK - 1):     # first and last slot of each third
        assert used >> sl & 1, sl
    assert Ns % CHUNK != 0 and max(np.diff(ms)) > CHUNK
    assert any(ms[m] // CHUNK != (ms[m + 1] - 1) // CHUNK for m in range(len(ms) - 1))
    circ = np.asarray(P["mem_circ"])
    assert any(circ[m] != circ[m + 1] for m in range(len(circ) - 1))
    mem = np.repeat(np.arange(len(ms) - 1), np.diff(ms))
    rect = (circ[mem] == 0) & (c1 != 0)
    assert rect.any() and np.all(c2[rect] != c1[rect])
    Xi = _planted_xi(P, shape)
    ref = reference(P, Xi, np.zeros(shape[1]), 0.0)
    for j, d in CANCEL:
        assert mk[j] & (1 if d == 0 else 2), (j, d)
        v = math.sqrt(ref["ss"][d][0][j])
        assert v < 1e-13 * math.sqrt(ref["smag"][d][j]), (j, d, v)
    # far member: the node-wise moment entries against the factored sums' magnitude
    jm = np.arange(ms[FAR_MEMBER], ms[FAR_MEMBER + 1])
    only = reference(P, Xi, np.zeros(shape[1]), 0.0, nodes=jm)
    assert only["MB"][5, 5] > 1e3 * abs(only["B"][5, 5]), (only["MB"][5, 5], only["B"][5, 5])
    nwl, cs = _slices(shape)
    e = np.sum(np.abs(Xi) ** 2, axis=0)
    assert e[(cs - 1) * nwl:].sum() > 0.99 * e.sum() and (cs == 1 or e[:nwl].sum() > 0)


def _plan_chunks(P):
    """k_fused_plan's drag-direction masks (raftk_fused2.cuh) restated: per chunk of CHUNK_NODES nodes, (direction mask
    cm, bit 3jj = axial, 3jj + 1 = transverse; accumulator slots used; reduction-round mask rm)."""
    cq, c1, c2 = (np.asarray(P[k]) for k in ("node_cd_q", "node_cd_p1", "node_cd_p2"))
    Ns = int(np.asarray(P["mem_start"])[-1])
    out = []
    for ch in range(-(-Ns // CHUNK)):
        cm = slots = 0
        for jj in range(CHUNK):
            j = ch * CHUNK + jj
            if j >= Ns:
                break
            q, p = cq[j] != 0, c1[j] != 0 or c2[j] != 0
            cm |= (int(q) | int(p) << 1) << (3 * jj)
            if q or p:
                slots |= 1 << jj
            if p:
                slots |= 1 << (10 + jj)
            if q and p:
                slots |= 1 << (20 + jj)
        out.append((cm, slots, sum(1 << rd for rd in range(4) if (slots >> (rd * 8)) & 0xff)))
    return out


def _walk_slots(cm, n):
    """The slots k_rao_fused2's RMS walk writes for a chunk of n nodes (transverse 1 at jj, transverse 2 at 10 + jj, axial
    at 20 + jj when the node has both, else at jj), and the slots its coefficient step reads back."""
    written = read = 0
    for jj in range(n):
        mk = (cm >> (3 * jj)) & 3
        if mk & 2:
            written |= (1 << jj) | (1 << (10 + jj))
            read |= (1 << jj) | (1 << (10 + jj))
        if mk & 1:
            written |= 1 << (20 + jj if mk & 2 else jj)
            read |= 1 << (20 + jj if mk & 2 else jj)
    return written, read


def _model(P, Xi, zeta, beta_deg, fault=None):
    """The linearisation modelled on the CPU in plain double, in the kernels' factored form, optionally with a fault."""
    mem, ls, fr, arm, circ = _nodes(P)
    ms = np.asarray(P["mem_start"])
    w = np.asarray(P["w"], dtype=float)
    u = _wave(P, zeta, beta_deg)
    armd = arm[0]
    if fault == "circ":
        circ = circ.copy()
        circ[mem == 4] = ~circ[mem == 4]
    cd = np.stack([np.asarray(P[k], dtype=float) for k in ("node_cd_q", "node_cd_p1", "node_cd_p2")])
    ss = []
    for d in range(3):
        dv = fr[:, d]
        V = np.concatenate([dv, np.cross(armd, dv)], 1)
        T = np.concatenate([np.zeros_like(dv), np.cross(fr[:, 0], dv)], 1)
        s = V @ Xi + ls[:, None] * (T @ Xi)
        v = u[d] - 1j * w[None, :] * s
        ss.append(np.sum(v.real ** 2 + v.imag ** 2, axis=1))
    b = np.zeros((3, len(ls)))
    for d in range(3):
        s = np.where(circ, ss[1] + ss[2], ss[d]) if d else ss[0]
        b[d] = cd[d] * np.sqrt(0.5 * s)
    if fault == "drop":
        b[:, 30] = 0.0
    B = np.zeros((6, 6))
    F = np.zeros((6, len(w)), dtype=complex)
    for m in range(len(ms) - 1):
        jm = np.arange(ms[m], ms[m + 1])
        a = armd[jm[0]]
        for d in range(3):
            dv = fr[jm[0], d]
            Vd = np.concatenate([dv, np.cross(a, dv)])
            Ud = np.concatenate([np.zeros(3), np.cross(fr[jm[0], 0], dv)])
            s0, s1, s2 = b[d, jm].sum(), (b[d, jm] * ls[jm]).sum(), (b[d, jm] * ls[jm] ** 2).sum()
            B += s0 * np.outer(Vd, Vd) + s1 * (np.outer(Vd, Ud) + np.outer(Ud, Vd)) + s2 * np.outer(Ud, Ud)
            F += Vd[:, None] * (b[d, jm] @ u[d, jm])[None, :] + Ud[:, None] * ((b[d, jm] * ls[jm]) @ u[d, jm])[None, :]
    if fault == "trans":
        B[:3, :3] *= 1 + 1e-9
    return B, F


@pytest.mark.parametrize("fault", [None, "drop", "circ", "trans"])
def test_modelled_faults_break_the_bounds(fault):
    """The CPU model of the kernels' algorithm meets the bounds with waves on (JONSWAP-like amplitudes, heading 37 deg);
    a dropped node, a swapped circular flag and the translational block off by 1e-9 each break them by more than 100x."""
    shape = KERNELS[0]
    P = _plant(shape[1])
    Xi = _planted_xi(P, shape)
    zeta = np.linspace(0.05, 1.2, shape[1])
    ref = reference(P, Xi, zeta, 37.0)
    B, F = _model(P, Xi, zeta, 37.0, fault)
    rb, rf = _ratios(B, F, ref)
    print("fault %s: |dB|/(u M) %.3g, |dF|/(u M) %.3g" % (fault, rb, rf))
    if fault is None:
        assert rb <= C_B and rf <= C_F, (rb, rf)
    elif fault == "trans":
        assert rb > 100 * C_B, rb
    else:
        assert rb > 100 * C_B and rf > 100 * C_F, (rb, rf)


def _loop_plan(shape, tol, n_iter):
    """Per case: (bin, DOF, k, sign, expected passes, converged) and Xi_init [nC, 6, nw] (module docstring)."""
    nw = shape[1]
    nwl, cs = _slices(shape)
    pos = sorted({b for r in range(cs) for b in (r * nwl, min(nw, (r + 1) * nwl) - 1)} | {nw - 1})
    rng = np.random.default_rng(int(-math.log10(tol) * 10) + nw)
    t2 = tol * tol
    plan, X = [], []
    ks = (0, 1, 3, n_iter + 2)
    c = 0
    for dof in range(6):
        for p in pos:
            k, sgn = ks[c % len(ks)], (-1, 1)[(c // len(ks)) % 2]
            x = t2 * (1 - 1e-6) * rng.uniform(0.0, 1.0, (6, nw)) * np.exp(2j * np.pi * rng.uniform(size=(6, nw)))
            x[dof, p] = t2 * 5.0 ** k * (1 + sgn * 1e-6) * np.exp(2j * np.pi * rng.uniform())
            passes = k + 1 if sgn < 0 else k + 2
            plan.append((p, dof, k, sgn, min(passes, n_iter + 1), int(passes <= n_iter + 1)))
            X.append(x)
            c += 1
    return plan, np.array(X)


def _relaxed(X, n):
    for _ in range(n):
        X = 0.2 * X.real + 1j * (0.2 * X.imag)
    return X


def test_loop_plan_predicts_the_reference_rule():
    """The reference's own rule |d| / (|x| + tol) < tol, run in NumPy on zero load from the planted iterates, gives the
    planned pass counts, and the planted (bin, DOF) sits at every DOF, at the first and last bin of every CTA and at the
    tail bin of each layout."""
    for shape in LOOP:
        for tol in TOLS:
            plan, X = _loop_plan(shape, tol, 10)
            nwl, cs = _slices(shape)
            assert {p for p, *_ in plan} >= {0, shape[1] - 1} | {r * nwl for r in range(cs)} | {r * nwl - 1 for r in range(1, cs)}
            assert {d for _, d, *_ in plan} == set(range(6)) and {k for _, _, k, *_ in plan} == {0, 1, 3, 12}
            for (p, dof, k, sgn, passes, conv), x in zip(plan[::5], X[::5]):
                last = x
                for it in range(11):
                    ok = np.all(np.abs(0.0 - last) / (0.0 + tol) < tol)
                    if ok or it == 10:
                        break
                    last = _relaxed(last, 1)
                assert (it + 1, int(ok)) == (passes, conv), (shape, tol, p, dof, k, sgn)


# ---- on the GPU -----------------------------------------------------------------------------------------------------
def _env(monkeypatch, shape):
    for k in ("RAFTK_FORCE_V1", "RAFTK_FUSED2_XCHG", "RAFTK_NO_DIRECT_D2H"):
        monkeypatch.delenv(k, raising=False)
    for k, v in shape[3].items():
        monkeypatch.setenv(k, v)


def _solve(monkeypatch, shape, designs, cases, n_iter, tol=0.01, xi_start=0.0, want=None):
    from raft_b200 import solver
    _env(monkeypatch, shape)
    if want is None:
        want = ("Xi", "status", "B_drag", "F_drag", "zeta") + (() if shape[4] == "v1" else ("Xi_last",))
    out = solver.solve_dynamics(solver.DesignBatch(designs), cases, n_iter=n_iter, tol=tol, xi_start=xi_start,
                                cluster_size=shape[2], want=want)
    return out, solver.last_dispatch()


def _linearise(monkeypatch, shape, P, Xi):
    """One pass from the planted iterate: n_iter = 0 with Xi_init on the fused kernels, hydro_linearization on v1.
    -> B_drag [nC, 6, 6], F_drag [nC, 6, nw], zeta [nC, nw]."""
    from raft_b200 import solver
    nC = len(SEA["Hs"])
    X = np.broadcast_to(Xi, (1, nC) + Xi.shape).copy()
    if shape[4] == "v1":
        _env(monkeypatch, shape)
        batch, ct = solver.DesignBatch(P), solver.CaseTable(SEA)
        out = solver.hydro_linearization(batch, ct, X)
        rec = solver.last_dispatch()
        assert rec["kernel"] == "v1", rec
        zeta = solver.hydro_excitation(batch, ct, want=("zeta",))["zeta"]
        return out["B_drag"][0], out["F_drag"][0], zeta
    out, rec = _solve(monkeypatch, shape, [P], solver.CaseTable(SEA, Xi_init=X), 0)
    _check_record(rec, shape)
    assert np.all(out["status"][0, :, 0] == 1), out["status"]
    return out["B_drag"][0], out["F_drag"][0], out["zeta"]


def _walk(P):
    return int(np.diff(np.asarray(P["mem_start"])).max())


WORST = {"B": 0.0, "F": 0.0, "Bwalk": 0.0, "Fwalk": 0.0}


def _check_bounds(rb, rf, walk, L, tag):
    """The bounds of the module docstring; walk: a fused kernel with waves on (ratios against (1 + L) u M)."""
    if walk:
        rb, rf = rb / (1.0 + L), rf / (1.0 + L)
    key = "walk" if walk else ""
    WORST["B" + key] = max(WORST["B" + key], rb)
    WORST["F" + key] = max(WORST["F" + key], rf)
    cb, cf = (C_B_WALK, C_F_WALK) if walk else (C_B, C_F)
    assert rb <= cb and rf <= cf, (tag, walk, rb, rf)


@gpu
@pytest.mark.parametrize("shape", KERNELS, ids=KID)
def test_planted_linearisation_vs_reference(shape, monkeypatch):
    """Families A and B: B_drag entry by entry and F_drag bin by bin within the bounds; F_drag exactly 0 without waves."""
    P = _plant(shape[1])
    Xi = _planted_xi(P, shape)
    B, F, zeta = _linearise(monkeypatch, shape, P, Xi)
    L = _walk(P)
    for c in range(len(SEA["Hs"])):
        waves = SEA["spec"][c] != SPEC_NONE
        if not waves:
            assert not np.any(zeta[c]) and not np.any(F[c]), c
        ref = reference(P, Xi, zeta[c], float(SEA["beta_deg"][c]))
        rb, rf = _ratios(B[c], F[c], ref)
        _check_bounds(rb, rf, waves and shape[4] != "v1", L, (shape[4], c))
    print("%s: worst %s" % (shape[4], WORST))


TRAIN_KERNELS = [s for s in KERNELS if s[4] != "v1" and not s[5]]


@gpu
@pytest.mark.parametrize("shape", TRAIN_KERNELS, ids=[s[4] for s in TRAIN_KERNELS])
def test_wave_trains_vs_reference(shape, monkeypatch):
    """A wave-train table on the planted design (test_dispatch_solve._train_table: two single-train cases and one case of
    three trains): every primary's B_drag and F_drag against the reference linearised about its Xi_last; every secondary
    train's F_drag bin by bin against the reference at its own zeta and heading with the primary's coefficients."""
    from raft_b200 import solver
    P = _plant(shape[1])
    table = _train_table()
    out, rec = _solve(monkeypatch, shape, [P], solver.CaseTable(table), 10)
    assert rec["kernel"] == shape[4] and rec["cluster_size"] == shape[2] and rec["trains"], rec
    assert np.all(out["status"][0, :, 2] == 0), out["status"]
    prim, beta, L = np.asarray(table["primary"]), np.asarray(table["beta_deg"], dtype=float), _walk(P)
    assert any(prim[c] != c for c in range(len(prim)))
    refs = {}
    for c in sorted(set(prim.tolist())):
        refs[c] = reference(P, out["Xi_last"][0, c], out["zeta"][c], beta[c])
        rb, rf = _ratios(out["B_drag"][0, c], out["F_drag"][0, c], refs[c])
        _check_bounds(rb, rf, True, L, (shape[4], "primary", c))
    for c in range(len(prim)):
        p = int(prim[c])
        if p == c:
            continue
        ref = reference(P, None, out["zeta"][c], beta[c], coef=(refs[p]["b"], refs[p]["bm"]))
        _, rf = _ratios(out["B_drag"][0, p], out["F_drag"][0, c], dict(ref, B=refs[p]["B"], MB=refs[p]["MB"]))
        _check_bounds(0.0, rf, True, L, (shape[4], "secondary", c))
    print("%s trains: worst %s" % (shape[4], WORST))


@gpu
def test_device_session_linearization_matches_host():
    """DeviceSession.linearization (v1 mode 1 on the device) equals the host entry bit for bit on the planted iterate."""
    import torch
    from raft_b200 import solver
    shape = KERNELS[-1]
    P = _plant(shape[1])
    Xi = _planted_xi(P, shape)
    nC = len(SEA["Hs"])
    X = np.broadcast_to(Xi, (1, nC) + Xi.shape).copy()
    host = solver.hydro_linearization(solver.DesignBatch(P), solver.CaseTable(SEA), X)
    sess = solver.DeviceSession(solver.DesignBatch(P), solver.CaseTable(SEA), tables=True)
    sess.excitation()
    dev = sess.linearization(torch.from_numpy(X).to(sess.device))
    torch.cuda.synchronize()
    assert solver.last_dispatch()["kernel"] == "v1"
    assert "B_drag" in dev
    for k in {"B_drag", "F_drag"} & set(dev):
        assert np.array_equal(dev[k].cpu().numpy(), host[k]), k


@gpu
@pytest.mark.parametrize("s", [-300, 300])
@pytest.mark.parametrize("shape", KERNELS, ids=KID)
def test_power_of_two_scaling_is_exact(shape, s, monkeypatch):
    """Spec NONE: Xi_init times 2^s gives B_drag times 2^s bit for bit, and F_drag stays exactly 0."""
    P = _plant(shape[1])
    Xi = _planted_xi(P, shape)
    B0, _, _ = _linearise(monkeypatch, shape, P, Xi)
    Bs, Fs, _ = _linearise(monkeypatch, shape, P, np.ldexp(Xi.real, s) + 1j * np.ldexp(Xi.imag, s))
    none = SEA["spec"] == SPEC_NONE
    assert np.array_equal(Bs[none], np.ldexp(B0[none], s)) and not np.any(Fs[none])


@gpu
@pytest.mark.parametrize("tol", TOLS)
@pytest.mark.parametrize("shape", LOOP, ids=LID)
def test_fixed_point_loop_is_exact(shape, tol, monkeypatch):
    """Zero load: passes, converged and Xi_last as the reference rule predicts, per planted (bin, DOF); v1 with the
    constant xi_start on every bin (the fused kernels the same through Xi_init, with identical pass counts)."""
    from raft_b200 import solver
    P = _design("cfg2", shape[1])
    n_iter = 10
    sea = lambda n: dict(Hs=np.ones(n), Tp=np.full(n, 10.0), gamma=np.zeros(n), beta_deg=np.zeros(n),   # noqa: E731
                         spec=np.full(n, SPEC_NONE, dtype=np.int32))
    consts = [(tol * tol * 5.0 ** k * (1 + sg * 1e-6), k, sg) for k in (0, 1, 3) for sg in (-1, 1)]
    for x0, k, sg in consts:
        passes = k + 1 if sg < 0 else k + 2
        if shape[4] == "v1":
            out, rec = _solve(monkeypatch, shape, [P], solver.CaseTable(sea(1)), n_iter, tol=tol, xi_start=x0)
        else:
            X = np.full((1, 1, 6, shape[1]), x0, dtype=complex)
            out, rec = _solve(monkeypatch, shape, [P], solver.CaseTable(sea(1), Xi_init=X), n_iter, tol=tol)
        _check_record(rec, shape)
        assert not np.any(out["Xi"])
        assert tuple(out["status"][0, 0, :3]) == (passes, 1, 0), (x0, k, sg, out["status"][0, 0])
    if shape[4] == "v1":
        return
    plan, X = _loop_plan(shape, tol, n_iter)
    out, rec = _solve(monkeypatch, shape, [P], solver.CaseTable(sea(len(plan)), Xi_init=X[None]), n_iter, tol=tol)
    _check_record(rec, shape)
    assert not np.any(out["Xi"])
    for c, (p, dof, k, sgn, passes, conv) in enumerate(plan):
        assert tuple(out["status"][0, c, :3]) == (passes, conv, 0), (c, p, dof, k, sgn, out["status"][0, c])
        last = _relaxed(X[c], passes - 1)
        assert np.array_equal(out["Xi_last"][0, c], last), (c, p, dof)


@gpu
@pytest.mark.parametrize("tol", [1e-70, 0.0])
@pytest.mark.parametrize("shape", LOOP, ids=LID)
def test_zero_iterate_at_the_smallest_tol(shape, tol, monkeypatch):
    """Zero load and a zero iterate: d = x = 0 at every bin.  At tol = RAFTK_TOL_MIN the reference rule converges on the
    first pass; at tol = 0 (0 / 0 < 0 is false) it never does, and the unit runs n_iter + 1 passes."""
    from raft_b200 import solver
    P = _design("cfg2", shape[1])
    sea = dict(Hs=np.ones(2), Tp=np.full(2, 10.0), gamma=np.zeros(2), beta_deg=np.zeros(2), spec=np.full(2, SPEC_NONE, dtype=np.int32))
    if shape[4] == "v1":
        ct = solver.CaseTable(sea)
    else:
        ct = solver.CaseTable(sea, Xi_init=np.zeros((1, 2, 6, shape[1]), dtype=complex))
    out, rec = _solve(monkeypatch, shape, [P], ct, 10, tol=tol, xi_start=0.0)
    _check_record(rec, shape)
    assert not np.any(out["Xi"])
    assert np.all(out["status"][0, :, :3] == ((1, 1, 0) if tol > 0 else (11, 0, 0))), out["status"]


@gpu
@pytest.mark.parametrize("tol", [1e-90, 1e-200, 9.9e-71, -0.01, float("nan")])
@pytest.mark.parametrize("shape", LOOP, ids=LID)
def test_tol_below_the_minimum_is_refused(shape, tol, monkeypatch):
    """A tol in (0, RAFTK_TOL_MIN), negative or NaN is refused before any launch.  Below ~1e-81 k_rao_fused2's
    d.d < (tol (|x| + tol))^2 underflowed to 0 < 0 at a still-water bin (d = x = 0), so such a unit never converged; below
    ~1e-162 k_rao_fused's |d| < tol |x| + tol^2 did too; and every kernel's d.d underflows for |d| < 1e-154, where it
    no longer decides as the reference's |d| / (|x| + tol) < tol does."""
    from raft_b200 import _lib, solver
    P = _design("cfg2", shape[1])
    sea = dict(Hs=np.ones(2), Tp=np.full(2, 10.0), gamma=np.zeros(2), beta_deg=np.zeros(2), spec=np.full(2, SPEC_NONE, dtype=np.int32))
    with pytest.raises(_lib.RaftkError, match="tol must be 0 or at least 1e-70"):
        _solve(monkeypatch, shape, [P], solver.CaseTable(sea), 10, tol=tol)
    assert solver.last_dispatch()["kernel"] == "none"


def _random_design(nw):
    """test_gpu_parity._random_design with three circular members (29 nodes) at cfg2's depth, on cfg2's grid."""
    from raft_b200 import grid
    from raft_b200.fowt import FOWT
    from test_dispatch_solve import MAX_FREQ
    from test_gpu_parity import _random_design as random_members
    rng = np.random.default_rng(30)
    design = random_members(rng, int(rng.integers(3, 5)))
    design["site"]["water_depth"] = 200.0
    m = 2e7
    mats = dict(M_struc=np.diag([m, m, m, m * 900, m * 900, m * 1500]), C_struc=np.zeros((6, 6)),
                C_hydro=np.diag([0, 0, 4e6, 2e9, 2e9, 0.0]), C_moor=np.diag([7e4, 7e4, 0, 0, 0, 1.2e8]), B_struc=np.zeros((6, 6)))
    f = FOWT(design, grid.make_w(0.3 / 100, 0.3), depth=200.0, matrices=mats)
    f.calcHydroConstants()
    return grid.regrid(f.pack(), nw, MAX_FREQ)


def _batch_designs(nw):
    """cfg2, the planted cfg2, cfg1 and a random design on cfg2's site and grid."""
    base = _design("cfg2", nw)
    cfg1 = dict(_design("cfg1", nw))
    cfg1["depth"], cfg1["k"] = base["depth"], base["k"]
    return [base, _plant(nw), cfg1, _random_design(nw)]


def test_batch_designs_differ():
    """The batch's designs share the grid and depth, and differ in member and node counts, circular/rectangular mixes and
    step classes."""
    from raft_b200 import solver
    ds = _batch_designs(201)
    assert all(np.array_equal(D["w"], ds[0]["w"]) and float(D["depth"]) == float(ds[0]["depth"]) for D in ds)
    assert len({len(D["mem_circ"]) for D in ds}) == 3 and len({int(D["mem_start"][-1]) for D in ds}) == 3
    assert len({tuple(np.asarray(D["mem_circ"]).tolist()) for D in ds}) >= 3
    classes = {(b.max_w_classes, b.max_h_classes, b.max_z_classes) for b in (solver.DesignBatch(D) for D in ds)}
    assert len(classes) >= 3, classes


@gpu
@pytest.mark.parametrize("shape", LOOP, ids=LID)
def test_heterogeneous_batch_is_bit_identical(shape, monkeypatch):
    """The four-design batch (different member and node counts, circular/rectangular mixes and step classes): every unit's
    Xi, Xi_last, status, B_drag and F_drag equal that design launched alone on the same kernel and cluster size."""
    from raft_b200 import solver
    designs = _batch_designs(shape[1])
    ct = solver.CaseTable({k: v[1:] for k, v in SEA.items()})
    both, rec = _solve(monkeypatch, shape, designs, ct, 10)
    assert rec["kernel"] == shape[4] and rec["cluster_size"] == shape[2], rec
    for d, Q in enumerate(designs):
        one, r1 = _solve(monkeypatch, shape, [Q], ct, 10)
        assert r1["kernel"] == shape[4] and r1["cluster_size"] == shape[2], (d, r1)
        for k in one:
            if k != "zeta":
                assert np.array_equal(both[k][d], one[k][0]), (d, k)
