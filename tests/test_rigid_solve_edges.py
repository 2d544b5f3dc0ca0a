"""The rigid solvers' 6x6 impedance solve (raftk_common.cuh solve6: LU with partial pivoting on |re| + |im|, the first
maximum winning, rows exchanged by register selects) against a high-precision reference of the same system, on inputs
that reach every pivot order, exact ties, ill-conditioned bins and the ends of the exponent range, in every rigid kernel.

The reference is the one of test_farm_edges and does not share the kernels' algorithm.  Each (design, case, bin) system
is rebuilt in NumPy from the solver's own outputs (B_drag, F_drag, F_iner, F_BEM) and the design tables, assembled as
the kernels do: fma(-w^2, M, C) with M = M0 + (A_w + op_A_w), C0 exactly, and w (B0 + B_drag + (B_w + op_B_w)).  Then
the normwise backward error eta <= ETA_C * n * u (u = 2^-53), and the forward error against the solution refined with
exact residuals <= FWD_C * n * kappa_inf(Z) * u, and <= FWD_CEIL on bins with kappa_inf(Z) <= 1e4, on every bin.

Inputs: cfg3 (BEM tables, so F_BEM is part of the load) regridded to each kernel's shape, drag-free (node_cd_* = 0: B_drag
and F_drag are zero and every bin is linear).
  * Planted impedances.  M0, B0 and C0 are zero and A_w = -Re Zt / w^2, B_w = Im Zt / w carry a target Zt, so that every
    kernel's assembly reduces to RN(-w^2 A_w) + i RN(w B_w), which NumPy reproduces bit for bit: the restated pivot rule
    sees the kernel's own Z.  Bin i belongs to a family by i % 8:
      0-4  pivot orders: Zt = P^T L U (|l| <= 0.5 in |re| + |im|, real diagonal of U), built so that the pivot of step k
           is row k + i % (6 - k).  All 15 exchanges (k, r > k) occur in every kernel, and neighbouring bins -- the lanes of
           a warp, and the bins one thread solves (t, t + T; the pair k_rao_fused2 holds) -- pivot differently;
      5    exact ties: at step k (columns < k upper triangular, exact zeros below), rows r1 < r2 (< r3) of column k hold
           (a, b), (b, a) and (a + b, 0) with |re| + |im| equal to the last bit; row r1 must win.  All 15 (k, r1) occur;
      6    ill conditioning: a rank-one perturbation delta of a singular matrix, kappa from 1e6 to 1e12;
      7    graded rows: force rows around 1e6 against moment rows around 1e12.
  * A physical case: cfg3 drag-free with C0[5, 5] = 0 (no yaw restoring: the lowest bins are nearly singular) and B_w
    zeroed at the bins around its heave and pitch resonances.
  * Operating points: the planted tables carried by op_A_w / op_B_w instead of A_w / B_w (op_impedance, which the fused
    kernels keep apart from their table branch); the result must equal the table branch bit for bit.
  * An exactly singular bin (a zero column) in one unit of a three-design launch: RAFTK_FLAG_SINGULAR in that unit's
    status word 2, every other unit bit-identical to the launch without it.

Kernels: fused128, fused256, fused256 with F0 in global memory, fused2-cluster, fused2-grid and v1 both natural and
forced, each reached by a shape the planner itself picks it for (asserted through solver.last_dispatch()), with ragged
slices.  Without a GPU the test proves, with the restated pivot rule on each kernel's own bin layout, that the inputs
reach those edges, checks the refinement against a 50-digit mpmath LU solve, and checks that the shipped fixtures take
no exchange outside (0, 4), (1, 3), (2, 4), (2, 5), (3, 5), (4, 5) (the seven with a case table take four of them), which
is why the planted inputs exist.

Measured on an H100 80GB HBM3 (700 W limit), over every test of this file: worst eta / (n u) = 0.308, worst
forward error / (n kappa u) = 0.194, worst forward error on bins with kappa <= 1e4 = 3.21e-15.  The bounds
keep about 10x of margin.

Scaling.  M0, B0, C0, A_w and B_w times 2^s: at s = 300 and 560, with the load unchanged, Xi must be 2^-s times the
unscaled Xi bit for bit; at s = -300 and -560 the explicit wave amplitudes zeta are scaled by 2^s as well, so the load
scales with Z and Xi must keep its bits.  Status flags stay 0.  (The pass count may differ: the convergence test
|d| < tol |x| + tol^2 has an absolute term.)  s = +-560 is a known defect, marked xfail(strict=True) so that it flips when
fixed: solve6 forms each pivot reciprocal from |p|^2, which overflows above |p| ~ 1.3e154 (a zero reciprocal: every Xi
comes out 0) and underflows below 1.5e-154 (NaN, RAFTK_FLAG_NAN), on every rigid kernel.  No SI-unit design gets near either.  The
fix of the dense LUs (raftk_misc.cuh piv_scale: p scaled by a power of two before |p|^2) is exact under scaling, but
applied to solve6 it moved the last bit of about 7 % of cfg2's Xi (the drag-free one-pass solve kept its bits, so the
code around the solve compiled differently) and cost 0.7 % of cfg2's step time, within the run-to-run spread; it is not
applied until it can be made bit-neutral."""
import math

import numpy as np
import pytest

from conftest import load_golden
from test_dispatch_solve import CLUSTER, FORCE, GRID, _check_record, _regrid_bem
from test_farm_edges import _errors, _pivot_rows, _refined, _residual, _two_prod

gpu = pytest.mark.gpu
U = 2.0 ** -53
N = 6
ETA_C = 3.0                  # eta <= ETA_C * n * u
FWD_C = 2.0                  # forward error <= FWD_C * n * kappa * u
FWD_CEIL = 3e-14             # forward error on bins with kappa_inf(Z) <= 1e4
RAFTK_FLAG_SINGULAR = 2
S = 2.0 ** 27                # planted impedance scale (~1.3e8, a platform's heave / surge order)
KAPPAS = [1e6, 1e7, 1e8, 1e9, 1e10, 1e11, 1e12]
EXCHANGES = {(k, r) for k in range(5) for r in range(k + 1, 6)}
TIES = {(k, r) for k in range(5) for r in range(k, 5)}           # (step, first tied row); a second tied row follows
FIXTURE_EXCHANGES = {(0, 4), (1, 3), (2, 4), (2, 5), (3, 5), (4, 5)}
FIXTURES = ["cfg1_OC3spar", "cfg2_VolturnUS-S_nw64", "cfg3_OC4semi-WAMIT_nw128", "test_OC3spar", "test_VolturnUS-S",
            "test_OC4semi-WAMIT_Coefs", "pin_VolturnUS-S-pointInertia"]

# (design, nw, cluster_size, environment, kernel, f0_global), as test_dispatch_solve.SHAPES picks them for cfg3
KERNELS = [("cfg3", 201, 2, {}, "fused128", False), ("cfg3", 333, 2, {}, "fused256", False),
           ("cfg3", 451, 1, {}, "fused256", True), ("cfg3", 501, 2, CLUSTER, "fused2-cluster", False),
           ("cfg3", 501, 2, GRID, "fused2-grid", False), ("cfg3", 601, 1, {}, "v1", False),
           ("cfg3", 333, 2, FORCE, "v1", False)]
KID = ["fused128", "fused256", "fused256-f0g", "fused2-cluster", "fused2-grid", "v1", "v1-forced"]
SEA = dict(Hs=np.array([6.0, 3.0]), Tp=np.array([12.0, 8.0]), gamma=np.zeros(2), beta_deg=np.array([0.0, 70.0]),
           spec=np.zeros(2, dtype=np.int32))
NC = 2


# ---- inputs ---------------------------------------------------------------------------------------------------------
def _cfg3(nw):
    P = _regrid_bem(load_golden("cfg3_OC4semi-WAMIT_nw128")[1], nw)
    for k in ("node_cd_q", "node_cd_p1", "node_cd_p2"):
        P[k] = np.zeros_like(P[k])
    return P


def _family(i):
    return ("piv", "piv", "piv", "piv", "piv", "tie", "ill", "graded")[i % 8]


def _pivot_seq(i):
    return [k + i % (6 - k) for k in range(5)]


def _crand(rng, shape, half):
    return rng.uniform(-half, half, size=shape) + 1j * rng.uniform(-half, half, size=shape)


def _zt_pivot(i, rng):
    """P^T L U: the pivot of step k is row _pivot_seq(i)[k], every other candidate at most half of it in |re| + |im|."""
    L = np.eye(N, dtype=complex) + np.tril(_crand(rng, (N, N), 0.25), -1)
    Um = np.triu(_crand(rng, (N, N), 0.5), 1) + np.diag(rng.uniform(1.0, 2.0, N))
    A = L @ Um
    seq = _pivot_seq(i)
    for k in reversed(range(5)):
        A[[k, seq[k]]] = A[[seq[k], k]]
    return S * A


def _tie_config(j):
    return sorted(TIES)[j % len(TIES)]


def _zt_tie(j, rng):
    """Step k of tie configuration j sees column k untouched (columns < k upper triangular, exact zeros below); its rows
    r1, r1 + 1 (, r1 + 2) hold the tied values (_tie_values, which _plant makes exact), the others at most 0.3 of them.
    -> (Zt, tied rows, k)."""
    k, r1 = _tie_config(j)
    A = _crand(rng, (N, N), 0.15)
    for c in range(k):
        A[c + 1:, c] = 0.0
        A[c, c] = 2.0
    for c in range(k + 1, N):
        A[c, c] += 1.0
    rows = list(range(r1, min(r1 + 3, N)))
    A[rows, k] = 1.0
    return S * A, rows, k


def _tie_values(j, rows, t, b):
    """(row, value) of the tied rows: (a, b), (b, a) and (a + b, 0) times S t, a = 1 - b, in an order that turns with j."""
    a = 1.0 - b
    pats = [complex(a, b), complex(b, a), complex(1.0, 0.0)]
    pats = pats[j % 3:] + pats[:j % 3]
    return [(r, S * t * v) for r, v in zip(rows, pats)]


def _zt_ill(j, rng):
    """U diag(2, 1.5, 1.2, 1, 0.8, delta) V^H, delta = 2 / kappa: a rank-one perturbation of a singular matrix."""
    Q1, _ = np.linalg.qr(_crand(rng, (N, N), 1.0))
    Q2, _ = np.linalg.qr(_crand(rng, (N, N), 1.0))
    s = np.array([2.0, 1.5, 1.2, 1.0, 0.8, 2.0 / KAPPAS[j % len(KAPPAS)]])
    return S * (Q1 * s) @ Q2.conj().T


def _zt_graded(rng):
    G = 2.0 * np.eye(N) + _crand(rng, (N, N), 0.6)
    return np.array([1e6] * 3 + [1e12] * 3)[:, None] * G


def _preimage(f, x, y0):
    """A double y within 8 ulps of y0 with f(y) == x exactly, or None."""
    ys, lo, hi = [y0], y0, y0
    for _ in range(8):
        lo, hi = np.nextafter(lo, -np.inf), np.nextafter(hi, np.inf)
        ys += [lo, hi]
    for y in ys:
        if f(y) == x:
            return y
    return None


def _plant(nw):
    """The planted design on the nw-bin grid: (design, [family per bin], {bin: info}).  info: the pivot sequence
    (pivot orders), (k, r1) (ties), the kappa target (ill) or None (graded)."""
    P = _cfg3(nw)
    P["M0"], P["B0"], P["C0"] = np.zeros((6, 6)), np.zeros((6, 6)), np.zeros((6, 6))
    w = np.asarray(P["w"], dtype=float)
    A_w, B_w = np.zeros((6, 6, nw)), np.zeros((6, 6, nw))
    fams, info = [], {}
    for i in range(nw):
        rng = np.random.default_rng(1000 + i)
        fam = _family(i)
        j = i // 8
        w1 = float(w[i])
        w2 = w1 * w1
        if fam == "piv":
            Zt, info[i] = _zt_pivot(i, rng), _pivot_seq(i)
        elif fam == "ill":
            Zt, info[i] = _zt_ill(j, rng), KAPPAS[j % len(KAPPAS)]
        elif fam == "graded":
            Zt, info[i] = _zt_graded(rng), None
        else:
            Zt, rows, k = _zt_tie(j, rng)
            info[i] = _tie_config(j)
        A_w[:, :, i] = -Zt.real / w2
        B_w[:, :, i] = Zt.imag / w1
        if fam == "tie":
            for c in range(k):                              # exact zeros below the diagonal of columns < k
                A_w[c + 1:, c, i] = 0.0
                B_w[c + 1:, c, i] = 0.0
            # tied values that both maps reach exactly: RN(-w^2 A) skips doubles where w^2 > 1, RN(w B) where w > 1
            for t, b in ((t, b) for b in np.arange(1, 32) / 64.0 for t in 1.0 + np.arange(64) / 64.0):
                hit = [(r, _preimage(lambda a: -(w2 * a), v.real, -v.real / w2), _preimage(lambda y: w1 * y, v.imag, v.imag / w1))
                       for r, v in _tie_values(j, rows, t, b)]
                if all(a is not None and y is not None for _, a, y in hit):
                    break
            else:
                raise AssertionError("no exact tie at bin %d" % i)
            for r, a, b in hit:
                A_w[r, k, i], B_w[r, k, i] = a, b
        fams.append(fam)
    P["A_w"], P["B_w"] = A_w, B_w
    return P, fams, info


def _physical(nw):
    """cfg3 drag-free, C0[5, 5] = 0, B_w zeroed within 3 bins of the heave and pitch resonances."""
    P = _cfg3(nw)
    P["C0"] = np.array(P["C0"], dtype=float)
    P["C0"][5, 5] = 0.0
    w = np.asarray(P["w"], dtype=float)
    B_w = np.array(P["B_w"], dtype=float)
    for d in (2, 4):
        r = P["C0"][d, d] - w ** 2 * (P["M0"][d, d] + P["A_w"][d, d])
        for i in np.nonzero(np.sign(r[1:]) != np.sign(r[:-1]))[0]:
            B_w[:, :, max(0, i - 3):i + 4] = 0.0
    P["B_w"] = B_w
    return P


def _singular(P, i=7, col=2):
    """P with column col of Z exactly zero at bin i."""
    Q = dict(P, A_w=np.array(P["A_w"]), B_w=np.array(P["B_w"]))
    Q["A_w"][:, col, i] = -np.asarray(P["M0"])[:, col]
    Q["B_w"][:, col, i] = -np.asarray(P["B0"])[:, col]
    return Q


def _layout(shape):
    """The kernel's bin layout: (bins per CTA, threads per CTA); a CTA's thread t solves local bins t, t + T, ..."""
    nw, cs, kernel = shape[1], shape[2], shape[4]
    return -(-nw // cs), (256 if kernel == "fused256" else 128)


def _neighbours(nw, nwl, T):
    """Bin pairs of one warp's neighbouring lanes, and of one thread."""
    lanes = [(i, i + 1) for i in range(nw - 1) if i // nwl == (i + 1) // nwl and (i % nwl) // 32 == ((i + 1) % nwl) // 32]
    thread = [(i, i + T) for i in range(nw - T) if i // nwl == (i + T) // nwl]
    return lanes, thread


# ---- the reference ----------------------------------------------------------------------------------------------------
def _fma(a, b, c):
    """Correctly rounded a * b + c, elementwise (Dekker's product, then math.fsum of the three exact terms)."""
    p, e = _two_prod(a, b)
    shape = np.broadcast(p, c).shape
    p, e, c = (np.broadcast_to(x, shape).ravel() for x in (p, e, c))
    return np.array([math.fsum(t) for t in zip(p, e, c)]).reshape(shape)


def _assemble(P, out, d, ops=None):
    """Z [nC, nw, 6, 6] and F [nC, nw, 6] of design d as the kernels build them, from the solver's outputs."""
    w = np.asarray(P["w"], dtype=float)
    nw = len(w)
    Z = np.zeros((NC, nw, 6, 6), dtype=complex)
    F = np.zeros((NC, nw, 6), dtype=complex)
    for c in range(NC):
        A = np.moveaxis(np.asarray(P["A_w"], dtype=float), -1, 0)
        B = np.moveaxis(np.asarray(P["B_w"], dtype=float), -1, 0)
        if ops is not None:
            A = A + np.moveaxis(ops["A_w"][ops["op"][c]], -1, 0)
            B = B + np.moveaxis(ops["B_w"][ops["op"][c]], -1, 0)
        M = np.asarray(P["M0"], dtype=float)[None] + A
        Bt = (np.asarray(P["B0"], dtype=float) + out["B_drag"][d, c])[None] + B
        Z[c] = _fma(-(w * w)[:, None, None], M, np.asarray(P["C0"], dtype=float)[None]) + 1j * (w[:, None, None] * Bt)
        F[c] = (out["F_drag"][d, c] + out["F_iner"][d, c] + out["F_BEM"][d, c]).T
    return Z, F


WORST = {"eta": 0.0, "fwd": 0.0, "ceil": 0.0}


def _check(Z, F, X, tag):
    """X [nC, 6, nw] against the reference on every (case, bin)."""
    for c in range(Z.shape[0]):
        for iw in range(Z.shape[1]):
            eta, fwd, kappa = _errors(Z[c, iw], F[c, iw], X[c, :, iw])
            WORST["eta"] = max(WORST["eta"], eta / (N * U))
            WORST["fwd"] = max(WORST["fwd"], fwd / (N * kappa * U))
            assert eta <= ETA_C * N * U, (tag, c, iw, eta / (N * U))
            assert fwd <= FWD_C * N * kappa * U, (tag, c, iw, fwd, kappa)
            if kappa <= 1e4:
                WORST["ceil"] = max(WORST["ceil"], fwd)
                assert fwd <= FWD_CEIL, (tag, c, iw, fwd, kappa)
    print("%s: worst eta/(n u) %.3g, fwd/(n kappa u) %.3g, fwd at kappa <= 1e4 %.3g" % (tag, WORST["eta"], WORST["fwd"], WORST["ceil"]))


def _planted_Z(P):
    """The kernels' Z of a planted design (M0 = B0 = C0 = 0, drag-free): RN(-w^2 A_w) + i RN(w B_w), exactly."""
    w = np.asarray(P["w"], dtype=float)
    return np.moveaxis(-((w * w) * P["A_w"]) + 1j * (w * P["B_w"]), -1, 0)


# ---- without a GPU: the inputs reach the edges -------------------------------------------------------------------------
@pytest.mark.parametrize("shape", KERNELS, ids=KID)
def test_planted_bins_reach_every_pivot_order_and_tie(shape):
    """With the kernels' pivot rule restated on the planted Z: every exchange (k, r > k) and every tie (k, r1) occurs; the
    pivot orders are the planned ones with a margin of at least 0.25 between the top two candidates; ties are exact and
    go to the first row; neighbouring bins of the kernel's layout pivot differently; the kappa targets are met."""
    nw = shape[1]
    P, fams, info = _plant(nw)
    Z = _planted_Z(P)
    assert np.array_equal(Z.real, _fma(-(P["w"] ** 2)[:, None, None], np.moveaxis(P["A_w"], -1, 0), 0.0))
    exch, ties, seqs, kap = set(), set(), {}, []
    for i in range(nw):
        rows = _pivot_rows(Z[i])
        seqs[i] = tuple(p for _, p, _ in rows[:5])
        if fams[i] == "piv":
            assert list(seqs[i]) == info[i], (i, seqs[i], info[i])
            assert min(m for _, _, m in rows[:5]) > 0.25, (i, rows)
            exch |= {(k, p) for k, p in enumerate(seqs[i]) if p > k}
        elif fams[i] == "tie":
            k, r1 = info[i]
            assert rows[k][1] == r1 and rows[k][2] == 0.0, (i, rows[k], info[i])
            ties.add((k, r1))
        elif fams[i] == "ill":
            kappa = np.linalg.cond(Z[i], np.inf)
            assert info[i] / 3 <= kappa <= info[i] * 30, (i, kappa, info[i])
            kap.append(kappa)
        else:
            assert np.linalg.cond(Z[i], np.inf) > 1e5
    assert exch == EXCHANGES and ties == TIES
    nwl, T = _layout(shape)
    lanes, thread = _neighbours(nw, nwl, T)
    lp = [(a, b) for a, b in lanes if fams[a] == fams[b] == "piv"]
    tp = [(a, b) for a, b in thread if fams[a] == fams[b] == "piv"]
    assert lp and bool(tp) == (nwl > T) and all(seqs[a] != seqs[b] for a, b in lp + tp)   # threads own one bin up to T
    assert max(kap) >= 1e12 / 3 and min(kap) <= 3e6
    print("%s nw=%d cs=%d T=%d: %d/15 exchanges, %d/15 ties (first row wins), %d lane pairs and %d thread pairs pivot "
          "differently, kappa_inf %.1e .. %.1e" % (shape[4], nw, shape[2], T, len(exch), len(ties), len(lp), len(tp), min(kap), max(kap)))


def test_physical_case_has_no_yaw_restoring_and_undamped_resonances():
    """The physical case zeroes C0[5, 5] and B_w at 13 or more bins around the heave and pitch resonances."""
    for nw in sorted({k[1] for k in KERNELS}):
        P = _physical(nw)
        assert P["C0"][5, 5] == 0.0 and np.count_nonzero(np.all(P["B_w"] == 0, axis=(0, 1))) >= 13, nw


def test_reference_against_mpmath():
    """The refined reference equals a 50-digit mpmath LU solve to 1e-30 on a pivot-order, a tie, a kappa = 1e12 and a
    graded bin, and the exact residual equals mpmath's."""
    import mpmath
    mpmath.mp.dps = 50
    P, fams, info = _plant(201)
    Z = _planted_Z(P)
    rng = np.random.default_rng(3)
    picks = [fams.index("piv"), fams.index("tie"), next(i for i in range(201) if fams[i] == "ill" and info[i] == 1e12),
             fams.index("graded")]
    for i in picks:
        F = (rng.normal(size=6) + 1j * rng.normal(size=6)) * 1e6
        xs = _refined(Z[i], F)
        M = mpmath.matrix([[mpmath.mpc(complex(v)) for v in row] for row in Z[i]])
        xm = mpmath.lu_solve(M, mpmath.matrix([mpmath.mpc(complex(v)) for v in F]))
        ref = [sum((mpmath.mpc(complex(x[r])) for x in xs), mpmath.mpc(0)) for r in range(6)]
        scale = max(abs(v) for v in xm)
        assert max(abs(ref[r] - xm[r]) for r in range(6)) / scale < 1e-30, (i, fams[i])
        x0 = xs[0] * (1 + 1e-9)
        res = _residual(Z[i], F, [x0])
        rm = [mpmath.mpc(complex(F[r])) - mpmath.fsum(M[r, j] * mpmath.mpc(complex(x0[j])) for j in range(6)) for r in range(6)]
        assert max(abs(complex(rm[r]) - res[r]) / max(abs(rm[r]), 1e-300) for r in range(6)) < 1e-15


def test_fixtures_reach_six_exchanges():
    """On the oracle's Z of every case of the shipped rigid fixtures with a case table: column 0 pivots on row 4 and column
    1 on row 3 in all but a few bins, no exact tie occurs, and no exchange outside six of the 15 is taken.  A select written wrong for any other
    exchange, or a tie broken the other way, would pass a suite that tests the solve on the fixtures alone."""
    from oracle import oracle as orc
    orc.build()
    seen, n_bins, n_04 = set(), 0, 0
    for name in FIXTURES:
        G, P = load_golden(name)
        od = orc.OracleDesign(P)
        for Hs, Tp, beta in G["ref_run_solve_cases"]:
            _, _, Z, _ = orc.solve_dynamics(od, 0, Hs, Tp, 0.0, beta, nIter=int(G["n_iter"]), want_Z=True)
            for z in Z:
                rows = _pivot_rows(z)
                n_bins += 1
                n_04 += rows[0][1] == 4 and rows[1][1] == 3
                assert min(m for _, _, m in rows[:5]) > 0.0, (name, rows)
                seen |= {(k, p) for k, p, _ in rows if p > k}
    assert seen <= FIXTURE_EXCHANGES and {(0, 4), (1, 3), (3, 5), (4, 5)} <= seen, sorted(seen)
    assert n_04 >= 0.99 * n_bins, (n_04, n_bins)
    print("fixtures: exchanges %s of 15; column 0 on row 4 and column 1 on row 3 in %d of %d bins" % (sorted(seen), n_04, n_bins))


# ---- on the GPU ---------------------------------------------------------------------------------------------------------
def _run(monkeypatch, shape, designs, cases):
    from raft_b200 import solver
    for k in ("RAFTK_FORCE_V1", "RAFTK_FUSED2_XCHG", "RAFTK_NO_DIRECT_D2H"):
        monkeypatch.delenv(k, raising=False)
    for k, v in shape[3].items():
        monkeypatch.setenv(k, v)
    out = solver.solve_dynamics(solver.DesignBatch(designs), cases, n_iter=10, cluster_size=shape[2],
                                want=("Xi", "status", "B_drag", "F_drag", "F_iner", "F_BEM"))
    _check_record(solver.last_dispatch(), shape)
    return out


def _zeta(nw, s=0):
    return np.full((NC, nw), np.ldexp(0.5, s))


@gpu
@pytest.mark.parametrize("shape", KERNELS, ids=KID)
def test_planted_and_physical_vs_reference(shape, monkeypatch):
    """Designs [planted, physical, planted]: every bin of both within the bounds, the third unit's bits those of the
    first; then the third design with a zero column at one bin: RAFTK_FLAG_SINGULAR there, the others' bits unchanged."""
    from raft_b200 import solver
    nw = shape[1]
    P, _, _ = _plant(nw)
    Q = _physical(nw)
    ct = solver.CaseTable(SEA, zeta=_zeta(nw))
    out = _run(monkeypatch, shape, [P, Q, P], ct)
    assert not np.any(out["status"][..., 2]), out["status"]
    assert not np.any(out["B_drag"]) and not np.any(out["F_drag"]) and np.any(out["F_BEM"])
    for d, D in ((0, P), (1, Q)):
        Z, F = _assemble(D, out, d)
        _check(Z, F, out["Xi"][d], "%s design %d" % (shape[4], d))
    assert np.array_equal(out["Xi"][2], out["Xi"][0])
    sing = _run(monkeypatch, shape, [P, Q, _singular(P)], ct)
    assert np.all(sing["status"][2, :, 2] & RAFTK_FLAG_SINGULAR), sing["status"][2]
    for k in ("Xi", "status"):
        assert np.array_equal(sing[k][:2], out[k][:2]), k


@gpu
@pytest.mark.parametrize("shape", KERNELS, ids=KID)
def test_operating_points_vs_reference(shape, monkeypatch):
    """The planted tables as one operating point shared by both cases, the design's own A_w / B_w zero: within the bounds,
    and bit-identical to the same tables in A_w / B_w."""
    from raft_b200 import solver
    nw = shape[1]
    P, _, _ = _plant(nw)
    ops = dict(op=np.zeros(NC, dtype=np.int32), A_w=P["A_w"][None], B_w=P["B_w"][None])
    P0 = dict(P, A_w=np.zeros_like(P["A_w"]), B_w=np.zeros_like(P["B_w"]))
    out = _run(monkeypatch, shape, [P0], solver.CaseTable(SEA, zeta=_zeta(nw), ops=ops))
    assert not np.any(out["status"][..., 2]), out["status"]
    Z, F = _assemble(P0, out, 0, ops=ops)
    _check(Z, F, out["Xi"][0], "%s operating point" % shape[4])
    tab = _run(monkeypatch, shape, [P], solver.CaseTable(SEA, zeta=_zeta(nw)))
    assert np.array_equal(out["Xi"], tab["Xi"])


OUT_OF_RANGE = pytest.mark.xfail(strict=True, reason="solve6 forms pivot reciprocals from |p|^2: zero above |p| ~ 1.3e154, "
                                  "inf below 1.5e-154 (module docstring)")
SCALES = (pytest.param(-560, marks=OUT_OF_RANGE), -300, 300, pytest.param(560, marks=OUT_OF_RANGE))


@gpu
@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("shape", KERNELS, ids=KID)
def test_power_of_two_scaling_is_exact(shape, s, monkeypatch):
    """Designs [planted, physical] with M0, B0, C0, A_w and B_w times 2^s (and zeta times 2^s for s < 0): Xi times 2^-s
    (the unscaled Xi for s < 0) bit for bit, flags 0."""
    from raft_b200 import solver
    nw = shape[1]
    designs = [_plant(nw)[0], _physical(nw)]
    base = _run(monkeypatch, shape, designs, solver.CaseTable(SEA, zeta=_zeta(nw)))
    X0 = base["Xi"]
    x = np.abs(np.concatenate([X0.real.ravel(), X0.imag.ravel()]))
    assert x[x > 0].min() * 2.0 ** -max(s, 0) > 1e-290
    scaled = [dict(D, **{k: np.ldexp(np.asarray(D[k], dtype=float), s) for k in ("M0", "B0", "C0", "A_w", "B_w")}) for D in designs]
    out = _run(monkeypatch, shape, scaled, solver.CaseTable(SEA, zeta=_zeta(nw, min(s, 0))))
    assert not np.any(out["status"][..., 2]), np.unique(out["status"][..., 2])
    ref = X0 if s < 0 else np.ldexp(X0.real, -s) + 1j * np.ldexp(X0.imag, -s)
    bad = ~((out["Xi"] == ref) | (np.isnan(out["Xi"]) & np.isnan(ref)))
    assert not np.any(bad), "%d of %d components differ, e.g. %r against %r" % (
        bad.sum(), bad.size, out["Xi"][bad][:2], ref[bad][:2])
