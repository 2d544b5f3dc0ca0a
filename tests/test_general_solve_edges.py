"""The generalised-DOF solves (raftk_general.cuh: k_gen_solve_blocked with its FD and OP instantiations, and
k_gen_train_solve) against a high-precision reference of the same system, on inputs that reach every pivot pattern of the
LU's thread layout, exact ties, ill-conditioned and graded bins, wave trains, a design axis, an exactly
singular bin and the ends of the exponent range, at n = 9, 40, 150 and 256.

The reference is the one of test_farm_edges and does not share the kernels' algorithm: the residual of the kernel's x is
computed exactly, the normwise backward error eta <= ETA_C * n * u (u = 2^-53) on every bin, and the forward error against
the solution refined with exact residuals <= FWD_C * n * kappa_inf(Z) * u, and <= FWD_CEIL on bins with kappa_inf(Z) <= 1e4,
on the bins test_farm_edges._sample picks (every bin at n = 9).

Inputs whose Z and F the kernels build exactly.  general_synth.design(n, nw) with every node's node_Imat, node_a_i and drag
coefficients zero (B_drag = F_drag = 0, F_iner = F_BEM + 0), M = B = C = 0 and the impedance planted on a full fd support
through A_w = -Re Zt / w^2, B_w = Im Zt / w: the kernels' Z is RN(-w^2 A_w) + i RN(w B_w), which NumPy reproduces bit for bit,
so the restated pivot rule sees the kernels' own Z.  The load is a BEM table (dense T0, explicit zeta); the F_BEM the call
returns is the kernels' right-hand side.  Drag-free, every pass solves the same system.  Bin i belongs to a family by i % 8:
  0-2  planted pivot sequences Zt = P^T L U, every other candidate at most 1/2 of the pivot in |re| + |im|: the pivot of
       step k is row k, row k + 1, a row in a later 8-column panel, a row 32-127 below (another warp), a row >= 128 below
       (the blocked kernel's second trip) or the last row, in turn;
  3-4  dominant pivots: the same with every other candidate at most 1e-6 of the pivot, so that any other choice leaves a
       backward error far above the bound;
  5    exact ties at one step k (columns < k upper triangular, exact zeros below) between rows of one warp, of different
       warps, and rows one thread of the blocked kernel reads on two trips; the first row must win;
  6    ill conditioning: a rank-one perturbation of a singular matrix, kappa_2 from 1e6 to 1e12;
  7    graded rows: translations 1e6, rotations 1e9, modal rows 1e-3 .. 1e9.
nw = 24 bins (16 at n = 256).  A physical case: general_synth's design with rotor and BEM tables on a support that crosses
the panels, drag-free, B_w zeroed within two bins of a resonance; its Z restated with an exact fma.

On the GPU, for each n (the LU kernel asserted through solver.last_dispatch()):
  * a train table (case 0 with two trains of different headings, case 1 with one): every primary and every secondary train
    (k_gen_train_solve: the primary's L, U and pivot rows with the secondary's own F_BEM) within the bounds;
  * the planted tables carried by op_A_w / op_B_w with A_w = B_w = 0 (the OP instantiations): Xi and status bit for bit;
  * a two-design batch (general_solve_dynamics_batch) with different planted tables: each design against its own reference;
  * A_w and B_w times 2^s, s in {-560, -300, 300, 560}, the load unchanged: Xi times 2^-s bit for bit; for s < 0 zeta times
    2^s as well, and Xi keeps its bits.  Status flags stay 0 (the pass count may differ: the convergence test
    |d| < tol (|x| + tol) has an absolute term).  Every pivot reciprocal and back-substitution quotient is formed at the
    pivot's scale (raftk_common.cuh piv_recip / piv_div), so |p|^2 neither overflows (above |p| ~ 1.3e154) nor underflows
    (below 1.5e-154);
  * one case of a three-case call with a zero column at one bin: RAFTK_FLAG_SINGULAR in its status word 2, the other cases
    bit-identical to the call without it, and solver.raise_on_flags raises.
Without a GPU the suite proves with the restated pivot rule that every pattern occurs at each n in the kernel's layout,
that a wrong pivot on a dominant bin leaves a backward error far above the bound, that the refinement agrees with a 50-digit
mpmath LU solve, and that every scaled input stays in the normal range.

Measured on an H100 80GB HBM3 (700 W limit), over every test of this file: worst eta / (n u) = 0.202, worst forward error
/ (n kappa u) = 0.221, worst forward error on bins with kappa <= 1e4 = 2.14e-15.  The bounds keep about 10x of margin.
Before the pivot scaling, s = +-560 failed on both kernels at every n (Xi zero above, NaN below), and a zero pivot was
reported as RAFTK_FLAG_NAN alone."""
import hashlib
import math

import numpy as np
import pytest

import general_synth as gs
from test_farm_edges import _pivot_rows, _refined, _residual, _sample
from test_rigid_solve_edges import _fma, _preimage, _tie_values

gpu = pytest.mark.gpu
U = 2.0 ** -53
ETA_C = 2.0                  # eta <= ETA_C * n * u
FWD_C = 2.0                  # forward error <= FWD_C * n * kappa * u
FWD_CEIL = 2e-14             # forward error on bins with kappa_inf(Z) <= 1e4
RAFTK_FLAG_SINGULAR = 2
S = 2.0 ** 27                # planted impedance scale, as test_rigid_solve_edges
SIZES = (9, 40, 150, 256)
KERNELS = [("gen-blocked", 128)]                               # (kernel, threads per CTA)
KID = ["blocked"]
FAMILIES = ("piv", "piv", "piv", "dom", "dom", "tie", "ill", "graded")
LMAX = {"piv": 0.5, "dom": 1e-6}                               # largest other candidate / pivot, in |re| + |im|
SCALES = (-560, -300, 300, 560)


def _nw(n):
    return 16 if n == 256 else 24


# ---- inputs ---------------------------------------------------------------------------------------------------------
def _crand(rng, shape, half):
    return rng.uniform(-half, half, size=shape) + 1j * rng.uniform(-half, half, size=shape)


def _pivot_seq(n, j):
    """Pivot row of every step k < n - 1 of planted bin j: the row itself, the next row, a row in the next 8-column panel, a
    row 32-127 below, one >= 128 below, the last row, in turn (an offset past the last row wraps into range)."""
    seq = []
    for k in range(n - 1):
        m = n - 1 - k
        opts = (0, 1, (k // 8 + 1) * 8 + k % 3 - k, 32 + (7 * k + 11 * j) % 96, 128 + (5 * k + 3 * j) % 128, m)
        o = opts[(k + j) % 6]
        seq.append(k + (o if o <= m else o % (m + 1)))
    return seq


def _zt_pivot(n, seq, lmax, rng):
    """P^T L U: the pivot of step k is row seq[k]; every other candidate of L's column k is at most lmax in |re| + |im|, one
    of them close to it, the rest small (so that L and U stay well conditioned at n = 256)."""
    L = np.eye(n, dtype=complex) + np.tril(_crand(rng, (n, n), 0.1 * lmax / math.sqrt(n)), -1)
    for k in range(n - 1):
        r = k + 1 + int(rng.integers(n - 1 - k))
        ph = rng.uniform(0.0, 2.0 * np.pi)
        L[r, k] = lmax * rng.uniform(0.8, 1.0) * complex(math.cos(ph), math.sin(ph)) / (abs(math.cos(ph)) + abs(math.sin(ph)))
    Um = np.triu(_crand(rng, (n, n), 0.3 / math.sqrt(n)), 1) + np.diag(rng.uniform(1.0, 2.0, n))
    A = L @ Um
    for k in reversed(range(n - 1)):
        A[[k, seq[k]]] = A[[seq[k], k]]
    return S * A


def _tie_configs(n):
    """(step k, offsets of the tied rows from k) of the tie bins at size n (one per tie bin, in order)."""
    return {9: [(0, (1, 2, 3)), (3, (1, 5)), (1, (0, 7))],
            40: [(0, (5, 37)), (2, (1, 33, 34)), (6, (0, 8, 33))],
            150: [(3, (2, 34, 130)), (0, (40, 130)), (10, (0, 1, 128))],
            256: [(3, (2, 34, 130)), (0, (40, 41, 130))]}[n]


def _zt_tie(n, k, offs, rng):
    """Step k sees column k untouched (columns < k upper triangular, exact zeros below); its rows k + offs are set to the tied
    values by _plant, every other candidate at most 0.3 of them."""
    A = _crand(rng, (n, n), 0.3 / math.sqrt(n))
    for c in range(k):
        A[c + 1:, c] = 0.0
        A[c, c] = 2.0
    for c in range(k + 1, n):
        A[c, c] += 1.0
    rows = [k + o for o in offs]
    A[rows, k] = 1.0
    return S * A, rows


def _zt_ill(n, kappa, rng):
    """U diag(2 .. 0.8, 2 / kappa) V^H: a rank-one perturbation of a singular matrix."""
    Q1, _ = np.linalg.qr(_crand(rng, (n, n), 1.0))
    Q2, _ = np.linalg.qr(_crand(rng, (n, n), 1.0))
    s = np.concatenate([np.linspace(2.0, 0.8, n - 1), [2.0 / kappa]])
    return S * (Q1 * s) @ Q2.conj().T


def _row_scales(n):
    """Translations 1e6, rotations 1e9, modal rows 1e-3, 1, 1e3, 1e6, 1e9 in turn."""
    return np.array([1e6] * 3 + [1e9] * 3 + [10.0 ** (-3 + 3 * ((r - 6) % 5)) for r in range(6, n)])


def _zt_graded(n, rng):
    return _row_scales(n)[:, None] * (2.0 * np.eye(n) + _crand(rng, (n, n), 1.0 / math.sqrt(n)))


def _plant(n, nw, seed=0):
    """Planted tables A_w, B_w [n, n, nw] and w on the design grid: (A_w, B_w, [family per bin], {bin: info}).  info: the
    pivot sequence (piv, dom), (k, tied rows) (tie), the kappa_2 target (ill), None (graded)."""
    w = np.asarray(gs.design(n, nw)[0]["w"], dtype=float)
    A_w, B_w = np.zeros((n, n, nw)), np.zeros((n, n, nw))
    fams = [FAMILIES[i % 8] for i in range(nw)]
    n_ill = fams.count("ill")
    kappas = np.logspace(6, 12, n_ill) if n_ill > 1 else np.array([1e12])
    info = {}
    for i in range(nw):
        rng = np.random.default_rng(100000 * seed + 1000 * n + i)
        fam, w1 = fams[i], float(w[i])
        w2 = w1 * w1
        j = fams[:i].count(fam)
        if fam in LMAX:
            info[i] = _pivot_seq(n, i)
            Zt = _zt_pivot(n, info[i], LMAX[fam], rng)
        elif fam == "ill":
            info[i] = float(kappas[j])
            Zt = _zt_ill(n, info[i], rng)
        elif fam == "graded":
            info[i], Zt = None, _zt_graded(n, rng)
        else:
            k, offs = _tie_configs(n)[j]
            Zt, rows = _zt_tie(n, k, offs, rng)
            info[i] = (k, rows)
        A_w[:, :, i] = -Zt.real / w2
        B_w[:, :, i] = Zt.imag / w1
        if fam == "tie":
            for c in range(k):                              # exact zeros below the diagonal of columns < k
                A_w[c + 1:, c, i] = 0.0
                B_w[c + 1:, c, i] = 0.0
            # tied values that both maps reach exactly: RN(-w^2 A) skips doubles where w^2 > 1, RN(w B) where w > 1
            for t, b in ((t, b) for b in np.arange(1, 32) / 64.0 for t in 1.0 + np.arange(64) / 64.0):
                hit = [(r, _preimage(lambda a: -(w2 * a), v.real, -v.real / w2), _preimage(lambda y: w1 * y, v.imag, v.imag / w1))
                       for r, v in _tie_values(j + seed, rows, t, b)]
                if all(a is not None and y is not None for _, a, y in hit):
                    break
            else:
                raise AssertionError("no exact tie at bin %d" % i)
            for r, a, y in hit:
                A_w[r, k, i], B_w[r, k, i] = a, y
    return A_w, B_w, fams, info


def _planted_Z(w, A_w, B_w):
    """The kernels' Z [nw, n, n] of planted tables (M = B = C = 0, drag-free): RN(-w^2 A_w) + i RN(w B_w), exactly."""
    return np.moveaxis(-((w * w) * A_w) + 1j * (w * B_w), -1, 0)


def _drag_free(P):
    P = dict(P)
    for k in ("node_Imat", "node_a_i", "node_Cd_q", "node_Cd_p1", "node_Cd_p2", "node_Cd_End"):
        P[k] = np.zeros_like(np.asarray(P[k], dtype=float))
    return P


def _design(n, seed=0):
    """The planted design: dict(P, M, B, Cm, fd) with M = B = C = 0 and the planted tables on the full support, and
    (fams, info)."""
    nw = _nw(n)
    P, M, B, _ = gs.design(n, nw)
    fd = gs.fd_tables(P, M, B, np.arange(n), seed=seed, bem="table", rotor=False)
    A_w, B_w, fams, info = _plant(n, nw, seed)
    fd.update(fd_idx=np.arange(n, dtype=np.int32), A_w=A_w, B_w=B_w)
    Z0 = np.zeros((n, n))
    return dict(P=_drag_free(P), M=Z0, B=Z0, Cm=Z0, fd=fd), fams, info


def _resonance(w, M, C):
    """(DOF, bin) of the first DOF whose C - w^2 M (M [n, n, nw]) changes sign between two bins."""
    for a in range(len(C)):
        r = C[a, a] - w ** 2 * M[a, a]
        hit = np.nonzero(np.sign(r[1:]) != np.sign(r[:-1]))[0]
        if len(hit):
            return int(a), int(hit[0])
    raise AssertionError("no resonance on the grid")


def _physical(n):
    """general_synth's design with rotor and BEM tables on support(n), drag-free, B_w zeroed within two bins of a
    resonance."""
    nw = _nw(n)
    P, M, B, Cm = gs.design(n, nw)
    idx = gs.support(n)
    fd = gs.fd_tables(P, M, B, idx, seed=n, bem="table")
    w = np.asarray(P["w"], dtype=float)
    Mw = M[:, :, None] + np.zeros(nw)
    Mw[np.ix_(idx, idx)] += fd["A_w"]
    a, i = _resonance(w, Mw, Cm)
    fd["B_w"] = np.array(fd["B_w"])
    fd["B_w"][:, :, max(0, i - 2):i + 3] = 0.0
    return dict(P=_drag_free(P), M=M, B=B, Cm=Cm, fd=fd), (a, i)


def _physical_Z(D):
    """The kernels' Z [nw, n, n] of a design with fd tables, drag-free (gen_impedance): fma(-w^2, M + A_w, C) + i w (B + B_w)
    on the support, fma(-w^2, M, C) + i w B elsewhere."""
    P, M, B, Cm, fd = D["P"], D["M"], D["B"], D["Cm"], D["fd"]
    w = np.asarray(P["w"], dtype=float)
    nw, idx = len(w), fd["fd_idx"]
    Mw, Bw = np.repeat(M[None], nw, axis=0), np.repeat(B[None], nw, axis=0)
    Mw[:, idx[:, None], idx[None, :]] = M[np.ix_(idx, idx)][None] + np.moveaxis(fd["A_w"], -1, 0)
    Bw[:, idx[:, None], idx[None, :]] = B[np.ix_(idx, idx)][None] + np.moveaxis(fd["B_w"], -1, 0)
    return _fma(-(w * w)[:, None, None], Mw, Cm[None]) + 1j * (w[:, None, None] * Bw)


def _trains():
    """Case 0 with two trains (headings 0 and 75 deg), case 1 with one: primary [0, 0, 2]."""
    from raft_b200 import packer
    table, _, _ = packer.pack_case_trains([
        dict(wave_spectrum=["JONSWAP"] * 2, wave_height=[6.0, 3.0], wave_period=[12.0, 8.0], wave_heading=[0.0, 75.0], wave_gamma=[0.0, 0.0]),
        dict(wave_spectrum="JONSWAP", wave_height=4.0, wave_period=10.0, wave_heading=30.0, wave_gamma=0.0)])
    return table


def _sea(nC):
    return dict(Hs=np.full(nC, 4.0), Tp=np.full(nC, 10.0), gamma=np.zeros(nC), beta_deg=np.linspace(0.0, 60.0, nC),
                spec=np.zeros(nC, dtype=np.int32))


def _zeta(nC, nw, s=0):
    """Unit-order wave amplitudes on every bin (JONSWAP's lowest bins are exactly zero)."""
    return np.full((nC, nw), np.ldexp(0.5, s))


# ---- the reference ----------------------------------------------------------------------------------------------------
WORST = {"eta": 0.0, "fwd": 0.0, "ceil": 0.0}
_REF = {}


def _errors_cached(z, f, x):
    """test_farm_edges._errors, the refined solution and kappa of each (Z, F) computed once: every call solves the
    same systems.  -> (eta, forward error, kappa_inf)."""
    key = hashlib.sha1(z.tobytes() + f.tobytes()).hexdigest()
    if key not in _REF:
        nZ = np.abs(z).sum(axis=1).max()
        _REF[key] = (_refined(z, f), nZ * np.abs(np.linalg.inv(z)).sum(axis=1).max())
    xs, kappa = _REF[key]
    d = x - xs[0]
    for t in xs[1:]:
        d = d - t
    return _eta(z, f, x), np.abs(d).max() / np.abs(xs[0]).max(), kappa


def _check(Z, F, X, tag):
    """X [n, nw] of one case against the reference of Z [nw, n, n], F [n, nw]: the backward error on every bin, the forward
    error on _sample's bins."""
    nw, n, _ = Z.shape
    fwd_bins = _sample(Z)
    for iw in range(nw):
        z, f, x = Z[iw], np.ascontiguousarray(F[:, iw]), X[:, iw]
        if iw not in fwd_bins:
            eta = _eta(z, f, x)
            WORST["eta"] = max(WORST["eta"], eta / (n * U))
            assert eta <= ETA_C * n * U, (tag, iw, eta / (n * U))
            continue
        eta, fwd, kappa = _errors_cached(z, f, x)
        WORST["eta"] = max(WORST["eta"], eta / (n * U))
        WORST["fwd"] = max(WORST["fwd"], fwd / (n * kappa * U))
        assert eta <= ETA_C * n * U, (tag, iw, eta / (n * U))
        assert fwd <= FWD_C * n * kappa * U, (tag, iw, fwd, kappa)
        if kappa <= 1e4:
            WORST["ceil"] = max(WORST["ceil"], fwd)
            assert fwd <= FWD_CEIL, (tag, iw, fwd, kappa)
    print("%s: worst eta/(n u) %.3g, fwd/(n kappa u) %.3g, fwd at kappa <= 1e4 %.3g" % (tag, WORST["eta"], WORST["fwd"], WORST["ceil"]))


def _lu_solve(Z, F, force=None):
    """x of Z x = F by LU with the kernels' pivot rule in double precision; ``force`` = (k, row) takes that row at step k."""
    A = np.array(Z, dtype=complex)
    b = np.array(F, dtype=complex)
    n = len(A)
    for k in range(n):
        t = np.abs(A[k:, k].real) + np.abs(A[k:, k].imag)
        p = k + int(np.argmax(t))
        if force is not None and force[0] == k:
            p = force[1]
        A[[k, p]] = A[[p, k]]
        b[[k, p]] = b[[p, k]]
        A[k + 1:, k] /= A[k, k]
        A[k + 1:, k + 1:] -= np.outer(A[k + 1:, k], A[k, k + 1:])
        b[k + 1:] -= A[k + 1:, k] * b[k]
    x = np.zeros(n, dtype=complex)
    for k in reversed(range(n)):
        x[k] = (b[k] - A[k, k + 1:] @ x[k + 1:]) / A[k, k]
    return x


def _eta(Z, F, x):
    r = _residual(Z, F, [x])
    return np.abs(r).max() / (np.abs(Z).sum(axis=1).max() * np.abs(x).max() + np.abs(F).max())


# ---- without a GPU: the inputs reach the edges -------------------------------------------------------------------------
def _pivot_cats(k, p, n, T):
    """What the pivot row p of step k is to a kernel whose CTA has T threads: thread (p - k) % T, trip (p - k) // T."""
    off = p - k
    cats = set()
    if off == 0:
        cats.add("self")
    if off == 1:
        cats.add("next")
    if p // 8 != k // 8:
        cats.add("panel")
    if (off % T) // 32 != 0:
        cats.add("warp")
    if off >= T:
        cats.add("trip")
    if p == n - 1:
        cats.add("last")
    return cats


def _tie_cats(k, rows, T):
    """'lanes' (two tied rows in one warp, different threads), 'warps' (in different warps), 'trips' (one thread, two trips)."""
    cats = set()
    for a in rows:
        for b in rows:
            if a < b:
                ta, tb = (a - k) % T, (b - k) % T
                cats.add("trips" if ta == tb else ("lanes" if ta // 32 == tb // 32 else "warps"))
    return cats


@pytest.mark.parametrize("n", SIZES)
def test_planted_bins_reach_every_pivot_pattern_and_tie(n):
    """With the kernels' pivot rule restated on the planted Z: the planned pivot rows with a margin of at least 0.45 (piv) or
    1 - 2e-6 (dom) between the top two candidates, covering, in each kernel's layout, the row itself, the next row, a row in
    another panel, another warp (n > 32), a second trip (the blocked kernel, n > 128) and the last row; exact ties won by the
    first row, between lanes, warps (n > 32) and trips (the blocked kernel, n > 128); the kappa targets of the ill bins."""
    nw = _nw(n)
    D, fams, info = _design(n)
    w = np.asarray(D["P"]["w"], dtype=float)
    Z = _planted_Z(w, D["fd"]["A_w"], D["fd"]["B_w"])
    assert np.array_equal(Z.real, _fma(-(w * w)[:, None, None], np.moveaxis(D["fd"]["A_w"], -1, 0), 0.0))
    cats = {T: set() for _, T in KERNELS}
    ties = {T: set() for _, T in KERNELS}
    kap = []
    for i in range(nw):
        rows = _pivot_rows(Z[i])
        if fams[i] in LMAX:
            assert [p for _, p, _ in rows[:-1]] == info[i], i
            margin = min(m for _, _, m in rows[:-1])
            assert margin > (0.45 if fams[i] == "piv" else 1.0 - 2e-6), (i, fams[i], margin)
            for T in cats:
                for k, p, _ in rows[:-1]:
                    cats[T] |= _pivot_cats(k, p, n, T)
        elif fams[i] == "tie":
            k, tied = info[i]
            assert rows[k][1] == tied[0] and rows[k][2] == 0.0, (i, rows[k], info[i])
            t = np.abs(Z[i, k:, k].real) + np.abs(Z[i, k:, k].imag)
            assert np.array_equal(np.nonzero(t == t.max())[0] + k, tied), (i, tied)
            assert np.sort(t)[-len(tied) - 1] <= 0.3 * t.max()
            for T in ties:
                ties[T] |= _tie_cats(k, tied, T)
        elif fams[i] == "ill":
            kappa = np.linalg.cond(Z[i])
            assert info[i] / 3 <= kappa <= info[i] * 3, (i, kappa, info[i])
            kap.append(kappa)
        else:
            assert np.linalg.cond(Z[i], np.inf) > 1e11
    for T in cats:
        want = {"self", "next", "panel", "last"} | ({"warp"} if n > 32 else set()) | ({"trip"} if n - 1 >= T else set())
        assert cats[T] == want, (n, T, sorted(cats[T]), sorted(want))
        want = {"lanes"} | ({"warps"} if n > 32 else set()) | ({"trips"} if n - 1 >= T else set())
        assert ties[T] == want, (n, T, sorted(ties[T]), sorted(want))
    assert min(kap) <= 3e6 and max(kap) >= 1e12 / 3
    print("n=%d: pivot patterns %s; ties %s; kappa_2 %.1e .. %.1e" % (n, {T: sorted(c) for T, c in cats.items()},
                                                                    {T: sorted(c) for T, c in ties.items()}, min(kap), max(kap)))


def test_a_wrong_pivot_fails_the_bound():
    """On a dominant-pivot bin at n = 40, LU with the second-best row taken at step 0 leaves a backward error more than 100x
    the bound; the right pivot stays within it."""
    n = 40
    D, fams, _ = _design(n)
    w = np.asarray(D["P"]["w"], dtype=float)
    Z = _planted_Z(w, D["fd"]["A_w"], D["fd"]["B_w"])
    rng = np.random.default_rng(7)
    for i in [i for i, f in enumerate(fams) if f == "dom"]:
        F = (rng.normal(size=n) + 1j * rng.normal(size=n)) * 1e6
        t = np.abs(Z[i, :, 0].real) + np.abs(Z[i, :, 0].imag)
        second = int(np.argsort(t)[-2])
        assert _eta(Z[i], F, _lu_solve(Z[i], F)) <= ETA_C * n * U
        eta = _eta(Z[i], F, _lu_solve(Z[i], F, force=(0, second)))
        assert eta > 100 * ETA_C * n * U, (i, eta / (ETA_C * n * U))
        print("bin %d: second-best pivot at step 0: eta = %.0fx the bound" % (i, eta / (ETA_C * n * U)))


def test_reference_against_mpmath():
    """At n = 40 the refined reference equals a 50-digit mpmath LU solve to 1e-30 on one bin of each family (the ill bin at
    kappa 1e12) and on the physical case's resonance bin; the exact residual equals mpmath's."""
    import mpmath
    mpmath.mp.dps = 50
    n = 40
    D, fams, info = _design(n)
    w = np.asarray(D["P"]["w"], dtype=float)
    Z = _planted_Z(w, D["fd"]["A_w"], D["fd"]["B_w"])
    Q, (_, ir) = _physical(n)
    picks = [(Z[fams.index(f)], f) for f in ("piv", "dom", "tie", "graded")]
    picks += [(Z[max((i for i in range(len(fams)) if fams[i] == "ill"), key=lambda i: info[i])], "ill"), (_physical_Z(Q)[ir], "physical")]
    rng = np.random.default_rng(3)
    for z, tag in picks:
        F = (rng.normal(size=n) + 1j * rng.normal(size=n)) * 1e6
        xs = _refined(z, F)
        M = mpmath.matrix([[mpmath.mpc(complex(v)) for v in row] for row in z])
        xm = mpmath.lu_solve(M, mpmath.matrix([mpmath.mpc(complex(v)) for v in F]))
        ref = [sum((mpmath.mpc(complex(x[r])) for x in xs), mpmath.mpc(0)) for r in range(n)]
        scale = max(abs(v) for v in xm)
        assert max(abs(ref[r] - xm[r]) for r in range(n)) / scale < 1e-30, tag
        x0 = xs[0] * (1 + 1e-9)
        res = _residual(z, F, [x0])
        rm = [mpmath.mpc(complex(F[r])) - mpmath.fsum(M[r, j] * mpmath.mpc(complex(x0[j])) for j in range(n)) for r in range(n)]
        assert max(abs(complex(rm[r]) - res[r]) / max(abs(rm[r]), 1e-300) for r in range(n)) < 1e-15, tag


def _in_range(a, s):
    a = np.abs(np.concatenate([np.asarray(a).real.ravel(), np.asarray(a).imag.ravel()]))
    a = a[a > 0]
    return a.min() * 2.0 ** s > 1e-290 and a.max() * 2.0 ** s < 1e300


@pytest.mark.parametrize("n", SIZES)
def test_scaled_inputs_stay_in_range(n):
    """A_w, B_w and the planted Z times 2^s, and zeta times 2^min(s, 0), keep every nonzero entry between 1e-290 and 1e300;
    the physical case leaves B_w zero on at least three bins around a resonance."""
    D, _, _ = _design(n)
    w = np.asarray(D["P"]["w"], dtype=float)
    Z = _planted_Z(w, D["fd"]["A_w"], D["fd"]["B_w"])
    for s in SCALES:
        for a in (D["fd"]["A_w"], D["fd"]["B_w"], Z):
            assert _in_range(a, s), (n, s)
        assert _in_range(_zeta(3, _nw(n), min(s, 0)), 0), (n, s)
    Q, (a, i) = _physical(n)
    assert np.count_nonzero(np.all(Q["fd"]["B_w"] == 0, axis=(0, 1))) >= 3, (n, a, i)


# ---- on the GPU ---------------------------------------------------------------------------------------------------------
def _solve(D, ct, kernel, fd=None):
    from raft_b200 import solver
    out = solver.general_solve_dynamics(D["P"], D["M"], D["B"], D["Cm"], ct, n_iter=10, fd=D["fd"] if fd is None else fd, F_BEM=True)
    rec = solver.last_dispatch()
    assert rec["family"] == "general" and rec["kernel"] == kernel, rec
    return out


def _check_trains(Z, Xi, st, Fb, primary, tag):
    """Every train of a call against the reference of its primary's Z with its own F_BEM."""
    for t, p in enumerate(primary):
        if p == t:
            assert st[t, 2] == 0 and st[t, 3] == 0, (tag, t, st[t])
        else:
            assert st[t].tolist() == [0, 1, 0, p + 1], (tag, t, st[t])
            assert np.any(Fb[t] != Fb[p])
        _check(Z, Fb[t], Xi[t], "%s train %d" % (tag, t))


@gpu
@pytest.mark.parametrize("kernel,T", KERNELS, ids=KID)
@pytest.mark.parametrize("n", SIZES)
def test_planted_trains_and_operating_points_vs_reference(n, kernel, T, monkeypatch):
    """The planted design with wave trains: every train within the bounds; the same tables as one operating point shared by
    every case, the design's own A_w / B_w zero: Xi and status bit for bit."""
    from raft_b200 import solver
    D, _, _ = _design(n)
    nw = _nw(n)
    table = _trains()
    ct = solver.CaseTable(table, zeta=_zeta(3, nw))
    Xi, st, Fb = _solve(D, ct, kernel)
    assert not np.any(st[:, 2]), st
    w = np.asarray(D["P"]["w"], dtype=float)
    _check_trains(_planted_Z(w, D["fd"]["A_w"], D["fd"]["B_w"]), Xi, st, Fb, table["primary"], "%s n=%d" % (kernel, n))
    fd = D["fd"]
    ops = dict(op=np.zeros(3, dtype=np.int32), A_w=fd["A_w"][None], B_w=fd["B_w"][None])
    fd0 = dict(fd, A_w=np.zeros_like(fd["A_w"]), B_w=np.zeros_like(fd["B_w"]))
    Xo, so, Fo = _solve(D, solver.CaseTable(table, zeta=_zeta(3, nw), ops=ops), kernel, fd=fd0)
    assert np.array_equal(Xo, Xi) and np.array_equal(so, st) and np.array_equal(Fo, Fb)


@gpu
@pytest.mark.parametrize("kernel,T", KERNELS, ids=KID)
@pytest.mark.parametrize("n", SIZES)
def test_physical_case_vs_reference(n, kernel, T, monkeypatch):
    """general_synth's design with rotor and BEM tables, drag-free, B_w zero around a resonance: two cases within the bounds
    of its Z restated with an exact fma."""
    from raft_b200 import solver
    D, _ = _physical(n)
    Xi, st, Fb = _solve(D, solver.CaseTable(_sea(2), zeta=_zeta(2, _nw(n))), kernel)
    assert not np.any(st[:, 2]), st
    Z = _physical_Z(D)
    for c in range(2):
        _check(Z, Fb[c], Xi[c], "%s n=%d physical case %d" % (kernel, n, c))


@gpu
@pytest.mark.parametrize("kernel,T", KERNELS, ids=KID)
@pytest.mark.parametrize("n", SIZES)
def test_design_axis_vs_reference(n, kernel, T, monkeypatch):
    """general_solve_dynamics_batch on two designs with different planted tables: each design against its own reference."""
    from raft_b200 import solver
    designs = [_design(n, seed=s)[0] for s in (1, 2)]
    nw = _nw(n)
    Xi, st, Fb = solver.general_solve_dynamics_batch(designs, solver.CaseTable(_sea(2), zeta=_zeta(2, nw)), n_iter=10, F_BEM=True)
    rec = solver.last_dispatch()
    assert rec["family"] == "general" and rec["kernel"] == kernel, rec
    assert not np.any(st[..., 2]), st
    for d, D in enumerate(designs):
        w = np.asarray(D["P"]["w"], dtype=float)
        Z = _planted_Z(w, D["fd"]["A_w"], D["fd"]["B_w"])
        for c in range(2):
            _check(Z, Fb[d, c], Xi[d, c], "%s n=%d design %d case %d" % (kernel, n, d, c))


@gpu
@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("kernel,T", KERNELS, ids=KID)
@pytest.mark.parametrize("n", SIZES)
def test_power_of_two_scaling_is_exact(n, kernel, T, s, monkeypatch):
    """A_w and B_w times 2^s (and zeta times 2^s for s < 0), with trains: Xi times 2^-s (the unscaled Xi for s < 0) bit for
    bit, flags 0."""
    from raft_b200 import solver
    D, _, _ = _design(n)
    nw = _nw(n)
    table = _trains()
    X0, st0, _ = _solve(D, solver.CaseTable(table, zeta=_zeta(3, nw)), kernel)
    assert not np.any(st0[:, 2])
    x = np.abs(np.concatenate([X0.real.ravel(), X0.imag.ravel()]))
    assert x[x > 0].min() * 2.0 ** -max(s, 0) > 1e-290 and x.max() * 2.0 ** -min(s, 0) < 1e300
    fd = dict(D["fd"], A_w=np.ldexp(D["fd"]["A_w"], s), B_w=np.ldexp(D["fd"]["B_w"], s))
    Xs, ss, _ = _solve(D, solver.CaseTable(table, zeta=_zeta(3, nw, min(s, 0))), kernel, fd=fd)
    assert not np.any(ss[:, 2]), ss
    assert np.array_equal(ss[:, 1], st0[:, 1]) and np.array_equal(ss[:, 3], st0[:, 3])
    ref = X0 if s < 0 else np.ldexp(X0.real, -s) + 1j * np.ldexp(X0.imag, -s)
    bad = ~((Xs == ref) | (np.isnan(Xs) & np.isnan(ref)))
    assert not np.any(bad), "%d of %d components differ, e.g. %r against %r" % (bad.sum(), bad.size, Xs[bad][:2], ref[bad][:2])


@gpu
@pytest.mark.parametrize("kernel,T", KERNELS, ids=KID)
@pytest.mark.parametrize("n", SIZES)
def test_a_singular_bin_is_flagged_singular(n, kernel, T, monkeypatch):
    """Three cases on operating points [0, 1, 0]; point 1 is the planted tables with column n // 2 zero at bin 1: case 1
    carries RAFTK_FLAG_SINGULAR in status word 2, cases 0 and 2 keep the bits of the call where every case runs point 0,
    and solver.raise_on_flags raises."""
    from raft_b200 import solver
    D, _, _ = _design(n)
    nw = _nw(n)
    fd = D["fd"]
    A1, B1 = np.array(fd["A_w"]), np.array(fd["B_w"])
    A1[:, n // 2, 1] = 0.0
    B1[:, n // 2, 1] = 0.0
    fd0 = dict(fd, A_w=np.zeros_like(fd["A_w"]), B_w=np.zeros_like(fd["B_w"]))
    tabs = dict(A_w=np.stack([fd["A_w"], A1]), B_w=np.stack([fd["B_w"], B1]))
    outs = []
    for op in ([0, 0, 0], [0, 1, 0]):
        ct = solver.CaseTable(_sea(3), zeta=_zeta(3, nw), ops=dict(tabs, op=np.array(op, dtype=np.int32)))
        outs.append(_solve(D, ct, kernel, fd=fd0))
    (X0, st0, _), (X1, st1, _) = outs
    assert not np.any(st0[:, 2]), st0
    assert st1[1, 2] & RAFTK_FLAG_SINGULAR and st1[1, 0] == 1, st1
    assert np.array_equal(X1[[0, 2]], X0[[0, 2]]) and np.array_equal(st1[[0, 2]], st0[[0, 2]])
    with pytest.raises(Exception):
        solver.raise_on_flags(st1)
