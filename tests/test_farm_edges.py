"""Every farm kernel's coupled solve against a high-precision reference of the same system, on arrays whose pivots cross
FOWT blocks, and the dense LUs' exactness under power-of-two scaling across the exponent range.

The reference is independent of the kernels' pivot order.  Each (farm, case, bin) system is rebuilt in NumPy from the
per-FOWT device outputs (B_drag, F_drag, F_iner, F_BEM), the design tables, the operating points, F_2nd and the array
matrices, assembled as farm_assemble does (it rounds -w^2 M + C without an fma: a few ulp per entry).  Then:
  * the residual F - Z x of the kernel's x is computed exactly (Dekker products, math.fsum per row), and the normwise
    backward error eta = |r|inf / (|Z|inf |x|inf + |F|inf) must stay below ETA_C * n * u (u = 2^-53);
  * the forward error is measured against the solution refined with those exact residuals until the last correction is
    below 1e-34 of the solution (the refinement is checked against a 40-digit mpmath LU solve on the CPU):
    |x - x*|inf / |x*|inf <= FWD_C * n * kappa_inf(Z) * u, and <= FWD_CEIL on bins with kappa_inf(Z) <= 1e4.  Every bin
    for 6N <= 30; above, the bins whose pivot crosses FOWT blocks (first two), the bin of largest kappa and every fourth.

Inputs.  A shared-mooring chain adds K = alpha * C0[0, 0] to both diagonal entries and -K to the coupling entries of the
surge and sway DOFs of neighbouring FOWTs, alpha in {1, 10}; the grid covers the coupled surge and sway resonances,
where the pivots of a FOWT's surge and sway columns come from its neighbour's rows.  A stiff link (alpha = 1e7) makes the
low-frequency bins ill-conditioned, kappa_inf(Z) above 1e8: alpha = 1e4 does not, because the pitch rows (C0[4, 4] ~ 5e9)
dominate |Z|inf until the link is stiffer than the pitch restoring (kappa stays below 1e7 there).  The CPU tests
restate the kernels' pivot rule (|re| + |im|, first maximum wins) and prove on the oracle's per-FOWT Z that these inputs
reach those edges.

Kernels: farm-warp (N = 1, 3, 4, and N = 2 with RAFTK_FARM_SMEM=1), farm-rows12 (N = 2), farm-block (N = 5 and N = 20: on
an H100 the 120 x 121 system, 232,320 bytes, still fits in shared memory) and farm-global (N = 21).

Measured on an H100 80GB HBM3 (700 W limit), over every test of this file: worst eta / (n u) = 0.104, worst forward error /
(n kappa u) = 0.038, worst forward error on bins with kappa <= 1e4 = 1.75e-15.  The bounds keep about 10x of margin.

Scaling.  Z -> 2^s Z with F unchanged must give X -> 2^-s X bit for bit with info = 0 for s in {-600, -300, 300, 560}, on
system_solve (sys-unblocked, sys-blocked, sys-global) and on the four farm kernels (the session's M0, B0, C0, B_drag,
A_w / B_w and array matrices scaled in place).  Every pivot reciprocal and back-substitution quotient is formed at the
pivot's scale (raftk_misc.cuh piv_recip / piv_div), so |p|^2 neither overflows nor underflows."""
import math
import os

import numpy as np
import pytest

from conftest import GOLDEN

gpu = pytest.mark.gpu
U = 2.0 ** -53
ETA_C = 1.0                  # eta <= ETA_C * n * u
FWD_C = 0.4                  # forward error <= FWD_C * n * kappa * u
FWD_CEIL = 2e-14             # forward error on bins with kappa_inf(Z) <= 1e4
NW, MAX_F = 32, 0.064        # 0.0126 .. 0.40 rad/s: the single-FOWT surge resonance (0.051) up to a chain's highest
ALPHAS = {"chain1": 1.0, "chain10": 10.0, "stiff": 1e7}
PER_FOWT = ("Xi", "status", "B_drag", "F_drag", "F_iner")
KERNELS = [(1, False, "farm-warp"), (2, False, "farm-rows12"), (2, True, "farm-warp"), (3, False, "farm-warp"),
           (4, False, "farm-warp"), (5, False, "farm-block"), (20, False, "farm-block"), (21, False, "farm-global")]
KID = ["N%d%s" % (N, "-smem" if smem else "") for N, smem, _ in KERNELS]


# ---- inputs ---------------------------------------------------------------------------------------------------------
def _fixture():
    z = np.load(os.path.join(GOLDEN, "farm_VolturnUS-S_farm_nw48.npz"))
    return [{k[len("P%d_" % i):]: z[k] for k in z.files if k.startswith("P%d_" % i)} for i in range(int(z["n_fowt"]))]


def _moved(P, dx):
    Q = dict(P)
    r = np.array([dx, 0.0, 0.0])
    for k in ("mem_rA", "node_r", "prp"):
        Q[k] = np.asarray(P[k], dtype=float) + r
    Q["x_ref"] = float(P["x_ref"]) + dx
    return Q


def _packs(N, tables=False, seed=0):
    """N FOWTs of the two-FOWT fixture, in turn, 1600 m apart on a row, on the NW-bin grid; ``tables``: seeded A_w / B_w /
    X_BEM (F_BEM in the load)."""
    from raft_b200 import grid
    base = [grid.regrid(P, NW, MAX_F) for P in _fixture()]
    packs = [_moved(base[i % 2], 1600.0 * (i - i % 2)) for i in range(N)]
    if tables:
        rng = np.random.default_rng(77 + seed)
        for i, P in enumerate(packs):
            d = np.diag(rng.uniform(0.5, 1.5, size=6))
            packs[i] = dict(P, A_w=(np.abs(P["M0"]) * 0.05 * d)[:, :, None] * rng.uniform(0.5, 1.0, size=NW)[None, None, :],
                            B_w=(np.abs(P["M0"]) * 0.01 * d)[:, :, None] * rng.uniform(0.0, 1.0, size=NW)[None, None, :],
                            bem_headings=np.array([0.0, 90.0, 180.0, 270.0]), heading_adjust=0.0,
                            X_BEM=(rng.normal(size=(4, 6, NW)) + 1j * rng.normal(size=(4, 6, NW))) * 2e5)
    return packs


def _link(N, alpha, c00):
    """Shared mooring lines between neighbouring FOWTs: +K on both diagonal entries, -K on the coupling entries of surge and
    sway, K = alpha * C0[0, 0]."""
    n = 6 * N
    C = np.zeros((n, n))
    K = alpha * c00
    for i in range(N - 1):
        for d in (0, 1):
            a, b = 6 * i + d, 6 * (i + 1) + d
            C[a, a] += K
            C[b, b] += K
            C[a, b] -= K
            C[b, a] -= K
    return C


def _cases(rows, primary=None):
    n = len(rows)
    d = dict(Hs=rows[:, 0], Tp=rows[:, 1], gamma=np.zeros(n), beta_deg=rows[:, 2], spec=np.zeros(n, dtype=np.int32))
    if primary is not None:
        d["primary"] = np.asarray(primary, dtype=np.int32)
    return d


CASES = np.array([[6.0, 12.0, 0.0], [3.0, 8.0, 70.0]])


def _zeta(nC):
    """Unit-order wave amplitudes on every bin (JONSWAP's lowest bins are exactly zero on this grid)."""
    return np.full((nC, NW), 0.5)


# ---- the reference ----------------------------------------------------------------------------------------------------
def _assemble(packs, out, cases, w, mats, f=0, N=None, ops=None, F2=None):
    """Z [nC, nw, n, n] and F [nC, nw, n] of farm f as farm_assemble builds them, from the per-FOWT device outputs."""
    N = len(packs) if N is None else N
    n, nw, nC = 6 * N, len(w), len(cases["Hs"])
    primary = cases.get("primary", np.arange(nC))
    Z = np.zeros((nC, nw, n, n), dtype=complex)
    F = np.zeros((nC, nw, n), dtype=complex)
    w2 = (w * w)[:, None, None]
    for c in range(nC):
        cp = int(primary[c])
        for i in range(N):
            d = f * N + i
            P = packs[d]
            M = np.broadcast_to(np.asarray(P["M0"], dtype=float)[None], (nw, 6, 6)).copy()
            B = np.broadcast_to((np.asarray(P["B0"], dtype=float) + out["B_drag"][d, cp])[None], (nw, 6, 6)).copy()
            if P.get("A_w") is not None:
                M += np.moveaxis(P["A_w"], -1, 0)
                B += np.moveaxis(P["B_w"], -1, 0)
            if ops is not None:
                k = int(ops["op"][c])
                A_op = ops["A_w"][k] if ops["A_w"].ndim == 4 else ops["A_w"][d, k]
                B_op = ops["B_w"][k] if ops["B_w"].ndim == 4 else ops["B_w"][d, k]
                M += np.moveaxis(A_op, -1, 0)
                B += np.moveaxis(B_op, -1, 0)
            s = slice(6 * i, 6 * i + 6)
            Z[c, :, s, s] = (np.asarray(P["C0"], dtype=float)[None] - w2 * M) + 1j * (w[:, None, None] * B)
            load = out["F_drag"][d, c] + out["F_iner"][d, c]
            if "F_BEM" in out:
                load = load + out["F_BEM"][d, c]
            if F2 is not None:
                load = load + F2[d, c]
            F[c, :, s] = load.T
        if mats.get("C_arr") is not None:
            Z[c] += mats["C_arr"][None]
        if mats.get("M_arr") is not None:
            Z[c] -= w2 * mats["M_arr"][None]
        if mats.get("B_arr") is not None:
            Z[c] += 1j * w[:, None, None] * mats["B_arr"][None]
    return Z, F


def _two_prod(a, b):
    """a * b = p + e exactly (Dekker; no overflow at these magnitudes)."""
    p = a * b
    s = 134217729.0
    ah = a * s
    ah = ah - (ah - a)
    al = a - ah
    bh = b * s
    bh = bh - (bh - b)
    bl = b - bh
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def _residual(Z, F, xs):
    """F - Z (xs[0] + xs[1] + ...) for one system, every component the correctly rounded exact value."""
    re, im = [F.real[:, None]], [F.imag[:, None]]
    for x in xs:
        for a, b, sg, dst in ((Z.real, x.real, -1.0, re), (Z.imag, x.imag, 1.0, re), (Z.real, x.imag, -1.0, im), (Z.imag, x.real, -1.0, im)):
            p, e = _two_prod(a, b[None, :])
            dst += [sg * p, sg * e]
    R, I = np.concatenate(re, axis=1), np.concatenate(im, axis=1)
    return np.array([complex(math.fsum(R[i]), math.fsum(I[i])) for i in range(len(F))])


def _refined(Z, F, iters=12):
    """x* of Z x = F as an unevaluated sum of double vectors: LAPACK's solve, refined with exact residuals until the last
    correction is below 1e-34 of the solution."""
    xs = [np.linalg.solve(Z, F)]
    for _ in range(iters):
        d = np.linalg.solve(Z, _residual(Z, F, xs))
        xs.append(d)
        if np.abs(d).max() <= 1e-34 * np.abs(xs[0]).max():
            return xs
    raise AssertionError("refinement did not converge (kappa %.1e)" % np.linalg.cond(Z, np.inf))


def _errors(Z, F, x):
    """-> (eta, forward error, kappa_inf) of the computed solution x of one system."""
    r = _residual(Z, F, [x])
    nZ = np.abs(Z).sum(axis=1).max()
    eta = np.abs(r).max() / (nZ * np.abs(x).max() + np.abs(F).max())
    xs = _refined(Z, F)
    d = x - xs[0]
    for t in xs[1:]:
        d = d - t
    fwd = np.abs(d).max() / np.abs(xs[0]).max()
    kappa = nZ * np.abs(np.linalg.inv(Z)).sum(axis=1).max()
    return eta, fwd, kappa


WORST = {"eta": 0.0, "fwd": 0.0, "ceil": 0.0}


def _sample(Z):
    """Bins of one case's Z [nw, n, n] that get the forward-error check."""
    nw, n, _ = Z.shape
    if n <= 30:
        return set(range(nw))
    cross = [iw for iw in range(nw) if any(p // 6 != k // 6 for k, p, _ in _pivot_rows(Z[iw]))]
    return set(cross[:2]) | {int(np.argmax([np.linalg.cond(z, np.inf) for z in Z]))} | set(range(0, nw, 4))


def _check(Z, F, X, tag):
    """X [nC, n, nw] (the kernel's Xi_sys rows) against the reference: the backward error on every (case, bin), the
    forward error on _sample's bins."""
    nC, nw, n, _ = Z.shape
    for c in range(nC):
        fwd_bins = _sample(Z[c])
        for iw in range(nw):
            if iw not in fwd_bins:
                r = _residual(Z[c, iw], F[c, iw], [X[c, :, iw]])
                eta = np.abs(r).max() / (np.abs(Z[c, iw]).sum(axis=1).max() * np.abs(X[c, :, iw]).max() + np.abs(F[c, iw]).max())
                WORST["eta"] = max(WORST["eta"], eta / (n * U))
                assert eta <= ETA_C * n * U, (tag, c, iw, eta / (n * U))
                continue
            eta, fwd, kappa = _errors(Z[c, iw], F[c, iw], X[c, :, iw])
            WORST["eta"] = max(WORST["eta"], eta / (n * U))
            WORST["fwd"] = max(WORST["fwd"], fwd / (n * kappa * U))
            assert eta <= ETA_C * n * U, (tag, c, iw, eta / (n * U))
            assert fwd <= FWD_C * n * kappa * U, (tag, c, iw, fwd, kappa)
            if kappa <= 1e4:
                WORST["ceil"] = max(WORST["ceil"], fwd)
                assert fwd <= FWD_CEIL, (tag, c, iw, fwd, kappa)
    print("%s: worst eta/(n u) %.3g, fwd/(n kappa u) %.3g, fwd at kappa <= 1e4 %.3g" % (tag, WORST["eta"], WORST["fwd"], WORST["ceil"]))


def _pivot_rows(Z):
    """The kernels' pivot rule restated: partial pivoting on |re| + |im|, first maximum wins.  -> [(step, row, margin)],
    margin = 1 - second largest candidate / largest."""
    A = np.array(Z, dtype=complex)
    n = len(A)
    out = []
    for k in range(n):
        t = np.abs(A[k:, k].real) + np.abs(A[k:, k].imag)
        p = k + int(np.argmax(t))
        top = np.sort(t)[::-1]
        out.append((k, p, 1.0 - (top[1] / top[0] if len(top) > 1 and top[0] > 0 else 0.0)))
        A[[k, p]] = A[[p, k]]
        A[k + 1:, k] /= A[k, k]
        A[k + 1:, k + 1:] -= np.outer(A[k + 1:, k], A[k, k + 1:])
    return out


def _oracle_Z(packs, cases, c=0, n_iter=10):
    """Per-FOWT Z [nw, 6, 6] and Xi of case c from the oracle."""
    from oracle import oracle as orc
    orc.build()
    Zs, Xs, passes = [], [], []
    for P in packs:
        r = orc.solve_dynamics(orc.OracleDesign(P), 0, cases["Hs"][c], cases["Tp"][c], 0.0, cases["beta_deg"][c], nIter=n_iter, want_Z=True)
        Xs.append(r[0])
        passes.append(r[1][0])
        Zs.append(r[2])
    return Zs, Xs, passes


def _oracle_system(Zs, C_arr):
    N = len(Zs)
    nw = Zs[0].shape[0]
    Z = np.zeros((nw, 6 * N, 6 * N), dtype=complex)
    for i, Zi in enumerate(Zs):
        Z[:, 6 * i:6 * i + 6, 6 * i:6 * i + 6] = Zi
    return Z + C_arr[None]


# ---- without a GPU: the inputs reach the edges -------------------------------------------------------------------------
@pytest.mark.parametrize("N,case", [(2, "chain1"), (2, "chain10"), (4, "chain1"), (4, "chain10")])
def test_shared_mooring_pivots_cross_fowt_blocks(N, case):
    """On the oracle's per-FOWT Z plus the chain, some bins take a pivot from another FOWT's rows, with a margin of more
    than 1e-8 between the top two candidates there: rounding cannot change the kernels' choice."""
    packs = _packs(N)
    Zs, _, _ = _oracle_Z(packs, _cases(CASES[:1]))
    Z = _oracle_system(Zs, _link(N, ALPHAS[case], packs[0]["C0"][0, 0]))
    crossing = 0
    for iw in range(NW):
        cross = [(k, p, m) for k, p, m in _pivot_rows(Z[iw]) if p // 6 != k // 6]
        if cross:
            crossing += 1
            assert min(m for _, _, m in cross) > 1e-8, (iw, cross)
    assert crossing >= 2, crossing


def test_stiff_link_reaches_its_condition_number():
    packs = _packs(2)
    Zs, _, _ = _oracle_Z(packs, _cases(CASES[:1]))
    kappa = [np.linalg.cond(Z, np.inf) for Z in _oracle_system(Zs, _link(2, ALPHAS["stiff"], packs[0]["C0"][0, 0]))]
    assert max(kappa) > 1e8 and sum(k > 1e7 for k in kappa) >= 3, ["%.1e" % k for k in kappa]
    weak = [np.linalg.cond(Z, np.inf) for Z in _oracle_system(Zs, _link(2, 1e4, packs[0]["C0"][0, 0]))]
    assert max(weak) < 1e7                                     # why the link is stiffer than alpha = 1e4


def test_reference_against_mpmath_and_lapack():
    """The refined reference equals a 40-digit mpmath LU solve to 1e-30 on a cross-pivoting and a stiff-link system, and
    equals numpy.linalg.solve to 1e-13 on well-conditioned ones; the exact residual equals mpmath's."""
    import mpmath
    mpmath.mp.dps = 40
    packs = _packs(2)
    Zs, _, _ = _oracle_Z(packs, _cases(CASES[:1]))
    rng = np.random.default_rng(4)
    for case, bins in (("chain10", (3, 7)), ("stiff", (0, 2))):
        Z = _oracle_system(Zs, _link(2, ALPHAS[case], packs[0]["C0"][0, 0]))
        for iw in bins:
            F = rng.normal(size=12) * 1e5 + 1j * rng.normal(size=12) * 1e5
            xs = _refined(Z[iw], F)
            M = mpmath.matrix([[mpmath.mpc(complex(v)) for v in row] for row in Z[iw]])
            xm = mpmath.lu_solve(M, mpmath.matrix([mpmath.mpc(complex(v)) for v in F]))
            ref = [sum((mpmath.mpc(complex(x[i])) for x in xs), mpmath.mpc(0)) for i in range(12)]
            scale = max(abs(v) for v in xm)
            assert max(abs(ref[i] - xm[i]) for i in range(12)) / scale < 1e-30, (case, iw)
            x0 = xs[0] * (1 + 1e-9)
            r = _residual(Z[iw], F, [x0])
            rm = [mpmath.mpc(complex(F[i])) - mpmath.fsum(M[i, j] * mpmath.mpc(complex(x0[j])) for j in range(12)) for i in range(12)]
            assert max(abs(complex(rm[i]) - r[i]) / max(abs(rm[i]), 1e-300) for i in range(12)) < 1e-15
    for iw in range(0, NW, 5):                                  # the plain two-FOWT array: kappa ~ 1e3 .. 1e5
        Z = _oracle_system(Zs, np.zeros((12, 12)))[iw] + np.eye(12) * 1e7
        if np.linalg.cond(Z, np.inf) > 1e3:
            continue
        F = rng.normal(size=12) + 1j * rng.normal(size=12)
        xs = _refined(Z, F)
        assert np.abs(xs[0] + xs[1] - np.linalg.solve(Z, F)).max() <= 1e-13 * np.abs(xs[0]).max()


def test_scaling_inputs_stay_in_range():
    """The scaled systems of the scaling tests keep every nonzero entry between 1e-290 and 1e300."""
    for n in (5, 49, 150):
        Z, F = _random_system(n, 3)
        _assert_in_range(Z, n)


def _assert_in_range(Z, tag):
    a = np.abs(np.concatenate([Z.real.ravel(), Z.imag.ravel()]))
    a = a[a > 0]
    for s in SCALES:
        assert a.min() * 2.0 ** s > 1e-290 and a.max() * 2.0 ** s < 1e300, (tag, s, a.min(), a.max())


# ---- on the GPU: every kernel against the reference --------------------------------------------------------------------
def _env(monkeypatch, smem):
    if smem:
        monkeypatch.setenv("RAFTK_FARM_SMEM", "1")
    else:
        monkeypatch.delenv("RAFTK_FARM_SMEM", raising=False)


def _run_farm(packs, cases, mats, kernel, want=PER_FOWT, n_fowt=None):
    from raft_b200 import solver
    batch = solver.DesignBatch(packs)
    if n_fowt is None:
        out = solver.solve_dynamics_farm(batch, cases, n_iter=10, want=want, **mats)
    else:
        out = solver.solve_dynamics_farm_batch(batch, cases, n_fowt, n_iter=10, want=want, **mats)
    rec = solver.last_dispatch()
    assert rec["family"] == "farm" and rec["kernel"] == kernel, rec
    assert not np.any(out["info"])
    return out


@gpu
@pytest.mark.parametrize("case", list(ALPHAS))
@pytest.mark.parametrize("N,smem,kernel", KERNELS, ids=KID)
def test_shared_mooring_vs_reference(N, smem, kernel, case, monkeypatch):
    from raft_b200 import solver
    _env(monkeypatch, smem)
    packs = _packs(N)
    cs = _cases(CASES)
    mats = dict(C_arr=_link(N, ALPHAS[case], packs[0]["C0"][0, 0]))
    out = _run_farm(packs, solver.CaseTable(cs, zeta=_zeta(2)), mats, kernel)
    Z, F = _assemble(packs, out, cs, packs[0]["w"], mats)
    _check(Z, F, out["Xi_sys"], "%s N=%d %s" % (kernel, N, case))


@gpu
@pytest.mark.parametrize("N,smem,kernel", KERNELS, ids=KID)
def test_every_feature_vs_reference(N, smem, kernel, monkeypatch):
    """M_arr (with a skew part) + B_arr (with a skew part) + the chain's C_arr, designs with A_w / B_w / X_BEM, F_2nd,
    primary and secondary wave trains and per-case operating points, on a batch of F = 3 farms with arr_shared 0 and 1."""
    from raft_b200 import solver
    from test_operating_points import _op_tables
    _env(monkeypatch, smem)
    Fm, n = 3, 6 * N
    packs = [P for f in range(Fm) for P in _packs(N, tables=True, seed=10 * N + f)]
    rng = np.random.default_rng(N)
    G = rng.normal(size=(n, n))
    S = rng.normal(size=(n, n))
    mats = dict(C_arr=_link(N, 10.0, packs[0]["C0"][0, 0]) + np.diag([5e4] * n), M_arr=(G @ G.T) * 2e3 / n + (S - S.T) * 5e2,
                B_arr=(G + G.T) * 1e3 + (S - S.T) * 4e3)
    rows = np.array([[6.0, 12.0, 0.0], [2.0, 7.0, 60.0], [4.0, 10.0, 200.0], [1.5, 6.0, 100.0]])
    cs = _cases(rows, primary=[0, 0, 2, 2])
    nC = len(rows)
    A, B = _op_tables(rng, packs[0], 2, Fm * N)
    ops = dict(op=np.array([0, 0, 1, 1], dtype=np.int32), A_w=A, B_w=B)
    F2 = rng.normal(size=(Fm * N, nC, 6, NW)) * 5e4
    want = PER_FOWT + ("F_BEM",)
    for shared in (1, 0):
        m = mats if shared else {k: np.stack([v * (1.0 + 0.1 * f) for f in range(Fm)]) for k, v in mats.items()}
        out = _run_farm(packs, solver.CaseTable(cs, zeta=_zeta(nC), F_2nd=F2, ops=ops), m, kernel, want=want, n_fowt=N)
        assert np.any(out["F_BEM"] != 0)
        for f in range(Fm):
            mf = {k: (v if shared else v[f]) for k, v in m.items()}
            Z, F = _assemble(packs, out, cs, packs[0]["w"], mf, f=f, N=N, ops=ops, F2=F2)
            assert np.any(Z != np.swapaxes(Z, -1, -2))              # non-symmetric
            _check(Z, F, out["Xi_sys"][f], "%s N=%d features shared=%d farm %d" % (kernel, N, shared, f))


@gpu
@pytest.mark.parametrize("N,smem,kernel", KERNELS, ids=KID)
def test_end_to_end_against_the_oracle(N, smem, kernel, monkeypatch):
    """The chain (alpha = 10) with the oracle's per-FOWT Z: pass counts identical, and the kernel's solution within the
    bounds of the system the oracle's Z and load define."""
    from raft_b200 import solver
    _env(monkeypatch, smem)
    packs = _packs(N)
    cs = _cases(CASES[:1])
    C_arr = _link(N, 10.0, packs[0]["C0"][0, 0])
    out = _run_farm(packs, solver.CaseTable(cs), dict(C_arr=C_arr), kernel)
    Zs, Xs, passes = _oracle_Z(packs, cs)
    assert np.array_equal(np.array(passes), out["status"][:, 0, 0])
    Z = _oracle_system(Zs, C_arr)
    F = np.concatenate([np.einsum("wab,bw->wa", Zi, Xi) for Zi, Xi in zip(Zs, Xs)], axis=1)
    keep = np.abs(F).max(axis=1) > 0                                   # JONSWAP is exactly zero on the lowest bins
    assert keep.sum() >= NW // 2
    Xo = out["Xi_sys"][0]
    for iw in np.nonzero(keep)[0]:
        xs = _refined(Z[iw], F[iw])
        kappa = np.linalg.cond(Z[iw], np.inf)
        err = np.abs(Xo[:, iw] - xs[0] - xs[1]).max() / np.abs(xs[0]).max()
        assert err <= 1e-9 + FWD_C * 6 * N * kappa * U, (iw, err, kappa)   # the oracle's Z and F are its own roundings


# ---- an exactly zero pivot ------------------------------------------------------------------------------------------------
def _session(packs, cs, nC):
    from raft_b200 import solver
    sess = solver.DeviceSession(solver.DesignBatch(packs), solver.CaseTable(cs, zeta=_zeta(nC)), device="cuda:0", want=PER_FOWT)
    sess.solve(n_iter=10)
    return sess


@gpu
@pytest.mark.parametrize("N,smem,kernel", [k for k in KERNELS if k[0] > 1], ids=KID[1:])
def test_a_pivot_that_cancels_to_zero(N, smem, kernel, monkeypatch):
    """Farm 1's last two FOWTs have nothing in yaw but a link C_arr = [[k, -k], [-k, k]] between them (k = 2^20): the
    elimination cancels the last pivot to exactly zero.  info[1] = 6N at every case and bin; the other farms keep their
    bits."""
    from raft_b200 import solver
    _env(monkeypatch, smem)
    Fm, n = 3, 6 * N
    packs = [P for f in range(Fm) for P in _packs(N)]
    C_arr = np.stack([_link(N, 1.0 + f, packs[0]["C0"][0, 0]) for f in range(Fm)])
    sess = _session(packs, _cases(CASES), 2)
    xi, info = sess.farm_response(C_arr=C_arr, n_fowt=N)
    assert solver.last_dispatch()["kernel"] == kernel
    good = xi.cpu().numpy().copy()
    assert not np.any(info.cpu().numpy())
    for d in (2 * N - 2, 2 * N - 1):
        for t in (sess.dt["M0"], sess.dt["B0"], sess.dt["C0"]):
            t.view(-1, 6, 6)[d, :, 5] = 0.0
            t.view(-1, 6, 6)[d, 5, :] = 0.0
        sess.out["B_drag"][d, :, :, 5] = 0.0
        sess.out["B_drag"][d, :, 5, :] = 0.0
    C1 = sess._farm_batch[1]["C_arr"][1]
    a, b = n - 7, n - 1
    k = 2.0 ** 20
    C1[:, a] = C1[a, :] = C1[:, b] = C1[b, :] = 0.0
    C1[a, a], C1[a, b], C1[b, a], C1[b, b] = k, -k, -k, k
    xi, info = sess.farm_response(n_fowt=N)
    assert solver.last_dispatch()["kernel"] == kernel
    info, xi = info.cpu().numpy(), xi.cpu().numpy()
    assert np.all(info[1] == n) and not np.any(info[0]) and not np.any(info[2]), np.unique(info[1])
    assert np.array_equal(xi[0], good[0]) and np.array_equal(xi[2], good[2])


# ---- the exponent range ----------------------------------------------------------------------------------------------------
SCALES = (-600, -300, 300, 560)


def _random_system(n, nw):
    rng = np.random.default_rng(n)
    Z = rng.uniform(0.5, 2.0, size=(nw, n, n)) * np.exp(2j * np.pi * rng.uniform(size=(nw, n, n)))
    Z[1::2] += 2 * np.sqrt(n) * np.eye(n)[None]
    F = rng.uniform(0.5, 2.0, size=(nw, n, 2)) * np.exp(2j * np.pi * rng.uniform(size=(nw, n, 2)))
    return Z, F


def _pow2(a, s):
    return np.ldexp(a.real, s) + 1j * np.ldexp(a.imag, s)


@gpu
@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("n,kernel", [(5, "sys-unblocked"), (49, "sys-blocked"), (150, "sys-global")])
def test_system_solve_is_exact_under_power_of_two_scaling(n, kernel, s):
    from raft_b200 import solver
    Z, F = _random_system(n, 3)
    _assert_in_range(Z, n)
    X0, info0 = solver.system_solve(Z, F)
    assert solver.last_dispatch()["kernel"] == kernel and not np.any(info0)
    x = np.abs(np.concatenate([X0.real.ravel(), X0.imag.ravel()]))
    assert x[x > 0].min() * 2.0 ** -s > 1e-290 and x.max() * 2.0 ** -s < 1e300
    Xs, info = solver.system_solve(_pow2(Z, s), F)
    assert solver.last_dispatch()["kernel"] == kernel
    assert not np.any(info), info
    assert np.array_equal(Xs, _pow2(X0, -s)), np.abs(Xs - _pow2(X0, -s)).max() / np.abs(_pow2(X0, -s)).max()


@gpu
@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("N,smem,kernel", [(2, False, "farm-rows12"), (2, True, "farm-warp"), (5, False, "farm-block"),
                                           (21, False, "farm-global")], ids=["N2", "N2-smem", "N5", "N21"])
def test_farm_kernels_are_exact_under_power_of_two_scaling(N, smem, kernel, s, monkeypatch):
    """The session's M0, B0, C0, B_drag, A_w / B_w and array matrices times 2^s, the load as it was: Xi_sys times 2^-s, bit
    for bit, info = 0."""
    import torch
    from raft_b200 import solver
    _env(monkeypatch, smem)
    n = 6 * N
    packs = _packs(N, tables=True, seed=N)
    cs = _cases(CASES)
    sess = solver.DeviceSession(solver.DesignBatch(packs), solver.CaseTable(cs, zeta=_zeta(2)), device="cuda:0",
                                want=PER_FOWT + ("F_BEM",))
    out = sess.solve(n_iter=10)
    rng = np.random.default_rng(5)
    G = rng.normal(size=(n, n))
    mats = dict(C_arr=_link(N, 10.0, packs[0]["C0"][0, 0]), M_arr=(G @ G.T) * 2e3 / n, B_arr=(G + G.T) * 1e3)
    xi, info = sess.farm_response(n_fowt=N, **mats)
    assert solver.last_dispatch()["kernel"] == kernel
    X0 = xi.cpu().numpy().copy()
    assert not np.any(info.cpu().numpy())
    host = {k: v.cpu().numpy() for k, v in out.items()}
    Z, _ = _assemble(packs, host, cs, packs[0]["w"], mats)
    _assert_in_range(Z, N)
    x = np.abs(np.concatenate([X0.real.ravel(), X0.imag.ravel()]))
    assert x[x > 0].min() * 2.0 ** -s > 1e-290 and x.max() * 2.0 ** -s < 1e300
    p = 2.0 ** s
    for k in ("M0", "B0", "C0", "A_w", "B_w"):
        sess.dt[k].mul_(p)
    sess.out["B_drag"].mul_(p)
    for t in sess._farm_batch[1].values():
        t.mul_(p)
    torch.cuda.synchronize()
    xi, info = sess.farm_response(n_fowt=N)
    assert solver.last_dispatch()["kernel"] == kernel
    Xs, info = xi.cpu().numpy(), info.cpu().numpy()
    assert not np.any(info), np.unique(info)
    ref = _pow2(X0, -s)
    assert np.array_equal(Xs, ref), np.nanmax(np.abs(Xs - ref)) / np.abs(ref).max()
