"""The eigen analysis (raftk_eigen.cuh) at the sizes, spectra and scalings the fixtures of test_eigen.py never reach, against a
high-precision reference of the same operation.

Reference: the eigenvalues and unit right / left eigenvectors of A = M^-1 C formed in mpmath at 40 digits from the exact FP64
inputs for n <= 24, LAPACK (scipy.linalg.eig) beyond.  Accuracy contract, per eigenvalue, with kappa_j = 1 / |y_j^H x_j| from
unit left and right vectors and cond(M) Skeel's condition number of M (the solve that forms A):
    |lam_j - lam_j^ref| <= C_LAM n eps ||A||_F kappa_j cond(M),
and, where mpmath is the reference, at most 10x LAPACK's own error (floor 4 eps ||A||_F kappa_j cond(M)).  Eigenvalues are paired
by a minimum-cost matching, which is the ascending pairing wherever they are apart.  Every system: finite outputs unless info
has RAFTK_EIG_SINGULAR / RAFTK_EIG_NOCONV, unit 2-norm modes, the largest component of a complex mode real, the residual
|Cv - lam Mv| / ((|C| + |lam| |M|) |v|) <= 1e-13, and for diagonalisable clusters the spanned subspaces of the reference.
Defective (Jordan) spectra are held to the eps^(1/k) perturbation bound instead.  Without a GPU: the reference's self-checks,
the planner's shared-memory boundary and the numpy restatement of the DOF claim against the reference's own code path."""
import time

import numpy as np
import pytest
import scipy.linalg
from scipy.optimize import linear_sum_assignment

from conftest import ROOT
from test_eigen import fixture, seeded, RIGID

gpu = pytest.mark.gpu
EPS = np.finfo(float).eps
C_LAM = 8.0                 # the constant of the per-eigenvalue bound
C_VEC = 8.0                 # the constant of the subspace bound
MP_NMAX = 24                # mpmath reference up to this n, LAPACK beyond
SINGULAR, NOCONV, COMPLEX = 8, 16, 4
MP_SECONDS = [0.0]


@pytest.fixture(scope="module", autouse=True)
def _report_mpmath_time():
    yield
    print("\ntest_eigen_edges: mpmath reference %.1f s" % MP_SECONDS[0])


# ---- the reference ---------------------------------------------------------------------------------------------------
_REF = {}


def skeel(M):
    return max(1.0, float(np.linalg.norm(np.abs(np.linalg.inv(M)) @ np.abs(M), np.inf)))


def _kappa(X, Y):
    """1 / |y^H x| of unit vectors: X columns right, Y rows left (y A = lam y)."""
    x = X / np.linalg.norm(X, axis=0)
    y = Y / np.linalg.norm(Y, axis=1)[:, None]
    return 1.0 / np.abs(np.einsum("ji,ij->j", y, x))


def reference(M, K, use_mp=None):
    """dict(lam, X (unit right vectors), kappa, normA, condM, exact, lapack, lapack_X) for A = M^-1 K."""
    M, K = np.asarray(M, dtype=float), np.asarray(K, dtype=float)
    key = (M.tobytes(), K.tobytes())
    if key in _REF:
        return _REF[key]
    n = len(M)
    A = np.linalg.solve(M, K)
    wl, vl, vr = scipy.linalg.eig(A, left=True, right=True)
    r = dict(lapack=wl, lapack_X=vr / np.linalg.norm(vr, axis=0), condM=skeel(M))
    if use_mp if use_mp is not None else n <= MP_NMAX:
        import mpmath
        t = time.perf_counter()
        with mpmath.workdps(40):
            Am = mpmath.inverse(mpmath.matrix(M.tolist())) * mpmath.matrix(K.tolist())
            E, EL, ER = mpmath.eig(Am, left=True, right=True)
            lam = np.array([complex(e) for e in E])
            X = np.array(ER.tolist(), dtype=complex)
            Y = np.array(EL.tolist(), dtype=complex)
            normA = float(mpmath.mnorm(Am, "f"))
        MP_SECONDS[0] += time.perf_counter() - t
        r.update(lam=lam, X=X / np.linalg.norm(X, axis=0), kappa=_kappa(X, Y), normA=normA, exact=True)
    else:
        r.update(lam=wl, X=r["lapack_X"], kappa=_kappa(vr, vl.conj().T), normA=float(np.linalg.norm(A)), exact=False)
    _REF[key] = r
    return r


def _pair(lam, ref_lam):
    """index into ref_lam for each lam: the minimum-cost matching (the ascending pairing wherever eigenvalues are apart)"""
    rows, cols = linear_sum_assignment(np.abs(np.asarray(lam)[:, None] - np.asarray(ref_lam)[None, :]))
    p = np.empty(len(lam), dtype=int)
    p[rows] = cols
    return p


def lam_tol(ref):
    n = len(ref["lam"])
    return C_LAM * n * EPS * ref["normA"] * ref["kappa"] * ref["condM"] * (1.0 if ref["exact"] else 2.0)


def check_eigenvalues(lam, ref, tol=None, lapack=None):
    """The per-eigenvalue bound, and 10x LAPACK's error where mpmath is the reference -> (pairing, worst err / bound).
    ``lapack``: LAPACK's eigenvalues of the same input, where that input is a transformation of the reference's system whose
    rounding the bound does not cover: then 10x LAPACK's error there is also accepted."""
    lam = np.asarray(lam, dtype=complex)
    p = _pair(lam, ref["lam"])
    err = np.abs(lam - ref["lam"][p])
    tol = (lam_tol(ref) if tol is None else tol)[p]
    wl = ref["lapack"] if lapack is None else lapack           # LAPACK's error for each reference eigenvalue
    pl = _pair(wl, ref["lam"])
    err_l = np.empty(len(lam))
    err_l[pl] = np.abs(wl - ref["lam"][pl])
    if lapack is not None:
        tol = np.maximum(tol, 10 * err_l[p])
    assert np.all(err <= tol), ("eigenvalue", np.max(err / tol), lam[np.argmax(err / tol)])
    if ref["exact"]:
        floor = 4 * EPS * ref["normA"] * ref["kappa"] * ref["condM"]
        lim = 10 * np.maximum(err_l, floor)[p]
        assert np.all(err <= lim), ("eigenvalue vs LAPACK", np.max(err / lim))
    return p, float(np.max(err / tol))


def _clusters(lam, tol):
    """groups of indices whose eigenvalues lie within tol_i + tol_j of each other (transitively)"""
    n = len(lam)
    parent = list(range(n))

    def find(a):
        while parent[a] != a:
            a = parent[a]
        return a
    for i in range(n):
        for j in range(i + 1, n):
            if abs(lam[i] - lam[j]) <= tol[i] + tol[j]:
                parent[find(i)] = find(j)
    groups = {}
    for i in range(n):
        groups.setdefault(find(i), []).append(i)
    return list(groups.values())


def sin_angle(Va, Vb):
    """sine of the largest principal angle between span(Va) and span(Vb) (same dimension)"""
    Qa, _ = np.linalg.qr(Va)
    Qb, _ = np.linalg.qr(Vb)
    return float(np.linalg.norm(Qa - Qb @ (Qb.conj().T @ Qa), 2))


def check_subspaces(V, p, ref, X=None, tol=None):
    """for each cluster of the reference, span(kernel modes) = span(reference vectors) to C_VEC n eps ||A|| cond(M) kappa / gap"""
    lamr = ref["lam"]
    X = ref["X"] if X is None else X
    tol = lam_tol(ref) if tol is None else tol
    n = len(lamr)
    kap = ref["kappa"].max()
    worst = 0.0
    for g in _clusters(lamr, 1e3 * tol):
        rest = np.setdiff1d(np.arange(n), g)
        if len(rest) == 0:
            continue
        gap = np.abs(lamr[g][:, None] - lamr[rest][None, :]).min()
        cols = [j for j in range(len(p)) if p[j] in g]
        s = sin_angle(V[:, cols], X[:, g])
        bound = max(C_VEC * n * EPS * ref["normA"] * ref["condM"] * kap / gap, 1e-12)
        assert s <= bound, ("subspace", g, s, bound)
        worst = max(worst, s / bound)
    return worst


def lapack_residual(M, K):
    w, V = np.linalg.eig(np.linalg.solve(M, K))
    return float((np.linalg.norm(K @ V - (M @ V) * w, axis=0) / (np.linalg.norm(K, 2) + np.abs(w) * np.linalg.norm(M, 2))).max())


def check_outputs(lam, V, info, M, K, res_tol=1e-13):
    """finite, unit 2-norm, complex modes' largest component real, residual <= res_tol (or all NaN with SINGULAR / NOCONV);
    the NaN slots of a DOF claim that left rows unclaimed are skipped"""
    lam, V = np.asarray(lam, dtype=complex), np.asarray(V, dtype=complex)
    if info & (SINGULAR | NOCONV):
        assert np.all(np.isnan(lam)) and np.all(np.isnan(V))
        return
    keep = ~np.isnan(lam.real)
    lam, V = lam[keep], V[:, keep]
    assert np.all(np.isfinite(lam)) and np.all(np.isfinite(V)), "non-finite outputs with info %d" % info
    nrm = np.linalg.norm(V, axis=0)
    assert np.all(np.abs(nrm - 1.0) <= 1e-14), ("norm", nrm)
    for j in np.flatnonzero(lam.imag != 0):
        a = np.abs(V[:, j])
        assert np.any((V[:, j].imag == 0.0) & (a >= a.max() * (1 - 4 * EPS))), ("phase", j)
    nC, nM = np.linalg.norm(K, 2), np.linalg.norm(M, 2)
    res = np.linalg.norm(K @ V - (M @ V) * lam[None, :], axis=0) / ((nC + np.abs(lam) * nM) * nrm)
    assert np.all(res <= res_tol), ("residual", res.max())
    return float(res.max())


def solve(M, K, sort="ascending", kernel=None):
    from raft_b200 import solver
    r = solver.solve_eigen(M, K, sort=sort)
    if kernel is not None:
        assert solver.last_dispatch()["kernel"] == kernel, (solver.last_dispatch()["kernel"], kernel)
    return r


def full_check(M, K, kernel, sort="ascending", ref=None, res_tol=1e-13):
    r = solve(M, K, sort, kernel)
    assert r["info"] & (SINGULAR | NOCONV) == 0, r["info"]
    check_outputs(r["lam"], r["modes"], r["info"], M, K, res_tol=res_tol)
    ref = reference(M, K) if ref is None else ref
    p, e = check_eigenvalues(r["lam"], ref)
    check_subspaces(np.asarray(r["modes"], dtype=complex), p, ref)
    return r, e


# ---- inputs ----------------------------------------------------------------------------------------------------------
def kernel_for(n):
    """the kernel the planner picks for n (n <= 12 k_eig_small; the slab holds H once it leaves shared memory)"""
    from raft_b200 import solver
    if n <= 12:
        return "eig-small"
    return "eig-cta-smem" if solver.eigen_workspace_bytes(1, n) == (2 * n * (n | 1) * 8 + 255) // 256 * 256 else "eig-cta-slab"


def smem_boundary():
    """(last n whose H fits in shared memory, first n in the slab), from the planner"""
    last = max(n for n in range(13, 400) if kernel_for(n) == "eig-cta-smem")
    return last, last + 1


def complex_system(n, seed):
    """M near I, a nonsymmetric K with complex-conjugate pairs (the first seed from `seed` that has one)"""
    for s in range(seed, seed + 100):
        rng = np.random.default_rng(s)
        M = np.eye(n) + 0.1 * np.diag(rng.uniform(size=n))
        K = rng.normal(size=(n, n)) * 5.0 + np.eye(n) * 3.0
        if np.any(np.linalg.eigvals(np.linalg.solve(M, K)).imag != 0):
            return M, K
    raise AssertionError("no complex pair")


def quasi_triangular(n, block, seed):
    """upper triangular with distinct diagonal 5, 6, ... and a trailing 2x2 block [[a, b], [c, d]]"""
    rng = np.random.default_rng(seed)
    T = np.triu(rng.uniform(-0.1, 0.1, size=(n, n)), 1) + np.diag(5.0 + np.arange(n))
    T[n - 2:, n - 2:] = np.array(block, dtype=float).reshape(2, 2)
    return T


LANV2 = {                                                        # eig_lanv2's branches
    "c0": [3.0, 1.5, 0.0, 2.0],                                  # upper triangular
    "b0": [2.0, 0.0, 1.5, 3.0],                                  # the swap
    "complex": [2.0, 3.0, -1.5, 2.0],                            # a = d, bc < 0
    "real_pair": [2.0, 3.0, 1.5, 2.0],                           # a = d, bc > 0
    "tiny_equal": [2.0, 1e-17, 1e-17, 2.0],                      # z < 4 ulp: equalise, then split into real eigenvalues
    "tiny_split": [2.0 + 2.0 ** -51, 1e-17, 1e-17, 2.0],         # a - d and bc tiny
    "tiny_complex": [2.0, 1e-17, -1e-17, 2.0],                   # z < 4 ulp, a complex pair
    "cancel": [3.0, 1.0, -(1.0 - 2.0 ** -53), 1.0],              # p^2 + bc cancels to 1 ulp: a nearly double real eigenvalue
    "lambda_I": [2.0, 0.0, 0.0, 2.0],
    "defective": [2.0, 1.0, 0.0, 2.0],
}


def jordan(n, lam):
    return lam * np.eye(n) + np.eye(n, k=1)


def orthogonal(n, seed):
    Q, R = np.linalg.qr(np.random.default_rng(seed).normal(size=(n, n)))
    return Q * np.sign(np.diag(R))


# ---- the DOF claim ---------------------------------------------------------------------------------------------------
def dof_claim(V, follow=None):
    """numpy restatement of the reference's DOF claim (raft_model.py:490-516): rows n-1..0 of |V| each take the column of
    their largest entry, the first on a tie; a column already taken is zeroed in that row and the search repeated, at most n
    times; the list of columns taken is reversed.  A row that takes nothing adds nothing, so the list can be shorter than n.
    ``follow``: columns in output order that a replay prefers among entries within 4 ulp of the row's maximum (the modes are
    the kernel's and its hypot may differ from numpy's by an ulp)."""
    mag = np.abs(np.asarray(V, dtype=complex))
    n = mag.shape[1]
    want = None if follow is None else list(follow)[::-1]
    taken = []
    for i in range(n - 1, -1, -1):
        row = mag[i].copy()
        for _ in range(n):
            top = row.max()
            j = int(np.argmax(row))
            if want is not None and len(taken) < len(want):
                near = np.flatnonzero(row >= top - 4 * np.spacing(top))
                k = want[len(taken)]
                if k in near and k not in taken:
                    j = k
                elif any(c in taken for c in near):
                    j = next(c for c in near if c in taken)
            if j in taken:
                row[j] = 0.0
            else:
                taken.append(j)
                break
    return taken[::-1]


def check_dof_order(M, K, kernel):
    """the kernel's DOF order against the restatement applied to its own modes (those of its ascending order) -> columns"""
    d = solve(M, K, "dof", kernel)
    a = solve(M, K, "ascending", kernel)
    ld, la = np.asarray(d["lam"], dtype=complex), np.asarray(a["lam"], dtype=complex)
    Vd, Va = np.asarray(d["modes"], dtype=complex), np.asarray(a["modes"], dtype=complex)
    cols = []
    for j in np.flatnonzero(~np.isnan(ld.real)):                 # the same internal column: bit-identical in both orders
        hit = [p for p in range(len(la)) if la[p] == ld[j] and np.array_equal(Va[:, p], Vd[:, j])]
        assert len(hit) == 1, (j, hit)
        cols.append(hit[0])
    nan = np.flatnonzero(np.isnan(ld.real))
    assert np.array_equal(nan, np.arange(len(cols), len(ld))) and np.all(np.isnan(Vd[:, nan]))
    assert dof_claim(Va, follow=cols) == cols, (dof_claim(Va, follow=cols), cols)
    return d, a, cols


# ==== without a GPU ===================================================================================================
@pytest.mark.parametrize("case", ["seeded6", "complex8", "wide12", "pivot6"])
def test_reference_lapack_meets_the_bound_against_mpmath(case):
    """the yardstick: LAPACK's eigenvalues meet the per-eigenvalue bound against mpmath, and kappa >= 1"""
    if case == "seeded6":
        M, K = (x[0] for x in seeded(6, 1, seed=11))
    elif case == "complex8":
        M, K = complex_system(8, 5)
    elif case == "wide12":                                       # eigenvalues from 1e-3 to 1e9
        Q = orthogonal(12, 3)
        M, K = np.eye(12), Q @ np.diag(np.logspace(-3, 9, 12)) @ Q.T + np.triu(np.ones((12, 12)), 1)
    else:
        M, K = pivoting_mass("perm", 6, 2)
    ref = reference(M, K)
    assert ref["exact"] and np.all(ref["kappa"] >= 1 - 1e-12)
    p, e = check_eigenvalues(ref["lapack"], ref)
    assert e <= 1.0
    check_subspaces(ref["lapack_X"], p, ref)


def test_reference_mpmath_vectors_are_eigenvectors():
    M, K = complex_system(6, 1)
    ref = reference(M, K)
    A = np.linalg.solve(M, K)
    assert np.abs(A @ ref["X"] - ref["X"] * ref["lam"]).max() <= 1e-13 * np.linalg.norm(A)


def test_shared_memory_boundary_from_the_planner():
    """H in shared memory up to the last n the opt-in limit holds, in the slab from the next n (an H100 without a device)"""
    from raft_b200 import solver
    last, first = smem_boundary()
    assert all(kernel_for(n) == "eig-cta-smem" for n in range(13, last + 1))
    assert all(kernel_for(n) == "eig-cta-slab" for n in range(first, first + 40))
    assert solver.eigen_workspace_bytes(1, first) == (3 * first * (first | 1) * 8 + 255) // 256 * 256
    assert all(solver.eigen_workspace_bytes(7, n) == 0 for n in range(1, 13))
    assert (last, first) == (167, 168)                           # 227 KB of opt-in shared memory per block on an H100


def test_dof_claim_restatement_by_hand():
    """the first-index tie, a claimed column zeroed and retried, and a row that claims nothing"""
    V = np.array([[0.5, 0.5, 0.0], [0.3, 0.9, 0.3], [0.7, 0.7, 0.1]])   # row 2 ties 0|1 -> 0; row 1 -> 1; row 0 -> 0, 1 taken,
    assert dof_claim(V) == [1, 0]                                         # column 2 zero there: argmax 0 again, nothing
    V = np.array([[0.1, 0.2, 0.9], [0.8, 0.1, 0.5], [0.1, 0.9, 0.2]])
    assert dof_claim(V) == [2, 0, 1]
    V = np.array([[0.0, 1.0, 0.0], [0.2, 0.3, 0.9], [0.0, 0.0, 1.0]])   # row 2 -> 2; row 1: 2 taken -> 1; row 0: 1 taken,
    assert dof_claim(V) == [0, 1, 2]                                      # then all zero: argmax 0, free -> 0
    V = np.array([[1.0, 0.2, 0.0], [0.5, 1.0, 0.0], [0.0, 1.0, 0.0]])
    assert dof_claim(V) == [0, 1]                                         # row 2 -> 1, row 1 -> 0, row 0 nothing
    # replaying a near tie: within 4 ulp either column is accepted
    V = np.array([[0.1, 0.2], [1.0, 1.0 + 2 * EPS]])
    assert dof_claim(V) == [0, 1] and dof_claim(V, follow=[1, 0]) == [1, 0]
    assert dof_claim(np.array([[0.1, 0.2], [1.0, 1.0 + 64 * EPS]]), follow=[1, 0]) == [0, 1]


def _claim_cases():
    rng = np.random.default_rng(21)
    out = []
    for n in (6, 12):
        M, K = seeded(n, 1, seed=n + 40)
        w, V = np.linalg.eig(np.linalg.solve(M[0], K[0]))
        out.append(("numpy-eig-%d" % n, w, V))
    M, K = complex_system(6, 9)
    w, V = np.linalg.eig(np.linalg.solve(M, K + 40.0 * M))         # the reference refuses eigenvalues with real part <= 0
    out.append(("numpy-eig-complex", w, V))
    w = np.arange(1.0, 7.0)
    V = np.eye(6) + 0.1 * rng.uniform(size=(6, 6))
    V[5, 2] = V[5, 4] = 1.5                                       # designed-in equal magnitudes: the first index wins
    V[3, 1] = V[3, 0] = 2.0
    out.append(("tie", w, V))
    V = np.eye(6)
    V[:4, :4] = [[1.0, 0.2, 0.0, 0.0], [0.5, 1.0, 0.0, 0.2], [0.0, 1.0, 0.0, 0.3], [0.3, 0.1, 1.0, 0.9]]
    V[4, 5] = 0.4
    out.append(("unclaimed", np.arange(1.0, 7.0), V))               # row 1's nonzeros only in columns already taken
    return out


@pytest.mark.parametrize("case", range(5))
def test_dof_claim_restatement_against_the_reference(case, monkeypatch):
    """the restatement against the reference's own Model.solveEigen on the same (eigenvalues, vectors), numpy's eig or designed"""
    import sys
    import types
    sys.path.insert(0, ROOT)
    from oracle import ref_harness as rh
    if not rh.reference_available():
        pytest.skip("reference tree not present")
    raft = rh.load_reference()
    rm = sys.modules[raft.Model.__module__]
    name, w, V = _claim_cases()[case]
    n = len(w)
    fake_np = types.SimpleNamespace(**{k: getattr(np, k) for k in dir(np) if not k.startswith("__")})
    fake_np.linalg = types.SimpleNamespace(eig=lambda A: (w.copy(), V.copy()), solve=np.linalg.solve)
    monkeypatch.setattr(rm, "np", fake_np)
    f = [types.SimpleNamespace(nDOF=6, M_struc=np.eye(6), A_hydro_morison=np.zeros((6, 6)), A_BEM=np.zeros((6, 6, 1)),
                               C_struc=np.eye(6) * 2, C_hydro=np.zeros((6, 6)), C_moor=np.zeros((6, 6)),
                               C_elast=np.zeros((6, 6)), yawstiff=0.0) for _ in range(n // 6)]
    model = types.SimpleNamespace(nDOF=n, fowtList=f, ms=None, results={})
    fns, modes = rm.Model.solveEigen(model)
    cols = dof_claim(V)
    np.testing.assert_array_equal(fns, np.sqrt(w[cols]) / 2.0 / np.pi)
    np.testing.assert_array_equal(modes, V[:, cols])
    if name == "unclaimed":
        assert len(cols) < n


# ==== on the GPU ======================================================================================================
SIZES = [1, 2, 3, 4, 5, 11, 12, 13, 31, 32, 33, 63, 64, 65, 127, 128, 129, "smem-last", "slab-first"]


def _size(n):
    if isinstance(n, str):
        last, first = smem_boundary()
        return last if n == "smem-last" else first
    return n


@gpu
@pytest.mark.parametrize("n", SIZES)
def test_sizes_against_the_reference(n):
    n = _size(n)
    kernel = kernel_for(n)
    nS = 2 if n <= 65 else 1
    M, K = seeded(n, nS, seed=1000 + n)
    worst = 0.0
    for s in range(nS):
        worst = max(worst, full_check(M[s], K[s], kernel)[1])
    if n >= 2:
        Mc, Kc = complex_system(n, 2000 + n)
        r, e = full_check(Mc, Kc, kernel)
        assert r["info"] & COMPLEX
        worst = max(worst, e)
    print("eigen edges n=%d (%s): worst |dlam| / bound %.2e" % (n, kernel, worst))


@gpu
@pytest.mark.parametrize("nS", [1, 31, 33, 65])
def test_small_kernel_partial_ctas(nS):
    """batches whose last 32-system CTA is partial: every system as it is alone, and as the reference has it"""
    M, K = seeded(6, nS, seed=500 + nS)
    Mc, Kc = complex_system(6, 77)
    M[nS // 2], K[nS // 2] = Mc, Kc
    r = solve(M, K, "ascending", "eig-small")
    for s in range(nS):
        one = solve(M[s:s + 1], K[s:s + 1], "ascending")
        lam = np.asarray(r["lam"][s], dtype=complex)
        assert np.array_equal(lam, np.asarray(one["lam"][0], dtype=complex))
        assert np.array_equal(np.asarray(r["modes"][s], dtype=complex), np.asarray(one["modes"][0], dtype=complex))
        assert r["info"][s] == one["info"][0]
        check_outputs(lam, r["modes"][s], r["info"][s], M[s], K[s])
    for s in (0, nS // 2, nS - 1):
        check_eigenvalues(r["lam"][s], reference(M[s], K[s]))


@gpu
@pytest.mark.parametrize("branch", list(LANV2))
@pytest.mark.parametrize("n", [2, 6, 40])
def test_lanv2_branches(n, branch):
    """each 2x2 standardisation, alone (n = 2) and as the trailing block of a quasi-triangular matrix (the TWO deflation
    rotates the rest of T and Q)"""
    T = np.array(LANV2[branch], dtype=float).reshape(2, 2) if n == 2 else quasi_triangular(n, LANV2[branch], n)
    M = np.eye(n)
    r = solve(M, T, "ascending", kernel_for(n))
    assert r["info"] & (SINGULAR | NOCONV) == 0
    check_outputs(r["lam"], r["modes"], r["info"], M, T)
    ref = reference(M, T)
    if branch == "defective":
        lam0 = 2.0
        tail = np.abs(np.asarray(r["lam"], dtype=complex) - lam0)
        assert np.sort(tail)[:2].max() <= 4 * np.sqrt(n * EPS * np.linalg.norm(T))
        return
    if branch in ("lambda_I", "tiny_equal", "tiny_split", "tiny_complex", "cancel"):
        # (nearly) double eigenvalues: kappa from the reference's own vectors is not a bound there; eps^(1/2)
        lam = np.asarray(r["lam"], dtype=complex)
        p = _pair(lam, ref["lam"])
        assert np.all(np.abs(lam - ref["lam"][p]) <= 4 * np.sqrt(n * EPS) * np.linalg.norm(T))
        return
    p, _ = check_eigenvalues(r["lam"], ref)
    check_subspaces(np.asarray(r["modes"], dtype=complex), p, ref)


def stalling(kind, n):
    if kind == "cyclic":                                         # eigenvalues 2 + the n-th roots of unity
        return np.roll(np.eye(n), 1, axis=0) + 2.0 * np.eye(n)
    Cm = np.zeros((n, n))                                        # companion of z^n - 2^n, shifted: 3 + 2 roots of unity
    Cm[1:, :-1] = np.eye(n - 1)
    Cm[0, -1] = 2.0 ** n
    return Cm + 3.0 * np.eye(n)


@gpu
@pytest.mark.parametrize("kind", ["cyclic", "companion"])
@pytest.mark.parametrize("n", [3, 4, 6, 12, 13, 40])
def test_stalling_shifts(kind, n):
    """matrices on which the standard Francis shifts stall: no NOCONV where LAPACK converges, and the §1 accuracy"""
    K = stalling(kind, n)
    M = np.eye(n)
    scipy.linalg.eigvals(K)                                      # LAPACK converges (raises otherwise)
    r = solve(M, K, "ascending", kernel_for(n))
    assert r["info"] & NOCONV == 0, r["info"]
    check_outputs(r["lam"], r["modes"], r["info"], M, K)
    ref = reference(M, K)
    p, _ = check_eigenvalues(r["lam"], ref)
    check_subspaces(np.asarray(r["modes"], dtype=complex), p, ref)


def pivoting_mass(kind, n, seed):
    """(M, K): M = P S with the diagonal never the pivot, a symmetric indefinite M, or an SPD M with cond ~ 1e12"""
    rng = np.random.default_rng(seed)
    _, K = seeded(n, 1, seed=seed + 7)
    K = K[0]
    Q = orthogonal(n, seed)
    if kind == "perm":
        B = rng.normal(size=(n, n))
        S = B @ B.T / n + np.eye(n) * 4.0
        M = np.roll(S, -1, axis=0)                               # row i of M is row i+1 of S: the big entry below the diagonal
    elif kind == "indefinite":
        d = rng.uniform(1.0, 3.0, size=n) * np.where(np.arange(n) % 3 == 1, -1.0, 1.0)
        M = (Q * d) @ Q.T
        M = (M + M.T) / 2
    else:
        M = (Q * np.logspace(0, 12, n)) @ Q.T
        M = (M + M.T) / 2
    return M, K


def _pivots(M):
    """the rows partial pivoting picks (first largest |a| of a column), as eig_solve_mc does"""
    X = np.array(M, dtype=float)
    n = len(X)
    out = []
    for k in range(n):
        p = k + int(np.argmax(np.abs(X[k:, k])))
        out.append(p)
        X[[k, p]] = X[[p, k]]
        X[k + 1:, k] /= X[k, k]
        X[k + 1:, k + 1:] -= np.outer(X[k + 1:, k], X[k, k + 1:])
    return out


@gpu
@pytest.mark.parametrize("kind", ["perm", "indefinite", "cond1e12"])
@pytest.mark.parametrize("n", [6, 12, 40, 200])
def test_pivoting_mass(kind, n):
    M, K = pivoting_mass(kind, n, n)
    if kind == "perm":
        assert all(p != k for k, p in enumerate(_pivots(M)[:-1]))
    # forming M^-1 C costs eps cond(M) in the residual of the pencil, for LAPACK as for the kernel
    r, _ = full_check(M, K, kernel_for(n), res_tol=max(1e-13, 10 * lapack_residual(M, K)))


@gpu
@pytest.mark.parametrize("copies", [2, 4, 24])
def test_identical_uncoupled_fowts(copies):
    """block-diagonal copies of one rigid fixture: every eigenvalue `copies` times, its eigenspace the copies of its mode"""
    z = fixture("OC3spar")
    M0, K0 = z["M_tot"], z["C_tot"]
    M, K = np.kron(np.eye(copies), M0), np.kron(np.eye(copies), K0)
    n = 6 * copies
    r = solve(M, K, "ascending", kernel_for(n))
    check_outputs(r["lam"], r["modes"], r["info"], M, K)
    r0 = reference(M0, K0)
    ref = dict(r0, lam=np.tile(r0["lam"], copies), kappa=np.tile(r0["kappa"], copies), X=np.kron(np.eye(copies), r0["X"]),
               normA=r0["normA"] * np.sqrt(copies), condM=skeel(M), exact=False)
    tol = lam_tol(ref)
    p = _pair(r["lam"], ref["lam"])
    assert np.all(np.abs(np.asarray(r["lam"]) - ref["lam"][p]) <= tol[p])
    check_subspaces(np.asarray(r["modes"], dtype=complex), p, ref, tol=tol)


@gpu
@pytest.mark.parametrize("hidden", [False, True])
@pytest.mark.parametrize("lam0", [1.0, 1e6])
@pytest.mark.parametrize("n", [12, 16, 22, 30, 64])
def test_jordan_blocks(n, lam0, hidden):
    """a defective eigenvalue of multiplicity n: finite unit modes with a small residual, eigenvalues to (n eps |A|)^(1/n)"""
    K = jordan(n, lam0)
    if hidden:
        Q = orthogonal(n, n)
        K = Q @ K @ Q.T
    M = np.eye(n)
    r = solve(M, K, "ascending", kernel_for(n))
    assert r["info"] & (SINGULAR | NOCONV) == 0, r["info"]
    check_outputs(r["lam"], r["modes"], r["info"], M, K)
    lam = np.asarray(r["lam"], dtype=complex)
    assert np.abs(lam - lam0).max() <= 4 * (n * EPS * np.linalg.norm(K)) ** (1.0 / n)
    if not hidden:
        assert np.all(lam == lam0)                               # T = J exactly: no rotation, no rounding


def _scaling(e_max, seed, n=6):
    return np.random.default_rng(seed).integers(-e_max, e_max + 1, size=n).astype(float)


@gpu
@pytest.mark.parametrize("e_max", [60, 300])
@pytest.mark.parametrize("how", ["similarity", "congruence"])
@pytest.mark.parametrize("name", RIGID)
def test_power_of_two_scaling(name, how, e_max):
    """D A D^-1 (M = I) and D M D, D C D (a change of units), D = 2^e, |e| <= e_max: the unscaled system's eigenvalues to its
    own bound, modes proportional to D v (similarity) or D^-1 v (congruence)"""
    z = fixture(name)
    M0, K0 = z["M_tot"], z["C_tot"]
    d = 2.0 ** _scaling(e_max, RIGID.index(name) + e_max)
    if how == "similarity":
        A0 = np.linalg.solve(M0, K0)
        ref = reference(np.eye(6), A0)
        M, K, X = np.eye(6), (d[:, None] * A0) / d[None, :], d[:, None] * ref["X"]
    else:
        ref = reference(M0, K0)
        M, K, X = d[:, None] * M0 * d[None, :], d[:, None] * K0 * d[None, :], ref["X"] / d[:, None]
    r = solve(M, K, "ascending", "eig-small")
    assert r["info"] & (SINGULAR | NOCONV) == 0
    check_outputs(r["lam"], r["modes"], r["info"], M, K)
    # balancing does not undo every such D exactly, and the degenerate roll / pitch pairs then split as they do in LAPACK
    wl, vl = np.linalg.eig(np.linalg.solve(M, K))
    p, _ = check_eigenvalues(r["lam"], ref, lapack=wl)
    X = X / np.linalg.norm(X, axis=0)
    V = np.asarray(r["modes"], dtype=complex)
    pl = _pair(wl, ref["lam"])
    lamr = ref["lam"]
    for j in range(6):                                          # modes of eigenvalues apart from the others
        if np.sort(np.abs(lamr - lamr[p[j]]))[1] < 1e-6 * np.abs(lamr).max():
            continue
        gap = np.sort(np.abs(lamr - lamr[p[j]]))[1]
        s_k = sin_angle(V[:, [j]], X[:, [p[j]]])
        s_l = sin_angle(vl[:, [int(np.flatnonzero(pl == p[j])[0])]], X[:, [p[j]]])
        bound = C_VEC * 6 * EPS * ref["normA"] * ref["condM"] * ref["kappa"].max() / gap
        assert s_k <= max(bound, 10 * s_l, 1e-12), (j, s_k, s_l, bound)


@gpu
def test_flexible_fixture_per_eigenvalue():
    """the rigid-body modes of the 150-DOF flexible FOWT held to their own accuracy, beside the tower modes"""
    z = fixture("VolturnUS-S-flexible")
    M, K = z["M_tot"], z["C_tot"]
    r, e = full_check(M, K, "eig-cta-smem")
    ref = reference(M, K)
    lam = np.asarray(r["lam"], dtype=complex)
    p = _pair(lam, ref["lam"])
    small = np.abs(ref["lam"][p]) < 1e-3 * np.abs(ref["lam"]).max()
    assert small.sum() >= 6
    print("flexible: worst |dlam| / bound %.2e, smallest eigenvalue rel err %.2e" % (
        e, np.max(np.abs(lam[small] - ref["lam"][p][small]) / np.abs(ref["lam"][p][small]))))


def _designed(V, w):
    return np.eye(len(w)), (V * w) @ np.linalg.inv(V)


@gpu
@pytest.mark.parametrize("case", ["seeded6", "seeded12", "seeded40", "complex6", "complex12", "tie6", "tie12"])
def test_dof_claim_order(case):
    """the kernel's DOF order is the restatement's on its own modes; conjugate pairs tie exactly and go first-index"""
    kind, n = case.rstrip("0123456789"), int(case.lstrip("abcdefghijklmnopqrstuvwxyz"))
    if kind == "seeded":
        M, K = (x[0] for x in seeded(n, 1, seed=300 + n))
    elif kind == "complex":
        M, K = complex_system(n, 400 + n)
    else:
        rng = np.random.default_rng(n)
        V = np.eye(n) + 0.05 * rng.uniform(size=(n, n))
        for i in range(0, n - 1, 2):                               # equal magnitudes between two columns in every other row
            V[i, i] = V[i, (i + 3) % n] = 1.0
        M, K = _designed(V, np.arange(1.0, n + 1.0) * 10.0)
    d, a, cols = check_dof_order(M, K, kernel_for(n))
    assert len(cols) == n
    lam = np.asarray(d["lam"], dtype=complex)
    for j in np.flatnonzero(lam.imag < 0):                        # the pair's +imag member is claimed first: it comes later
        k = np.flatnonzero(lam == np.conj(lam[j]))
        assert len(k) == 1 and k[0] > j, (j, k)


def unclaimed_system():
    """M = I and A block upper triangular with lower-triangular 2x2 diagonal blocks: eig_lanv2 swaps each block exactly, so
    the modes keep exact zeros and a row can find its nonzeros only in columns already claimed"""
    A = np.array([[1.0, 0.0, 0.0, 0.0, 0.0, 0.0],
                  [0.0, 2.0, 0.0, 0.0, 0.0, 0.0],
                  [0.0, 0.0, 3.0, 0.0, 0.7, 0.0],
                  [0.0, 0.0, 5.0, 4.0, 0.3, 0.9],
                  [0.0, 0.0, 0.0, 0.0, 5.0, 0.0],
                  [0.0, 0.0, 0.0, 0.0, 3.0, 6.0]])
    return np.eye(6), A


@gpu
def test_dof_claim_unclaimed_rows():
    from raft_b200 import solver
    M, K = unclaimed_system()
    d, a, cols = check_dof_order(M, K, "eig-small")
    assert len(cols) < 6 and np.isnan(np.asarray(d["lam"], dtype=complex)[len(cols):]).all()
    fns, modes = solver.eigen_fns_modes(M, K, "dof")
    assert np.array_equal(fns, np.sqrt(np.asarray(a["lam"])[cols]) / 2 / np.pi) and np.array_equal(modes, np.asarray(a["modes"])[:, cols])


@gpu
@pytest.mark.parametrize("sort", ["dof", "ascending"])
@pytest.mark.parametrize("n", [6, 40, 200])
def test_modes_false_is_bit_identical(n, sort):
    from raft_b200 import solver
    M, K = seeded(n, 3, seed=900 + n)
    Mc, Kc = complex_system(n, 950 + n)
    M[1], K[1] = Mc, Kc
    a = solver.solve_eigen(M, K, sort=sort, modes=True)
    b = solver.solve_eigen(M, K, sort=sort, modes=False)
    assert solver.last_dispatch()["kernel"] == kernel_for(n) and b["modes"] is None
    assert np.array_equal(a["lam"], b["lam"], equal_nan=True) and np.array_equal(a["info"], b["info"])
