// raftk_eigen.cuh -- natural frequencies and mode shapes (raftk_eigen_*, Model.solveEigen / FOWT.solveEigen,
// raft_model.py:436-547, raft_fowt.py:1646-1729): eigenvalues and right eigenvectors of A = M^-1 C for a batch of systems.
//
// One algorithm per system (Golub & Van Loan, Matrix Computations, 4th ed.: 3.4, 7.4-7.6), in FP64:
//   1. LU of M with partial pivoting (first largest |a| of a column), A = M^-1 C by forward and back substitution;
//   2. Parlett-Reinsch balancing by powers of two (no permutation): exact, no rounding;
//   3. Householder reduction to upper Hessenberg form, Q accumulated;
//   4. Francis double-shift implicit QR to real Schur form T = Q^T A Q (deflation on small subdiagonals, exceptional shifts
//      every 10th iteration, 2x2 blocks standardised), at most 30 n iterations in total;
//   5. eigenvectors of T by back-substitution (real eigenvalues and complex-conjugate pairs; the partial vector rescaled by a
//      power of two before a step could grow it past 2^400, as LAPACK's dtrevc rescales), back-transformed with Q,
//      un-balanced, scaled to unit 2-norm (the norm recomputed with max-abs scaling when the sum of squares leaves
//      [2^-900, 2^900]); a complex vector is rotated so that its largest component is real;
//   6. the output order: ascending (real part, then imaginary part; stable) or the DOF claim of the reference.
// The storage of one system is a set of accessors (EigSys) and the work is written as loops over `tid += nt` with sync()
// between phases, so the same device functions run one system per thread (k_eig_small: nt = 1, sync a no-op, working set
// interleaved across the 32 lanes of a CTA in shared memory) and one system per CTA (k_eig_cta: rows and columns of each
// reflector and bulge step shared by the CTA's threads; scalar decisions made by thread 0 and broadcast through shared memory).
// Every reduction is in a fixed order, so a system's result depends on neither the batch nor the number of resident CTAs.

#define EIG_SMALL_NMAX 12          // k_eig_small takes n <= 12: rigid designs and two-FOWT farms
#define EIG_SMALL_T 32             // systems (threads) per k_eig_small CTA
#define EIG_CTA_T 128              // threads per k_eig_cta CTA
#define EIG_NSC 8                  // broadcast scalars per system

// per-system vectors: doubles scale[n], wr[n], wi[n], w[n], sc[EIG_NSC]; ints claim[n], ord[n], isc[EIG_NSC]
__host__ __device__ inline int eig_vec_doubles(int n) { return 4 * n + EIG_NSC; }
__host__ __device__ inline int eig_vec_ints(int n) { return 2 * n + EIG_NSC; }
__host__ __device__ inline int eig_ld(int n) { return n | 1; }     // odd row stride: row-parallel shared-memory access without bank conflicts

template <int ES, bool CTA>
struct EigSys {
    int n, ld;
    double *h, *q, *x;      // [n][ld] each, element stride ES: H (A, then T), Q (then the eigenvectors), X (LU of M, then T's eigenvectors)
    double *dv;
    int *iv;
    int tid, nt;
    __device__ double &H(int i, int j) const { return h[(i * ld + j) * ES]; }
    __device__ double &Q(int i, int j) const { return q[(i * ld + j) * ES]; }
    __device__ double &X(int i, int j) const { return x[(i * ld + j) * ES]; }
    __device__ double &scale(int i) const { return dv[i * ES]; }
    __device__ double &wr(int i) const { return dv[(n + i) * ES]; }
    __device__ double &wi(int i) const { return dv[(2 * n + i) * ES]; }
    __device__ double &w(int i) const { return dv[(3 * n + i) * ES]; }
    __device__ double &sc(int i) const { return dv[(4 * n + i) * ES]; }
    __device__ int &claim(int i) const { return iv[i * ES]; }
    __device__ int &ord(int i) const { return iv[(n + i) * ES]; }
    __device__ int &isc(int i) const { return iv[(2 * n + i) * ES]; }
    __device__ bool lead() const { return tid == 0; }
    __device__ void sync() const { if (CTA) __syncthreads(); }
};

#define EIG_ULP 2.220446049250313e-16                  // eps * base (LAPACK dlamch('P'))
#define EIG_SAFMIN 2.2250738585072014e-308
#define EIG_SFMIN1 (EIG_SAFMIN / EIG_ULP)
#define EIG_SFMAX1 (1.0 / EIG_SFMIN1)
#define EIG_SFMIN2 (EIG_SFMIN1 * 2.0)
#define EIG_SFMAX2 (1.0 / EIG_SFMIN2)
#define EIG_GROW_LOG2 400                               // a back-substitution step keeps |quotient| * max(1, |column of T|) below 2^400 |pivot|

// (i, j) over [r0, r1) x [c0, c1), shared by the threads of a system
template <class S, class F> __device__ __forceinline__ void eig_par2(const S &s, int r0, int r1, int c0, int c1, F f)
{
    const int w = c1 - c0;
    if (w <= 0 || r1 <= r0) return;
    if (s.nt == 1) {
        for (int i = r0; i < r1; i++)
            for (int j = c0; j < c1; j++) f(i, j);
    } else {
        const int tot = (r1 - r0) * w;
        for (int e = s.tid; e < tot; e += s.nt) f(r0 + e / w, c0 + e % w);
    }
}

// 1. load, LU of M with partial pivoting, H = M^-1 C.  Returns RAFTK_EIG_SINGULAR on an exactly zero pivot.
template <class S> __device__ int eig_solve_mc(const S &s, const double *M, const double *C)
{
    const int n = s.n;
    eig_par2(s, 0, n, 0, n, [&](int i, int j) { s.X(i, j) = M[i * n + j]; s.H(i, j) = C[i * n + j]; });
    s.sync();
    for (int k = 0; k < n; k++) {
        if (s.lead()) {
            int p = k;
            double best = fabs(s.X(k, k));
            for (int i = k + 1; i < n; i++) {
                const double a = fabs(s.X(i, k));
                if (a > best) { best = a; p = i; }
            }
            s.isc(0) = p;
            s.isc(1) = best == 0.0;
        }
        s.sync();
        const int p = s.isc(0), zero = s.isc(1);
        s.sync();
        if (zero) return RAFTK_EIG_SINGULAR;
        if (p != k)
            for (int j = s.tid; j < n; j += s.nt) {
                double t = s.X(k, j); s.X(k, j) = s.X(p, j); s.X(p, j) = t;
                t = s.H(k, j); s.H(k, j) = s.H(p, j); s.H(p, j) = t;
            }
        s.sync();
        const double d = s.X(k, k);
        for (int i = k + 1 + s.tid; i < n; i += s.nt) s.X(i, k) /= d;
        s.sync();
        eig_par2(s, k + 1, n, k + 1, n, [&](int i, int j) { s.X(i, j) -= s.X(i, k) * s.X(k, j); });
        s.sync();
    }
    for (int j = s.tid; j < n; j += s.nt) {                 // one right-hand side (column of C) per thread
        for (int i = 1; i < n; i++) {
            double t = s.H(i, j);
            for (int k = 0; k < i; k++) t -= s.X(i, k) * s.H(k, j);
            s.H(i, j) = t;
        }
        for (int i = n - 1; i >= 0; i--) {
            double t = s.H(i, j);
            for (int k = i + 1; k < n; k++) t -= s.X(i, k) * s.H(k, j);
            s.H(i, j) = t / s.X(i, i);
        }
    }
    s.sync();
    return 0;
}

// 2. balancing: row i / f and column i * f with f a power of two, while that cuts ||row|| + ||col|| below 0.95 of itself
template <class S> __device__ void eig_balance(const S &s)
{
    const int n = s.n;
    for (int i = s.tid; i < n; i += s.nt) s.scale(i) = 1.0;
    for (int sweep = 0; sweep < 64; sweep++) {
        if (s.lead()) s.isc(2) = 0;
        s.sync();
        for (int i = 0; i < n; i++) {
            if (s.lead()) {
                double c = 0.0, r = 0.0, ca = 0.0, ra = 0.0;
                for (int k = 0; k < n; k++) {
                    const double a = s.H(k, i), b = s.H(i, k);
                    c += a * a; r += b * b;
                    ca = fmax(ca, fabs(a)); ra = fmax(ra, fabs(b));
                }
                c = sqrt(c); r = sqrt(r);
                double f = 1.0;
                if (c != 0.0 && r != 0.0) {
                    const double s0 = c + r;
                    double g = r / 2.0;
                    while (c < g && fmax(f, fmax(c, ca)) < EIG_SFMAX2 && fmin(r, fmin(g, ra)) > EIG_SFMIN2) {
                        f *= 2.0; c *= 2.0; ca *= 2.0; r /= 2.0; g /= 2.0; ra /= 2.0;
                    }
                    g = c / 2.0;
                    while (g >= r && fmax(r, ra) < EIG_SFMAX2 && fmin(fmin(f, c), fmin(g, ca)) > EIG_SFMIN2) {
                        f /= 2.0; c /= 2.0; g /= 2.0; ca /= 2.0; r *= 2.0; ra *= 2.0;
                    }
                    const double si = s.scale(i);
                    if (c + r >= 0.95 * s0) f = 1.0;
                    else if (f < 1.0 && si < 1.0 && f * si <= EIG_SFMIN1) f = 1.0;
                    else if (f > 1.0 && si > 1.0 && si >= EIG_SFMAX1 / f) f = 1.0;
                }
                if (f != 1.0) { s.scale(i) *= f; s.isc(2) = 1; }
                s.sc(0) = f;
            }
            s.sync();
            const double f = s.sc(0);
            if (f != 1.0) {
                const double g = 1.0 / f;
                for (int k = s.tid; k < n; k += s.nt)
                    if (k != i) { s.H(i, k) *= g; s.H(k, i) *= f; }
            }
            s.sync();
        }
        const int more = s.isc(2);
        s.sync();
        if (!more) break;
    }
}

// 3. Hessenberg reduction H <- Q^T H Q, Q = P_0 P_1 ... P_{n-3}
template <class S> __device__ void eig_hessenberg(const S &s)
{
    const int n = s.n;
    eig_par2(s, 0, n, 0, n, [&](int i, int j) { s.Q(i, j) = i == j ? 1.0 : 0.0; });
    s.sync();
    for (int k = 0; k + 2 < n; k++) {
        if (s.lead()) {                                     // P_k = I - tau v v^T, v = [1, w(k+2..)] on rows k+1..n-1
            const double alpha = s.H(k + 1, k);
            double xn = 0.0;
            for (int i = k + 2; i < n; i++) xn += s.H(i, k) * s.H(i, k);
            xn = sqrt(xn);
            double tau = 0.0;
            s.w(k + 1) = 1.0;
            if (xn != 0.0) {
                const double beta = -copysign(hypot(alpha, xn), alpha);
                tau = (beta - alpha) / beta;
                const double r = 1.0 / (alpha - beta);
                for (int i = k + 2; i < n; i++) s.w(i) = s.H(i, k) * r;
                s.H(k + 1, k) = beta;
            }
            for (int i = k + 2; i < n; i++) s.H(i, k) = 0.0;
            s.sc(0) = tau;
        }
        s.sync();
        const double tau = s.sc(0);
        if (tau != 0.0) {
            for (int r = s.tid; r < 2 * n; r += s.nt) {     // from the right: every row of H and of Q, columns k+1..n-1
                const bool hq = r < n;
                const int rr = hq ? r : r - n;
                double t = 0.0;
                for (int j = k + 1; j < n; j++) t += (hq ? s.H(rr, j) : s.Q(rr, j)) * s.w(j);
                t *= tau;
                for (int j = k + 1; j < n; j++) {
                    if (hq) s.H(rr, j) -= t * s.w(j);
                    else s.Q(rr, j) -= t * s.w(j);
                }
            }
            s.sync();
            for (int c = k + 1 + s.tid; c < n; c += s.nt) { // from the left: rows k+1..n-1, columns k+1..n-1
                double t = 0.0;
                for (int i = k + 1; i < n; i++) t += s.w(i) * s.H(i, c);
                t *= tau;
                for (int i = k + 1; i < n; i++) s.H(i, c) -= t * s.w(i);
            }
        }
        s.sync();
    }
}

// standardised Schur factorisation of a real 2x2 block [a b; c d] = [cs -sn; sn cs] [aa bb; cc dd] [cs sn; -sn cs]:
// c = 0 for real eigenvalues, a = d and b c < 0 for a complex pair; (rt1r, rt1i), (rt2r, rt2i) the eigenvalues, rt1i >= 0
__device__ inline void eig_lanv2(double &a, double &b, double &c, double &d, double &rt1r, double &rt1i, double &rt2r, double &rt2i,
                                 double &cs, double &sn)
{
    if (c == 0.0) {
        cs = 1.0; sn = 0.0;
    } else if (b == 0.0) {                                  // swap rows and columns
        cs = 0.0; sn = 1.0;
        const double t = d; d = a; a = t; b = -c; c = 0.0;
    } else if ((a - d) == 0.0 && (b > 0.0) != (c > 0.0)) {
        cs = 1.0; sn = 0.0;
    } else {
        const double temp = a - d;
        double p = 0.5 * temp;
        const double bcmax = fmax(fabs(b), fabs(c));
        const double bcmis = fmin(fabs(b), fabs(c)) * copysign(1.0, b) * copysign(1.0, c);
        double scale = fmax(fabs(p), bcmax);
        double z = (p / scale) * p + (bcmax / scale) * bcmis;
        if (z >= 4.0 * EIG_ULP) {                           // real eigenvalues
            z = p + copysign(sqrt(scale) * sqrt(z), p);
            a = d + z;
            d = d - (bcmax / z) * bcmis;
            const double tau = hypot(c, z);
            cs = z / tau; sn = c / tau;
            b = b - c; c = 0.0;
        } else {                                            // complex or nearly equal real eigenvalues: equalise the diagonal
            const double sigma = b + c;
            const double tau = hypot(sigma, temp);
            cs = sqrt(0.5 * (1.0 + fabs(sigma) / tau));
            sn = -(p / (tau * cs)) * copysign(1.0, sigma);
            const double aa = a * cs + b * sn, bb = -a * sn + b * cs, cc = c * cs + d * sn, dd = -c * sn + d * cs;
            a = aa * cs + cc * sn; b = bb * cs + dd * sn; c = -aa * sn + cc * cs; d = -bb * sn + dd * cs;
            const double t2 = 0.5 * (a + d);
            a = t2; d = t2;
            if (c != 0.0) {
                if (b != 0.0) {
                    if ((b > 0.0) == (c > 0.0)) {           // real eigenvalues: reduce to upper triangular
                        const double sab = sqrt(fabs(b)), sac = sqrt(fabs(c));
                        p = copysign(sab * sac, c);
                        const double t3 = 1.0 / sqrt(fabs(b + c));
                        a = t2 + p; d = t2 - p;
                        b = b - c; c = 0.0;
                        const double cs1 = sab * t3, sn1 = sac * t3;
                        const double t4 = cs * cs1 - sn * sn1;
                        sn = cs * sn1 + sn * cs1; cs = t4;
                    }
                } else {
                    b = -c; c = 0.0;
                    const double t4 = cs; cs = -sn; sn = t4;
                }
            }
        }
    }
    rt1r = a; rt2r = d;
    if (c == 0.0) { rt1i = 0.0; rt2i = 0.0; }
    else { rt1i = sqrt(fabs(b)) * sqrt(fabs(c)); rt2i = -rt1i; }
}

// Householder reflector of length nr <= 3 (LAPACK dlarfg): v <- [1, v1/(v0-beta), ...], returns tau, v0 <- beta
__device__ inline double eig_larfg(int nr, double &v0, double &v1, double &v2)
{
    const double xn = nr == 3 ? hypot(v1, v2) : (nr == 2 ? fabs(v1) : 0.0);
    if (xn == 0.0) return 0.0;
    const double beta = -copysign(hypot(v0, xn), v0);
    const double tau = (beta - v0) / beta;
    const double r = 1.0 / (v0 - beta);
    v1 *= r;
    if (nr == 3) v2 *= r;
    v0 = beta;
    return tau;
}

// 4. real Schur form: H <- T, Q <- Q Z, eigenvalues in wr / wi.  Returns RAFTK_EIG_NOCONV after 30 n iterations.
template <class S> __device__ int eig_schur(const S &s)
{
    const int n = s.n;
    const double smlnum = EIG_SAFMIN * ((double)n / EIG_ULP);
    const int itmax = 30 * n;
    int its = 0, kdefl = 0, i = n - 1, l = 0;
    enum { SWEEP = 0, ONE = 1, TWO = 2, FAIL = 3 };
    while (i >= 0) {
        if (s.lead()) {
            int k;
            for (k = i; k > l; k--) {                       // a negligible subdiagonal (Ahues & Tisseur's test)
                const double hk = fabs(s.H(k, k - 1));
                if (hk <= smlnum) break;
                double tst = fabs(s.H(k - 1, k - 1)) + fabs(s.H(k, k));
                if (tst == 0.0) {
                    if (k - 2 >= 0) tst += fabs(s.H(k - 1, k - 2));
                    if (k + 1 <= n - 1) tst += fabs(s.H(k + 1, k));
                }
                if (hk <= EIG_ULP * tst) {
                    const double ab = fmax(hk, fabs(s.H(k - 1, k))), ba = fmin(hk, fabs(s.H(k - 1, k)));
                    const double dkk = fabs(s.H(k - 1, k - 1) - s.H(k, k));
                    const double aa = fmax(fabs(s.H(k, k)), dkk), bb = fmin(fabs(s.H(k, k)), dkk);
                    const double sa = aa + ab;
                    if (ba * (ab / sa) <= fmax(smlnum, EIG_ULP * (bb * (aa / sa)))) break;
                }
            }
            const int lk = k;
            if (lk > 0) s.H(lk, lk - 1) = 0.0;
            int act = SWEEP, m = lk;
            if (lk == i) {
                act = ONE;
                s.wr(i) = s.H(i, i); s.wi(i) = 0.0;
            } else if (lk == i - 1) {
                act = TWO;
                double a = s.H(i - 1, i - 1), b = s.H(i - 1, i), c = s.H(i, i - 1), d = s.H(i, i), cs, sn;
                eig_lanv2(a, b, c, d, s.wr(i - 1), s.wi(i - 1), s.wr(i), s.wi(i), cs, sn);
                s.H(i - 1, i - 1) = a; s.H(i - 1, i) = b; s.H(i, i - 1) = c; s.H(i, i) = d;
                s.sc(0) = cs; s.sc(1) = sn;
            } else if (its >= itmax) {
                act = FAIL;
            } else {
                const int kd = kdefl + 1;
                double h11, h12, h21, h22;
                if (kd % 20 == 0) {                         // exceptional shift at the bottom of the active block
                    const double e = fabs(s.H(i, i - 1)) + fabs(s.H(i - 1, i - 2));
                    h11 = 0.75 * e + s.H(i, i); h12 = -0.4375 * e; h21 = e; h22 = h11;
                } else if (kd % 10 == 0) {                  // exceptional shift at its top
                    const double e = fabs(s.H(lk + 1, lk)) + fabs(s.H(lk + 2, lk + 1));
                    h11 = 0.75 * e + s.H(lk, lk); h12 = -0.4375 * e; h21 = e; h22 = h11;
                } else {
                    h11 = s.H(i - 1, i - 1); h21 = s.H(i, i - 1); h12 = s.H(i - 1, i); h22 = s.H(i, i);
                }
                double rt1r, rt1i, rt2r, rt2i;
                const double e = fabs(h11) + fabs(h12) + fabs(h21) + fabs(h22);
                if (e == 0.0) {
                    rt1r = rt1i = rt2r = rt2i = 0.0;
                } else {
                    h11 /= e; h21 /= e; h12 /= e; h22 /= e;
                    const double tr = (h11 + h22) / 2.0;
                    const double det = (h11 - tr) * (h22 - tr) - h12 * h21;
                    const double rtdisc = sqrt(fabs(det));
                    if (det >= 0.0) {                       // complex-conjugate shifts
                        rt1r = tr * e; rt2r = rt1r; rt1i = rtdisc * e; rt2i = -rt1i;
                    } else {                                // real shifts: the one closer to h22, twice
                        rt1r = tr + rtdisc; rt2r = tr - rtdisc;
                        if (fabs(rt1r - h22) <= fabs(rt2r - h22)) { rt1r *= e; rt2r = rt1r; }
                        else { rt2r *= e; rt1r = rt2r; }
                        rt1i = rt2i = 0.0;
                    }
                }
                double v0 = 0.0, v1 = 0.0, v2 = 0.0;
                for (m = i - 2; m >= lk; m--) {             // two consecutive small subdiagonals
                    double h21s = s.H(m + 1, m);
                    double sm = fabs(s.H(m, m) - rt2r) + fabs(rt2i) + fabs(h21s);
                    h21s = s.H(m + 1, m) / sm;
                    v0 = h21s * s.H(m, m + 1) + (s.H(m, m) - rt1r) * ((s.H(m, m) - rt2r) / sm) - rt1i * (rt2i / sm);
                    v1 = h21s * (s.H(m, m) + s.H(m + 1, m + 1) - rt1r - rt2r);
                    v2 = h21s * s.H(m + 2, m + 1);
                    sm = fabs(v0) + fabs(v1) + fabs(v2);
                    v0 /= sm; v1 /= sm; v2 /= sm;
                    if (m == lk) break;
                    const double h00 = fabs(s.H(m, m - 1)) * (fabs(v1) + fabs(v2));
                    const double h01 = fabs(v0) * (fabs(s.H(m - 1, m - 1)) + fabs(s.H(m, m)) + fabs(s.H(m + 1, m + 1)));
                    if (h00 <= EIG_ULP * h01) break;
                }
                s.sc(2) = v0; s.sc(3) = v1; s.sc(4) = v2;
            }
            s.isc(0) = act; s.isc(1) = lk; s.isc(2) = m;
        }
        s.sync();
        const int act = s.isc(0), lk = s.isc(1), m0 = s.isc(2);
        s.sync();
        if (act == FAIL) return RAFTK_EIG_NOCONV;
        if (act == ONE || act == TWO) {
            if (act == TWO) {                               // apply the block's rotation to the rest of T and to Q
                const double cs = s.sc(0), sn = s.sc(1);
                for (int r = s.tid; r < 2 * n; r += s.nt) {
                    const bool hq = r < n;
                    const int rr = hq ? r : r - n;
                    if (hq && rr > i) {                     // rows i-1, i; column rr
                        const double x = s.H(i - 1, rr), y = s.H(i, rr);
                        s.H(i - 1, rr) = cs * x + sn * y; s.H(i, rr) = cs * y - sn * x;
                    }
                    if (hq && rr < i - 1) {                 // columns i-1, i; row rr
                        const double x = s.H(rr, i - 1), y = s.H(rr, i);
                        s.H(rr, i - 1) = cs * x + sn * y; s.H(rr, i) = cs * y - sn * x;
                    }
                    if (!hq) {
                        const double x = s.Q(rr, i - 1), y = s.Q(rr, i);
                        s.Q(rr, i - 1) = cs * x + sn * y; s.Q(rr, i) = cs * y - sn * x;
                    }
                }
                s.sync();
            }
            kdefl = 0; l = 0;
            i = lk - 1;
            continue;
        }
        its++; kdefl++; l = lk;
        for (int k = m0; k <= i - 1; k++) {                 // chase the bulge from m0 to the bottom of the active block
            const int nr = min(3, i - k + 1);
            if (s.lead()) {
                double v0, v1, v2;
                if (k > m0) { v0 = s.H(k, k - 1); v1 = s.H(k + 1, k - 1); v2 = nr == 3 ? s.H(k + 2, k - 1) : 0.0; }
                else { v0 = s.sc(2); v1 = s.sc(3); v2 = s.sc(4); }
                const double t1 = eig_larfg(nr, v0, v1, v2);
                if (k > m0) {
                    s.H(k, k - 1) = v0; s.H(k + 1, k - 1) = 0.0;
                    if (k < i - 1) s.H(k + 2, k - 1) = 0.0;
                } else if (m0 > lk) {
                    s.H(k, k - 1) *= (1.0 - t1);
                }
                s.sc(5) = t1; s.sc(6) = v1; s.sc(7) = nr == 3 ? v2 : 0.0;
            }
            s.sync();
            const double t1 = s.sc(5), v1 = s.sc(6), v2 = s.sc(7), t2 = t1 * v1, t3 = t1 * v2;
            for (int j = k + s.tid; j < n; j += s.nt) {     // rows k..k+nr-1 from the left
                if (nr == 3) {
                    const double sm = s.H(k, j) + v1 * s.H(k + 1, j) + v2 * s.H(k + 2, j);
                    s.H(k, j) -= sm * t1; s.H(k + 1, j) -= sm * t2; s.H(k + 2, j) -= sm * t3;
                } else {
                    const double sm = s.H(k, j) + v1 * s.H(k + 1, j);
                    s.H(k, j) -= sm * t1; s.H(k + 1, j) -= sm * t2;
                }
            }
            s.sync();
            const int rh = min(k + 3, i) + 1;               // columns k..k+nr-1 from the right: rows 0..min(k+3,i) of H, all of Q
            for (int r = s.tid; r < rh + n; r += s.nt) {
                const bool hq = r < rh;
                const int rr = hq ? r : r - rh;
                double &a0 = hq ? s.H(rr, k) : s.Q(rr, k);
                double &a1 = hq ? s.H(rr, k + 1) : s.Q(rr, k + 1);
                if (nr == 3) {
                    double &a2 = hq ? s.H(rr, k + 2) : s.Q(rr, k + 2);
                    const double sm = a0 + v1 * a1 + v2 * a2;
                    a0 -= sm * t1; a1 -= sm * t2; a2 -= sm * t3;
                } else {
                    const double sm = a0 + v1 * a1;
                    a0 -= sm * t1; a1 -= sm * t2;
                }
            }
            s.sync();
        }
    }
    return 0;
}

// complex scalar helpers of the back-substitution (Smith's division)
struct EigC { double r, i; };
__device__ inline EigC eig_cdiv(EigC a, EigC b)
{
    if (fabs(b.i) <= fabs(b.r)) {
        const double e = b.i / b.r, f = b.r + b.i * e;
        return {(a.r + a.i * e) / f, (a.i - a.r * e) / f};
    }
    const double e = b.r / b.i, f = b.i + b.r * e;
    return {(a.r * e + a.i) / f, (a.i * e - a.r) / f};
}
__device__ inline EigC eig_csub(EigC a, EigC b) { return {a.r - b.r, a.i - b.i}; }
__device__ inline EigC eig_cmul(EigC a, EigC b) { return {a.r * b.r - a.i * b.i, a.r * b.i + a.i * b.r}; }
__device__ inline double eig_cabs1(EigC a) { return fabs(a.r) + fabs(a.i); }

// x = (A - lam I)^-1 b for a 2x2 block, complete pivoting; pivots below smin are replaced by smin (as LAPACK's dlaln2)
__device__ inline void eig_solve2(double a00, double a01, double a10, double a11, EigC lam, double smin, EigC &b0, EigC &b1)
{
    EigC A[4] = {{a00 - lam.r, -lam.i}, {a01, 0.0}, {a10, 0.0}, {a11 - lam.r, -lam.i}};
    int p = 0;
    for (int t = 1; t < 4; t++)
        if (eig_cabs1(A[t]) > eig_cabs1(A[p])) p = t;
    if (eig_cabs1(A[p]) < smin) {
        b0 = {b0.r / smin, b0.i / smin}; b1 = {b1.r / smin, b1.i / smin};
        return;
    }
    const int pr = p >> 1, pc = p & 1;                      // move the pivot to (0, 0)
    const EigC u00 = A[pr * 2 + pc], u01 = A[pr * 2 + (1 - pc)], l0 = A[(1 - pr) * 2 + pc], l1 = A[(1 - pr) * 2 + (1 - pc)];
    const EigC r0 = pr ? b1 : b0, r1 = pr ? b0 : b1;
    const EigC l10 = eig_cdiv(l0, u00);
    EigC u11 = eig_csub(l1, eig_cmul(l10, u01));
    if (eig_cabs1(u11) < smin) u11 = {smin, 0.0};
    const EigC y1 = eig_csub(r1, eig_cmul(l10, r0));
    const EigC x1 = eig_cdiv(y1, u11);
    const EigC x0 = eig_cdiv(eig_csub(r0, eig_cmul(u01, x1)), u00);
    if (pc) { b0 = x1; b1 = x0; } else { b0 = x0; b1 = x1; }
}

// eigenvector of T for eigenvalue ki (real) or the pair (ki-1, ki) into X(:, ki) (real) or X(:, ki-1) + i X(:, ki), rows 0..ki.
// w(j) holds the largest |T(k, j)|, k < j.  Dividing by a pivot near smin grows the partial vector by up to 1 / smin per step
// (a Jordan block overflows after about 20 steps), so before a step whose quotient times max(1, w) could pass 2^400 |pivot| the
// vector is scaled down by a power of two; the unit-norm scaling later makes the result independent of that scale.
template <bool CPX, class S> __device__ void eig_trevc(const S &s, int ki)
{
    const int n = s.n;
    const int kr = CPX ? ki - 1 : ki;                       // column of the real part; the imaginary part is in column ki
    const EigC lam = {s.wr(kr), CPX ? sqrt(fabs(s.H(ki, ki - 1))) * sqrt(fabs(s.H(ki - 1, ki))) : 0.0};
    const double smin = fmax(EIG_ULP * (fabs(lam.r) + fabs(lam.i)), EIG_SAFMIN * ((double)n / EIG_ULP));
    auto get = [&](int k) -> EigC { return {s.X(k, kr), CPX ? s.X(k, ki) : 0.0}; };
    auto put = [&](int k, EigC v) { s.X(k, kr) = v.r; if (CPX) s.X(k, ki) = v.i; };
    auto guard = [&](double xa, double g, double da) {     // rescale so that xa max(1, g) < 2^EIG_GROW_LOG2 da
        g = fmax(1.0, g);
        if (!(xa * g > scalbn(da, EIG_GROW_LOG2))) return;
        const double f = scalbn(1.0, ilogb(da) + EIG_GROW_LOG2 - ilogb(xa) - ilogb(g) - 2);
        for (int k = 0; k <= ki; k++) { s.X(k, kr) *= f; if (CPX) s.X(k, ki) *= f; }
    };
    int top;
    if (CPX) {
        EigC a, b;
        if (fabs(s.H(ki - 1, ki)) >= fabs(s.H(ki, ki - 1))) { a = {1.0, 0.0}; b = {0.0, lam.i / s.H(ki - 1, ki)}; }
        else { a = {-lam.i / s.H(ki, ki - 1), 0.0}; b = {0.0, 1.0}; }
        put(ki - 1, a); put(ki, b);
        for (int k = 0; k < ki - 1; k++) put(k, {-a.r * s.H(k, ki - 1), -b.i * s.H(k, ki)});
        top = ki - 2;
    } else {
        s.X(ki, ki) = 1.0;
        for (int k = 0; k < ki; k++) s.X(k, ki) = -s.H(k, ki);
        top = ki - 1;
    }
    for (int j = top; j >= 0;) {
        if (j > 0 && s.H(j, j - 1) != 0.0) {                // 2x2 diagonal block (j-1, j): |x| <= 8 |b| / smin
            guard(fmax(eig_cabs1(get(j - 1)), eig_cabs1(get(j))), fmax(s.w(j - 1), s.w(j)), 0.125 * smin);
            EigC b0 = get(j - 1), b1 = get(j);
            eig_solve2(s.H(j - 1, j - 1), s.H(j - 1, j), s.H(j, j - 1), s.H(j, j), lam, smin, b0, b1);
            put(j - 1, b0); put(j, b1);
            for (int k = 0; k < j - 1; k++) {
                const EigC v = get(k);
                put(k, {v.r - b0.r * s.H(k, j - 1) - b1.r * s.H(k, j), v.i - b0.i * s.H(k, j - 1) - b1.i * s.H(k, j)});
            }
            j -= 2;
        } else {
            EigC d = {s.H(j, j) - lam.r, -lam.i};
            if (eig_cabs1(d) < smin) d = {smin, 0.0};
            guard(eig_cabs1(get(j)), s.w(j), eig_cabs1(d));
            const EigC y = eig_cdiv(get(j), d);
            put(j, y);
            for (int k = 0; k < j; k++) {
                const EigC v = get(k);
                put(k, {v.r - y.r * s.H(k, j), v.i - y.i * s.H(k, j)});
            }
            j -= 1;
        }
    }
    if (CPX) { s.X(ki, kr) = 0.0; s.X(ki - 1, ki) = 0.0; }
}

// 5. eigenvectors into Q (LAPACK's real layout: a pair (c, c+1) is Q(:,c) +- i Q(:,c+1)), un-balanced, unit 2-norm, phase
template <class S> __device__ void eig_vectors(const S &s)
{
    const int n = s.n;
    for (int j = s.tid; j < n; j += s.nt) {                 // the growth bound of each back-substitution step
        double g = 0.0;
        for (int k = 0; k < j; k++) g = fmax(g, fabs(s.H(k, j)));
        s.w(j) = g;
    }
    s.sync();
    for (int k = s.tid; k < n; k += s.nt) {                 // one eigenvector (or pair) per thread
        if (s.wi(k) == 0.0) eig_trevc<false>(s, k);
        else if (s.wi(k) < 0.0) eig_trevc<true>(s, k);
    }
    s.sync();
    for (int r = s.tid; r < n; r += s.nt) {                 // V = Q X, in place from the last column down; then D V
        for (int c = n - 1; c >= 0; c--) {
            if (s.wi(c) < 0.0) {
                double re = 0.0, im = 0.0;
                for (int k = 0; k <= c; k++) { re += s.Q(r, k) * s.X(k, c - 1); im += s.Q(r, k) * s.X(k, c); }
                s.Q(r, c - 1) = re; s.Q(r, c) = im;
                c--;
            } else {
                double re = 0.0;
                for (int k = 0; k <= c; k++) re += s.Q(r, k) * s.X(k, c);
                s.Q(r, c) = re;
            }
        }
        const double d = s.scale(r);
        for (int c = 0; c < n; c++) s.Q(r, c) *= d;
    }
    s.sync();
    for (int c = s.tid; c < n; c += s.nt) {
        if (s.wi(c) == 0.0) {
            double nn = 0.0;
            for (int r = 0; r < n; r++) nn += s.Q(r, c) * s.Q(r, c);
            double f = 1.0 / sqrt(nn);
            if (!(nn >= 0x1p-900 && nn <= 0x1p+900)) {      // the sum of squares over- or underflows: scale by the largest entry
                double amax = 0.0;
                for (int r = 0; r < n; r++) amax = fmax(amax, fabs(s.Q(r, c)));
                const int e = ilogb(amax);
                double t = 0.0;
                for (int r = 0; r < n; r++) { const double v = scalbn(s.Q(r, c), -e); t += v * v; }
                f = scalbn(1.0 / sqrt(t), -e);
            }
            for (int r = 0; r < n; r++) s.Q(r, c) *= f;
        } else if (s.wi(c) > 0.0) {
            double n0 = 0.0, n1 = 0.0;
            for (int r = 0; r < n; r++) { n0 += s.Q(r, c) * s.Q(r, c); n1 += s.Q(r, c + 1) * s.Q(r, c + 1); }
            double f = 1.0 / hypot(sqrt(n0), sqrt(n1));
            if (!(n0 + n1 >= 0x1p-900 && n0 + n1 <= 0x1p+900)) {     // as for a real vector
                double amax = 0.0;
                for (int r = 0; r < n; r++) amax = fmax(amax, fmax(fabs(s.Q(r, c)), fabs(s.Q(r, c + 1))));
                const int e = ilogb(amax);
                double t = 0.0;
                for (int r = 0; r < n; r++) {
                    const double u = scalbn(s.Q(r, c), -e), v = scalbn(s.Q(r, c + 1), -e);
                    t += u * u + v * v;
                }
                f = scalbn(1.0 / sqrt(t), -e);
            }
            int kmax = 0;
            double best = -1.0;
            for (int r = 0; r < n; r++) {
                s.Q(r, c) *= f; s.Q(r, c + 1) *= f;
                const double m2 = s.Q(r, c) * s.Q(r, c) + s.Q(r, c + 1) * s.Q(r, c + 1);
                if (m2 > best) { best = m2; kmax = r; }
            }
            const double fx = s.Q(kmax, c), gx = s.Q(kmax, c + 1);   // rotate the largest component onto the real axis
            double cs = 1.0, sn = 0.0;
            if (gx != 0.0) {
                if (fx == 0.0) { cs = 0.0; sn = copysign(1.0, gx); }
                else { const double d = hypot(fx, gx); cs = fabs(fx) / d; sn = gx / copysign(d, fx); }
            }
            for (int r = 0; r < n; r++) {
                const double x = s.Q(r, c), y = s.Q(r, c + 1);
                s.Q(r, c) = cs * x + sn * y; s.Q(r, c + 1) = cs * y - sn * x;
            }
            s.Q(kmax, c + 1) = 0.0;
        }
    }
    s.sync();
}

// component r of eigenvector c (complex)
template <class S> __device__ __forceinline__ EigC eig_vec(const S &s, int r, int c)
{
    const double w = s.wi(c);
    if (w == 0.0) return {s.Q(r, c), 0.0};
    if (w > 0.0) return {s.Q(r, c), s.Q(r, c + 1)};
    return {s.Q(r, c - 1), -s.Q(r, c)};
}

// 6. output order into ord(): ascending (real part, then imaginary part; stable), or the reference's DOF claim
// (raft_model.py:490-516): rows n-1..0 of |V| each claim the column of their largest entry (first index on a tie), an
// already claimed column is zeroed and the search repeated, and the list is reversed.  A row that claims nothing within n
// tries leaves its slot -1 (the reference then returns fewer modes).  Flags into isc(3).
template <class S> __device__ void eig_order(const S &s, int sort)
{
    const int n = s.n;
    if (s.lead()) {
        int flags = 0;
        for (int k = 0; k < n; k++) {
            if (s.wi(k) != 0.0) flags |= RAFTK_EIG_COMPLEX;
            if (!(s.wr(k) > 0.0)) flags |= RAFTK_EIG_NONPOSITIVE;
        }
        if (sort == RAFTK_EIG_SORT_ASCENDING) {
            for (int k = 0; k < n; k++) {
                const int o = k;
                int j = k;
                while (j > 0) {
                    const int p = s.ord(j - 1);
                    const bool less = s.wr(o) < s.wr(p) || (s.wr(o) == s.wr(p) && s.wi(o) < s.wi(p));
                    if (!less) break;
                    s.ord(j) = p; j--;
                }
                s.ord(j) = o;
            }
        } else {
            for (int k = 0; k < n; k++) { s.claim(k) = 0; s.ord(k) = -1; }
            int cnt = 0;
            for (int i = n - 1; i >= 0; i--) {
                for (int c = 0; c < n; c++) { const EigC v = eig_vec(s, i, c); s.w(c) = hypot(v.r, v.i); }
                for (int t = 0; t < n; t++) {
                    int ind = 0;
                    for (int c = 1; c < n; c++)
                        if (s.w(c) > s.w(ind)) ind = c;
                    if (s.claim(ind)) s.w(ind) = 0.0;
                    else { s.claim(ind) = 1; s.ord(cnt++) = ind; break; }
                }
            }
            for (int a = 0, b = cnt - 1; a < b; a++, b--) { const int t = s.ord(a); s.ord(a) = s.ord(b); s.ord(b) = t; }
        }
        s.isc(3) = flags;
    }
    s.sync();
}

// the whole analysis of system `sys`; `flags` gathers the RAFTK_EIG_* bits, written by the caller's lead thread
template <class S> __device__ int eig_system(const S &s, const raftk_eigen &e, int sys)
{
    const int n = s.n;
    const size_t nn = (size_t)n * n;
    const double *M = e.M + sys * nn, *C = e.C + sys * nn;
    int flags = 0;
    for (int i = 0; i < n; i++)
        if (M[i * n + i] < 1.0 || C[i * n + i] < 1.0) flags |= RAFTK_EIG_SMALL_DIAG;
    int rc = eig_solve_mc(s, M, C);
    if (!rc) {
        eig_balance(s);
        eig_hessenberg(s);
        rc = eig_schur(s);
    }
    double *lam = e.lam + sys * (size_t)n * 2;
    double *modes = e.modes ? e.modes + sys * nn * 2 : nullptr;
    if (rc) {                                               // no spectrum: NaN outputs, the flag says why
        for (int j = s.tid; j < n; j += s.nt) lam[2 * j] = lam[2 * j + 1] = CUDART_NAN;
        if (modes)
            for (size_t t = s.tid; t < 2 * nn; t += s.nt) modes[t] = CUDART_NAN;
        s.sync();
        return flags | rc;
    }
    eig_vectors(s);
    eig_order(s, e.sort);
    flags |= s.isc(3);
    for (int j = s.tid; j < n; j += s.nt) {
        const int c = s.ord(j);
        lam[2 * j] = c < 0 ? CUDART_NAN : s.wr(c);
        lam[2 * j + 1] = c < 0 ? CUDART_NAN : s.wi(c);
    }
    if (modes)
        eig_par2(s, 0, n, 0, n, [&](int r, int j) {
            const int c = s.ord(j);
            const EigC v = c < 0 ? EigC{CUDART_NAN, CUDART_NAN} : eig_vec(s, r, c);
            modes[(r * (size_t)n + j) * 2] = v.r;
            modes[(r * (size_t)n + j) * 2 + 1] = v.i;
        });
    s.sync();
    return flags;
}

// one system per thread, n <= 12; thread t's working set interleaved at stride EIG_SMALL_T in dynamic shared memory
__global__ void __launch_bounds__(EIG_SMALL_T) k_eig_small(const raftk_eigen e)
{
    extern __shared__ double eig_smem[];
    const int n = e.n, ld = eig_ld(n), lane = threadIdx.x;
    const int sys = blockIdx.x * EIG_SMALL_T + lane;
    if (sys >= e.n_systems) return;
    EigSys<EIG_SMALL_T, false> s;
    s.n = n; s.ld = ld; s.tid = 0; s.nt = 1;
    const int mat = n * ld;
    s.h = eig_smem + lane;
    s.q = s.h + (size_t)mat * EIG_SMALL_T;
    s.x = s.q + (size_t)mat * EIG_SMALL_T;
    s.dv = s.x + (size_t)mat * EIG_SMALL_T;
    s.iv = reinterpret_cast<int *>(eig_smem + (size_t)(3 * mat + eig_vec_doubles(n)) * EIG_SMALL_T) + lane;
    e.info[sys] = eig_system(s, e, sys);
}

// one system per CTA, persistent CTAs walking the system list; Q and X in the CTA's workspace slab, H in shared memory
// (H_SMEM) or in the slab
template <bool H_SMEM>
__global__ void __launch_bounds__(EIG_CTA_T) k_eig_cta(const raftk_eigen e, double *ws, size_t slab_doubles)
{
    extern __shared__ double eig_smem[];
    const int n = e.n, ld = eig_ld(n), mat = n * ld;
    EigSys<1, true> s;
    s.n = n; s.ld = ld; s.tid = threadIdx.x; s.nt = blockDim.x;
    double *slab = ws + blockIdx.x * slab_doubles;
    s.q = slab;
    s.x = slab + mat;
    s.dv = eig_smem;
    s.iv = reinterpret_cast<int *>(eig_smem + eig_vec_doubles(n));
    s.h = H_SMEM ? eig_smem + eig_vec_doubles(n) + (eig_vec_ints(n) + 1) / 2 : slab + 2 * (size_t)mat;
    for (int sys = blockIdx.x; sys < e.n_systems; sys += gridDim.x) {
        const int f = eig_system(s, e, sys);
        if (s.lead()) e.info[sys] = f;
        __syncthreads();
    }
}
