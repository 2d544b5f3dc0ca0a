// raftk_lu.cuh -- the dense complex LU with partial pivoting of every system factored in shared or global memory
// (k_system_solve*, k_farm_response*, k_gen_solve_blocked, k_gen_train_solve; included by raftk.cu only).
// One numerical contract for all of them: the pivot of column k is the first maximum of |re| + |im| over rows k..n-1 (LAPACK
// izamax), and every element receives its rank-1 updates in ascending k, so that the column-at-a-time and the blocked
// factorisations round alike, whatever the thread count, panel width or placement.  Pivot reciprocals and back-substitution
// quotients are taken at the pivot's own scale: piv_recip / piv_div (raftk_common.cuh).
// A group of T threads works on one system: one warp when T = 32 (no CTA-wide barrier), else the whole CTA.
// Loops strided by the group size stay rolled (#pragma unroll 1): unrolled, they cost the in-place kernels enough registers
// to lose a CTA per SM.
#pragma once

template <int T> __device__ __forceinline__ void gsync() { if (T == 32) __syncwarp(); else __syncthreads(); }

// v -= l u
__device__ __forceinline__ void cmsub(double2 &v, const double2 l, const double2 u)
{
    v.x -= l.x * u.x - l.y * u.y; v.y -= l.x * u.y + l.y * u.x;
}

// multiplier v / pivot, from the pivot's reciprocal ri
__device__ __forceinline__ double2 lu_mult(const double2 v, const double2 ri)
{
    return make_double2(v.x * ri.x - v.y * ri.y, v.x * ri.y + v.y * ri.x);
}

// Pivot row of the column x[r * ld], rows j..m-1.  Threads 0..S-1 scan it and a warp butterfly reduces (the lower row wins a
// tie).  S = 32: every lane of the warp ends on the winner.  S > 32: the per-warp winners go through best_s / idx_s and every
// thread finishes the reduction itself, so all S end on the same row; a __syncthreads() must separate the return from the
// next call's writes to the slots.
template <int S>
__device__ __forceinline__ int lu_pivot_row(const double2 *x, int ld, int j, int m, int tid, double *best_s, int *idx_s)
{
    double best = -1.0; int p = j;
#pragma unroll 1
    for (int r = j + tid; r < m; r += S) {
        const double2 v = x[r * ld];
        const double t = fabs(v.x) + fabs(v.y);
        if (t > best) { best = t; p = r; }
    }
    for (int o = 16; o >= 1; o >>= 1) {
        const double ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int op = __shfl_xor_sync(0xffffffffu, p, o);
        if (ob > best || (ob == best && op < p)) { best = ob; p = op; }
    }
    if constexpr (S > 32) {
        if ((tid & 31) == 0) { best_s[tid >> 5] = best; idx_s[tid >> 5] = p; }
        __syncthreads();
        best = best_s[0]; p = idx_s[0];
#pragma unroll
        for (int q = 1; q < S / 32; q++) if (best_s[q] > best || (best_s[q] == best && idx_s[q] < p)) { best = best_s[q]; p = idx_s[q]; }
    }
    return p;
}

// Shared slots of a factorisation in place: the current column's pivot row and reciprocal, and the info word.
struct LuSlots { int *piv; double2 *rinv; int *bad; };

// Shared slots of a factorisation with a staged panel: the per-warp winners of the T-thread pivot search, the panel's pivot
// rows (panel-relative) and the info word.
template <int T, int PWMAX> struct LuStaged {
    double best[T / 32];
    int idx[T / 32];
    int piv[PWMAX];
    int bad;
};

// One elimination step in place on column col of the augmented system A [n][nc]: pivot search by the group's first warp,
// swap of the whole rows, multipliers.
template <int T>
__device__ __forceinline__ void lu_pivot_step(double2 *A, int n, int nc, int col, int gtid, LuSlots S)
{
    if (gtid < 32) {
        const int p = lu_pivot_row<32>(A + col, nc, col, n, gtid, nullptr, nullptr);
        if (gtid == 0) {
            *S.piv = p;
            bool zero;
            *S.rinv = piv_recip(A[p * nc + col], zero);
            if (zero && *S.bad == 0) *S.bad = col + 1;
        }
    }
    gsync<T>();
    const int p = *S.piv;
    if (p != col) for (int t = gtid; t < nc; t += T) { const double2 tmp = A[col * nc + t]; A[col * nc + t] = A[p * nc + t]; A[p * nc + t] = tmp; }
    gsync<T>();
    const double2 ri = *S.rinv;
#pragma unroll 1
    for (int r = col + 1 + gtid; r < n; r += T) A[r * nc + col] = lu_mult(A[r * nc + col], ri);
    gsync<T>();
}

// Column-at-a-time LU in place of the augmented system A [n][nc], the right-hand sides eliminated along: small systems, where
// one panel per column is the right shape.  Returns k + 1 of the first zero pivot, else 0.
template <int T>
__device__ __forceinline__ int lu_unblocked(double2 *A, int n, int nc, int gtid, LuSlots S)
{
    if (gtid == 0) *S.bad = 0;
    for (int k = 0; k < n; k++) {
        lu_pivot_step<T>(A, n, nc, k, gtid, S);
        const int rows = n - k - 1, cols = nc - k - 1;
#pragma unroll 1
        for (int t = gtid; t < rows * cols; t += T) {
            const int r = k + 1 + t / cols, cidx = k + 1 + t % cols;
            const double2 l = A[r * nc + k], u = A[k * nc + cidx];
            double2 v = A[r * nc + cidx];
            cmsub(v, l, u);
            A[r * nc + cidx] = v;
        }
        gsync<T>();
    }
    return *S.bad;
}

// Blocked right-looking LU of the augmented system [A | B]: A [n][lda] (columns 0..n-1), B [n][ldb] (the nrhs right-hand
// sides, columns n..n+nrhs-1), one CTA of T threads.  Per panel of pw columns:
//   1. the panel is factored column by column: pivot, interchange, multipliers, update of the panel's own columns;
//   2. one thread per column right of the panel applies the panel's interchanges there and solves the row block against the
//      unit-lower panel head;
//   3. the trailing matrix takes the panel's pw rank-1 updates from a 4 x 2 register tile per thread: every element is loaded
//      and stored once per panel, so the panel width divides the traffic to the matrix.
// STAGE_PANEL = false: [A | B] is in shared memory (B = A + n, ldb = lda), the panel is factored in place with S = the LuSlots,
//   and each interchange swaps whole rows.
// STAGE_PANEL = true: [A | B] is in global memory (L2-resident while the CTA works on it); the panel is factored in the shared
//   scratch Ps [n][pw] with S = LuStaged<T, >= pw>, and its interchanges reach the columns right of it only: the factored A's
//   columns left of each panel keep the rows they had when that panel was done.  piv (or NULL) receives the pivot rows.
// STAGE_ROWS (with STAGE_PANEL): the row block is solved in the shared scratch Us [pw][n + nrhs] and the trailing update reads
//   it there.
// Returns k + 1 of the first zero pivot, else 0.  Every thread of the CTA takes part.
template <int T, bool STAGE_PANEL, bool STAGE_ROWS, class Sh>
__device__ __forceinline__ int lu_blocked(double2 *A, int lda, double2 *B, int ldb, int n, int nrhs, int pw, Sh &S,
                                          double2 *Ps = nullptr, double2 *Us = nullptr, int *piv = nullptr)
{
    static_assert(STAGE_PANEL || !STAGE_ROWS, "the row block is staged with the panel");
    using Ix = typename std::conditional<STAGE_PANEL, size_t, int>::type;
    const int tid = threadIdx.x, nc = n + nrhs;
    // column col of [A | B] from row 0, and its leading dimension
    auto column = [&](int col, Ix &ld) -> double2 * {
        if constexpr (!STAGE_PANEL) { ld = lda; return A + col; }
        ld = col < n ? (Ix)lda : (Ix)ldb;
        return col < n ? A + col : B + (col - n);
    };
    // multiplier of row kb + r in the panel's column j
    auto lmul = [&](int kb, int r, int j) -> double2 {
        if constexpr (STAGE_PANEL) return Ps[r * pw + j];
        else return A[(kb + r) * lda + kb + j];
    };
    if constexpr (STAGE_PANEL) { if (tid == 0) S.bad = 0; } else { if (tid == 0) *S.bad = 0; }
    for (int kb = 0; kb < n; kb += pw) {
        const int nb = min(pw, n - kb), m = n - kb, c0 = kb + nb;
        // ---- 1. the panel ---------------------------------------------------------------------------------------------
        if constexpr (STAGE_PANEL) {
#pragma unroll 1
            for (int t = tid; t < m * nb; t += T) { const int r = t / nb, j = t - r * nb; Ps[r * pw + j] = A[(size_t)(kb + r) * lda + kb + j]; }
            __syncthreads();
            for (int j = 0; j < nb; j++) {
                const int p = lu_pivot_row<T>(Ps + j, pw, j, m, tid, S.best, S.idx);
                bool zero;
                const double2 ri = piv_recip(Ps[p * pw + j], zero);
                __syncthreads();                                       // pivot and reduction slots read by all before they change
                if (tid == 0) {
                    S.piv[j] = p;
                    if (piv) piv[kb + j] = kb + p;
                    if (zero && S.bad == 0) S.bad = kb + j + 1;
                }
                if (p != j && tid < nb) { const double2 t1 = Ps[j * pw + tid]; Ps[j * pw + tid] = Ps[p * pw + tid]; Ps[p * pw + tid] = t1; }
                __syncthreads();
#pragma unroll 1
                for (int r = j + 1 + tid; r < m; r += T) {             // multiplier, then the panel's columns right of j
                    const double2 l = lu_mult(Ps[r * pw + j], ri);
                    Ps[r * pw + j] = l;
                    for (int b = j + 1; b < nb; b++) { double2 x = Ps[r * pw + b]; cmsub(x, l, Ps[j * pw + b]); Ps[r * pw + b] = x; }
                }
                __syncthreads();
            }
#pragma unroll 1
            for (int t = tid; t < m * nb; t += T) { const int r = t / nb, j = t - r * nb; A[(size_t)(kb + r) * lda + kb + j] = Ps[r * pw + j]; }
        } else {
            for (int j = 0; j < nb; j++) {
                const int col = kb + j;
                lu_pivot_step<T>(A, n, lda, col, tid, S);
                const int rows = n - col - 1, cols = c0 - col - 1;
#pragma unroll 1
                for (int t = tid; t < rows * cols; t += T) {
                    const int r = col + 1 + t / cols, cidx = col + 1 + t % cols;
                    const double2 l = A[r * lda + col], u = A[col * lda + cidx];
                    double2 v = A[r * lda + cidx];
                    cmsub(v, l, u);
                    A[r * lda + cidx] = v;
                }
                __syncthreads();
            }
        }
        // ---- 2. interchanges and the row block's unit-lower solve, one thread per column -------------------------------------
        const int ncol = nc - c0;
#pragma unroll 1
        for (int b = tid; b < ncol; b += T) {
            Ix ld;
            double2 *x = column(c0 + b, ld);
            x += (Ix)kb * ld;                                          // rows kb.. of the column
            if constexpr (STAGE_PANEL)
                for (int j = 0; j < nb; j++) {
                    const int p = S.piv[j];
                    if (p != j) { const double2 t1 = x[j * ld]; x[j * ld] = x[p * ld]; x[p * ld] = t1; }
                }
            double2 *u = x;
            Ix lu = ld;
            if constexpr (STAGE_ROWS) {
                for (int j = 0; j < nb; j++) Us[j * nc + b] = x[j * ld];
                u = Us + b; lu = nc;
            }
            for (int j = 0; j < nb; j++) {
                const double2 uj = u[j * lu];
                for (int r = j + 1; r < nb; r++) { double2 v = u[r * lu]; cmsub(v, lmul(kb, r, j), uj); u[r * lu] = v; }
            }
            if constexpr (STAGE_ROWS) for (int j = 0; j < nb; j++) x[j * ld] = Us[j * nc + b];
        }
        __syncthreads();
        // ---- 3. trailing update, 4 x 2 register tile, updates in elimination order -------------------------------------------
        const int m2 = n - c0, tr = (m2 + 3) / 4, tc = (ncol + 1) / 2;
#pragma unroll 1
        for (int t = tid; t < tr * tc; t += T) {
            const int r0 = 4 * (t / tc), b0 = 2 * (t - (t / tc) * tc);
            double2 *cp[2];
            Ix ld[2];
#pragma unroll
            for (int y = 0; y < 2; y++) cp[y] = column(min(c0 + b0 + y, nc - 1), ld[y]);
            double2 acc[4][2];
#pragma unroll
            for (int x = 0; x < 4; x++)
#pragma unroll
                for (int y = 0; y < 2; y++)
                    acc[x][y] = !STAGE_PANEL ? cp[y][min(c0 + r0 + x, n - 1) * ld[y]]              // in shared memory: clamped reads
                              : (r0 + x < m2 && b0 + y < ncol) ? cp[y][(c0 + r0 + x) * ld[y]] : make_double2(0.0, 0.0);
            for (int j = 0; j < nb; j++) {
                double2 l[4], u[2];
#pragma unroll
                for (int x = 0; x < 4; x++) l[x] = lmul(kb, min(nb + r0 + x, m - 1), j);
#pragma unroll
                for (int y = 0; y < 2; y++) u[y] = STAGE_ROWS ? Us[j * nc + min(b0 + y, ncol - 1)] : cp[y][(kb + j) * ld[y]];
#pragma unroll
                for (int x = 0; x < 4; x++)
#pragma unroll
                    for (int y = 0; y < 2; y++) cmsub(acc[x][y], l[x], u[y]);
            }
#pragma unroll
            for (int x = 0; x < 4; x++)
#pragma unroll
                for (int y = 0; y < 2; y++)
                    if (r0 + x < m2 && b0 + y < ncol) cp[y][(c0 + r0 + x) * ld[y]] = acc[x][y];
        }
        __syncthreads();
    }
    if constexpr (STAGE_PANEL) return S.bad; else return *S.bad;
}

// Back substitution of the upper triangle of A [n][lda] into the nrhs right-hand sides B [n][ldb], row by row from the bottom,
// the updates spread over the group of T threads.  Ix: int in shared memory, size_t in global memory.
template <int T, class Ix>
__device__ __forceinline__ void lu_back_subst(const double2 *A, Ix lda, double2 *B, Ix ldb, int n, int nrhs, int gtid)
{
    for (int r = n - 1; r >= 0; r--) {
        const double2 pv = A[r * lda + r];
#pragma unroll 1
        for (int rh = gtid; rh < nrhs; rh += T) B[r * ldb + rh] = piv_div(B[r * ldb + rh], pv);
        gsync<T>();
#pragma unroll 1
        for (int t = gtid; t < r * nrhs; t += T) {
            const int rr = t / nrhs, rh = t - rr * nrhs;
            const double2 a = A[rr * lda + r], x = B[r * ldb + rh];
            double2 b = B[rr * ldb + rh];
            cmsub(b, a, x);
            B[rr * ldb + rh] = b;
        }
        gsync<T>();
    }
}
