// raftk_misc.cuh -- k_system_solve (farm 6N system), k_response_stats, k_fp64_peak (included by raftk.cu only).
#pragma once

// ------------------------------------------------------------------------------------------------
// K3: dense complex solve per frequency (farm system response).  One CTA per frequency, matrix in
// shared memory, LU with partial pivoting (raftk_lu.cuh: column at a time up to n = 24, else in panels of 8 columns), nrhs
// right-hand sides.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_system_solve(int n, int nrhs, double2 *Z, double2 *F, int *info)
{
    extern __shared__ __align__(16) double smem_raw[];
    double2 *A = reinterpret_cast<double2 *>(smem_raw);              // [n][n+nrhs] augmented
    __shared__ int piv_s, bad_s;
    __shared__ double2 rinv_s;
    LuSlots S{&piv_s, &rinv_s, &bad_s};
    const int iw = blockIdx.x, tid = threadIdx.x, nc = n + nrhs;
    double2 *Zg = Z + (size_t)iw * n * n, *Fg = F + (size_t)iw * n * nrhs;
    for (int t = tid; t < n * n; t += blockDim.x) A[(t / n) * nc + (t % n)] = Zg[t];
    for (int t = tid; t < n * nrhs; t += blockDim.x) A[(t / nrhs) * nc + n + (t % nrhs)] = Fg[t];
    __syncthreads();
    const int bad = n > 24 ? lu_blocked<128, false, false>(A, nc, A + n, nc, n, nrhs, 8, S) : lu_unblocked<128>(A, n, nc, tid, S);
    lu_back_subst<128>(A, nc, A + n, nc, n, nrhs, tid);
    for (int t = tid; t < n * nrhs; t += blockDim.x) Fg[t] = A[(t / nrhs) * nc + n + (t % nrhs)];
    if (tid == 0 && info) info[iw] = bad;
}

// ------------------------------------------------------------------------------------------------
// K3b: farm system response straight from the per-FOWT solves (raft_model.py:1164-1236):
// Z_sys = blockdiag_i(-w^2 (M0_i + A_w,i) + i w (B0_i + B_drag_i + B_w,i) + C0_i) + (-w^2 M_arr + i w B_arr + C_arr),
// F = F_BEM_i + F_iner_i + F_drag_i (+ F_2nd_i) stacked, Xi_sys = Z_sys^-1 F.  Everything is read from device-resident
// outputs of the drag-linearisation solve: no host assembly of Z, no per-case transfer of nw n^2 complex numbers.
// WARP = true : small systems (6N <= 24), one WARP per (frequency, case), up to FARM_WPC systems per CTA, no CTA-wide barriers;
// WARP = false: one CTA per (frequency, case) of 256 threads, blocked LU in panels of 8 columns.
// A call solves nF farms of N FOWTs each (one farm: nF = 1): design f * N + i is FOWT i of farm f.  The shared-memory and
// register kernels take the farm from blockIdx.z, so the systems a CTA packs along the frequency axis belong to one farm and
// a ragged last group ends at nw; k_farm_response_global walks (farm, case, frequency) systems.
// ------------------------------------------------------------------------------------------------
struct FarmParams {
    int N, nC, nw, nF;
    size_t arr_stride;                          // doubles between two farms' array matrices: (6N)^2, or 0 when every farm shares one set
    const double *B_drag;                       // [nF * N][nC][36]
    const double2 *F_drag, *F_iner, *F_BEM;     // [nF * N][nC][6][nw]; F_BEM may be NULL
    const double *M_arr, *B_arr, *C_arr;        // [nF or 1][6N][6N] or NULL
    double2 *Xi;                                // [nF][nC][6N][nw]
    int *info;                                  // [nF][nC][nw] or NULL
};
#define FARM_WPC 4

// A ragged batch (raftk_farm_ragged): one launch per kernel class over that class's farms, blockIdx.z (or the system walk)
// indexing the class's run of descriptors.  A descriptor holds what a uniform batch derives from the farm index: the first
// design, N, the offsets of the farm's Xi_sys / info rows and array matrices, and (k_farm_response_global) the panel width
// glu_plan gives its 6N, so that every farm is factored exactly as a uniform batch of its N would factor it.
struct FarmDesc {
    int d0, N, pw, _pad;
    size_t xo, io, ao;                          // complex elements of Xi, words of info, doubles of M_arr / B_arr / C_arr
};
struct FarmRagParams : FarmParams {
    const FarmDesc *fd;                         // [nF]: this class's farms
    size_t slab;                                // double2 elements between two CTAs' slabs (k_farm_response_global)
};
template <bool RAG> using FarmArg = typename std::conditional<RAG, FarmRagParams, FarmParams>::type;

// Farm f of a launch: N, first design, array-matrix offset, the base of its Xi / info and its row there for case c.  A
// uniform batch derives them from f (the expressions its kernels always used), a ragged one reads f's descriptor.
template <bool RAG, class Prm> __device__ __forceinline__ int farm_n(const Prm &P, int f)
{
    if constexpr (RAG) return P.fd[f].N; else return P.N;
}
template <bool RAG, class Prm> __device__ __forceinline__ size_t farm_d0(const Prm &P, int f)
{
    if constexpr (RAG) return (size_t)P.fd[f].d0; else return (size_t)f * P.N;
}
template <bool RAG, class Prm> __device__ __forceinline__ size_t farm_ao(const Prm &P, int f)
{
    if constexpr (RAG) return P.fd[f].ao; else return (size_t)f * P.arr_stride;
}
template <bool RAG, class Prm> __device__ __forceinline__ double2 *farm_xi(const Prm &P, int f)
{
    if constexpr (RAG) return P.Xi + P.fd[f].xo; else return P.Xi;
}
template <bool RAG, class Prm> __device__ __forceinline__ int *farm_info(const Prm &P, int f)
{
    if constexpr (RAG) return P.info ? P.info + P.fd[f].io : nullptr; else return P.info;
}
template <bool RAG, class Prm> __device__ __forceinline__ size_t farm_row(const Prm &P, int f, int c)
{
    if constexpr (RAG) return (size_t)c; else return (size_t)f * P.nC + c;
}
// k_farm_response_global: double2 elements between two CTAs' slabs, and farm f's panel width (a uniform launch's `pw`)
template <bool RAG, class Prm> __device__ __forceinline__ size_t farm_slab(const Prm &P)
{
    if constexpr (RAG) return P.slab; else return (size_t)6 * P.N * (6 * P.N + 1);
}
template <bool RAG, class Prm> __device__ __forceinline__ int farm_pw(const Prm &P, int f, int pw)
{
    if constexpr (RAG) return P.fd[f].pw; else return pw;
}

// The frequency-dependent terms of design i's block entry e at bin iw for a case c with an operating point: the design's
// A_w / B_w plus the operating point's (tab_term), added to M and B.  (A secondary train's operating point is its primary's:
// raftk_cases.op.)
__device__ __forceinline__ void farm_op_terms(const DesignsDev &D, const CasesDev &Cs, size_t i, int c, int e, int iw, double &M, double &B)
{
    const size_t nw = D.nw, o = (size_t)e * nw + iw;
    const double *Aw = D.A_w ? D.A_w + i * 36 * nw : nullptr, *Bw = D.B_w ? D.B_w + i * 36 * nw : nullptr;
    M += tab_term(Aw, op_table(Cs, Cs.op_A_w, i, c, (int)nw), o);
    B += tab_term(Bw, op_table(Cs, Cs.op_B_w, i, c, (int)nw), o);
}

// Assembly of one (farm, case c, frequency iw) system, shared by k_farm_response and k_farm_response_global: Z_sys into
// A [n][nc] (nc = n + 1) and the right-hand side into its column n, spread over the gsize threads of a group.
// OP: the case table carries operating points (cases.op) -- the farm kernels take it in instantiations of their own, so that
// the calls without them compile as before.
template <bool OP, bool RAG = false, class Prm = FarmParams>
__device__ __forceinline__ void farm_assemble(const DesignsDev &D, const CasesDev &Cs, const Prm &P, int farm, int c, int iw, double2 *A,
                                              int gtid, int gsize)
{
    const int n = 6 * farm_n<RAG>(P, farm), nc = n + 1, nw = P.nw;
    const double w = D.w[iw], w2 = w * w;
    const int cp = Cs.primary ? Cs.primary[c] : c;                   // secondary wave trains use their primary's damping
    const size_t d0 = farm_d0<RAG>(P, farm), ao = farm_ao<RAG>(P, farm);
    for (int t = gtid; t < n * n; t += gsize) {
        const int a = t / n, b = t % n, j = b / 6;
        const size_t i = d0 + a / 6;                                 // design of block row a
        double zr = 0.0, zi = 0.0;
        if (a / 6 == j) {
            const int e = 6 * (a % 6) + (b - 6 * j);
            double M = D.M0[(size_t)i * 36 + e], B = D.B0[(size_t)i * 36 + e] + P.B_drag[((size_t)i * P.nC + cp) * 36 + e];
            if (OP) farm_op_terms(D, Cs, i, c, e, iw, M, B);
            else if (D.A_w) { M += D.A_w[((size_t)i * 36 + e) * nw + iw]; B += D.B_w[((size_t)i * 36 + e) * nw + iw]; }
            zr = fma(-w2, M, D.C0[(size_t)i * 36 + e]);
            zi = w * B;
        }
        if (P.C_arr) zr += P.C_arr[ao + t];
        if (P.M_arr) zr -= w2 * P.M_arr[ao + t];
        if (P.B_arr) zi += w * P.B_arr[ao + t];
        A[a * nc + b] = make_double2(zr, zi);
    }
    for (int a = gtid; a < n; a += gsize) {
        const int e = a % 6;
        const size_t o = (((d0 + a / 6) * P.nC + c) * 6 + e) * nw + iw;
        double2 f = P.F_drag[o];
        const double2 h = P.F_iner[o];
        f.x += h.x; f.y += h.y;
        if (P.F_BEM) { const double2 q = P.F_BEM[o]; f.x += q.x; f.y += q.y; }
        if (Cs.F_2nd) f.x += Cs.F_2nd[o];
        A[a * nc + n] = f;
    }
}

// RAG: one class of a ragged batch, blockIdx.z indexing its descriptors; shared memory sized for the class's largest N
template <bool WARP, bool OP = false, bool RAG = false>
__global__ void __launch_bounds__(WARP ? 32 * FARM_WPC : 256) k_farm_response(DesignsDev D, CasesDev Cs, FarmArg<RAG> P)
{
    extern __shared__ __align__(16) double smem_raw[];
    __shared__ int piv_s[FARM_WPC], bad_s[FARM_WPC];
    __shared__ double2 rinv_s[FARM_WPC];
    const int n = 6 * farm_n<RAG>(P, blockIdx.z), nc = n + 1, nw = P.nw;
    const int g = WARP ? (int)(threadIdx.x >> 5) : 0, gtid = WARP ? (int)(threadIdx.x & 31) : (int)threadIdx.x;
    const int gsize = WARP ? 32 : (int)blockDim.x;
    const int iw = WARP ? (int)(blockIdx.x * (blockDim.x >> 5)) + g : (int)blockIdx.x, c = blockIdx.y, f = blockIdx.z;
    if (iw >= nw) return;                                            // (warp-uniform; no CTA-wide barrier follows in the WARP variant)
    double2 *A = reinterpret_cast<double2 *>(smem_raw) + (size_t)g * n * nc;
    const size_t u = farm_row<RAG>(P, f, c);                         // row of Xi and info
    LuSlots S{&piv_s[g], &rinv_s[g], &bad_s[g]};
    farm_assemble<OP, RAG>(D, Cs, P, f, c, iw, A, gtid, gsize);
    constexpr int T = WARP ? 32 : 256;
    gsync<T>();
    int bad;
    if constexpr (WARP) bad = lu_unblocked<T>(A, n, nc, gtid, S);
    else bad = lu_blocked<T, false, false>(A, nc, A + n, nc, n, 1, 8, S);
    lu_back_subst<T>(A, nc, A + n, nc, n, 1, gtid);
    double2 *Xi = farm_xi<RAG>(P, f);
    int *info = farm_info<RAG>(P, f);
    for (int a = gtid; a < n; a += gsize) Xi[(u * n + a) * nw + iw] = A[a * nc + n];
    if (gtid == 0 && info) info[u * nw + iw] = bad;
}

// ------------------------------------------------------------------------------------------------
// K3d: dense solves whose augmented system does not fit in one CTA's shared memory (farms of 20 and more FOWTs, any n for
// raftk_system_solve).  The system stays in global memory (L2-resident while the CTA works on it) and lu_blocked factors it
// with its panel staged in shared memory (raftk_lu.cuh), pw columns wide (glu_plan); back substitution of the nrhs
// right-hand sides follows.  Every thread of the CTA takes part; each kernel loops over its systems with persistent CTAs, so
// a result depends on nothing but the system itself.
// ------------------------------------------------------------------------------------------------
#define GLU_T 256
#define GLU_PWMAX 16

// farm system response of k_farm_response (same assembly) for any N: persistent CTAs, CTA b owns slab b of the workspace
// ([6N][6N+1] double2) and solves the (farm, case, frequency) systems b, b + gridDim.x, ... of the nF * nC * nw in all.
// RAG: the farms of one class of a ragged batch, each with its own N and panel width (its descriptor); slabs P.slab elements
// apart (the class's largest N) and the panel sized for the largest n * pw by the launch
template <bool OP = false, bool RAG = false>
__global__ void __launch_bounds__(GLU_T, 2) k_farm_response_global(DesignsDev D, CasesDev Cs, FarmArg<RAG> P, double2 *ws, int pw)
{
    extern __shared__ __align__(16) double smem_raw[];
    __shared__ LuStaged<GLU_T, GLU_PWMAX> S;
    double2 *Ps = reinterpret_cast<double2 *>(smem_raw);
    const int nw = P.nw;
    double2 *A = ws + (size_t)blockIdx.x * farm_slab<RAG>(P);
    const long long nsys = (long long)P.nF * P.nC * nw;
    for (long long s = blockIdx.x; s < nsys; s += gridDim.x) {
        const long long fc = s / nw;                                   // f * nC + c
        const int iw = (int)(s - fc * nw), f = (int)(fc / P.nC), c = (int)(fc - (long long)f * P.nC);
        const int n = 6 * farm_n<RAG>(P, f), nc = n + 1;
        const size_t u = farm_row<RAG>(P, f, c);                       // row of Xi and info
        double2 *Xi = farm_xi<RAG>(P, f);
        int *info = farm_info<RAG>(P, f);
        farm_assemble<OP, RAG>(D, Cs, P, f, c, iw, A, threadIdx.x, GLU_T);
        __syncthreads();
        const int bad = lu_blocked<GLU_T, true, false>(A, nc, A + n, nc, n, 1, farm_pw<RAG>(P, f, pw), S, Ps);
        lu_back_subst<GLU_T>(A, (size_t)nc, A + n, (size_t)nc, n, 1, threadIdx.x);
        for (int a = threadIdx.x; a < n; a += GLU_T) Xi[(u * n + a) * nw + iw] = A[(size_t)a * nc + n];
        if (threadIdx.x == 0 && info) info[u * nw + iw] = bad;
        __syncthreads();                                               // the slab is rewritten by the next system
    }
}

// raftk_system_solve for any n: Z [nw][n][n] factored in place, F [nw][n][nrhs] overwritten with the solutions
__global__ void __launch_bounds__(GLU_T, 2) k_system_solve_global(int n, int nw, int nrhs, int pw, double2 *Z, double2 *F, int *info)
{
    extern __shared__ __align__(16) double smem_raw[];
    __shared__ LuStaged<GLU_T, GLU_PWMAX> S;
    double2 *Ps = reinterpret_cast<double2 *>(smem_raw);
    for (int iw = blockIdx.x; iw < nw; iw += gridDim.x) {
        double2 *A = Z + (size_t)iw * n * n, *B = F + (size_t)iw * n * nrhs;
        const int bad = lu_blocked<GLU_T, true, false>(A, n, B, nrhs, n, nrhs, pw, S, Ps);
        lu_back_subst<GLU_T>(A, (size_t)n, B, (size_t)nrhs, n, nrhs, threadIdx.x);
        if (threadIdx.x == 0 && info) info[iw] = bad;
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------
// K3c: farm system response for the two-FOWT array (6N = 12; the template also builds for 18 / 24, where it needs 188 / 238
// registers and is not launched): the augmented system lives in REGISTERS, one lane per row.
// A group of LPS lanes (16 for 6N = 12: two systems per warp; 32 above) owns one (frequency, case) system; lane r holds row r
// (N6 matrix entries + the right-hand side).  Elimination step k (fully unrolled, so every register index is static):
// pivot = first maximum of |re| + |im| over rows >= k (butterfly over the group, LAPACK izamax tie-break), ONE shuffle per
// entry moves the pivot row to everybody and old row k to the pivot's lane, every row below k eliminates itself.  No shared
// memory, no barriers; back substitution broadcasts one unknown per step.  Same assembly arithmetic as k_farm_response.
// ------------------------------------------------------------------------------------------------
template <int N6, bool OP = false, bool RAG = false>
__global__ void __launch_bounds__(128) k_farm_rows(DesignsDev D, CasesDev Cs, FarmArg<RAG> P)
{
    constexpr int LPS = N6 <= 16 ? 16 : 32, SPW = 32 / LPS, NC = N6 + 1;
    const int nw = P.nw, lane = threadIdx.x & 31, r = lane & (LPS - 1);
    const int sys = ((int)blockIdx.x * ((int)blockDim.x >> 5) + ((int)threadIdx.x >> 5)) * SPW + lane / LPS;
    const int c = blockIdx.y, f = blockIdx.z;
    const bool live = sys < nw;                        // a group beyond the grid keeps shuffling with its neighbours but never stores
    const int iw = live ? sys : nw - 1;
    const bool row_ok = r < N6;
    const int a = row_ok ? r : 0;
    const double w = D.w[iw], w2 = w * w;
    const int cp = Cs.primary ? Cs.primary[c] : c;
    const int ib = a / 6, ea = a - 6 * ib;             // block row of the system; its design is FOWT ib of farm f
    // (a ragged class of this kernel holds farms with 6N = N6 only)
    const size_t i = farm_d0<RAG>(P, f) + ib, ao = farm_ao<RAG>(P, f), u = farm_row<RAG>(P, f, c);
    double2 row[NC];
#pragma unroll
    for (int b = 0; b < N6; b++) {
        double zr = 0.0, zi = 0.0;
        if (b / 6 == ib) {
            const int e = 6 * ea + (b - 6 * (b / 6));
            double M = D.M0[(size_t)i * 36 + e], B = D.B0[(size_t)i * 36 + e] + P.B_drag[((size_t)i * P.nC + cp) * 36 + e];
            if (OP) farm_op_terms(D, Cs, i, c, e, iw, M, B);
            else if (D.A_w) { M += D.A_w[((size_t)i * 36 + e) * nw + iw]; B += D.B_w[((size_t)i * 36 + e) * nw + iw]; }
            zr = fma(-w2, M, D.C0[(size_t)i * 36 + e]);
            zi = w * B;
        }
        const size_t t = ao + a * N6 + b;
        if (P.C_arr) zr += P.C_arr[t];
        if (P.M_arr) zr -= w2 * P.M_arr[t];
        if (P.B_arr) zi += w * P.B_arr[t];
        row[b] = make_double2(zr, zi);
    }
    {
        const size_t o = (((size_t)i * P.nC + c) * 6 + ea) * nw + iw;
        double2 f = P.F_drag[o];
        const double2 h = P.F_iner[o];
        f.x += h.x; f.y += h.y;
        if (P.F_BEM) { const double2 q = P.F_BEM[o]; f.x += q.x; f.y += q.y; }
        if (Cs.F_2nd) f.x += Cs.F_2nd[o];
        row[N6] = f;
    }
    int bad = 0;
    double2 myinv = make_double2(0.0, 0.0);
    static_for<0, N6>([&](auto K) {
        constexpr int k = decltype(K)::value;
        double best = (row_ok && r >= k) ? fabs(row[k].x) + fabs(row[k].y) : -1.0;
        int p = r;
#pragma unroll
        for (int o = LPS / 2; o >= 1; o >>= 1) {
            const double ob = __shfl_xor_sync(0xffffffffu, best, o, LPS);
            const int op = __shfl_xor_sync(0xffffffffu, p, o, LPS);
            if (ob > best || (ob == best && op < p)) { best = ob; p = op; }
        }
        // one shuffle per entry: the pivot's lane fetches old row k, every other lane the pivot row
        const int src = (r == p) ? k : p;
        double2 piv[NC];
        static_for<k, NC>([&](auto J) {
            constexpr int j = decltype(J)::value;
            double2 t;
            t.x = __shfl_sync(0xffffffffu, row[j].x, src, LPS);
            t.y = __shfl_sync(0xffffffffu, row[j].y, src, LPS);
            if (r == p) { piv[j] = row[j]; row[j] = t; }
            else { piv[j] = t; if (r == k) row[j] = t; }
        });
        // 1 / p at the pivot's scale (piv_recip), one division per step: q = p sc, 1 / |q|^2 times sc, times q
        const double sc = piv_scale(piv[k]);
        const double2 q = make_double2(piv[k].x * sc, piv[k].y * sc);
        const double den = q.x * q.x + q.y * q.y;
        double2 ri = make_double2(0.0, 0.0);
        if (den > 0.0) { const double inv = 1.0 / den * sc; ri = make_double2(q.x * inv, -q.y * inv); }
        else if (bad == 0) bad = k + 1;
        if (r == k) myinv = ri;                          // 1 / U_kk stays with row k for the back substitution
        if (row_ok && r > k) {
            const double2 v = row[k];
            const double2 l = make_double2(v.x * ri.x - v.y * ri.y, v.x * ri.y + v.y * ri.x);
            static_for<k + 1, NC>([&](auto J) {
                constexpr int j = decltype(J)::value;
                row[j].x -= l.x * piv[j].x - l.y * piv[j].y;
                row[j].y -= l.x * piv[j].y + l.y * piv[j].x;
            });
        }
    });
    // back substitution: lane k multiplies by the reciprocal of its diagonal kept from the elimination, everybody above subtracts
    double2 x = make_double2(0.0, 0.0);
    static_for<0, N6>([&](auto KK) {
        constexpr int k = N6 - 1 - decltype(KK)::value;
        const double2 pv = row[k], s = row[N6];
        const double2 xk_own = make_double2(s.x * myinv.x - s.y * myinv.y, s.x * myinv.y + s.y * myinv.x);      // only lane k's value is used
        double2 xk;
        xk.x = __shfl_sync(0xffffffffu, xk_own.x, k, LPS);
        xk.y = __shfl_sync(0xffffffffu, xk_own.y, k, LPS);
        if (r == k) x = xk;
        if (r < k) {
            row[N6].x -= pv.x * xk.x - pv.y * xk.y;
            row[N6].y -= pv.x * xk.y + pv.y * xk.x;
        }
    });
    double2 *Xi = farm_xi<RAG>(P, f);
    int *info = farm_info<RAG>(P, f);
    if (live && row_ok) Xi[(u * N6 + r) * nw + iw] = x;
    if (live && r == 0 && info) info[u * nw + iw] = bad;
}

// K3e: a rank's farms of a sharded batch (raftk_farm_batch_response_gather_dev, raftk_farm_ragged_response_gather_dev) to the
// other ranks' copies after their solve.  The rank's farms are contiguous, so their
// Xi_sys, info and per-FOWT status are three contiguous runs, stored at the same offsets of every copy: blockIdx.y = p; Xi_sys
// and info where X[p] / I[p] are set, the status rows to every S[p]
struct FarmFlatPeer {
    int n_peers;
    size_t nx, ni, ns;                          // complex elements of Xi_sys, info words, status words of this rank's farms
    const double2 *Xi;
    const int *info, *status;
    double2 *X[RAFTK_MAX_PEERS];
    int *I[RAFTK_MAX_PEERS];
    int *S[RAFTK_MAX_PEERS];
};
__global__ void __launch_bounds__(256) k_farm_publish(FarmFlatPeer P)
{
    const int p = blockIdx.y;
    const size_t stride = (size_t)gridDim.x * 256, t0 = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (double2 *x = P.X[p]) for (size_t t = t0; t < P.nx; t += stride) x[t] = P.Xi[t];
    if (int *d = P.I[p]) for (size_t t = t0; t < P.ni; t += stride) d[t] = P.info[t];
    if (int *d = P.S[p]) for (size_t t = t0; t < P.ns; t += stride) d[t] = P.status[t];
}

// std = sqrt(1/2 sum_w |Y|^2) of one 128-thread CTA from each thread's partial sum s: warp shuffles, then the four warps
// in a fixed order (the same reduction tree for every statistics kernel)
__device__ __forceinline__ void block_rms_tail(double s, double (&part)[4], int tid, double *out)
{
    for (int o = 16; o >= 1; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((tid & 31) == 0) part[tid >> 5] = s;
    __syncthreads();
    if (tid == 0) *out = sqrt(0.5 * (((part[0] + part[1]) + part[2]) + part[3]));
}

// ------------------------------------------------------------------------------------------------
// K4: response statistics (std, PSD) -- one CTA per (unit, dof), fixed-order block reduction over frequency
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_response_stats(int nw, double dw, int rot_deg, const double2 *Xi, double *sd, double *psd)
{
    __shared__ double part[4];
    const int row = blockIdx.x, dof = row % 6, tid = threadIdx.x;
    const double scale = (rot_deg && dof >= 3) ? (180.0 / CUDART_PI) : 1.0;      // np.rad2deg
    const double2 *x = Xi + (size_t)row * nw;
    double s = 0.0;
    for (int i = tid; i < nw; i += 128) {
        const double re = x[i].x * scale, im = x[i].y * scale;
        const double a2 = re * re + im * im;
        s += a2;
        if (psd) psd[(size_t)row * nw + i] = 0.5 * a2 / dw;
    }
    block_rms_tail(s, part, tid, sd + row);
}

// ------------------------------------------------------------------------------------------------
// K5: output-channel statistics -- every channel of saveTurbineOutputs beyond the platform DOFs (nacelle accelerations,
// tower-base moment, raft_fowt.py:2401-2444, 2504-2538) is a linear functional of the response:
// Y(w) = sum_dof coef[design][ch][dof][w] * Xi[design][case][dof][w].  One CTA per (design, case, channel).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_channel_stats(int nC, int nch, int nw, double dw, const double2 *coef, const double2 *Xi,
                                                       double *sd, double *psd, double2 *amp)
{
    __shared__ double part[4];
    const int row = blockIdx.x, ch = row % nch, unit = row / nch, d = unit / nC, tid = threadIdx.x;
    const double2 *cf = coef + ((size_t)d * nch + ch) * 6 * nw;
    const double2 *x = Xi + (size_t)unit * 6 * nw;
    double s = 0.0;
    for (int i = tid; i < nw; i += 128) {
        double yr = 0.0, yi = 0.0;
#pragma unroll
        for (int a = 0; a < 6; a++) {
            const double2 c = cf[(size_t)a * nw + i], v = x[(size_t)a * nw + i];
            yr += c.x * v.x - c.y * v.y; yi += c.x * v.y + c.y * v.x;
        }
        const double a2 = yr * yr + yi * yi;
        s += a2;
        if (psd) psd[(size_t)row * nw + i] = 0.5 * a2 / dw;
        if (amp) amp[(size_t)row * nw + i] = make_double2(yr, yi);
    }
    block_rms_tail(s, part, tid, sd + row);
}

// ------------------------------------------------------------------------------------------------
// K5g: output channels of a FOWT with generalised DOFs (raftk_general_channel_stats_*): real functionals of the reduced
// response, Y(w) = w^wpow[ch] sum_b R[ch][b] Xi[unit][b][w] (PRP motions, nacelle accelerations, tower-base internal
// loads; raft_fowt.py:2299-2604).  One CTA per (unit, channel).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_general_channel_stats(int n, int nch, int nw, double dw, const double *w, const double *R,
                                                               const int *wpow, const double2 *Xi, double *sd, double *psd, double2 *amp)
{
    __shared__ double part[4];
    const int row = blockIdx.x, ch = row % nch, unit = row / nch, tid = threadIdx.x;
    const double *r = R + (size_t)ch * n;
    const double2 *x = Xi + (size_t)unit * n * nw;
    const int p = wpow[ch];
    double s = 0.0;
    for (int i = tid; i < nw; i += 128) {
        double yr = 0.0, yi = 0.0;
        for (int b = 0; b < n; b++) {
            const double c = r[b];
            const double2 v = x[(size_t)b * nw + i];
            yr = fma(c, v.x, yr); yi = fma(c, v.y, yi);
        }
        if (p == 2) { const double w2 = w[i] * w[i]; yr *= w2; yi *= w2; }
        else if (p == 1) { const double w1 = w[i]; yr *= w1; yi *= w1; }
        const double a2 = yr * yr + yi * yi;
        s += a2;
        if (psd) psd[(size_t)row * nw + i] = 0.5 * a2 / dw;
        if (amp) amp[(size_t)row * nw + i] = make_double2(yr, yi);
    }
    block_rms_tail(s, part, tid, sd + row);
}

// ------------------------------------------------------------------------------------------------
// K5f: output channels of farm batches (raftk_farm_channel_stats_*): mooring tensions and any other real functional of the
// coupled response, Y[f,r,ch,w] = w^wpow[ch] sum_b R_f[ch][b] Xi_sys[f][r][b][w] (raft_model.py:371-433 applies J_arr to
// Xi_sys, raft_fowt.py:2355-2399 J_moor to a FOWT's PRP motions).  k_general_channel_stats re-reads a unit's whole Xi for
// every channel; here one CTA per (farm, row, bin tile) stages the tile's n x tile bins of Xi_sys in shared memory once (or
// reads them from L2 when not even one bin fits) and computes every channel from it.  Each Y is the fma chain over
// b = 0..n-1 of k_general_channel_stats and |Y|^2 the same expression, so with k_farm_channel_reduce (that kernel's
// thread-strided sum and block_rms_tail) every std, PSD and amplitude is bit-identical to k_general_channel_stats' on the
// same R and Xi, whatever the tile width and the batch.
// ------------------------------------------------------------------------------------------------
// Xi tile staging shared by the tiled reductions (k_farm_channels, k_fatigue_moments, k_stress_moments): with SMEM the CTA's
// T threads copy the tile's P.n x tw bins, x the tile's bin 0 of column 0 (stride P.nw between columns), to xs [P.n][tw]
template <bool SMEM, int T, class Prm>
__device__ __forceinline__ void stage_xi_tile(const Prm &P, double2 *xs, const double2 *x, int tw, int tid)
{
    if (SMEM) {
        for (int k = tid; k < P.n * tw; k += T) {
            const int b = k / tw, i = k - b * tw;
            xs[k] = x[(size_t)b * P.nw + i];
        }
        __syncthreads();
    }
}

#define FARM_CH_T 256
#define FARM_CH_B 4             // channels per thread
struct FarmChParams {
    int n, nch, nw, n_rows, tile, n_tiles;
    size_t r_stride;            // doubles between two farms' R; 0: one R for every farm
    const double *w, *R;
    const double2 *Xi;          // [F, n_rows, n, nw]
    double *a2;                 // |Y|^2 [F, n_rows, nch, nw]: the psd output or the workspace
    double2 *amp;               // [F, n_rows, nch, nw] or NULL
    unsigned wbits[RAFTK_FARM_CH_MAX / 16];
};

// A ragged batch's farm (raftk_farm_ragged_channel_stats_*): its n = 6N_f, channel count and first channel, and where its
// Xi_sys block (complex elements) and R_f (doubles) start.  Its output rows start at n_rows * ch0.
struct FarmChDesc {
    int n, nch, ch0, _pad;
    size_t xo, ro;
};
struct FarmChRagParams : FarmChParams {
    const FarmChDesc *fd;                               // [F]
};
template <bool RAG> using FarmChArg = typename std::conditional<RAG, FarmChRagParams, FarmChParams>::type;
// Farm f's n, channel count, Xi tile base, R_f and first output row for row fr = f * n_rows + r; a uniform batch derives them
// from P (the expressions its kernel always used), a ragged one from f's descriptor
template <bool RAG, class Prm> __device__ __forceinline__ int farmch_n(const Prm &P, int f)
{
    if constexpr (RAG) return P.fd[f].n; else return P.n;
}
template <bool RAG, class Prm> __device__ __forceinline__ int farmch_nch(const Prm &P, int f)
{
    if constexpr (RAG) return P.fd[f].nch; else return P.nch;
}
template <bool RAG, class Prm> __device__ __forceinline__ const double2 *farmch_xi(const Prm &P, size_t fr, int f, int i0)
{
    if constexpr (RAG) return P.Xi + P.fd[f].xo + (fr - (size_t)f * P.n_rows) * P.fd[f].n * P.nw + i0;
    else return P.Xi + fr * (size_t)P.n * P.nw + i0;
}
template <bool RAG, class Prm> __device__ __forceinline__ const double *farmch_r(const Prm &P, int f)
{
    if constexpr (RAG) return P.R + P.fd[f].ro; else return P.R + (size_t)f * P.r_stride;
}
template <bool RAG, class Prm> __device__ __forceinline__ size_t farmch_row0(const Prm &P, size_t fr, int f)
{
    if constexpr (RAG) return (size_t)P.n_rows * P.fd[f].ch0 + (fr - (size_t)f * P.n_rows) * P.fd[f].nch;
    else return fr * P.nch;
}
template <bool RAG, class Prm> __device__ __forceinline__ int farmch_ch0(const Prm &P, int f)
{
    if constexpr (RAG) return P.fd[f].ch0; else return 0;
}
struct XiTileShape { int n, nw; };

template <bool SMEM>
__global__ void __launch_bounds__(FARM_CH_T) k_farm_channels(const __grid_constant__ FarmChParams P)
{
    extern __shared__ double2 xs[];                     // [n][tw] when SMEM
    const int tid = threadIdx.x;
    const int t = (int)(blockIdx.x % (unsigned)P.n_tiles);
    const size_t fr = blockIdx.x / (unsigned)P.n_tiles;    // farm * n_rows + row
    const int f = (int)(fr / (size_t)P.n_rows);
    const int i0 = t * P.tile, tw = min(P.tile, P.nw - i0);
    const double2 *x = P.Xi + fr * (size_t)P.n * P.nw + i0;
    stage_xi_tile<SMEM, FARM_CH_T>(P, xs, x, tw, tid);
    // a thread computes FARM_CH_B channels of one bin: each Xi value read feeds FARM_CH_B independent chains (every chain
    // still runs over b = 0..n-1 in order); a warp's threads share their channels, so the R loads are broadcasts
    const double *Rf = P.R + (size_t)f * P.r_stride;
    const int nchb = (P.nch + FARM_CH_B - 1) / FARM_CH_B;
    for (int k = tid; k < nchb * tw; k += FARM_CH_T) {
        const int c0 = (k / tw) * FARM_CH_B, i = k - (k / tw) * tw;
        const double *r[FARM_CH_B];
        double yr[FARM_CH_B], yi[FARM_CH_B];
#pragma unroll
        for (int j = 0; j < FARM_CH_B; j++) { r[j] = Rf + (size_t)min(c0 + j, P.nch - 1) * P.n; yr[j] = 0.0; yi[j] = 0.0; }
        for (int b = 0; b < P.n; b++) {
            const double2 v = SMEM ? xs[b * tw + i] : x[(size_t)b * P.nw + i];
#pragma unroll
            for (int j = 0; j < FARM_CH_B; j++) {
                const double c = r[j][b];
                yr[j] = fma(c, v.x, yr[j]); yi[j] = fma(c, v.y, yi[j]);
            }
        }
        const int iw = i0 + i;
#pragma unroll
        for (int j = 0; j < FARM_CH_B; j++) {
            const int ch = c0 + j;
            if (ch >= P.nch) break;
            double re = yr[j], im = yi[j];
            const int p = (P.wbits[ch >> 4] >> ((ch & 15) * 2)) & 3;
            if (p == 2) { const double w2 = P.w[iw] * P.w[iw]; re *= w2; im *= w2; }
            else if (p == 1) { const double w1 = P.w[iw]; re *= w1; im *= w1; }
            const size_t o = (fr * P.nch + ch) * P.nw + iw;
            P.a2[o] = re * re + im * im;
            if (P.amp) P.amp[o] = make_double2(re, im);
        }
    }
}

// k_farm_channels for a ragged batch (raftk_farm_ragged_channel_stats_*): one tile width for every farm (the largest n's),
// each farm's n, channels and offsets from its descriptor, the same per-channel arithmetic.  Kept apart from k_farm_channels
// so that the uniform kernel compiles as before.
template <bool SMEM, bool RAG = true>
__global__ void __launch_bounds__(FARM_CH_T) k_farm_channels_ragged(const __grid_constant__ FarmChRagParams P)
{
    extern __shared__ double2 xs[];                     // [n][tw] when SMEM
    const int tid = threadIdx.x;
    const int t = (int)(blockIdx.x % (unsigned)P.n_tiles);
    const size_t fr = blockIdx.x / (unsigned)P.n_tiles;    // farm * n_rows + row
    const int f = (int)(fr / (size_t)P.n_rows);
    const int i0 = t * P.tile, tw = min(P.tile, P.nw - i0);
    const double2 *x = farmch_xi<RAG>(P, fr, f, i0);
    const int n = farmch_n<RAG>(P, f), nch = farmch_nch<RAG>(P, f);
    stage_xi_tile<SMEM, FARM_CH_T>(XiTileShape{n, P.nw}, xs, x, tw, tid);
    // a thread computes FARM_CH_B channels of one bin: each Xi value read feeds FARM_CH_B independent chains (every chain
    // still runs over b = 0..n-1 in order); a warp's threads share their channels, so the R loads are broadcasts
    const double *Rf = farmch_r<RAG>(P, f);
    const int nchb = (nch + FARM_CH_B - 1) / FARM_CH_B;
    for (int k = tid; k < nchb * tw; k += FARM_CH_T) {
        const int c0 = (k / tw) * FARM_CH_B, i = k - (k / tw) * tw;
        const double *r[FARM_CH_B];
        double yr[FARM_CH_B], yi[FARM_CH_B];
#pragma unroll
        for (int j = 0; j < FARM_CH_B; j++) { r[j] = Rf + (size_t)min(c0 + j, nch - 1) * n; yr[j] = 0.0; yi[j] = 0.0; }
        for (int b = 0; b < n; b++) {
            const double2 v = SMEM ? xs[b * tw + i] : x[(size_t)b * P.nw + i];
#pragma unroll
            for (int j = 0; j < FARM_CH_B; j++) {
                const double c = r[j][b];
                yr[j] = fma(c, v.x, yr[j]); yi[j] = fma(c, v.y, yi[j]);
            }
        }
        const int iw = i0 + i;
#pragma unroll
        for (int j = 0; j < FARM_CH_B; j++) {
            const int ch = c0 + j, cw = farmch_ch0<RAG>(P, f) + ch;
            if (ch >= nch) break;
            double re = yr[j], im = yi[j];
            const int p = (P.wbits[cw >> 4] >> ((cw & 15) * 2)) & 3;
            if (p == 2) { const double w2 = P.w[iw] * P.w[iw]; re *= w2; im *= w2; }
            else if (p == 1) { const double w1 = P.w[iw]; re *= w1; im *= w1; }
            const size_t o = (farmch_row0<RAG>(P, fr, f) + ch) * P.nw + iw;
            P.a2[o] = re * re + im * im;
            if (P.amp) P.amp[o] = make_double2(re, im);
        }
    }
}

// std = sqrt(1/2 sum_w |Y|^2) and PSD = 1/2 |Y|^2 / dw per (farm, row, channel): one 128-thread CTA per row, summing a2 in
// k_general_channel_stats' thread-strided order.  psd may be a2 itself (each thread rewrites the bins it read).
__global__ void __launch_bounds__(128) k_farm_channel_reduce(int nw, double dw, const double *a2, double *sd, double *psd)
{
    __shared__ double part[4];
    const size_t row = blockIdx.x;
    const int tid = threadIdx.x;
    double s = 0.0;
    for (int i = tid; i < nw; i += 128) {
        const double v = a2[row * nw + i];
        s += v;
        if (psd) psd[row * nw + i] = 0.5 * v / dw;
    }
    block_rms_tail(s, part, tid, sd + row);
}

// ------------------------------------------------------------------------------------------------
// FP64 FMA peak micro-kernel
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_fp64_peak(double *out, int iters)
{
    double a0 = threadIdx.x * 1e-3, a1 = a0 + 1, a2 = a0 + 2, a3 = a0 + 3, a4 = a0 + 4, a5 = a0 + 5, a6 = a0 + 6, a7 = a0 + 7;
    const double b = 1.0000001, c = 1e-9;
    for (int i = 0; i < iters; i++) {
        a0 = fma(a0, b, c); a1 = fma(a1, b, c); a2 = fma(a2, b, c); a3 = fma(a3, b, c);
        a4 = fma(a4, b, c); a5 = fma(a5, b, c); a6 = fma(a6, b, c); a7 = fma(a7, b, c);
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = a0 + a1 + a2 + a3 + a4 + a5 + a6 + a7;
}

// ------------------------------------------------------------------------------------------------
// K6: cross-GPU arrival barrier of the fused exchange (raftk_peer_barrier_dev).  Thread p tells rank p that this
// rank's stores of `epoch` are complete (they were issued by earlier kernels of this stream, so they are performed
// before this kernel starts; the release store orders the flag behind them at system scope), then waits for
// rank p's flag in the local copy.  Bounded spin: a dead peer sets *timeout_flag instead of hanging the GPU.
// ------------------------------------------------------------------------------------------------
struct PeerFlags { int n, rank; unsigned epoch; unsigned *flags[RAFTK_MAX_PEERS]; };

__global__ void k_peer_barrier(PeerFlags F, int *timeout_flag)
{
    const int p = threadIdx.x;
    if (p >= F.n) return;
    __threadfence_system();
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(F.flags[p] + F.rank), "r"(F.epoch) : "memory");
    const unsigned *mine = F.flags[F.rank] + p;
    const long long t0 = clock64();
    for (;;) {
        unsigned v;
        asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(mine) : "memory");
        if ((int)(v - F.epoch) >= 0) break;
        if (clock64() - t0 > 8000000000LL) { if (timeout_flag) *timeout_flag = 1; break; }     // ~4 s at 1.9 GHz
        __nanosleep(200);
    }
}
