// raftk_common.cuh -- device-side structures and routines shared by all kernels (included by raftk.cu only).
#pragma once

// ------------------------------------------------------------------------------------------------
// device helpers
// ------------------------------------------------------------------------------------------------
#define SOLVE_THREADS 128
#define CHUNK_NODES 10          // nodes per register-accumulator chunk in the RMS pass (3*10 <= 32)
#define MEM_STRIDE 24           // doubles per member in shared memory
// step classes of the fused solvers (DESIGN.md section 5): node spacings whose keys agree to STEP_RTOL (relative to the
// node's own key) share one set of factors; a key at or below STEP_ZERO in every component is no step (identity row).
// First-node depths agree to Z0_RTOL * max(1, |z0|).  The host-side hints (solver.py, batch_builder.py,
// raftk_builder.h) count with the same constants.
#define STEP_RTOL 5e-14
#define STEP_ZERO 1e-14
#define Z0_RTOL 1e-12

struct DesignsDev {
    int nD, nw, max_nodes, max_members, n_bem_head;
    double depth, rho, g, dw;
    const double *w, *k;
    const int *member_offset;
    const double *mem_frame, *mem_rA, *mem_arm;
    const int *mem_node_start, *mem_circ;
    const double *node_ls, *node_cd_q, *node_cd_p1, *node_cd_p2, *node_in_q, *node_in_p1, *node_in_p2, *node_pa;
    const double2 *node_in_p1_w, *node_in_p2_w;
    const double *M0, *B0, *C0, *A_w, *B_w;
    const double *bem_headings, *X_BEM, *bem_xyh;
    int max_rotors;                                  // submerged rotors (raftk_designs.rot_*), 0: none
    const int *rot_count;
    const double *rot_r3, *rot_G;
};

struct CasesDev {
    int nC;
    const double *Hs, *Tp, *gamma, *beta_deg, *zeta_in;
    const int *spec;
    const int *primary;     // [nC] or NULL: case whose drag linearisation this case reuses (secondary wave trains)
    const double *F_2nd;    // [nD][nC][6][nw] real second-order force amplitudes added to F_BEM + F_iner, or NULL
    const int *op;          // [nC] operating point of every case, or NULL (raftk_cases.op)
    int n_op, op_shared;
    const double *op_A_w, *op_B_w;   // [nD or 1][n_op][36][nw]
};

// The operating-point table `tab` (op_A_w or op_B_w) of unit (design d, case c), or NULL without operating points.
__device__ __forceinline__ const double *op_table(const CasesDev &Cs, const double *tab, size_t d, int c, int nw)
{
    return Cs.op ? tab + ((Cs.op_shared ? 0 : d * Cs.n_op) + (size_t)Cs.op[c]) * 36 * nw : nullptr;
}

// Frequency-dependent term at table offset e: the design's (dt) plus the operating point's (ot), summed before either meets
// M0 / B0, so that a call with operating points equals one with the point's tables summed into A_w / B_w, bit for bit.
// At least one of dt, ot is non-NULL.
__device__ __forceinline__ double tab_term(const double *dt, const double *ot, size_t e)
{
    return ot ? (dt ? dt[e] + ot[e] : ot[e]) : dt[e];
}

// The fused solvers' impedance at bin i for a unit with an operating point (Ao, Bo; DESIGN: the design's Aw, Bw too), the
// same arithmetic as their table branch with tab_term's sums: ar + i ai = C - w^2 (M + A) + i w (B + B_w).  Ms, Bs, Cm: the
// unit's 6x6 mass, damping (drag included) and stiffness.  Kept apart from the table branch so that the solves without
// operating points compile as before.
template <bool DESIGN>
__device__ __forceinline__ void op_impedance(double (&ar)[6][6], double (&ai)[6][6], const double *Ms, const double *Bs, const double *Cm,
                                             const double *Aw, const double *Bw, const double *Ao, const double *Bo, int i, int nw,
                                             double w, double w2)
{
#pragma unroll
    for (int a = 0; a < 6; a++)
#pragma unroll
        for (int b = 0; b < 6; b++) {
            const size_t e = (size_t)(6 * a + b) * nw + i;
            const double M = Ms[6 * a + b] + (DESIGN ? Aw[e] + Ao[e] : Ao[e]);
            const double B = Bs[6 * a + b] + (DESIGN ? Bw[e] + Bo[e] : Bo[e]);
            ar[a][b] = fma(-w2, M, Cm[6 * a + b]);
            ai[a][b] = w * B;
        }
}

// The fused solvers' impedance at bin i without operating points: with the design's frequency-dependent added mass and
// damping tables Aw, Bw (BEM, aero) when Aw is non-NULL, else from the constant matrices alone.
__device__ __forceinline__ void impedance(double (&ar)[6][6], double (&ai)[6][6], const double *Ms, const double *Bs, const double *Cm,
                                          const double *Aw, const double *Bw, int i, int nw, double w, double w2)
{
    if (Aw) {
#pragma unroll
        for (int a = 0; a < 6; a++)
#pragma unroll
            for (int b = 0; b < 6; b++) {
                const double M = Ms[6 * a + b] + Aw[(size_t)(6 * a + b) * nw + i];
                const double B = Bs[6 * a + b] + Bw[(size_t)(6 * a + b) * nw + i];
                ar[a][b] = fma(-w2, M, Cm[6 * a + b]);
                ai[a][b] = w * B;
            }
    } else {
#pragma unroll
        for (int a = 0; a < 6; a++)
#pragma unroll
            for (int b = 0; b < 6; b++) {
                ar[a][b] = fma(-w2, Ms[6 * a + b], Cm[6 * a + b]);
                ai[a][b] = w * Bs[6 * a + b];
            }
    }
}

struct Work {          // workspace views for one chunk of designs [d0, d0+nDc)
    int d0, nDc;
    double2 *depth_tab;   // [nDc][max_nodes][nw]           (C, S)
    double2 *phase_tab;   // [nDc][nC][max_nodes][nw]       zeta*w*E
    double2 *F0;          // [nDc][nC][6][nw]               F_BEM + F_iner
    double *zeta;         // [nC][nw]
};

// depth functions of helpers.py:207-222 (k == 0 / k h > 89.4 / general)
__device__ __forceinline__ void depth_funcs(double k, double h, double z, double &S_, double &C_, double &P_)
{
    if (k == 0.0) { S_ = 1.0; C_ = 99999.0; P_ = 99999.0; }
    else if (k * h > 89.4) {
        double e = exp(k * z);
        S_ = e; C_ = e; P_ = e + exp(-k * (z + 2.0 * h));
    } else {
        double sh = sinh(k * h);
        S_ = sinh(k * (z + h)) / sh;
        C_ = cosh(k * (z + h)) / sh;
        P_ = cosh(k * (z + h)) / cosh(k * h);
    }
}


// sum of 32 per-lane value arrays across the warp: on return lane l holds the warp total of v[l].
// Fixed butterfly order -> deterministic.  (V-1 shuffles instead of 5V.)
__device__ __forceinline__ double warp_multi_reduce32(double (&v)[32])
{
    const unsigned lane = threadIdx.x & 31u;
#pragma unroll
    for (int half = 16; half >= 1; half >>= 1) {
        const bool up = (lane & half) != 0;
#pragma unroll
        for (int t = 0; t < half; t++) {
            const double keep = up ? v[t + half] : v[t];
            const double send = up ? v[t] : v[t + half];
            v[t] = keep + __shfl_xor_sync(0xffffffffu, send, half);
        }
    }
    return v[0];
}

// compile-time loop: indices are constants, so register arrays never fall back to local memory
// (ptxas/NVVM give up on "#pragma unroll" for the triple LU nest and then index dynamically).
template <int B, int E, class F>
__device__ __forceinline__ void static_for(F &&f)
{
    if constexpr (B < E) {
        f(std::integral_constant<int, B>{});
        static_for<B + 1, E>(f);
    }
}

// Pivot reciprocals and back-substitution quotients of the dense LUs in global and shared memory (the farm and system solves,
// the generalised-DOF solves) are formed at the pivot's own scale: p is multiplied by sc = 2^-e, e the binary exponent of
// max(|re|, |im|), before |p|^2 is taken, and the result by sc again.  |p|^2 alone overflows above |p| ~ 1.3e154 (a zero
// reciprocal: nothing eliminated) and underflows below 1.5e-154 (a false zero pivot).  Power-of-two scaling is exact, so
// wherever the unscaled formula stayed in the normal range the bits are the same.  sc is built from the exponent field,
// clamped to [1, 2045] so that it stays a normal double (a subnormal or zero pivot takes 2^1022, one at or above 2^1022
// takes 2^-1022); a zero pivot still gives |q|^2 = 0, and inf / NaN go through as before.
__device__ __forceinline__ double piv_scale(const double2 p)
{
    const int eb = min(max((__double2hiint(fmax(fabs(p.x), fabs(p.y))) >> 20) & 0x7ff, 1), 2045);
    return __hiloint2double((2046 - eb) << 20, 0);
}

// 1 / p, and 0 for a zero pivot (zero set)
__device__ __forceinline__ double2 piv_recip(const double2 p, bool &zero)
{
    const double sc = piv_scale(p);
    const double2 q = make_double2(p.x * sc, p.y * sc);
    const double den = q.x * q.x + q.y * q.y;
    zero = !(den > 0.0);
    return zero ? make_double2(0.0, 0.0) : make_double2(q.x / den * sc, -q.y / den * sc);
}

// s / p
__device__ __forceinline__ double2 piv_div(const double2 s, const double2 p)
{
    const double sc = piv_scale(p);
    const double2 q = make_double2(p.x * sc, p.y * sc);
    const double den = q.x * q.x + q.y * q.y;
    return make_double2((s.x * q.x + s.y * q.y) / den * sc, (s.y * q.x - s.x * q.y) / den * sc);
}

// 6x6 complex solve in registers: LU with partial pivoting (|re|+|im| metric, as LAPACK izamax),
// forward elimination applied to b on the fly, back substitution.  Returns false on a zero pivot.
__device__ __forceinline__ bool solve6(double (&ar)[6][6], double (&ai)[6][6], double (&br)[6], double (&bi)[6])
{
    double rr[6], ri[6];
    bool ok = true;
    static_for<0, 6>([&](auto K) {
        constexpr int k = decltype(K)::value;
        int p = k;
        double best = fabs(ar[k][k]) + fabs(ai[k][k]);
        static_for<k + 1, 6>([&](auto I) {
            constexpr int i = decltype(I)::value;
            const double t = fabs(ar[i][k]) + fabs(ai[i][k]);
            if (t > best) { best = t; p = i; }
        });
        if (best == 0.0) ok = false;
        // (rows are always selected, not guarded by a warp vote "does any lane pivot here?")
        static_for<k + 1, 6>([&](auto I) {
            constexpr int i = decltype(I)::value;
            // row swap as register selects (a dynamic row index would push the matrix to local memory)
            const bool sw = (p == i);
            static_for<k, 6>([&](auto J) {
                constexpr int j = decltype(J)::value;
                const double r1 = ar[k][j], r2 = ar[i][j], i1 = ai[k][j], i2 = ai[i][j];
                ar[k][j] = sw ? r2 : r1; ar[i][j] = sw ? r1 : r2;
                ai[k][j] = sw ? i2 : i1; ai[i][j] = sw ? i1 : i2;
            });
            const double r1 = br[k], r2 = br[i], i1 = bi[k], i2 = bi[i];
            br[k] = sw ? r2 : r1; br[i] = sw ? r1 : r2;
            bi[k] = sw ? i2 : i1; bi[i] = sw ? i1 : i2;
        });
        const double pr = ar[k][k], pi = ai[k][k];
        const double inv = 1.0 / (pr * pr + pi * pi);
        rr[k] = pr * inv; ri[k] = -pi * inv;
        static_for<k + 1, 6>([&](auto I) {
            constexpr int i = decltype(I)::value;
            const double lr = ar[i][k] * rr[k] - ai[i][k] * ri[k];
            const double li = ar[i][k] * ri[k] + ai[i][k] * rr[k];
            static_for<k + 1, 6>([&](auto J) {
                constexpr int j = decltype(J)::value;
                ar[i][j] -= lr * ar[k][j] - li * ai[k][j];
                ai[i][j] -= lr * ai[k][j] + li * ar[k][j];
            });
            br[i] -= lr * br[k] - li * bi[k];
            bi[i] -= lr * bi[k] + li * br[k];
        });
    });
    static_for<0, 6>([&](auto II) {
        constexpr int i = 5 - decltype(II)::value;
        double sr = br[i], si = bi[i];
        static_for<i + 1, 6>([&](auto J) {
            constexpr int j = decltype(J)::value;
            sr -= ar[i][j] * br[j] - ai[i][j] * bi[j];
            si -= ar[i][j] * bi[j] + ai[i][j] * br[j];
        });
        br[i] = sr * rr[i] - si * ri[i];
        bi[i] = sr * ri[i] + si * rr[i];
    });
    return ok;
}
