// raftk_stress.cuh -- tower-base axial stress around the circumference (raftk_stress_ring_*).
//
// For unit u, case c and ring (a tower base) with the fore-aft moment a and the side-side moment b of the project's channel
// definitions (real rows: Y = w^wpow R Xi[col0 ..]; complex per-bin coefficients: Y = sum_b coef[b,w] Xi[col0 + b, w]), over the
// rows h of the case (its wave trains), the thin-wall axial stress sigma(theta) = c (a cos theta - b sin theta), c = (d/2) / Izz
// / 1e6 (MPa), Izz = pi/8 t d^3, has the spectral moments
//   lambda_k(theta) = c^2 (cos^2 S_aa,k - 2 sin cos S_ab,k + sin^2 S_bb,k),
//   S_aa,k = sum_h sum_j w_j^k 1/2 |a|^2, S_bb,k the same of b, S_ab,k = sum_h sum_j w_j^k 1/2 Re(a conj(b)),  k = 0, 1, 2, 4.
// So the response is walked once for the 3 x 4 sums, whatever the number of angles.
//
// k_stress_moments: one CTA per (unit, row, bin tile), built like k_fatigue_moments: the tile of Xi staged in shared memory
// (read from L2 when not even one chunk fits), a warp per (ring, FAT_CHUNK-bin chunk), one bin per lane, the chunk's twelve
// sums reduced with a fixed shuffle tree.  Tiles are whole chunks of the tile rule the two share (moment_tile), so a chunk's
// partial sums do not depend on the tile width.
// k_stress_finish: one thread per (unit, case, ring, angle) sums the chunk partials of the case's rows in (row, chunk) order,
// forms lambda_k(theta) and gives std, avg, max, min and the DEL through fatigue_del, the closed form k_fatigue_finish
// applies.  k_stress_hot: one thread per (unit, case, ring): the argmax angles of std and DEL over the grid, and the largest
// std over the circle, c sqrt(mu), mu the larger eigenvalue of [[S_aa,0, S_ab,0], [S_ab,0, S_bb,0]].  k_stress_psd: one thread
// per (unit, case, ring, bin), the per-bin PSD sum_h 1/2 |sigma_h|^2 / dw of every angle.
// No atomics anywhere: a result does not depend on which units, cases, rings or angles share the call, or on the tile width.
#pragma once

#define STR_T 256
#define STR_FIN_T 128
#define STR_NS 12               // sums per (ring, chunk): {aa, bb, ab} x {w^0, w^1, w^2, w^4}
#define STR_LAUNCH_CASES 64     // cases per finish / hot / PSD launch: their row table travels in the launch parameters

struct StrParams {
    // response and channels
    int n, n_r, nw, n_rows, n_rings, n_ch, tile, n_tiles, n_chunks;
    size_t r_stride;                    // real form: doubles between two units' R (0: shared)
    size_t cf_ustride, cf_rstride;      // complex form: coefficients between two units / two rows (0: shared)
    const double *w, *R;
    const double2 *coef, *Xi;           // Xi [U, n_rows, n, nw]
    double *part;                       // [U, n_rows, n_chunks, n_rings, STR_NS]
    // reductions
    int n_cases, n_angles, method, c0, nc;
    double c2, c, f_eq, m, dw;          // m = 0: no DEL
    const double *mean;                 // [U, n_cases, n_rings, n_ch] or NULL
    double *std, *avg, *mx, *mn, *DEL, *wd, *hot, *psd;
    int *info;
    int col0[RAFTK_STRESS_RING_MAX];
    unsigned wbits[RAFTK_STRESS_RING_MAX * 2 / 16];
    int row0[STR_LAUNCH_CASES + 1];
    double p[STR_LAUNCH_CASES];         // case weights
    double angle[RAFTK_STRESS_ANGLE_MAX];
};

// fore-aft (a) and side-side (b) amplitudes of ring `ring` at bin iw of row (u, r), b = 0 with one channel; x points at
// column 0 of the row's bin iw (stride nw between columns), or at the staged tile (stride xs_stride)
template <bool COEF>
__device__ __forceinline__ void stress_ab(const StrParams &P, size_t u, size_t r, int ring, int iw, const double2 *x, int xs_stride,
                                          double2 &a, double2 &b)
{
    double ar = 0.0, ai = 0.0, br = 0.0, bi = 0.0;
    const bool two = P.n_ch == 2;
    const double2 *xc = x + (size_t)P.col0[ring] * xs_stride;
    if (COEF) {
        const double2 *ca = P.coef + u * P.cf_ustride + r * P.cf_rstride + (size_t)ring * P.n_ch * P.n_r * P.nw + iw;
        const double2 *cb = ca + (size_t)P.n_r * P.nw;
        for (int k = 0; k < P.n_r; k++) {
            const double2 v = xc[(size_t)k * xs_stride];
            const double2 f = ca[(size_t)k * P.nw];
            ar += f.x * v.x - f.y * v.y; ai += f.x * v.y + f.y * v.x;
            if (two) {
                const double2 s = cb[(size_t)k * P.nw];
                br += s.x * v.x - s.y * v.y; bi += s.x * v.y + s.y * v.x;
            }
        }
    } else {
        const double *ra = P.R + u * P.r_stride + (size_t)ring * P.n_ch * P.n_r, *rb = ra + P.n_r;
        for (int k = 0; k < P.n_r; k++) {
            const double2 v = xc[(size_t)k * xs_stride];
            ar = fma(ra[k], v.x, ar); ai = fma(ra[k], v.y, ai);
            if (two) { br = fma(rb[k], v.x, br); bi = fma(rb[k], v.y, bi); }
        }
        const double w1 = P.w[iw];
        const int pa = (P.wbits[ring >> 3] >> ((ring & 7) * 4)) & 3, pb = (P.wbits[ring >> 3] >> ((ring & 7) * 4 + 2)) & 3;
        const double fa = pa == 2 ? w1 * w1 : (pa == 1 ? w1 : 1.0), fb = pb == 2 ? w1 * w1 : (pb == 1 ? w1 : 1.0);
        if (pa) { ar *= fa; ai *= fa; }
        if (pb) { br *= fb; bi *= fb; }
    }
    a = make_double2(ar, ai);
    b = make_double2(br, bi);
}

template <bool SMEM, bool COEF>
__global__ void __launch_bounds__(STR_T) k_stress_moments(const __grid_constant__ StrParams P)
{
    extern __shared__ double2 xs[];                     // [n][tw] when SMEM
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int t = (int)(blockIdx.x % (unsigned)P.n_tiles);
    const size_t ur = blockIdx.x / (unsigned)P.n_tiles;    // unit * n_rows + row
    const size_t u = ur / (size_t)P.n_rows, r = ur - u * P.n_rows;
    const int i0 = t * P.tile, tw = min(P.tile, P.nw - i0);
    const double2 *x = P.Xi + ur * (size_t)P.n * P.nw + i0;
    stage_xi_tile<SMEM, STR_T>(P, xs, x, tw, tid);
    const int n_ck = (tw + FAT_CHUNK - 1) / FAT_CHUNK;
    for (int k = warp; k < P.n_rings * n_ck; k += STR_T / 32) {
        const int ring = k / n_ck, ck = k - ring * n_ck;
        const int i = ck * FAT_CHUNK + lane, iw = i0 + i;
        const bool live = i < tw;
        double2 a = make_double2(0.0, 0.0), b = a;
        if (live) {
            if (SMEM) stress_ab<COEF>(P, u, r, ring, iw, xs + i, tw, a, b);
            else stress_ab<COEF>(P, u, r, ring, iw, x + i, P.nw, a, b);
        }
        const double w1 = live ? P.w[iw] : 0.0, w2 = w1 * w1, w4 = w2 * w2;
        const double p[3] = {0.5 * (a.x * a.x + a.y * a.y), 0.5 * (b.x * b.x + b.y * b.y), 0.5 * (a.x * b.x + a.y * b.y)};
        double s[STR_NS];
#pragma unroll
        for (int j = 0; j < 3; j++) { s[4 * j] = p[j]; s[4 * j + 1] = w1 * p[j]; s[4 * j + 2] = w2 * p[j]; s[4 * j + 3] = w4 * p[j]; }
        for (int sh = 16; sh >= 1; sh >>= 1) {
#pragma unroll
            for (int j = 0; j < STR_NS; j++) s[j] += __shfl_xor_sync(0xffffffffu, s[j], sh);
        }
        if (lane < STR_NS) {
            double v = s[0];
#pragma unroll
            for (int j = 1; j < STR_NS; j++) if (lane == j) v = s[j];
            P.part[((ur * P.n_chunks + (size_t)(i0 / FAT_CHUNK + ck)) * P.n_rings + ring) * STR_NS + lane] = v;
        }
    }
}

// the twelve sums of (unit u, ring) over rows r0 .. r1-1, in (row, chunk) order
__device__ __forceinline__ void stress_sums(const StrParams &P, size_t u, int r0, int r1, int ring, double S[STR_NS])
{
#pragma unroll
    for (int j = 0; j < STR_NS; j++) S[j] = 0.0;
    for (int r = r0; r < r1; r++) {
        const double *q = P.part + (((u * P.n_rows + r) * P.n_chunks) * P.n_rings + ring) * STR_NS;
        for (int j = 0; j < P.n_chunks; j++, q += (size_t)P.n_rings * STR_NS) {
#pragma unroll
            for (int v = 0; v < STR_NS / 4; v++) {
                const double4 d = *reinterpret_cast<const double4 *>(q + 4 * v);
                S[4 * v] += d.x; S[4 * v + 1] += d.y; S[4 * v + 2] += d.z; S[4 * v + 3] += d.w;
            }
        }
    }
}

__global__ void __launch_bounds__(STR_FIN_T) k_stress_finish(const __grid_constant__ StrParams P, size_t n_threads)
{
    const size_t g = (size_t)blockIdx.x * STR_FIN_T + threadIdx.x;
    if (g >= n_threads) return;
    const int ia = (int)(g % (unsigned)P.n_angles);
    const int ring = (int)((g / (unsigned)P.n_angles) % (unsigned)P.n_rings);
    const int cl = (int)((g / ((size_t)P.n_angles * P.n_rings)) % (unsigned)P.nc);
    const size_t u = g / ((size_t)P.n_angles * P.n_rings * P.nc);
    const int c = P.c0 + cl;
    double S[STR_NS];
    stress_sums(P, u, P.row0[cl], P.row0[cl + 1], ring, S);
    double sn, cs;
    sincos(P.angle[ia], &sn, &cs);
    const double qa = cs * cs, qb = sn * sn, qab = 2.0 * sn * cs;
    double l[4];
#pragma unroll
    for (int k = 0; k < 4; k++) l[k] = P.c2 * (qa * S[k] - qab * S[8 + k] + qb * S[4 + k]);
    const size_t cr = (u * P.n_cases + c) * P.n_rings + ring, o = cr * P.n_angles + ia;
    const double sd = sqrt(fmax(l[0], 0.0));
    double avg = 0.0;
    if (P.mean) {
        const double *mu = P.mean + cr * P.n_ch;
        avg = P.c * (cs * mu[0] - (P.n_ch == 2 ? sn * mu[1] : 0.0));
    }
    P.std[o] = sd; P.avg[o] = avg; P.mx[o] = avg + 3.0 * sd; P.mn[o] = avg - 3.0 * sd;
    if (P.m > 0.0) fatigue_del(P, l[0], l[1], l[2], l[3], &P.m, cl, o);
}

// argmax over the grid of std (and DEL) and the largest std over the circle, for (unit, case, ring):
// hot = {angle of max std, max std, angle of max DEL, max DEL, exact max std, its angle in [0, pi)}
__global__ void __launch_bounds__(STR_FIN_T) k_stress_hot(const __grid_constant__ StrParams P, size_t n_threads)
{
    const size_t g = (size_t)blockIdx.x * STR_FIN_T + threadIdx.x;
    if (g >= n_threads) return;
    const int ring = (int)(g % (unsigned)P.n_rings);
    const int cl = (int)((g / (unsigned)P.n_rings) % (unsigned)P.nc);
    const size_t u = g / ((size_t)P.n_rings * P.nc);
    const size_t cr = (u * P.n_cases + P.c0 + cl) * P.n_rings + ring;
    const double *sd = P.std + cr * P.n_angles;
    int js = 0, jd = 0;
    for (int j = 1; j < P.n_angles; j++) if (sd[j] > sd[js]) js = j;
    double *h = P.hot + cr * 6;
    h[0] = P.angle[js]; h[1] = sd[js];
    if (P.m > 0.0) {
        const double *dl = P.DEL + cr * P.n_angles;
        for (int j = 1; j < P.n_angles; j++) if (dl[j] > dl[jd]) jd = j;
        h[2] = P.angle[jd]; h[3] = dl[jd];
    } else {
        h[2] = 0.0; h[3] = 0.0;
    }
    double S[STR_NS];
    stress_sums(P, u, P.row0[cl], P.row0[cl + 1], ring, S);
    const double half = 0.5 * (S[0] - S[4]), A = sqrt(half * half + S[8] * S[8]);
    const double mu = 0.5 * (S[0] + S[4]) + A;
    double th = A > 0.0 ? 0.5 * atan2(-S[8], half) : 0.0;     // maximiser of (S_aa - S_bb)/2 cos 2t - S_ab sin 2t
    if (th < 0.0) th += CUDART_PI;
    h[4] = P.c * sqrt(fmax(mu, 0.0)); h[5] = th;
}

// lifetime hot spot of (unit, ring): the argmax angle of DEL_life [U, n_rings, n_angles] -> hot [U, n_rings, 2] (angle, DEL)
__global__ void __launch_bounds__(STR_FIN_T) k_stress_hot_life(const __grid_constant__ StrParams P, const double *DEL_life, size_t n_threads)
{
    const size_t g = (size_t)blockIdx.x * STR_FIN_T + threadIdx.x;
    if (g >= n_threads) return;
    const double *dl = DEL_life + g * P.n_angles;
    int jd = 0;
    for (int j = 1; j < P.n_angles; j++) if (dl[j] > dl[jd]) jd = j;
    P.hot[g * 2] = P.angle[jd]; P.hot[g * 2 + 1] = dl[jd];
}

// per-bin stress PSD of every angle, [U, n_cases, n_rings, n_angles, nw]: sum over the case's rows of 1/2 |sigma|^2 / dw
template <bool COEF>
__global__ void __launch_bounds__(STR_FIN_T) k_stress_psd(const __grid_constant__ StrParams P, size_t n_threads)
{
    const size_t g = (size_t)blockIdx.x * STR_FIN_T + threadIdx.x;
    if (g >= n_threads) return;
    const int iw = (int)(g % (unsigned)P.nw);
    const int ring = (int)((g / (unsigned)P.nw) % (unsigned)P.n_rings);
    const int cl = (int)((g / ((size_t)P.nw * P.n_rings)) % (unsigned)P.nc);
    const size_t u = g / ((size_t)P.nw * P.n_rings * P.nc);
    double paa = 0.0, pbb = 0.0, pab = 0.0;
    for (int r = P.row0[cl]; r < P.row0[cl + 1]; r++) {
        double2 a, b;
        stress_ab<COEF>(P, u, r, ring, iw, P.Xi + ((u * P.n_rows + r) * P.n) * P.nw + iw, P.nw, a, b);
        paa += 0.5 * (a.x * a.x + a.y * a.y); pbb += 0.5 * (b.x * b.x + b.y * b.y); pab += 0.5 * (a.x * b.x + a.y * b.y);
    }
    const double f = P.c2 / P.dw;
    double *o = P.psd + (((u * P.n_cases + P.c0 + cl) * P.n_rings + ring) * P.n_angles) * P.nw + iw;
    for (int ia = 0; ia < P.n_angles; ia++) {
        double sn, cs;
        sincos(P.angle[ia], &sn, &cs);
        o[(size_t)ia * P.nw] = f * (cs * cs * paa - 2.0 * sn * cs * pab + sn * sn * pbb);
    }
}
