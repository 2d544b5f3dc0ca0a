// raftk_fatigue.cuh -- spectral fatigue damage-equivalent loads (raftk_fatigue_*).
//
// For unit u, case c and channel ch, with the rows h of the case (its wave trains) and the channel amplitude Y_h(w) of the
// project's channel definitions (real rows: Y = w^wpow R Xi; complex per-bin coefficients: Y = sum_b coef[b,w] Xi[b,w]):
//   lambda_k = sum_h sum_j w_j^k 1/2 |Y_h(w_j)|^2,  k = 0, 1, 2, 4        (rad/s, one-sided, getRMS's discrete rule)
// then Dirlik's (or the narrow-band) closed form of the stress-range moment E[S^m] and the damage rate d = E[P] E[S^m],
// DEL = (d / f_eq)^(1/m), and optionally DEL_life = (sum_c p_c d_c / (f_eq sum_c p_c))^(1/m).
//
// k_fatigue_moments: one CTA per (unit, row, bin tile) stages the tile's n x tile bins of Xi in shared memory (as
// k_farm_channels does; Xi is read from L2 when not even one chunk of bins fits).  A warp takes FAT_CH_B channels of one
// chunk of FAT_CHUNK bins, one bin per lane, and reduces the chunk's four moment sums with a fixed shuffle tree.  Tiles
// are whole chunks, so a chunk's partial sums do not depend on the tile width.
// k_fatigue_finish: one thread per (unit, case, channel) sums the chunk partials of the case's rows in (row, chunk) order
// and applies the closed form in the log domain.  k_fatigue_life: one thread per (unit, channel) sums p_c d_c over the cases
// in order, scaled by the largest term.
// No atomics anywhere: a result does not depend on which units, cases or channels share the call, or on the tile width.
#pragma once

#define FAT_T 256
#define FAT_CHUNK 32            // bins per partial sum: one warp, one bin per lane
#define FAT_CH_B 4              // channels per warp item
#define FAT_FIN_T 128
#define FAT_LAUNCH_CHUNK 256    // cases and channels per finish / life launch: their tables travel in the launch parameters

struct FatMomParams {
    int n, nch, nw, n_rows, tile, n_tiles, n_chunks;
    size_t r_stride;            // real form: doubles between two units' R (0: shared)
    size_t cf_ustride, cf_rstride;   // complex form: coefficients between two units / two rows (0: shared)
    const double *w, *R;
    const double2 *coef, *Xi;   // Xi [U, n_rows, n, nw]
    double *part;               // [U, n_rows, n_chunks, nch, 4]
    unsigned wbits[RAFTK_FATIGUE_CH_MAX / 16];
};

template <bool SMEM, bool COEF>
__global__ void __launch_bounds__(FAT_T) k_fatigue_moments(const __grid_constant__ FatMomParams P)
{
    extern __shared__ double2 xs[];                     // [n][tw] when SMEM
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int t = (int)(blockIdx.x % (unsigned)P.n_tiles);
    const size_t ur = blockIdx.x / (unsigned)P.n_tiles;    // unit * n_rows + row
    const size_t u = ur / (size_t)P.n_rows, r = ur - u * P.n_rows;
    const int i0 = t * P.tile, tw = min(P.tile, P.nw - i0);
    const double2 *x = P.Xi + ur * (size_t)P.n * P.nw + i0;
    stage_xi_tile<SMEM, FAT_T>(P, xs, x, tw, tid);
    const int nchb = (P.nch + FAT_CH_B - 1) / FAT_CH_B;
    const int n_ck = (tw + FAT_CHUNK - 1) / FAT_CHUNK;
    for (int k = warp; k < nchb * n_ck; k += FAT_T / 32) {
        const int cg = k / n_ck, ck = k - cg * n_ck;
        const int i = ck * FAT_CHUNK + lane, iw = i0 + i;
        const bool live = i < tw;
        const int c0 = cg * FAT_CH_B;
        double yr[FAT_CH_B], yi[FAT_CH_B];
#pragma unroll
        for (int j = 0; j < FAT_CH_B; j++) { yr[j] = 0.0; yi[j] = 0.0; }
        if (live) {
            if (COEF) {
                const double2 *cf[FAT_CH_B];
#pragma unroll
                for (int j = 0; j < FAT_CH_B; j++)
                    cf[j] = P.coef + u * P.cf_ustride + r * P.cf_rstride + (size_t)min(c0 + j, P.nch - 1) * P.n * P.nw + iw;
                for (int b = 0; b < P.n; b++) {
                    const double2 v = SMEM ? xs[b * tw + i] : x[(size_t)b * P.nw + i];
#pragma unroll
                    for (int j = 0; j < FAT_CH_B; j++) {
                        const double2 c = cf[j][(size_t)b * P.nw];
                        yr[j] += c.x * v.x - c.y * v.y; yi[j] += c.x * v.y + c.y * v.x;
                    }
                }
            } else {
                const double *rr[FAT_CH_B];
#pragma unroll
                for (int j = 0; j < FAT_CH_B; j++) rr[j] = P.R + u * P.r_stride + (size_t)min(c0 + j, P.nch - 1) * P.n;
                for (int b = 0; b < P.n; b++) {
                    const double2 v = SMEM ? xs[b * tw + i] : x[(size_t)b * P.nw + i];
#pragma unroll
                    for (int j = 0; j < FAT_CH_B; j++) {
                        const double c = rr[j][b];
                        yr[j] = fma(c, v.x, yr[j]); yi[j] = fma(c, v.y, yi[j]);
                    }
                }
            }
        }
        const double w1 = live ? P.w[iw] : 0.0, w2 = w1 * w1, w4 = w2 * w2;
        const size_t o = ((ur * P.n_chunks + (size_t)(i0 / FAT_CHUNK + ck)) * P.nch) * 4;
#pragma unroll
        for (int j = 0; j < FAT_CH_B; j++) {
            const int ch = c0 + j;
            if (ch >= P.nch) break;                     // warp-uniform
            double re = yr[j], im = yi[j];
            if (!COEF) {
                const int p = (P.wbits[ch >> 4] >> ((ch & 15) * 2)) & 3;
                if (p == 2) { re *= w2; im *= w2; }
                else if (p == 1) { re *= w1; im *= w1; }
            }
            const double a = 0.5 * (re * re + im * im);
            double s0 = a, s1 = w1 * a, s2 = w2 * a, s4 = w4 * a;
            for (int sh = 16; sh >= 1; sh >>= 1) {
                s0 += __shfl_xor_sync(0xffffffffu, s0, sh);
                s1 += __shfl_xor_sync(0xffffffffu, s1, sh);
                s2 += __shfl_xor_sync(0xffffffffu, s2, sh);
                s4 += __shfl_xor_sync(0xffffffffu, s4, sh);
            }
            if (lane == 0) {
                double *q = P.part + o + (size_t)ch * 4;
                q[0] = s0; q[1] = s1; q[2] = s2; q[3] = s4;
            }
        }
    }
}

struct FatFinParams {
    int n_rows, n_cases, nch, n_chunks, method;
    int c0, nc, k0, nk;         // the launch's cases c0 .. c0+nc-1 and channels k0 .. k0+nk-1
    double f_eq;
    const double *part;
    double *moments, *DEL, *wd; // wd [U, n_cases, nch]: log(p_c d_c) for the lifetime sum, or NULL
    int *info;
    int row0[FAT_LAUNCH_CHUNK + 1];
    double m[FAT_LAUNCH_CHUNK], p[FAT_LAUNCH_CHUNK];
};

// log of the damage rate d (1/s) of moments l0, l1, l2, l4 (l0 > 0, l2 > 0) for Woehler exponent m, evaluated in the log
// domain so that neither (2 sqrt(l0))^m nor Gamma(1+m) overflows before the 1/m root; sets RAFTK_FATIGUE_NARROWBAND in *info
// when the narrow-band form was used
__device__ __forceinline__ double fatigue_log_rate(double l0, double l1, double l2, double l4, double m, int method, int *info)
{
    const double log_2pi = 1.8378770664093453, ln2 = 0.6931471805599453;
    if (method == RAFTK_FATIGUE_DIRLIK) {
        const double xm = (l1 / l0) * sqrt(l2 / l4), g = l2 / sqrt(l0 * l4);
        const double D1 = 2.0 * (xm - g * g) / (1.0 + g * g);
        const double den = 1.0 - g - D1 + D1 * D1;
        const double R = (g - xm - D1 * D1) / den;
        const double D2 = den / (1.0 - R), D3 = 1.0 - D1 - D2;
        const double Q = 1.25 * (g - D3 - D2 * R) / D1;
        const double inner = D2 * pow(fabs(R), m) + D3;
        const bool ok = 1.0 - g >= RAFTK_FATIGUE_NB_SWITCH && isfinite(D1) && D1 > 0.0 && isfinite(Q) && Q > 0.0 && isfinite(R) && R > 0.0
                        && inner > 0.0;
        if (ok) {
            // log of the bracket D1 Q^m Gamma(1+m) + 2^(m/2) Gamma(1+m/2) (D2 |R|^m + D3), larger term first
            const double t1 = log(D1) + m * log(Q) + lgamma(1.0 + m);
            const double t2 = 0.5 * m * ln2 + lgamma(1.0 + 0.5 * m) + log(inner);
            const double hi = fmax(t1, t2), lo = fmin(t1, t2);
            const double lb = hi + log1p(exp(lo - hi));
            return 0.5 * log(l4 / l2) - log_2pi + m * (ln2 + 0.5 * log(l0)) + lb;
        }
    }
    *info |= RAFTK_FATIGUE_NARROWBAND;
    return 0.5 * log(l2 / l0) - log_2pi + m * (ln2 + 0.5 * log(2.0 * l0)) + lgamma(1.0 + 0.5 * m);
}

// DEL = (d / P.f_eq)^(1/m) of moments l0, l1, l2, l4 into P.DEL[o] and P.info[o] (RAFTK_FATIGUE_ZERO when l0 or l2 is 0), and
// log(p_c d_c) of the weight p_c = P.p[cl] of local case cl into P.wd[o] for the lifetime sum when P.wd is given; shared by
// k_fatigue_finish and k_stress_finish.  The exponent *mp is read only where it is used, which keeps both kernels' code as it
// was before they shared this.
template <class Prm>
__device__ __forceinline__ void fatigue_del(const Prm &P, double l0, double l1, double l2, double l4, const double *mp, int cl, size_t o)
{
    int info = 0;
    double ld = -CUDART_INF, del = 0.0;
    if (!(l0 > 0.0) || !(l2 > 0.0)) {
        info = RAFTK_FATIGUE_ZERO;
    } else {
        const double m = *mp;
        ld = fatigue_log_rate(l0, l1, l2, l4, m, P.method, &info);
        del = exp((ld - log(P.f_eq)) / m);
    }
    P.DEL[o] = del;
    P.info[o] = info;
    if (P.wd) P.wd[o] = P.p[cl] > 0.0 ? log(P.p[cl]) + ld : -CUDART_INF;
}

__global__ void __launch_bounds__(FAT_FIN_T) k_fatigue_finish(const __grid_constant__ FatFinParams P, size_t n_threads)
{
    const size_t g = (size_t)blockIdx.x * FAT_FIN_T + threadIdx.x;
    if (g >= n_threads) return;
    const int kl = (int)(g % (unsigned)P.nk);
    const int cl = (int)((g / (unsigned)P.nk) % (unsigned)P.nc);
    const size_t u = g / ((size_t)P.nk * P.nc);
    const int ch = P.k0 + kl, c = P.c0 + cl;
    double l0 = 0.0, l1 = 0.0, l2 = 0.0, l4 = 0.0;
    for (int r = P.row0[cl]; r < P.row0[cl + 1]; r++) {
        const double *q = P.part + ((u * P.n_rows + r) * P.n_chunks * P.nch + ch) * 4;
        for (int j = 0; j < P.n_chunks; j++, q += (size_t)P.nch * 4) {
            const double4 v = *reinterpret_cast<const double4 *>(q);
            l0 += v.x; l1 += v.y; l2 += v.z; l4 += v.w;
        }
    }
    const size_t o = (u * P.n_cases + c) * P.nch + ch;
    if (P.moments) {
        double *q = P.moments + o * 4;
        q[0] = l0; q[1] = l1; q[2] = l2; q[3] = l4;
    }
    fatigue_del(P, l0, l1, l2, l4, &P.m[kl], cl, o);
}

struct FatLifeParams {
    int n_cases, nch, k0, nk;
    double log_fw;              // log(f_eq * sum_c p_c)
    const double *wd;           // log(p_c d_c) [U, n_cases, nch]
    double *DEL_life;
    double m[FAT_LAUNCH_CHUNK];
};

// DEL_life = (sum_c p_c d_c / (f_eq sum_c p_c))^(1/m) from log(p_c d_c), scaled by the largest term: two passes over the
// cases in order
__global__ void __launch_bounds__(FAT_FIN_T) k_fatigue_life(const __grid_constant__ FatLifeParams P, size_t n_threads)
{
    const size_t g = (size_t)blockIdx.x * FAT_FIN_T + threadIdx.x;
    if (g >= n_threads) return;
    const int kl = (int)(g % (unsigned)P.nk);
    const size_t u = g / (unsigned)P.nk;
    const int ch = P.k0 + kl;
    const double *x = P.wd + u * P.n_cases * P.nch + ch;
    double mx = -CUDART_INF;
    for (int c = 0; c < P.n_cases; c++) mx = fmax(mx, x[(size_t)c * P.nch]);
    double s = 0.0;
    if (mx > -CUDART_INF)
        for (int c = 0; c < P.n_cases; c++) s += exp(x[(size_t)c * P.nch] - mx);
    P.DEL_life[u * P.nch + ch] = mx > -CUDART_INF ? exp((mx + log(s) - P.log_fw) / P.m[kl]) : 0.0;
}
