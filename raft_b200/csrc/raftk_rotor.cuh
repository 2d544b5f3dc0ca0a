// raftk_rotor.cuh -- rotor speed, generator torque and blade pitch statistics (raftk_rotor_stats_*).
//
// FOWT.saveTurbineOutputs (raft_fowt.py:2610-2679), per rotor ir of an operating turbine (aeroServoMod > 1, inflow > 0):
//   phi_h(w)    = C(w) XiHub[h, ir](w)                 for every wave train h              (:2643-2644)
//   phi_last(w) = C(w) (0 - V_w(w) / (j w))            the last, all-zero row of Model.Xi  (:2646)
//   omega  = j w phi,  torque = (j w kp_tau + ki_tau) phi,  bPitch = (j w kp_beta + ki_beta) phi   (:2649-2651)
//   std = sqrt(1/2 sum_rows sum_w |.|^2), PSD(w) = 1/2 sum_rows |.|^2 / dw   (getRMS / getPSD, helpers.py:678-700)
// omega in rpm through the reference's radps2rpm (/0.1047, helpers.py:32-33), bPitch in degrees (rad2deg, :25-26).
// XiHub[h, ir] is a real functional of the response: y = sum_b R[rot][b] Xi[unit][row][col0[rot] + b].  Each channel is
// a complex factor times phi, so per bin  sum_rows |channel|^2 = |factor|^2 |C|^2 (sum_rows |y|^2 + |V_w|^2 / w^2).
// One 128-thread CTA per (unit, case, rotor), threads strided over bins; the rows of the case, the fma chain over b and the
// block reduction run in a fixed order, so a result does not depend on which units, cases or rotors share the call.
#pragma once

#define ROTOR_T 128
#define ROTOR_CHUNK 256         // cases and rotors per launch: their col0 / case_row0 travel in the launch parameters

struct RotorParams {
    int n_rows, n_dof, nw, n_r;
    int n_cases, n_rot;         // output strides
    int c0, nc, k0, nk;         // the launch's cases c0 .. c0+nc-1 and rotors k0 .. k0+nk-1
    size_t r_stride;            // doubles between two units' R (0: shared)
    size_t tf_stride;           // (case, rotor) entries between two units' C / V_w / gains (0: shared)
    double dw;
    const double *w, *R, *gains;
    const double2 *Xi, *C, *Vw;
    double *sd, *psd;
    int col0[ROTOR_CHUNK];
    int row0[ROTOR_CHUNK + 1];  // case_row0[c0 .. c0+nc]
};

__global__ void __launch_bounds__(ROTOR_T) k_rotor_stats(const __grid_constant__ RotorParams P)
{
    __shared__ double part[3][4];
    const int tid = threadIdx.x;
    const int kl = (int)(blockIdx.x % (unsigned)P.nk);
    const int cl = (int)((blockIdx.x / (unsigned)P.nk) % (unsigned)P.nc);
    const size_t u = blockIdx.x / ((unsigned)P.nk * (unsigned)P.nc);
    const int k = P.k0 + kl, c = P.c0 + cl;
    const size_t t = u * P.tf_stride + (size_t)c * P.n_rot + k;         // (case, rotor) entry of the tables
    const double2 *Cf = P.C + t * P.nw, *Vw = P.Vw + t * P.nw;
    const double kp_t = P.gains[4 * t], ki_t = P.gains[4 * t + 1], kp_b = P.gains[4 * t + 2], ki_b = P.gains[4 * t + 3];
    const double *R = P.R + u * P.r_stride + (size_t)k * P.n_r;
    const size_t row_sz = (size_t)P.n_dof * P.nw;
    const double2 *x = P.Xi + u * P.n_rows * row_sz + (size_t)P.col0[kl] * P.nw;
    const int r0 = P.row0[cl], r1 = P.row0[cl + 1];
    const double rpm = 1.0 / 0.1047, deg = 57.29577951308232;           // radps2rpm(1), rad2deg(1)
    const size_t o = ((u * P.n_cases + c) * P.n_rot + k) * 3;
    double s0 = 0.0, s1 = 0.0, s2 = 0.0;
    for (int i = tid; i < P.nw; i += ROTOR_T) {
        double y2 = 0.0;                                                  // sum over the case's trains of |XiHub|^2
        for (int r = r0; r < r1; r++) {
            const double2 *xr = x + (size_t)r * row_sz + i;
            double yr = 0.0, yi = 0.0;
            for (int b = 0; b < P.n_r; b++) {
                const double cb = R[b];
                const double2 v = xr[(size_t)b * P.nw];
                yr = fma(cb, v.x, yr); yi = fma(cb, v.y, yi);
            }
            y2 += yr * yr + yi * yi;
        }
        const double wi = P.w[i], w2 = wi * wi;
        const double2 cf = Cf[i], vw = Vw[i];
        const double a = (cf.x * cf.x + cf.y * cf.y) * (y2 + (vw.x * vw.x + vw.y * vw.y) / w2);   // sum_rows |phi|^2
        const double om = w2 * a, tq = (ki_t * ki_t + w2 * (kp_t * kp_t)) * a, bp = (ki_b * ki_b + w2 * (kp_b * kp_b)) * a;
        s0 += om; s1 += tq; s2 += bp;
        if (P.psd) {
            double *p = P.psd + o * P.nw + i;
            p[0] = rpm * rpm * (0.5 * om / P.dw);
            p[P.nw] = 0.5 * tq / P.dw;
            p[2 * (size_t)P.nw] = deg * deg * (0.5 * bp / P.dw);
        }
    }
    // block_rms_tail's order for each of the three sums
    for (int sh = 16; sh >= 1; sh >>= 1) {
        s0 += __shfl_xor_sync(0xffffffffu, s0, sh);
        s1 += __shfl_xor_sync(0xffffffffu, s1, sh);
        s2 += __shfl_xor_sync(0xffffffffu, s2, sh);
    }
    if ((tid & 31) == 0) { part[0][tid >> 5] = s0; part[1][tid >> 5] = s1; part[2][tid >> 5] = s2; }
    __syncthreads();
    if (tid < 3) {
        const double s = ((part[tid][0] + part[tid][1]) + part[tid][2]) + part[tid][3];
        const double rms = sqrt(0.5 * s);
        P.sd[o + tid] = tid == 0 ? rms / 0.1047 : (tid == 1 ? rms : rms * deg);
    }
}
