// raftk_general.cuh -- Model.solveDynamics for FOWTs with generalised degrees of freedom (flexible members, nDOF up to 256;
// raft_fowt.py:1854-1857, 1886-1888, 1913-1929 and raft_model.py:1052-1142)  (included by raftk.cu only).  Validated on
// the GPU against the reference's 150-DOF VolturnUS-S-flexible run (tests/test_general_dofs.py).
//
// The checker (oracle/raft_oracle.c: ro_general_*) is pinned to the reference's VolturnUS-S-flexible pickles and a 150-DOF
// solveDynamics run; these kernels restate the same bookkeeping: every strip node j carries the 6 x n block Tn_j of fowt.T
// of its structural node and its offset rr_j from it; node motion = Tn_j Xi, node load -> Tn_j^T [f ; rr_j x f].
// Launch sequence per call (no host synchronisation; cases that have converged skip their CTAs):
//   k_gen_wave      (case, node, w)   wave kinematics u, inertial node load f6 = [f ; rr x f]
//   k_gen_bem       (case, w)         BEM tables only: 6-component BEM force (full DOFs 0-5) of every case and train
//   k_gen_project   (case, dof, w)    F = sum_j Tn_j^T f6_j   (F_BEM = T0^T f_BEM; F_iner = F_BEM + sum_j Tn_j^T f6_j; F_drag)
//   k_gen_add_2nd   (case, 0-5, w)    QTF only: F_iner += F_2nd on reduced DOFs 0-5 (F_2nd from the k_qtf_* kernels, before)
//   per pass:
//   k_gen_node_pass (case, node)      node velocity from Tn_j XiLast, RMS over w, linearised Bmat_j, drag load f6
//   k_gen_bdrag     (case, row)       B_drag = sum_j Tn_j^T B6_j Tn_j
//   k_gen_project                     F_drag
//   k_gen_solve     (case, w)         Z = -w^2 M + i w (B + B_drag) + C, dense complex LU with partial pivoting, Xi;
//                                     on the support of the frequency-dependent terms M + A_w(w) and B + B_w(w) (gen_impedance)
//   k_gen_relax     (case)            convergence bookkeeping, XiLast = 0.2 XiLast + 0.8 Xi
// Wave trains (cases.primary): a secondary train takes no part in the loop (done at init); after it
//   k_gen_node_pass<true>   (case, node)   drag node load from the PRIMARY's last Bmat and the train's own u
//   k_gen_project                          F_drag of the secondaries
//   k_gen_train_solve (case, w)            Xi = Z_p^-1 (F_iner + F_drag) from the primary's LU factors left in W.Z and W.piv:
//                                          row interchanges, unit-lower and upper triangular solves, O(n^2) per system
#pragma once

struct GenDev {
    int n, nw, Ns;
    double depth, dw;
    const double *w, *k;
    const double *node_r;        // [Ns][3]
    const double *node_frame;    // [Ns][9]  q, p1, p2 of the node's member
    const int *node_circ;        // [Ns]
    const double *node_Imat;     // [Ns][9]
    const double2 *node_Imat_w;  // [Ns][9][nw] MacCamy-Fuchs, or NULL
    const double *node_a_i;      // [Ns] signed end area
    const double *node_cd;       // [Ns][4]  a_q Cd_q, a_p1 Cd_p1, a_p2 Cd_p2, a_End Cd_End
    const double *Tn;            // [Ns][6][n]
    const double *rr;            // [Ns][3]
    const double *M, *B, *C;     // [n][n]
    double rho;
};

// frequency-dependent terms (raftk_general_fd), a parameter of their own so that every kernel of the constant-matrix solve
// keeps its parameter layout; n_fd = 0 / n_bem_head = 0 without them
struct GenFdDev {
    int n_fd, n_bem_head;
    const int *fd_idx;           // [n_fd] strictly increasing reduced DOFs
    const double *A_w, *B_w;     // [n_fd][n_fd][nw]
    const double *bem_headings;  // [n_bem_head] deg
    const double2 *X_BEM;        // [n_bem_head][6][nw] heading-relative
    const double *T0;            // [6][n] rows 0..5 of fowt.T
    double x_ref, y_ref, hadj;
    double2 *fb6;                // [nC][6][nw] workspace: BEM force in full DOFs 0-5
    const double2 *F_BEM;        // [nC][n][nw] BEM force in reduced DOFs, added to F_iner
};

struct GenWork {                 // per-call workspace views
    double2 *u;                  // [nC][Ns][3][nw]
    double2 *f6;                 // [nC][Ns][6][nw]   node loads (inertial pass, then drag passes)
    double2 *F_iner, *F_drag;    // [nC][n][nw]
    double2 *XiLast;             // [nC][n][nw]
    double *Bmat;                // [nC][Ns][9]
    double *B_drag;              // [nC][n][n]
    double2 *Z;                  // [nC][nw][n][n+1]  augmented systems; after a case's last pass its LU factors (LAPACK layout)
    int *piv;                    // [nC][nw][n]       pivot row of every elimination step of that factorisation
    int *flags;                  // [nC][4]: done, pass_not_converged, passes, nan
};

// k_gen_wave: grid (ceil(nw/128), Ns, nC), block 128
__global__ void __launch_bounds__(128) k_gen_wave(GenDev D, CasesDev Cs, GenWork W)
{
    const int i = blockIdx.x * 128 + threadIdx.x, j = blockIdx.y, c = blockIdx.z;
    if (i >= D.nw) return;
    const int nw = D.nw;
    const double w = D.w[i], k = D.k[i], h = D.depth;
    const double beta = Cs.beta_deg[c] * (CUDART_PI / 180.0);
    const double zeta0 = sea_state_zeta(Cs, c, i, nw, w, D.dw);
    const double *r = D.node_r + 3 * j, *q = D.node_frame + 9 * j, *rr = D.rr + 3 * j;
    double sb, cb, sp, cp;
    sincos(beta, &sb, &cb);
    sincos(-(k * (cb * r[0] + sb * r[1])), &sp, &cp);
    const double zr = zeta0 * cp, zi = zeta0 * sp;              // zeta at the node (helpers.py:200)
    double S_, C_, P_;
    depth_funcs(k, h, r[2], S_, C_, P_);
    // u = (w zeta C cos b, w zeta C sin b, i w zeta S); ud = i w u; pDyn = rho g zeta P (rho, g: the call's defaults 1025, 9.81)
    double2 u[3], ud[3];
    u[0] = make_double2(w * zr * C_ * cb, w * zi * C_ * cb);
    u[1] = make_double2(w * zr * C_ * sb, w * zi * C_ * sb);
    u[2] = make_double2(-w * zi * S_, w * zr * S_);
    for (int a = 0; a < 3; a++) ud[a] = make_double2(-w * u[a].y, w * u[a].x);
    const double pr = 1025.0 * 9.81 * zr * P_, pi = 1025.0 * 9.81 * zi * P_;
    double2 f[3];
    for (int a = 0; a < 3; a++) {
        double fr = 0.0, fi = 0.0;
        for (int b = 0; b < 3; b++) {
            if (D.node_Imat_w) {
                const double2 m = D.node_Imat_w[((size_t)j * 9 + 3 * a + b) * nw + i];
                fr += m.x * ud[b].x - m.y * ud[b].y; fi += m.x * ud[b].y + m.y * ud[b].x;
            } else {
                const double m = D.node_Imat[9 * j + 3 * a + b];
                fr += m * ud[b].x; fi += m * ud[b].y;
            }
        }
        f[a] = make_double2(fr + pr * D.node_a_i[j] * q[a], fi + pi * D.node_a_i[j] * q[a]);
    }
    const size_t ub = (((size_t)c * D.Ns + j) * 3) * nw + i, fb = (((size_t)c * D.Ns + j) * 6) * nw + i;
    for (int a = 0; a < 3; a++) { W.u[ub + (size_t)a * nw] = u[a]; W.f6[fb + (size_t)a * nw] = f[a]; }
    // moments rr x f (translateForce3to6DOF)
    W.f6[fb + (size_t)3 * nw] = make_double2(rr[1] * f[2].x - rr[2] * f[1].x, rr[1] * f[2].y - rr[2] * f[1].y);
    W.f6[fb + (size_t)4 * nw] = make_double2(rr[2] * f[0].x - rr[0] * f[2].x, rr[2] * f[0].y - rr[0] * f[2].y);
    W.f6[fb + (size_t)5 * nw] = make_double2(rr[0] * f[1].x - rr[1] * f[0].x, rr[0] * f[1].y - rr[1] * f[0].y);
}

// k_gen_project: F[c][dof][i] = sum_j sum_b T_j[b][dof] f6_j[b][i] over Ns loads f6 [nC][Ns][6][nw] with their 6 x n blocks
// T [Ns][6][n]: the strip nodes' Tn and node loads (BEM = false), or T0 and the BEM force of k_gen_bem (BEM = true, Ns = 1);
// plus X.F_BEM with ADD (F_iner = F_BEM + ...).  grid (ceil(nw/128), n, nC), block 128.  sec_only (the primary map)
// restricts it to the secondary trains.
template <bool BEM, bool ADD>
__global__ void __launch_bounds__(128) k_gen_project(GenDev D, GenWork W, double2 *F, int skip_done, const int *sec_only, GenFdDev X)
{
    const int i = blockIdx.x * 128 + threadIdx.x, dof = blockIdx.y, c = blockIdx.z;
    if (i >= D.nw || (skip_done && W.flags[4 * c]) || (sec_only && sec_only[c] == c)) return;
    const int nw = D.nw, n = D.n;
    double sr = 0.0, si = 0.0;
    for (int j = 0; j < (BEM ? 1 : D.Ns); j++) {
        const double *T = (BEM ? X.T0 : D.Tn) + (size_t)j * 6 * n + dof;
        const double2 *f = (BEM ? X.fb6 : W.f6) + (((size_t)c * (BEM ? 1 : D.Ns) + j) * 6) * nw + i;
#pragma unroll
        for (int b = 0; b < 6; b++) {
            const double t = T[(size_t)b * n];
            const double2 v = f[(size_t)b * nw];
            sr = fma(t, v.x, sr); si = fma(t, v.y, si);
        }
    }
    if constexpr (ADD) { const double2 a = X.F_BEM[((size_t)c * n + dof) * nw + i]; sr = a.x + sr; si = a.y + si; }
    F[((size_t)c * n + dof) * nw + i] = make_double2(sr, si);
}

// k_gen_bem: grid (ceil(nw/128), nC), block 128: BEM excitation of every case (secondary trains with their own heading and
// sea state, raft_model.py:1200-1236) in full DOFs 0-5, from the rigid solvers' bem_excitation_table
__global__ void __launch_bounds__(128) k_gen_bem(GenDev D, CasesDev Cs, GenFdDev X)
{
    const int i = blockIdx.x * 128 + threadIdx.x, c = blockIdx.y;
    if (i >= D.nw) return;
    const int nw = D.nw;
    const double beta = Cs.beta_deg[c] * (CUDART_PI / 180.0);
    double sb, cb;
    sincos(beta, &sb, &cb);
    const double zeta = sea_state_zeta(Cs, c, i, nw, D.w[i], D.dw);
    double Br[6], Bi[6];
    bem_excitation_table(X.bem_headings, X.n_bem_head, X.X_BEM, nw, X.x_ref, X.y_ref, X.hadj, i, D.k[i], beta, sb, cb, zeta, Br, Bi);
    double2 *f = X.fb6 + (size_t)c * 6 * nw + i;
#pragma unroll
    for (int a = 0; a < 6; a++) f[(size_t)a * nw] = make_double2(Br[a], Bi[a]);
}

// k_gen_add_2nd: grid (ceil(nw/128), 6, nC), block 128: the second-order force of every case and train (real amplitudes
// [nC][6][nw] of k_qtf_tiles / k_qtf_force) added to reduced rows 0-5 of F_iner, which already hold F_BEM + F_iner:
// (F_BEM + F_iner) + F_2nd (raft_model.py:1048, 1212; lumped on the first 6 DOFs, :1034)
__global__ void __launch_bounds__(128) k_gen_add_2nd(GenDev D, GenWork W, const double *F2)
{
    const int i = blockIdx.x * 128 + threadIdx.x, a = blockIdx.y, c = blockIdx.z;
    if (i >= D.nw) return;
    double2 &f = W.F_iner[((size_t)c * D.n + a) * D.nw + i];
    f.x = f.x + F2[((size_t)c * 6 + a) * D.nw + i];
}

// DOF -> position on the support of the frequency-dependent terms (-1 off it), built once per CTA in shared memory
__device__ __forceinline__ void gen_fd_map(const GenDev &D, const GenFdDev &X, int *fdpos, int tid, int nthr)
{
    for (int t = tid; t < D.n; t += nthr) fdpos[t] = -1;
    __syncthreads();
    for (int t = tid; t < X.n_fd; t += nthr) fdpos[X.fd_idx[t]] = t;
    __syncthreads();
}

// impedance entry t = a n + b at frequency i (raft_model.py:1086).  On the support: M + A_w and (B + B_w) + B_drag with the
// rigid solver's grouping (raftk_fused.cuh); elsewhere the constant-matrix expression.  FD = false (n_fd = 0) is the
// constant-matrix kernel as it was, instruction for instruction: no map, no branch
template <bool FD>
__device__ __forceinline__ double2 gen_impedance(const GenDev &D, const GenFdDev &X, const int *fdpos, const double *Bd, int t, int i, double w,
                                                 double w2)
{
    if constexpr (FD) {
        const int pa = fdpos[t / D.n], pb = fdpos[t % D.n];
        if (pa >= 0 && pb >= 0) {
            const size_t e = ((size_t)pa * X.n_fd + pb) * D.nw + i;
            const double M = D.M[t] + X.A_w[e], B = (D.B[t] + X.B_w[e]) + Bd[t];
            return make_double2(fma(-w2, M, D.C[t]), w * B);
        }
    }
    return make_double2(fma(-w2, D.M[t], D.C[t]), w * (D.B[t] + Bd[t]));
}

// k_gen_node_pass: grid (Ns, nC), block 128: RMS of the relative velocity components over w (raft_member.py:2071-2090),
// Bmat (:2092-2116), then the drag node load f6 = [Bmat u ; rr x (Bmat u)] (:2122-2124).
// TRAIN: secondary trains only, Bmat taken from their primary's last pass (calcDragExcitation(ih), raft_fowt.py:1940-1957).
template <bool TRAIN>
__global__ void __launch_bounds__(128) k_gen_node_pass(GenDev D, GenWork W, const int *primary)
{
    __shared__ double red[4][4];
    __shared__ double bm[9];
    const int j = blockIdx.x, c = blockIdx.y, tid = threadIdx.x, nw = D.nw, n = D.n;
    const double *rr = D.rr + 3 * j;
    const double2 *u = W.u + (((size_t)c * D.Ns + j) * 3) * nw;
    if constexpr (TRAIN) {
        const int p = primary[c];
        if (p == c) return;
        if (tid < 9) bm[tid] = W.Bmat[((size_t)p * D.Ns + j) * 9 + tid];
    } else {
    if (W.flags[4 * c]) return;
    const double *q = D.node_frame + 9 * j, *p1 = q + 3, *p2 = q + 6, *T = D.Tn + (size_t)j * 6 * n;
    const double2 *X = W.XiLast + (size_t)c * n * nw;
    double sq = 0.0, sp = 0.0, sp1 = 0.0, sp2 = 0.0;
    for (int i = tid; i < nw; i += 128) {
        double2 xn[6];
        for (int a = 0; a < 6; a++) {                       // Xi_nodes = node.T @ Xi (raft_fowt.py:1921)
            double sr = 0.0, si = 0.0;
            for (int b = 0; b < n; b++) { const double t = T[(size_t)a * n + b]; const double2 x = X[(size_t)b * nw + i]; sr = fma(t, x.x, sr); si = fma(t, x.y, si); }
            xn[a] = make_double2(sr, si);
        }
        // getKinematics: dr = x + theta x rr ; v = i w dr
        double2 dr[3];
        dr[0] = make_double2(xn[0].x + (-xn[5].x * rr[1] + xn[4].x * rr[2]), xn[0].y + (-xn[5].y * rr[1] + xn[4].y * rr[2]));
        dr[1] = make_double2(xn[1].x + ( xn[5].x * rr[0] - xn[3].x * rr[2]), xn[1].y + ( xn[5].y * rr[0] - xn[3].y * rr[2]));
        dr[2] = make_double2(xn[2].x + (-xn[4].x * rr[0] + xn[3].x * rr[1]), xn[2].y + (-xn[4].y * rr[0] + xn[3].y * rr[1]));
        const double w = D.w[i];
        double2 vr[3];
        for (int a = 0; a < 3; a++) { const double2 uu = u[(size_t)a * nw + i]; vr[a] = make_double2(uu.x + w * dr[a].y, uu.y - w * dr[a].x); }   // u - i w dr
        double2 aq = make_double2(0, 0), a1 = aq, a2 = aq;
        for (int a = 0; a < 3; a++) {
            aq.x += vr[a].x * q[a]; aq.y += vr[a].y * q[a]; a1.x += vr[a].x * p1[a]; a1.y += vr[a].y * p1[a]; a2.x += vr[a].x * p2[a]; a2.y += vr[a].y * p2[a];
        }
        for (int a = 0; a < 3; a++) {
            const double vqx = aq.x * q[a], vqy = aq.y * q[a], vpx = vr[a].x - vqx, vpy = vr[a].y - vqy;
            sq += vqx * vqx + vqy * vqy; sp += vpx * vpx + vpy * vpy;
            sp1 += (a1.x * p1[a]) * (a1.x * p1[a]) + (a1.y * p1[a]) * (a1.y * p1[a]);
            sp2 += (a2.x * p2[a]) * (a2.x * p2[a]) + (a2.y * p2[a]) * (a2.y * p2[a]);
        }
    }
    double v4[4] = { sq, sp, sp1, sp2 };
    for (int t = 0; t < 4; t++) {
        for (int o = 16; o >= 1; o >>= 1) v4[t] += __shfl_xor_sync(0xffffffffu, v4[t], o);
        if ((tid & 31) == 0) red[tid >> 5][t] = v4[t];
    }
    __syncthreads();
    if (tid == 0) {
        double s[4];
        for (int t = 0; t < 4; t++) s[t] = ((red[0][t] + red[1][t]) + red[2][t]) + red[3][t];
        const double vq = sqrt(0.5 * s[0]);
        const double v1 = D.node_circ[j] ? sqrt(0.5 * s[1]) : sqrt(0.5 * s[2]);
        const double v2 = D.node_circ[j] ? v1 : sqrt(0.5 * s[3]);
        const double cc = sqrt(8.0 / CUDART_PI) * 0.5 * D.rho;
        const double *cd = D.node_cd + 4 * j;
        const double Bq = cc * vq * cd[0], Bp1 = cc * v1 * cd[1], Bp2 = cc * v2 * cd[2], Be = cc * vq * cd[3];
        for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) {
            const double m = (Bq * (q[a] * q[b]) + Bp1 * (p1[a] * p1[b]) + Bp2 * (p2[a] * p2[b])) + Be * (q[a] * q[b]);
            bm[3 * a + b] = m;
            W.Bmat[((size_t)c * D.Ns + j) * 9 + 3 * a + b] = m;
        }
    }
    }
    __syncthreads();
    double2 *f6 = W.f6 + (((size_t)c * D.Ns + j) * 6) * nw;
    for (int i = tid; i < nw; i += 128) {
        double2 f[3];
        for (int a = 0; a < 3; a++) {
            double fr = 0.0, fi = 0.0;
            for (int b = 0; b < 3; b++) { const double2 uu = u[(size_t)b * nw + i]; fr += bm[3 * a + b] * uu.x; fi += bm[3 * a + b] * uu.y; }
            f[a] = make_double2(fr, fi);
            f6[(size_t)a * nw + i] = f[a];
        }
        f6[(size_t)3 * nw + i] = make_double2(rr[1] * f[2].x - rr[2] * f[1].x, rr[1] * f[2].y - rr[2] * f[1].y);
        f6[(size_t)4 * nw + i] = make_double2(rr[2] * f[0].x - rr[0] * f[2].x, rr[2] * f[0].y - rr[0] * f[2].y);
        f6[(size_t)5 * nw + i] = make_double2(rr[0] * f[1].x - rr[1] * f[0].x, rr[0] * f[1].y - rr[1] * f[0].y);
    }
}

// translateMatrix3to6DOF(Bmat, rr) (helpers.py:537-560): [[B, B H], [(B H)^T, H B H^T]] with H = getH(rr)
__host__ __device__ __forceinline__ void gen_B6(const double *Bm, const double *r, double (&B6)[6][6])
{
    const double H[3][3] = { { 0, r[2], -r[1] }, { -r[2], 0, r[0] }, { r[1], -r[0], 0 } };
    double BH[3][3], HB[3][3];
    for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) {
        double s = 0, t = 0;
        for (int l = 0; l < 3; l++) { s += Bm[3 * a + l] * H[l][b]; t += H[a][l] * Bm[3 * l + b]; }
        BH[a][b] = s; HB[a][b] = t;
    }
    for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) {
        double s = 0;
        for (int l = 0; l < 3; l++) s += HB[a][l] * H[b][l];
        B6[a][b] = Bm[3 * a + b]; B6[a][3 + b] = BH[a][b]; B6[3 + a][b] = BH[b][a]; B6[3 + a][3 + b] = s;
    }
}

// k_gen_bdrag: B_drag[c][r][cc] = sum_j sum_{a,l} Tn_j[a][r] B6_j[a][l] Tn_j[l][cc].  grid (n, nC), block 128
__global__ void __launch_bounds__(128) k_gen_bdrag(GenDev D, GenWork W)
{
    __shared__ double tb[6];
    const int r = blockIdx.x, c = blockIdx.y, tid = threadIdx.x, n = D.n;
    if (W.flags[4 * c]) return;
    double acc[2] = { 0.0, 0.0 };                            // columns tid and tid + 128 (n <= 256)
    for (int j = 0; j < D.Ns; j++) {
        const double *T = D.Tn + (size_t)j * 6 * n;
        if (tid < 6) {                                       // tb[l] = sum_a Tn[a][r] B6[a][l]
            double B6[6][6];
            gen_B6(W.Bmat + ((size_t)c * D.Ns + j) * 9, D.rr + 3 * j, B6);
            double s = 0.0;
            for (int a = 0; a < 6; a++) s += T[(size_t)a * n + r] * B6[a][tid];
            tb[tid] = s;
        }
        __syncthreads();
        for (int e = 0; e < 2; e++) {
            const int cc = tid + 128 * e;
            if (cc < n) { double s = 0.0; for (int l = 0; l < 6; l++) s += tb[l] * T[(size_t)l * n + cc]; acc[e] += s; }
        }
        __syncthreads();
    }
    for (int e = 0; e < 2; e++) { const int cc = tid + 128 * e; if (cc < n) W.B_drag[((size_t)c * n + r) * n + cc] = acc[e]; }
}

// k_gen_solve: grid (nw, nC), block 256.  Augmented system [Z | F] (n x (n+1)) in global memory (L2-resident), right-looking
// LU with partial pivoting on |re| + |im| (LAPACK izamax), back substitution; writes Xi and the convergence verdict.
template <bool FD>
__global__ void __launch_bounds__(256) k_gen_solve(GenDev D, GenWork W, double2 *Xi, double tol, GenFdDev X)
{
    __shared__ double pv[8];
    __shared__ int pi_[8];
    __shared__ double2 piv;
    __shared__ int prow, bad;
    __shared__ int fdpos[FD ? 256 : 1];
    const int i = blockIdx.x, c = blockIdx.y, tid = threadIdx.x, n = D.n, nw = D.nw, nc = n + 1;
    if (W.flags[4 * c]) return;
    double2 *A = W.Z + ((size_t)c * nw + i) * (size_t)n * nc;
    const double w = D.w[i], w2 = w * w;
    const double *Bd = W.B_drag + (size_t)c * n * n;
    if constexpr (FD) gen_fd_map(D, X, fdpos, tid, 256);
    for (int t = tid; t < n * n; t += 256) {
        const int a = t / n, b = t % n;
        A[(size_t)a * nc + b] = gen_impedance<FD>(D, X, fdpos, Bd, t, i, w, w2);
    }
    for (int a = tid; a < n; a += 256) {
        const double2 f1 = W.F_iner[((size_t)c * n + a) * nw + i], f2 = W.F_drag[((size_t)c * n + a) * nw + i];
        A[(size_t)a * nc + n] = make_double2(f1.x + f2.x, f1.y + f2.y);
    }
    if (tid == 0) bad = 0;
    __syncthreads();
    for (int k = 0; k < n; k++) {
        // pivot search in column k, rows k..n-1 (first maximum wins, like izamax)
        double best = -1.0; int bi = k;
        for (int r = k + tid; r < n; r += 256) { const double2 v = A[(size_t)r * nc + k]; const double m = fabs(v.x) + fabs(v.y); if (m > best) { best = m; bi = r; } }
        for (int o = 16; o >= 1; o >>= 1) {
            const double ob = __shfl_xor_sync(0xffffffffu, best, o); const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
        }
        if ((tid & 31) == 0) { pv[tid >> 5] = best; pi_[tid >> 5] = bi; }
        __syncthreads();
        if (tid == 0) {
            double b0 = pv[0]; int r0 = pi_[0];
            for (int t = 1; t < 8; t++) if (pv[t] > b0 || (pv[t] == b0 && pi_[t] < r0)) { b0 = pv[t]; r0 = pi_[t]; }
            prow = r0;
            W.piv[((size_t)c * nw + i) * n + k] = r0;
            if (!(b0 > 0.0)) bad = 1;
        }
        __syncthreads();
        const int p = prow;
        // whole rows, so that L ends in LAPACK's layout (k_gen_train_solve reuses these factors)
        if (p != k) for (int b = tid; b < nc; b += 256) { const double2 t1 = A[(size_t)k * nc + b]; A[(size_t)k * nc + b] = A[(size_t)p * nc + b]; A[(size_t)p * nc + b] = t1; }
        __syncthreads();
        if (tid == 0) { const double2 a = A[(size_t)k * nc + k]; const double dd = a.x * a.x + a.y * a.y; piv = make_double2(a.x / dd, -a.y / dd); }
        __syncthreads();
        const double2 ip = piv;
        // multipliers l_r = a_rk / a_kk, then trailing update a_rb -= l_r a_kb (b = k+1 .. n incl. the right-hand side)
        for (int r = k + 1 + tid; r < n; r += 256) { const double2 a = A[(size_t)r * nc + k]; A[(size_t)r * nc + k] = make_double2(a.x * ip.x - a.y * ip.y, a.x * ip.y + a.y * ip.x); }
        __syncthreads();
        const int rows = n - k - 1, cols = nc - k - 1;
        for (int t = tid; t < rows * cols; t += 256) {
            const int r = k + 1 + t / cols, b = k + 1 + t % cols;
            const double2 l = A[(size_t)r * nc + k], ak = A[(size_t)k * nc + b];
            double2 v = A[(size_t)r * nc + b];
            v.x -= l.x * ak.x - l.y * ak.y; v.y -= l.x * ak.y + l.y * ak.x;
            A[(size_t)r * nc + b] = v;
        }
        __syncthreads();
    }
    // back substitution on the last column
    for (int k = n - 1; k >= 0; k--) {
        if (tid == 0) {
            const double2 a = A[(size_t)k * nc + k], b = A[(size_t)k * nc + n];
            const double dd = a.x * a.x + a.y * a.y;
            A[(size_t)k * nc + n] = make_double2((b.x * a.x + b.y * a.y) / dd, (b.y * a.x - b.x * a.y) / dd);
        }
        __syncthreads();
        const double2 x = A[(size_t)k * nc + n];
        for (int r = tid; r < k; r += 256) {
            const double2 a = A[(size_t)r * nc + k];
            double2 b = A[(size_t)r * nc + n];
            b.x -= a.x * x.x - a.y * x.y; b.y -= a.x * x.y + a.y * x.x;
            A[(size_t)r * nc + n] = b;
        }
        __syncthreads();
    }
    int notconv = 0, nan = 0;
    for (int a = tid; a < n; a += 256) {
        const double2 x = A[(size_t)a * nc + n], l = W.XiLast[((size_t)c * n + a) * nw + i];
        Xi[((size_t)c * n + a) * nw + i] = x;
        if (isnan(x.x) || isnan(x.y)) nan = 1;
        const double dx = x.x - l.x, dy = x.y - l.y;
        if (!(sqrt(dx * dx + dy * dy) / (sqrt(x.x * x.x + x.y * x.y) + tol) < tol)) notconv = 1;     // raft_model.py:1101-1102
    }
    if (notconv) atomicOr(&W.flags[4 * c + 1], 1);
    if (nan || bad) atomicOr(&W.flags[4 * c + 3], 1);
}

// k_gen_solve_blocked: grid (nw, nC), block 256.  Same system, same pivot rule and the same elimination order as
// k_gen_solve, organised as a blocked right-looking LU (LAPACK zgetrf's structure) so that the work is done on chip:
//   per block of GB columns:  panel (rows kb.., GB columns) factored in SHARED memory with partial pivoting; its row swaps
//   applied to the rest of the rows; the GB x (rest) row block solved against the unit-lower panel head in shared memory;
//   trailing update A22 -= L21 U12 with a 4 x 2 register tile per thread -- every A22 element is loaded once, receives its
//   GB rank-1 contributions IN ELIMINATION ORDER (k ascending, the rounding sequence of the unblocked algorithm) and is
//   stored once.  Traffic to the L2-resident matrix drops by GB (16) against the unblocked kernel's one pass per column;
//   9 Mflop per 150 x 150 system then run from registers and shared memory.
#define GB 8
#define GT 128
template <bool FD>
__global__ void __launch_bounds__(GT, 4) k_gen_solve_blocked(GenDev D, GenWork W, double2 *Xi, double tol, GenFdDev X)
{
    extern __shared__ __align__(16) double smem_raw[];
    __shared__ double pv[GT / 32];
    __shared__ int pi_[GT / 32];
    __shared__ int bad;
    __shared__ int pivrow[GB];
    __shared__ int fdpos[FD ? 256 : 1];
    const int i = blockIdx.x, c = blockIdx.y, tid = threadIdx.x, n = D.n, nw = D.nw, nc = n + 1;
    if (W.flags[4 * c]) return;
    double2 *P = reinterpret_cast<double2 *>(smem_raw);          // panel  [n][GB]   (rows kb.. stored from 0)
    double2 *U = P + (size_t)n * GB;                             // row block [GB][nc]
    double2 *A = W.Z + ((size_t)c * nw + i) * (size_t)n * nc;
    const double w = D.w[i], w2 = w * w;
    const double *Bd = W.B_drag + (size_t)c * n * n;
    if constexpr (FD) gen_fd_map(D, X, fdpos, tid, GT);
    for (int t = tid; t < n * n; t += GT) {
        const int a = t / n, b = t % n;
        A[(size_t)a * nc + b] = gen_impedance<FD>(D, X, fdpos, Bd, t, i, w, w2);
    }
    for (int a = tid; a < n; a += GT) {
        const double2 f1 = W.F_iner[((size_t)c * n + a) * nw + i], f2 = W.F_drag[((size_t)c * n + a) * nw + i];
        A[(size_t)a * nc + n] = make_double2(f1.x + f2.x, f1.y + f2.y);
    }
    if (tid == 0) bad = 0;
    __syncthreads();
    for (int kb = 0; kb < n; kb += GB) {
        const int nb = min(GB, n - kb), m = n - kb;
        // ---- 1. panel into shared memory ------------------------------------------------------------------------
        for (int t = tid; t < m * nb; t += GT) { const int r = t / nb, j = t % nb; P[r * GB + j] = A[(size_t)(kb + r) * nc + kb + j]; }
        __syncthreads();
        // ---- 2. unblocked LU of the panel (pivot on |re| + |im|, first maximum wins, like izamax) ---------------------
        for (int j = 0; j < nb; j++) {
            double best = -1.0; int bi = j;
            for (int r = j + tid; r < m; r += GT) { const double2 v = P[r * GB + j]; const double mg = fabs(v.x) + fabs(v.y); if (mg > best) { best = mg; bi = r; } }
            for (int o = 16; o >= 1; o >>= 1) {
                const double ob = __shfl_xor_sync(0xffffffffu, best, o); const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
            }
            if ((tid & 31) == 0) { pv[tid >> 5] = best; pi_[tid >> 5] = bi; }
            __syncthreads();
            // every thread finishes the reduction itself (same winner everywhere) and reads the pivot before rows move
            double b0 = pv[0]; int p = pi_[0];
#pragma unroll
            for (int t = 1; t < GT / 32; t++) if (pv[t] > b0 || (pv[t] == b0 && pi_[t] < p)) { b0 = pv[t]; p = pi_[t]; }
            const double2 a = P[p * GB + j];
            const double dd = a.x * a.x + a.y * a.y;
            const double2 ip = make_double2(a.x / dd, -a.y / dd);
            if (tid == 0) { pivrow[j] = p; W.piv[((size_t)c * nw + i) * n + kb + j] = kb + p; if (!(b0 > 0.0)) bad = 1; }
            __syncthreads();
            if (p != j && tid < nb) { const double2 t1 = P[j * GB + tid]; P[j * GB + tid] = P[p * GB + tid]; P[p * GB + tid] = t1; }
            __syncthreads();
            // multipliers and the update of the panel's remaining columns in one sweep: thread per row
            const int cols = nb - j - 1;
            for (int r = j + 1 + tid; r < m; r += GT) {
                const double2 v = P[r * GB + j];
                const double2 l = make_double2(v.x * ip.x - v.y * ip.y, v.x * ip.y + v.y * ip.x);
                P[r * GB + j] = l;
                for (int b = 0; b < cols; b++) {
                    const double2 ak = P[j * GB + j + 1 + b];
                    double2 x = P[r * GB + j + 1 + b];
                    x.x -= l.x * ak.x - l.y * ak.y; x.y -= l.x * ak.y + l.y * ak.x;
                    P[r * GB + j + 1 + b] = x;
                }
            }
            __syncthreads();
        }
        // ---- 3. panel back to the matrix; its row swaps applied, in order, to the columns outside the panel -------
        for (int t = tid; t < m * nb; t += GT) { const int r = t / nb, j = t % nb; A[(size_t)(kb + r) * nc + kb + j] = P[r * GB + j]; }
        for (int col = tid; col < nc; col += GT) {
            if (col >= kb && col < kb + nb) continue;
            for (int j = 0; j < nb; j++) {
                const int p = pivrow[j];
                if (p != j) { const double2 t1 = A[(size_t)(kb + j) * nc + col]; A[(size_t)(kb + j) * nc + col] = A[(size_t)(kb + p) * nc + col]; A[(size_t)(kb + p) * nc + col] = t1; }
            }
        }
        __syncthreads();
        // ---- 4. row block U12 = L11^-1 A12 (unit lower triangular solve per column, elimination order) -----------------
        const int c0 = kb + nb, ncol = nc - c0;
        for (int t = tid; t < nb * ncol; t += GT) { const int j = t / ncol, b = t % ncol; U[j * nc + b] = A[(size_t)(kb + j) * nc + c0 + b]; }
        __syncthreads();
        for (int b = tid; b < ncol; b += GT) {
            for (int j = 0; j < nb; j++) {
                const double2 uj = U[j * nc + b];
                for (int r = j + 1; r < nb; r++) {
                    const double2 l = P[r * GB + j];
                    double2 v = U[r * nc + b];
                    v.x -= l.x * uj.x - l.y * uj.y; v.y -= l.x * uj.y + l.y * uj.x;
                    U[r * nc + b] = v;
                }
            }
        }
        __syncthreads();
        for (int t = tid; t < nb * ncol; t += GT) { const int j = t / ncol, b = t % ncol; A[(size_t)(kb + j) * nc + c0 + b] = U[j * nc + b]; }
        // ---- 5. trailing update A22 -= L21 U12: 4 x 2 register tile per thread, contributions in elimination order --
        const int m2 = m - nb;
        const int tr = (m2 + 3) / 4, tc = (ncol + 1) / 2;
        for (int t = tid; t < tr * tc; t += GT) {
            const int r0 = 4 * (t / tc), b0 = 2 * (t % tc);
            double2 acc[4][2];
#pragma unroll
            for (int x = 0; x < 4; x++)
#pragma unroll
                for (int y = 0; y < 2; y++)
                    acc[x][y] = (r0 + x < m2 && b0 + y < ncol) ? A[(size_t)(c0 + r0 + x) * nc + c0 + b0 + y] : make_double2(0.0, 0.0);
            for (int j = 0; j < nb; j++) {
                double2 l[4], u[2];
#pragma unroll
                for (int x = 0; x < 4; x++) l[x] = P[min(nb + r0 + x, m - 1) * GB + j];
#pragma unroll
                for (int y = 0; y < 2; y++) u[y] = U[j * nc + min(b0 + y, ncol - 1)];
#pragma unroll
                for (int x = 0; x < 4; x++)
#pragma unroll
                    for (int y = 0; y < 2; y++) {
                        acc[x][y].x -= l[x].x * u[y].x - l[x].y * u[y].y;
                        acc[x][y].y -= l[x].x * u[y].y + l[x].y * u[y].x;
                    }
            }
#pragma unroll
            for (int x = 0; x < 4; x++)
#pragma unroll
                for (int y = 0; y < 2; y++)
                    if (r0 + x < m2 && b0 + y < ncol) A[(size_t)(c0 + r0 + x) * nc + c0 + b0 + y] = acc[x][y];
        }
        __syncthreads();
    }
    // back substitution on the last column
    for (int k = n - 1; k >= 0; k--) {
        if (tid == 0) {
            const double2 a = A[(size_t)k * nc + k], b = A[(size_t)k * nc + n];
            const double dd = a.x * a.x + a.y * a.y;
            A[(size_t)k * nc + n] = make_double2((b.x * a.x + b.y * a.y) / dd, (b.y * a.x - b.x * a.y) / dd);
        }
        __syncthreads();
        const double2 x = A[(size_t)k * nc + n];
        for (int r = tid; r < k; r += GT) {
            const double2 a = A[(size_t)r * nc + k];
            double2 b = A[(size_t)r * nc + n];
            b.x -= a.x * x.x - a.y * x.y; b.y -= a.x * x.y + a.y * x.x;
            A[(size_t)r * nc + n] = b;
        }
        __syncthreads();
    }
    int notconv = 0, nan = 0;
    for (int a = tid; a < n; a += GT) {
        const double2 x = A[(size_t)a * nc + n], l = W.XiLast[((size_t)c * n + a) * nw + i];
        Xi[((size_t)c * n + a) * nw + i] = x;
        if (isnan(x.x) || isnan(x.y)) nan = 1;
        const double dx = x.x - l.x, dy = x.y - l.y;
        if (!(sqrt(dx * dx + dy * dy) / (sqrt(x.x * x.x + x.y * x.y) + tol) < tol)) notconv = 1;     // raft_model.py:1101-1102
    }
    if (notconv) atomicOr(&W.flags[4 * c + 1], 1);
    if (nan || bad) atomicOr(&W.flags[4 * c + 3], 1);
}

// k_gen_init: grid (nC), block 256: XiLast = XiStart (raft_model.py:999), flags = 0; secondary trains start done
__global__ void __launch_bounds__(256) k_gen_init(GenDev D, GenWork W, double xi_start, const int *primary)
{
    const int c = blockIdx.x, tid = threadIdx.x;
    const size_t tot = (size_t)D.n * D.nw;
    double2 *L = W.XiLast + (size_t)c * tot;
    for (size_t t = tid; t < tot; t += 256) L[t] = make_double2(xi_start, 0.0);
    if (tid < 4) W.flags[4 * c + tid] = (tid == 0 && primary && primary[c] != c) ? 1 : 0;
}

// k_gen_train_solve: grid (nw, nC), block 128, secondary trains only: Xi = Z_p^-1 (F_iner + F_drag) with the LU factors of the
// primary's last pass (L unit lower, U upper, row interchanges piv applied in elimination order; raft_model.py:1200-1236)
__global__ void __launch_bounds__(128) k_gen_train_solve(GenDev D, GenWork W, const int *primary, double2 *Xi)
{
    __shared__ double2 b[256];
    const int i = blockIdx.x, c = blockIdx.y, tid = threadIdx.x, n = D.n, nw = D.nw, nc = n + 1;
    const int p = primary[c];
    if (p == c) return;
    const double2 *A = W.Z + ((size_t)p * nw + i) * (size_t)n * nc;
    const int *pv = W.piv + ((size_t)p * nw + i) * n;
    for (int a = tid; a < n; a += 128) {
        const double2 f1 = W.F_iner[((size_t)c * n + a) * nw + i], f2 = W.F_drag[((size_t)c * n + a) * nw + i];
        b[a] = make_double2(f1.x + f2.x, f1.y + f2.y);
    }
    __syncthreads();
    if (tid == 0)
        for (int k = 0; k < n; k++) { const int q = pv[k]; if (q != k) { const double2 t = b[k]; b[k] = b[q]; b[q] = t; } }
    __syncthreads();
    for (int k = 0; k < n - 1; k++) {                           // L y = P b
        const double2 x = b[k];
        for (int r = k + 1 + tid; r < n; r += 128) {
            const double2 l = A[(size_t)r * nc + k];
            double2 v = b[r];
            v.x -= l.x * x.x - l.y * x.y; v.y -= l.x * x.y + l.y * x.x;
            b[r] = v;
        }
        __syncthreads();
    }
    for (int k = n - 1; k >= 0; k--) {                          // U x = y, as the back substitution of k_gen_solve*
        if (tid == 0) {
            const double2 a = A[(size_t)k * nc + k], v = b[k];
            const double dd = a.x * a.x + a.y * a.y;
            b[k] = make_double2((v.x * a.x + v.y * a.y) / dd, (v.y * a.x - v.x * a.y) / dd);
        }
        __syncthreads();
        const double2 x = b[k];
        for (int r = tid; r < k; r += 128) {
            const double2 a = A[(size_t)r * nc + k];
            double2 v = b[r];
            v.x -= a.x * x.x - a.y * x.y; v.y -= a.x * x.y + a.y * x.x;
            b[r] = v;
        }
        __syncthreads();
    }
    int nan = 0;
    for (int a = tid; a < n; a += 128) {
        const double2 x = b[a];
        Xi[((size_t)c * n + a) * nw + i] = x;
        if (isnan(x.x) || isnan(x.y)) nan = 1;
    }
    if (nan) atomicOr(&W.flags[4 * c + 3], 1);
}

// k_gen_relax: grid (nC), block 256: close the pass (raft_model.py:1098-1133)
__global__ void __launch_bounds__(256) k_gen_relax(GenDev D, GenWork W, const double2 *Xi)
{
    __shared__ int st[2];
    const int c = blockIdx.x, tid = threadIdx.x;
    if (W.flags[4 * c]) return;
    if (tid == 0) { st[0] = W.flags[4 * c + 1]; st[1] = W.flags[4 * c + 3]; }
    __syncthreads();
    const int notconv = st[0], nan = st[1];
    if (!nan && notconv) {
        const size_t tot = (size_t)D.n * D.nw;
        double2 *L = W.XiLast + (size_t)c * tot;
        const double2 *X = Xi + (size_t)c * tot;
        for (size_t t = tid; t < tot; t += 256) L[t] = make_double2(0.2 * L[t].x + 0.8 * X[t].x, 0.2 * L[t].y + 0.8 * X[t].y);
    }
    __syncthreads();
    if (tid == 0) {
        W.flags[4 * c + 2] += 1;                              // passes
        if (nan || !notconv) W.flags[4 * c] = nan ? 2 : 1;   // done: 1 converged, 2 NaN
        W.flags[4 * c + 1] = 0;
    }
}

// status rows for the caller: passes, converged, flags (RAFTK_FLAG_NAN), 0; a secondary train: 0, 1, flags, primary + 1
__global__ void __launch_bounds__(128) k_gen_status(int nC, const int *flags, const int *primary, int *status)
{
    const int c = blockIdx.x * 128 + threadIdx.x;
    if (c >= nC) return;
    const int p = primary ? primary[c] : c;
    status[4 * c + 0] = flags[4 * c + 2];
    status[4 * c + 1] = flags[4 * c] == 1 ? 1 : 0;
    status[4 * c + 2] = (flags[4 * c] == 2 || flags[4 * c + 3]) ? RAFTK_FLAG_NAN : 0;
    status[4 * c + 3] = p != c ? p + 1 : 0;
}
