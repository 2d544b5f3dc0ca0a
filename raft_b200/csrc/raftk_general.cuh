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
//   k_gen_solve_blocked (case, w)     Z = -w^2 M + i w (B + B_drag) + C, dense complex LU with partial pivoting, Xi;
//                                     on the support of the frequency-dependent terms M + A_w(w) and B + B_w(w) (gen_impedance),
//                                     plus the case's operating point there when the case table carries them (OP)
//   k_gen_relax     (case)            convergence bookkeeping, XiLast = 0.2 XiLast + 0.8 Xi
// Wave trains (cases.primary): a secondary train takes no part in the loop (done at init); after it
//   k_gen_node_pass<true>   (case, node)   drag node load from the PRIMARY's last Bmat and the train's own u
//   k_gen_project                          F_drag of the secondaries
//   k_gen_train_solve (case, w)            Xi = Z_p^-1 (F_iner + F_drag) from the primary's LU factors left in W.Z and W.piv:
//                                          row interchanges, unit-lower and upper triangular solves, O(n^2) per system
#pragma once

struct GenDev {
    int n, nw, Ns;               // Ns: node rows per unit in the workspace (a design batch: its largest design's count)
    int u0, nCt;                 // unit u of a launch is unit u0 + u of the call = design d * nCt + case c (gen_unit)
    const int *node_off;         // [nD+1] CSR node offsets of a design batch, or NULL: one design of Ns nodes
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
    const double *M, *B, *C;     // [nD][n][n]
    double rho;
};

// unit u of a launch -> its design d, case c (index into the whole case table), first node j0 and node count Ns.  Node-indexed
// grids run over the largest count of the chunk; blocks past their design's count return.
struct GenUnit { int d, c, j0, Ns; };
__device__ __forceinline__ GenUnit gen_unit(const GenDev &D, int u)
{
    GenUnit U;
    const int t = D.u0 + u;
    U.d = t / D.nCt; U.c = t - U.d * D.nCt;
    U.j0 = D.node_off ? D.node_off[U.d] : 0;
    U.Ns = D.node_off ? D.node_off[U.d + 1] - U.j0 : D.Ns;
    return U;
}

// frequency-dependent terms (raftk_general_fd), a parameter of their own so that every kernel of the constant-matrix solve
// keeps its parameter layout; n_fd = 0 / n_bem_head = 0 without them.  Tables carry a leading design axis [nD].
struct GenFdDev {
    int n_fd, n_bem_head;
    const int *fd_idx;           // [nD][n_fd] strictly increasing reduced DOFs
    const double *A_w, *B_w;     // [nD][n_fd][n_fd][nw]
    const double *bem_headings;  // [nD][n_bem_head] deg
    const double2 *X_BEM;        // [nD][n_bem_head][6][nw] heading-relative
    const double *T0;            // [nD][6][n] rows 0..5 of fowt.T
    double x_ref, y_ref, hadj;
    const double *x_ref_d, *y_ref_d, *hadj_d;   // [nD] per design, or NULL: x_ref, y_ref, hadj for every design
    double2 *fb6;                // [nC][6][nw] workspace: BEM force in full DOFs 0-5
    const double2 *F_BEM;        // [nC][n][nw] BEM force in reduced DOFs, added to F_iner
};

// per-case operating points (raftk_cases.op) on the support of fd_idx: GenFdDev plus the case table's op column and the tables
// [nD or 1][n_op][n_fd][n_fd][nw].  Only the OP instantiations of k_gen_solve_blocked take it, so that every other kernel keeps its
// parameter layout.
struct GenFdOpDev : GenFdDev {
    const int *op;               // [nC of the whole table] operating point of every case
    int n_op, op_shared;         // op_shared: one set of tables for every design
    const double *op_A_w, *op_B_w;
};
template <bool OP> using GenFdArg = typename std::conditional<OP, GenFdOpDev, GenFdDev>::type;

struct GenWork {                 // per-call workspace views
    double2 *u;                  // [nC][Ns][3][nw]
    double2 *f6;                 // [nC][Ns][6][nw]   node loads (inertial pass, then drag passes)
    double2 *F_iner, *F_drag;    // [nC][n][nw]
    double2 *XiLast;             // [nC][n][nw]
    double *Bmat;                // [nC][Ns][9]
    double *B_drag;              // [nC][n][n]
    double2 *Z;                  // [nC][nw][n][n+1]  augmented systems; after a case's last pass its LU factors (lu_blocked's
                                 //                   layout: the columns of each panel of GB keep the rows they had then)
    int *piv;                    // [nC][nw][n]       pivot row (of the whole system) of every elimination step of that factorisation
    int *flags;                  // [nC][4]: done, pass_not_converged, passes, RAFTK_FLAG_NAN | RAFTK_FLAG_SINGULAR (a zero pivot)
};

// k_gen_wave: grid (ceil(nw/128), Ns, nC), block 128
__global__ void __launch_bounds__(128) k_gen_wave(GenDev D, CasesDev Cs, GenWork W)
{
    const int i = blockIdx.x * 128 + threadIdx.x, j = blockIdx.y, un = blockIdx.z;
    if (i >= D.nw) return;
    const GenUnit U = gen_unit(D, un);
    if (j >= U.Ns) return;
    const int nw = D.nw, c = U.c, jn = U.j0 + j;
    const double w = D.w[i], k = D.k[i], h = D.depth;
    const double beta = Cs.beta_deg[c] * (CUDART_PI / 180.0);
    const double zeta0 = sea_state_zeta(Cs, c, i, nw, w, D.dw);
    const double *r = D.node_r + 3 * jn, *q = D.node_frame + 9 * jn, *rr = D.rr + 3 * jn;
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
                const double2 m = D.node_Imat_w[((size_t)jn * 9 + 3 * a + b) * nw + i];
                fr += m.x * ud[b].x - m.y * ud[b].y; fi += m.x * ud[b].y + m.y * ud[b].x;
            } else {
                const double m = D.node_Imat[9 * jn + 3 * a + b];
                fr += m * ud[b].x; fi += m * ud[b].y;
            }
        }
        f[a] = make_double2(fr + pr * D.node_a_i[jn] * q[a], fi + pi * D.node_a_i[jn] * q[a]);
    }
    const size_t ub = (((size_t)un * D.Ns + j) * 3) * nw + i, fb = (((size_t)un * D.Ns + j) * 6) * nw + i;
    for (int a = 0; a < 3; a++) { W.u[ub + (size_t)a * nw] = u[a]; W.f6[fb + (size_t)a * nw] = f[a]; }
    // moments rr x f (translateForce3to6DOF)
    W.f6[fb + (size_t)3 * nw] = make_double2(rr[1] * f[2].x - rr[2] * f[1].x, rr[1] * f[2].y - rr[2] * f[1].y);
    W.f6[fb + (size_t)4 * nw] = make_double2(rr[2] * f[0].x - rr[0] * f[2].x, rr[2] * f[0].y - rr[0] * f[2].y);
    W.f6[fb + (size_t)5 * nw] = make_double2(rr[0] * f[1].x - rr[1] * f[0].x, rr[0] * f[1].y - rr[1] * f[0].y);
}

// k_gen_project: F[c][dof][i] = sum_j sum_b T_j[b][dof] f6_j[b][i] over Ns loads f6 [nC][Ns][6][nw] with their 6 x n blocks
// T [Ns][6][n]: the strip nodes' Tn and node loads (BEM = false), or T0 and the BEM force of k_gen_bem (BEM = true, Ns = 1);
// plus X.F_BEM with ADD (F_iner = F_BEM + ...).  grid (ceil(nw/128), n, units), block 128.  sec_only (the primary map)
// restricts it to the secondary trains.
template <bool BEM, bool ADD>
__global__ void __launch_bounds__(128) k_gen_project(GenDev D, GenWork W, double2 *F, int skip_done, const int *sec_only, GenFdDev X)
{
    const int i = blockIdx.x * 128 + threadIdx.x, dof = blockIdx.y, c = blockIdx.z;
    if (i >= D.nw || (skip_done && W.flags[4 * c]) || (sec_only && sec_only[c] == c)) return;
    const int nw = D.nw, n = D.n;
    const GenUnit U = gen_unit(D, c);
    double sr = 0.0, si = 0.0;
    for (int j = 0; j < (BEM ? 1 : U.Ns); j++) {
        const double *T = (BEM ? X.T0 + (size_t)U.d * 6 * n : D.Tn + (size_t)(U.j0 + j) * 6 * n) + dof;
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

// k_gen_bem: grid (ceil(nw/128), units), block 128: BEM excitation of every case (secondary trains with their own heading and
// sea state, raft_model.py:1200-1236) in full DOFs 0-5, from the rigid solvers' bem_excitation_table
__global__ void __launch_bounds__(128) k_gen_bem(GenDev D, CasesDev Cs, GenFdDev X)
{
    const int i = blockIdx.x * 128 + threadIdx.x, u = blockIdx.y;
    if (i >= D.nw) return;
    const int nw = D.nw;
    const GenUnit U = gen_unit(D, u);
    const int c = U.c, d = U.d, nh = X.n_bem_head;
    const double beta = Cs.beta_deg[c] * (CUDART_PI / 180.0);
    double sb, cb;
    sincos(beta, &sb, &cb);
    const double zeta = sea_state_zeta(Cs, c, i, nw, D.w[i], D.dw);
    double Br[6], Bi[6];
    bem_excitation_table(X.bem_headings + (size_t)d * nh, nh, X.X_BEM + (size_t)d * nh * 6 * nw, nw, X.x_ref_d ? X.x_ref_d[d] : X.x_ref,
                         X.y_ref_d ? X.y_ref_d[d] : X.y_ref, X.hadj_d ? X.hadj_d[d] : X.hadj, i, D.k[i], beta, sb, cb, zeta, Br, Bi);
    double2 *f = X.fb6 + (size_t)u * 6 * nw + i;
#pragma unroll
    for (int a = 0; a < 6; a++) f[(size_t)a * nw] = make_double2(Br[a], Bi[a]);
}

// k_gen_add_2nd: grid (ceil(nw/128), 6, units), block 128: the second-order force of every case and train (real amplitudes
// [nC][6][nw] of k_qtf_tiles / k_qtf_force) added to reduced rows 0-5 of F_iner, which already hold F_BEM + F_iner:
// (F_BEM + F_iner) + F_2nd (raft_model.py:1048, 1212; lumped on the first 6 DOFs, :1034)
__global__ void __launch_bounds__(128) k_gen_add_2nd(GenDev D, GenWork W, const double *F2)
{
    const int i = blockIdx.x * 128 + threadIdx.x, a = blockIdx.y, c = blockIdx.z;
    if (i >= D.nw) return;
    double2 &f = W.F_iner[((size_t)c * D.n + a) * D.nw + i];
    f.x = f.x + F2[((size_t)c * 6 + a) * D.nw + i];
}

// DOF -> position on the support of design d's frequency-dependent terms (-1 off it), built once per CTA in shared memory
__device__ __forceinline__ void gen_fd_map(const GenDev &D, const GenFdDev &X, int d, int *fdpos, int tid, int nthr)
{
    const int *idx = X.fd_idx + (size_t)d * X.n_fd;
    for (int t = tid; t < D.n; t += nthr) fdpos[t] = -1;
    __syncthreads();
    for (int t = tid; t < X.n_fd; t += nthr) fdpos[idx[t]] = t;
    __syncthreads();
}

// one design's constant matrices and frequency-dependent tables
struct GenMats { const double *M, *B, *C, *A_w, *B_w; };
__device__ __forceinline__ GenMats gen_mats(const GenDev &D, const GenFdDev &X, int d)
{
    const size_t nn = (size_t)D.n * D.n, ff = (size_t)X.n_fd * X.n_fd * D.nw;
    GenMats G;
    G.M = D.M + d * nn; G.B = D.B + d * nn; G.C = D.C + d * nn;
    G.A_w = X.A_w ? X.A_w + d * ff : nullptr; G.B_w = X.B_w ? X.B_w + d * ff : nullptr;
    return G;
}

// the operating-point tables of unit U (design d, case U.c of the whole table): op_A_w / op_B_w at [op_shared ? 0 : d][op[c]]
__device__ __forceinline__ void gen_op_tables(const GenDev &D, const GenFdOpDev &X, const GenUnit &U, const double *&Ao, const double *&Bo)
{
    const size_t ff = (size_t)X.n_fd * X.n_fd * D.nw, o = ((X.op_shared ? 0 : (size_t)U.d * X.n_op) + (size_t)X.op[U.c]) * ff;
    Ao = X.op_A_w + o; Bo = X.op_B_w + o;
}

// impedance entry t = a n + b at frequency i (raft_model.py:1086).  On the support: M + A_w and (B + B_w) + B_drag with the
// rigid solver's grouping (raftk_fused.cuh); elsewhere the constant-matrix expression.  FD = false (n_fd = 0) is the
// constant-matrix kernel as it was, instruction for instruction: no map, no branch.  OP: the case's operating point (Ao, Bo
// on the same support) summed with the design's table first, M + (A_w + Ao) and (B + (B_w + Bo)) + B_drag, so that a call
// with operating points equals one with each point's tables summed into fd.A_w / fd.B_w, bit for bit.
template <bool FD, bool OP = false>
__device__ __forceinline__ double2 gen_impedance(const GenDev &D, const GenFdDev &X, const GenMats &G, const int *fdpos, const double *Bd, int t,
                                                 int i, double w, double w2, const double *Ao = nullptr, const double *Bo = nullptr)
{
    if constexpr (FD) {
        const int pa = fdpos[t / D.n], pb = fdpos[t % D.n];
        if (pa >= 0 && pb >= 0) {
            const size_t e = ((size_t)pa * X.n_fd + pb) * D.nw + i;
            const double M = G.M[t] + (OP ? G.A_w[e] + Ao[e] : G.A_w[e]), B = (G.B[t] + (OP ? G.B_w[e] + Bo[e] : G.B_w[e])) + Bd[t];
            return make_double2(fma(-w2, M, G.C[t]), w * B);
        }
    }
    return make_double2(fma(-w2, G.M[t], G.C[t]), w * (G.B[t] + Bd[t]));
}

// k_gen_node_pass: grid (Ns, units), block 128: RMS of the relative velocity components over w (raft_member.py:2071-2090),
// Bmat (:2092-2116), then the drag node load f6 = [Bmat u ; rr x (Bmat u)] (:2122-2124).
// TRAIN: secondary trains only, Bmat taken from their primary's last pass (calcDragExcitation(ih), raft_fowt.py:1940-1957).
template <bool TRAIN>
__global__ void __launch_bounds__(128) k_gen_node_pass(GenDev D, GenWork W, const int *primary)
{
    __shared__ double red[4][4];
    __shared__ double bm[9];
    const int j = blockIdx.x, c = blockIdx.y, tid = threadIdx.x, nw = D.nw, n = D.n;
    const GenUnit U = gen_unit(D, c);
    if (j >= U.Ns) return;
    const int jn = U.j0 + j;
    const double *rr = D.rr + 3 * jn;
    const double2 *u = W.u + (((size_t)c * D.Ns + j) * 3) * nw;
    if constexpr (TRAIN) {
        const int p = primary[c];
        if (p == c) return;
        if (tid < 9) bm[tid] = W.Bmat[((size_t)p * D.Ns + j) * 9 + tid];
    } else {
    if (W.flags[4 * c]) return;
    const double *q = D.node_frame + 9 * jn, *p1 = q + 3, *p2 = q + 6, *T = D.Tn + (size_t)jn * 6 * n;
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
        const double v1 = D.node_circ[jn] ? sqrt(0.5 * s[1]) : sqrt(0.5 * s[2]);
        const double v2 = D.node_circ[jn] ? v1 : sqrt(0.5 * s[3]);
        const double cc = sqrt(8.0 / CUDART_PI) * 0.5 * D.rho;
        const double *cd = D.node_cd + 4 * jn;
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

// k_gen_bdrag: B_drag[c][r][cc] = sum_j sum_{a,l} Tn_j[a][r] B6_j[a][l] Tn_j[l][cc].  grid (n, units), block 128
__global__ void __launch_bounds__(128) k_gen_bdrag(GenDev D, GenWork W)
{
    __shared__ double tb[6];
    const int r = blockIdx.x, c = blockIdx.y, tid = threadIdx.x, n = D.n;
    if (W.flags[4 * c]) return;
    const GenUnit U = gen_unit(D, c);
    double acc[2] = { 0.0, 0.0 };                            // columns tid and tid + 128 (n <= 256)
    for (int j = 0; j < U.Ns; j++) {
        const double *T = D.Tn + (size_t)(U.j0 + j) * 6 * n;
        if (tid < 6) {                                       // tb[l] = sum_a Tn[a][r] B6[a][l]
            double B6[6][6];
            gen_B6(W.Bmat + ((size_t)c * D.Ns + j) * 9, D.rr + 3 * (U.j0 + j), B6);
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

// k_gen_solve_blocked: grid (nw, units), block GT.  Augmented system [Z | F] (n x (n+1)) assembled in global memory
// (L2-resident), factored by lu_blocked in panels of GB columns with the panel and the row block staged in shared memory
// (raftk_lu.cuh): every element loaded once per panel, 9 Mflop per 150 x 150 system run from registers and shared memory.
// Back substitution, then Xi and the convergence verdict.  The factors and pivot rows stay in W.Z / W.piv for the secondary
// trains (k_gen_train_solve).  OP (with FD): the case table carries operating points (GenFdOpDev); an instantiation of its
// own, so that the solves without them compile as before.
#define GB 8
#define GT 128
template <bool FD, bool OP = false>
__global__ void __launch_bounds__(GT, 4) k_gen_solve_blocked(GenDev D, GenWork W, double2 *Xi, double tol, GenFdArg<OP> X)
{
    static_assert(FD || !OP, "operating points live on the support of the frequency-dependent terms");
    extern __shared__ __align__(16) double smem_raw[];
    __shared__ LuStaged<GT, GB> S;
    __shared__ int fdpos[FD ? 256 : 1];
    const int i = blockIdx.x, c = blockIdx.y, tid = threadIdx.x, n = D.n, nw = D.nw, nc = n + 1;
    if (W.flags[4 * c]) return;
    const GenUnit Un = gen_unit(D, c);
    const int d = Un.d;
    const GenMats G = gen_mats(D, X, d);
    const double *Ao = nullptr, *Bo = nullptr;
    if constexpr (OP) gen_op_tables(D, X, Un, Ao, Bo);
    double2 *P = reinterpret_cast<double2 *>(smem_raw);          // panel  [n][GB]   (rows kb.. stored from 0)
    double2 *U = P + (size_t)n * GB;                             // row block [GB][nc]
    double2 *A = W.Z + ((size_t)c * nw + i) * (size_t)n * nc;
    const double w = D.w[i], w2 = w * w;
    const double *Bd = W.B_drag + (size_t)c * n * n;
    if constexpr (FD) gen_fd_map(D, X, d, fdpos, tid, GT);
    for (int t = tid; t < n * n; t += GT) {
        const int a = t / n, b = t % n;
        A[(size_t)a * nc + b] = gen_impedance<FD, OP>(D, X, G, fdpos, Bd, t, i, w, w2, Ao, Bo);
    }
    for (int a = tid; a < n; a += GT) {
        const double2 f1 = W.F_iner[((size_t)c * n + a) * nw + i], f2 = W.F_drag[((size_t)c * n + a) * nw + i];
        A[(size_t)a * nc + n] = make_double2(f1.x + f2.x, f1.y + f2.y);
    }
    __syncthreads();
    const int bad = lu_blocked<GT, true, true>(A, nc, A + n, nc, n, 1, GB, S, P, U, W.piv + ((size_t)c * nw + i) * n);
    lu_back_subst<GT>(A, (size_t)nc, A + n, (size_t)nc, n, 1, tid);
    int notconv = 0, nan = 0;
    for (int a = tid; a < n; a += GT) {
        const double2 x = A[(size_t)a * nc + n], l = W.XiLast[((size_t)c * n + a) * nw + i];
        Xi[((size_t)c * n + a) * nw + i] = x;
        if (isnan(x.x) || isnan(x.y)) nan = 1;
        const double dx = x.x - l.x, dy = x.y - l.y;
        if (!(sqrt(dx * dx + dy * dy) / (sqrt(x.x * x.x + x.y * x.y) + tol) < tol)) notconv = 1;     // raft_model.py:1101-1102
    }
    if (notconv) atomicOr(&W.flags[4 * c + 1], 1);
    if (nan || bad) atomicOr(&W.flags[4 * c + 3], (nan ? RAFTK_FLAG_NAN : 0) | (bad ? RAFTK_FLAG_SINGULAR : 0));
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
// primary's last pass (raft_model.py:1200-1236): the unit-lower solve applies each panel's interchanges (W.piv) as it reaches
// the panel's first column, which is where k_gen_solve_blocked applied them to the right-hand side, so that every element
// receives the same updates in the same order; then the upper solve.  A zero diagonal of U (the primary's singular bin)
// sets RAFTK_FLAG_SINGULAR in the secondary's flag word 3 as well.
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
    for (int k = 0; k < n - 1; k++) {                           // L y = P b
        if (k % GB == 0) {
            if (tid == 0)
                for (int j = k; j < min(k + GB, n); j++) { const int q = pv[j]; if (q != j) { const double2 t = b[j]; b[j] = b[q]; b[q] = t; } }
            __syncthreads();
        }
        const double2 x = b[k];
        for (int r = k + 1 + tid; r < n; r += 128) { double2 v = b[r]; cmsub(v, A[(size_t)r * nc + k], x); b[r] = v; }
        __syncthreads();
    }
    int zero = 0;                                               // a zero diagonal of U
    for (int k = tid; k < n; k += 128) { const double2 a = A[(size_t)k * nc + k]; if (a.x == 0.0 && a.y == 0.0) zero = 1; }
    lu_back_subst<128>(A, (size_t)nc, b, (size_t)1, n, 1, tid);                 // U x = y
    int nan = 0;
    for (int a = tid; a < n; a += 128) {
        const double2 x = b[a];
        Xi[((size_t)c * n + a) * nw + i] = x;
        if (isnan(x.x) || isnan(x.y)) nan = 1;
    }
    if (nan || zero) atomicOr(&W.flags[4 * c + 3], (nan ? RAFTK_FLAG_NAN : 0) | (zero ? RAFTK_FLAG_SINGULAR : 0));
}

// k_gen_relax: grid (nC), block 256: close the pass (raft_model.py:1098-1133)
__global__ void __launch_bounds__(256) k_gen_relax(GenDev D, GenWork W, const double2 *Xi)
{
    __shared__ int st[2];
    const int c = blockIdx.x, tid = threadIdx.x;
    if (W.flags[4 * c]) return;
    if (tid == 0) { st[0] = W.flags[4 * c + 1]; st[1] = W.flags[4 * c + 3]; }
    __syncthreads();
    const int notconv = st[0], nan = st[1];                   // NaN or a zero pivot: the unit stops
    if (!nan && notconv) {
        const size_t tot = (size_t)D.n * D.nw;
        double2 *L = W.XiLast + (size_t)c * tot;
        const double2 *X = Xi + (size_t)c * tot;
        for (size_t t = tid; t < tot; t += 256) L[t] = make_double2(0.2 * L[t].x + 0.8 * X[t].x, 0.2 * L[t].y + 0.8 * X[t].y);
    }
    __syncthreads();
    if (tid == 0) {
        W.flags[4 * c + 2] += 1;                              // passes
        if (nan || !notconv) W.flags[4 * c] = nan ? 2 : 1;   // done: 1 converged, 2 NaN or a zero pivot
        W.flags[4 * c + 1] = 0;
    }
}

// Streamed tables and design batches (raftk_general_solve_dynamics_stream_*, raftk_general_batch_solve_dynamics_*): the
// units (design, case), design-major, run in chunks of whole train groups, each chunk the sequence above on units u0 .. u0+m-1
// (GenDev.u0; outputs advanced to unit u0).  Around it:
//   k_gen_chunk_primary (unit)   cases.primary of the chunk as chunk-local units (a primary lies in its train's design)
//   k_gen_status_rebase (unit)   status word 3 of the chunk's secondaries back to the primary's case index + 1
__global__ void __launch_bounds__(128) k_gen_chunk_primary(int m, int u0, int nCt, const int *primary, int *local)
{
    const int t = blockIdx.x * 128 + threadIdx.x;
    if (t >= m) return;
    const int c = (u0 + t) % nCt;
    local[t] = t - c + primary[c];
}

__global__ void __launch_bounds__(128) k_gen_status_rebase(int m, int u0, int nCt, int *status)
{
    const int t = blockIdx.x * 128 + threadIdx.x;
    if (t < m && status[4 * t + 3] != 0) status[4 * t + 3] += (u0 + t) % nCt - t;
}

// raftk_general_publish_dev: rank p's gathered rows for this call, X[p] complex [rows][n][nw] and S[p] int [rows][4] (NULL: no
// status); status word 3 of a secondary train is shifted by primary_base (shard-local primary + 1 -> the whole table's)
struct GenPublish {
    size_t elems;
    int rows, primary_base;
    double2 *X[RAFTK_MAX_PEERS];
    int *S[RAFTK_MAX_PEERS];
};

// status rows for the caller: passes, converged, flags (flag word 3: RAFTK_FLAG_NAN, RAFTK_FLAG_SINGULAR), 0; a secondary
// train: 0, 1, flags, primary + 1
__global__ void __launch_bounds__(128) k_gen_status(int nC, const int *flags, const int *primary, int *status)
{
    const int c = blockIdx.x * 128 + threadIdx.x;
    if (c >= nC) return;
    const int p = primary ? primary[c] : c;
    status[4 * c + 0] = flags[4 * c + 2];
    status[4 * c + 1] = flags[4 * c] == 1 ? 1 : 0;
    status[4 * c + 2] = flags[4 * c + 3] & (RAFTK_FLAG_NAN | RAFTK_FLAG_SINGULAR);
    status[4 * c + 3] = p != c ? p + 1 : 0;
}
