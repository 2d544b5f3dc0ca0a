// raftk_tables.cuh -- v1 kernels with global wave-kinematics tables: k_depth_table, k_excitation, k_drag_solve.
// They serve the stand-alone calcHydroExcitation / calcHydroLinearization entry points and are the fallback of
// raftk_solve_dynamics when a frequency slice does not fit on chip (included by raftk.cu only).
#pragma once

// ------------------------------------------------------------------------------------------------
// K0: depth table.  grid (ceil(nw/128), members of the chunk), block 128
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_depth_table(DesignsDev D, Work W)
{
    // blockIdx.y = local design, blockIdx.z unused; loop over the design's members and nodes
    const int dl = blockIdx.y, d = W.d0 + dl;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= D.nw) return;
    const int m0 = D.member_offset[d], m1 = D.member_offset[d + 1];
    const int nbase = D.mem_node_start[m0];
    const double k = D.k[i], h = D.depth;
    for (int m = m0; m < m1; m++) {
        const double qz = D.mem_frame[9 * m + 2], zA = D.mem_rA[3 * m + 2];
        const int j0 = D.mem_node_start[m], j1 = D.mem_node_start[m + 1];
        for (int j = j0; j < j1; j++) {
            double z = zA + D.node_ls[j] * qz;
            double S_, C_, P_;
            depth_funcs(k, h, z, S_, C_, P_);
            W.depth_tab[((size_t)dl * D.max_nodes + (j - nbase)) * D.nw + i] = make_double2(C_, S_);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// K1: excitation.  grid (ceil(nw/128), nC, nDc), block 128, thread = frequency
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ double jonswap(double w, double Hs, double Tp, double Gamma)
{
    // helpers.py:733-760
    if (!(Gamma != 0.0)) {
        double t = Tp / sqrt(Hs);
        if (t <= 3.6) Gamma = 5.0;
        else if (t >= 5.0) Gamma = 1.0;
        else Gamma = exp(5.75 - 1.15 * t);
    }
    const double f = 0.5 / CUDART_PI * w;
    const double fpOvrf4 = pow(Tp * f, -4.0);
    const double C = 1.0 - (0.287 * log(Gamma));
    const double Sigma = (f <= 1.0 / Tp) ? 0.07 : 0.09;
    const double t = (f * Tp - 1.0) / Sigma;
    const double Alpha = exp(-0.5 * t * t);
    return 0.5 / CUDART_PI * C * 0.3125 * Hs * Hs * fpOvrf4 / f * exp(-1.25 * fpOvrf4) * pow(Gamma, Alpha);
}

// wave spectrum of one case at one frequency (raft_fowt.py:1758-1772); explicit amplitudes: S = zeta^2 / (2 dw)
__device__ __forceinline__ double sea_state_S(const CasesDev &Cs, int c, int i, int nw, double w, double dw)
{
    if (Cs.zeta_in) { const double z = Cs.zeta_in[(size_t)c * nw + i]; return z * z / (2.0 * dw); }
    const int spec = Cs.spec[c];
    if (spec == RAFTK_SPEC_JONSWAP) return jonswap(w, Cs.Hs[c], Cs.Tp[c], Cs.gamma[c]);
    if (spec == RAFTK_SPEC_UNIT) return 1.0;
    if (spec == RAFTK_SPEC_CONSTANT) return Cs.Hs[c];
    return 0.0;
}

// wave amplitude of one case at one frequency: explicit table or spectrum -> zeta = sqrt(2 S dw) (raft_fowt.py:1759-1774)
__device__ __forceinline__ double sea_state_zeta(const CasesDev &Cs, int c, int i, int nw, double w, double dw)
{
    if (Cs.zeta_in) return Cs.zeta_in[(size_t)c * nw + i];
    return sqrt(2.0 * sea_state_S(Cs, c, i, nw, w, dw) * dw);
}

// BEM excitation at frequency i for heading beta from one heading-relative coefficient table X [nhs][6][nw] on headings hd:
// bracket the heading with wrap-around, interpolate, rotate back to the global frame, scale by the wave amplitude and the
// array phase offset of (xr, yr) (raft_fowt.py:1796-1849).  Br/Bi receive the 6 complex force components (full DOFs 0-5).
// Shared by the rigid solvers (bem_excitation below) and the generalised-DOF solve (k_gen_bem).
__device__ __forceinline__ void bem_excitation_table(const double *hd, int nhs, const double2 *X, int nw, double xr, double yr,
                                                     double hadj, int i, double k, double beta, double sb, double cb, double zeta,
                                                     double (&Br)[6], double (&Bi)[6])
{
    double bdeg = fmod(beta * (180.0 / CUDART_PI) - hadj, 360.0);
    if (bdeg < 0) bdeg += 360.0;                                   // python's % is non-negative
    int i1 = 0, i2 = 0; double f2 = 0;
    if (bdeg <= hd[0]) {
        const double hlast = hd[nhs - 1] - 360.0;
        i1 = nhs - 1; i2 = 0; f2 = (bdeg - hlast) / (hd[0] - hlast);
    } else if (bdeg >= hd[nhs - 1]) {
        const double hfirst = hd[0] + 360.0;
        i1 = nhs - 1; i2 = 0; f2 = (bdeg - hd[nhs - 1]) / (hfirst - hd[nhs - 1]);
    } else {
        for (int t = 0; t < nhs - 1; t++) if (hd[t + 1] > bdeg) { i1 = t; i2 = t + 1; f2 = (bdeg - hd[t]) / (hd[t + 1] - hd[t]); break; }
    }
    const double f1 = 1.0 - f2;
    double Xr[6], Xi_[6];
#pragma unroll
    for (int a = 0; a < 6; a++) {
        const double2 x1 = X[((size_t)i1 * 6 + a) * nw + i], x2 = X[((size_t)i2 * 6 + a) * nw + i];
        Xr[a] = x1.x * f1 + x2.x * f2; Xi_[a] = x1.y * f1 + x2.y * f2;
    }
    double Rr[6], Ri[6];
    Rr[0] = Xr[0] * cb - Xr[1] * sb; Ri[0] = Xi_[0] * cb - Xi_[1] * sb;
    Rr[1] = Xr[0] * sb + Xr[1] * cb; Ri[1] = Xi_[0] * sb + Xi_[1] * cb;
    Rr[2] = Xr[2];                   Ri[2] = Xi_[2];
    Rr[3] = Xr[3] * cb - Xr[4] * sb; Ri[3] = Xi_[3] * cb - Xi_[4] * sb;
    Rr[4] = Xr[3] * sb + Xr[4] * cb; Ri[4] = Xi_[3] * sb + Xi_[4] * cb;
    Rr[5] = Xr[5];                   Ri[5] = Xi_[5];
    double sp, cp;
    sincos(-(k * (xr * cb + yr * sb)), &sp, &cp);
    const double pr = zeta * cp, pi = zeta * sp;
#pragma unroll
    for (int a = 0; a < 6; a++) { Br[a] = Rr[a] * pr - Ri[a] * pi; Bi[a] = Rr[a] * pi + Ri[a] * pr; }
}

// BEM excitation of design d of a rigid batch: its table, headings and (x_ref, y_ref, heading_adjust)
__device__ __forceinline__ void bem_excitation(const DesignsDev &D, int d, int i, double k, double beta, double sb, double cb,
                                               double zeta, double (&Br)[6], double (&Bi)[6])
{
    const int nhs = D.n_bem_head, nw = D.nw;
    bem_excitation_table(D.bem_headings, nhs, reinterpret_cast<const double2 *>(D.X_BEM) + (size_t)d * nhs * 6 * nw, nw,
                         D.bem_xyh[3 * d], D.bem_xyh[3 * d + 1], D.bem_xyh[3 * d + 2], i, k, beta, sb, cb, zeta, Br, Bi);
}

// Inertial wave excitation of design d's submerged rotors at bin i (raft_fowt.py:1859-1888), added to Fr + i Fi: the wave
// acceleration ud = i w u of getWaveKin at each hub r3 (helpers.py:188-236; phase from the hub's global x, y, depth terms at
// z = r3[2]) through the packed G [6][3] (raftk_designs.rot_G).  The reference applies the term after its wave-train loop,
// with the train index left at the last train, so only the last row of each group of Cs.primary gets it (groups are
// contiguous, primary first; without primary every row is its own group).
__device__ __forceinline__ void rotor_excitation(const DesignsDev &D, const CasesDev &Cs, int d, int c, int i, double k, double w,
                                                 double beta, double sb, double cb, double zeta, double (&Fr)[6], double (&Fi)[6])
{
    if (Cs.primary && c + 1 < Cs.nC && Cs.primary[c + 1] != c + 1) return;
    const int n = D.rot_count[d];
    for (int r = 0; r < n; r++) {
        const size_t e = (size_t)d * D.max_rotors + r;
        const double *r3 = D.rot_r3 + 3 * e, *G = D.rot_G + 18 * e;
        double S_, C_, P_;
        depth_funcs(k, D.depth, r3[2], S_, C_, P_);
        double se, ce;
        sincos(-(k * (cb * r3[0] + sb * r3[1])), &se, &ce);     // local elevation zeta (ce + i se)
        // u = w zeta_l (C cb, C sb, i S); ud = i w u
        const double a = w * w * zeta;
        const double hr = a * C_ * cb, vr = a * C_ * sb, zr = a * S_;
        const double ur[3] = {-hr * se, -vr * se, -zr * ce}, ui[3] = {hr * ce, vr * ce, -zr * se};
#pragma unroll
        for (int t = 0; t < 6; t++) {
            Fr[t] += G[3 * t] * ur[0] + G[3 * t + 1] * ur[1] + G[3 * t + 2] * ur[2];
            Fi[t] += G[3 * t] * ui[0] + G[3 * t + 1] * ui[1] + G[3 * t + 2] * ui[2];
        }
    }
}

struct ExcOut { double2 *F_iner, *F_BEM; double *zeta; };

__global__ void __launch_bounds__(128) k_excitation(DesignsDev D, CasesDev Cs, Work W, ExcOut O)
{
    const int c = blockIdx.y, dl = blockIdx.z, d = W.d0 + dl;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= D.nw) return;
    const int nw = D.nw;
    const double w = D.w[i], k = D.k[i];

    const double zeta = sea_state_zeta(Cs, c, i, nw, w, D.dw);
    if (dl == 0) {
        W.zeta[(size_t)c * nw + i] = zeta;
        if (O.zeta && W.d0 == 0) O.zeta[(size_t)c * nw + i] = zeta;
    }
    const double beta = Cs.beta_deg[c] * (CUDART_PI / 180.0);   // np.deg2rad
    double sb, cb;
    sincos(beta, &sb, &cb);
    const double zw = zeta * w;

    const int m0 = D.member_offset[d], m1 = D.member_offset[d + 1];
    const int nbase = D.mem_node_start[m0];
    const size_t unit = (size_t)dl * Cs.nC + c;
    double2 *ptab = W.phase_tab + unit * D.max_nodes * nw;
    const double2 *dtab = W.depth_tab + (size_t)dl * D.max_nodes * nw;

    double Fr[6] = {0, 0, 0, 0, 0, 0}, Fi[6] = {0, 0, 0, 0, 0, 0};
    for (int m = m0; m < m1; m++) {
        const double *fr = D.mem_frame + 9 * m;
        const double q0 = fr[0], q1 = fr[1], q2 = fr[2], p10 = fr[3], p11 = fr[4], p12 = fr[5], p20 = fr[6], p21 = fr[7], p22 = fr[8];
        const double xA = D.mem_rA[3 * m], yA = D.mem_rA[3 * m + 1], zA = D.mem_rA[3 * m + 2];
        const double hq = q0 * cb + q1 * sb, h1 = p10 * cb + p11 * sb, h2 = p20 * cb + p21 * sb;
        const int j0 = D.mem_node_start[m], j1 = D.mem_node_start[m + 1];
        double Aqr = 0, Aqi = 0, A1r = 0, A1i = 0, A2r = 0, A2i = 0, L1r = 0, L1i = 0, L2r = 0, L2i = 0;
        for (int j = j0; j < j1; j++) {
            const double ls = D.node_ls[j];
            const double x = xA + ls * q0, y = yA + ls * q1;
            double se, ce;
            sincos(-(k * (cb * x + sb * y)), &se, &ce);          // E = exp(-i k (x cos b + y sin b))
            const double er = zw * ce, ei = zw * se;             // zeta*w*E
            ptab[(size_t)(j - nbase) * nw + i] = make_double2(er, ei);
            const double2 cs = dtab[(size_t)(j - nbase) * nw + i];
            const double inq = D.node_in_q[j], pa = D.node_pa[j];
            double in1 = D.node_in_p1[j], in2 = D.node_in_p2[j], in1i = 0.0, in2i = 0.0;
            if (D.node_in_p1_w) {                                 // MacCamy-Fuchs: complex, per frequency
                const double2 v1 = D.node_in_p1_w[(size_t)j * nw + i], v2 = D.node_in_p2_w[(size_t)j * nw + i];
                in1 = v1.x; in1i = v1.y; in2 = v2.x; in2i = v2.y;
            }
            if (inq != 0.0 || in1 != 0.0 || in2 != 0.0 || in1i != 0.0 || in2i != 0.0 || pa != 0.0) {
                // c_d = zeta w E (C h_d + i S d_z); inertial force coefficient along d: i w in_d c_d
                double gr, gi, cr, ci;
                gr = cs.x * hq; gi = cs.y * q2; cr = er * gr - ei * gi; ci = er * gi + ei * gr;
                double fqr = -w * inq * ci, fqi = w * inq * cr;
                gr = cs.x * h1; gi = cs.y * p12; cr = er * gr - ei * gi; ci = er * gi + ei * gr;
                const double f1r = -w * (in1 * ci + in1i * cr), f1i = w * (in1 * cr - in1i * ci);
                gr = cs.x * h2; gi = cs.y * p22; cr = er * gr - ei * gi; ci = er * gi + ei * gr;
                const double f2r = -w * (in2 * ci + in2i * cr), f2i = w * (in2 * cr - in2i * ci);
                if (pa != 0.0) {                                  // dynamic pressure on end area (member:1988)
                    double S_, C_, P_;
                    depth_funcs(k, D.depth, zA + ls * q2, S_, C_, P_);
                    fqr += pa * P_ * zeta * ce; fqi += pa * P_ * zeta * se;
                }
                Aqr += fqr; Aqi += fqi; A1r += f1r; A1i += f1i; A2r += f2r; A2i += f2i;
                L1r += ls * f1r; L1i += ls * f1i; L2r += ls * f2r; L2i += ls * f2i;
            }
        }
        const double *arm = D.mem_arm + 3 * m;
        const double a0 = arm[0], a1 = arm[1], a2 = arm[2];
        // a x q, a x p1, a x p2
        const double aq0 = a1 * q2 - a2 * q1, aq1 = a2 * q0 - a0 * q2, aq2 = a0 * q1 - a1 * q0;
        const double b10 = a1 * p12 - a2 * p11, b11 = a2 * p10 - a0 * p12, b12 = a0 * p11 - a1 * p10;
        const double b20 = a1 * p22 - a2 * p21, b21 = a2 * p20 - a0 * p22, b22 = a0 * p21 - a1 * p20;
        Fr[0] += q0 * Aqr + p10 * A1r + p20 * A2r;  Fi[0] += q0 * Aqi + p10 * A1i + p20 * A2i;
        Fr[1] += q1 * Aqr + p11 * A1r + p21 * A2r;  Fi[1] += q1 * Aqi + p11 * A1i + p21 * A2i;
        Fr[2] += q2 * Aqr + p12 * A1r + p22 * A2r;  Fi[2] += q2 * Aqi + p12 * A1i + p22 * A2i;
        Fr[3] += aq0 * Aqr + b10 * A1r + b20 * A2r + p20 * L1r - p10 * L2r;
        Fi[3] += aq0 * Aqi + b10 * A1i + b20 * A2i + p20 * L1i - p10 * L2i;
        Fr[4] += aq1 * Aqr + b11 * A1r + b21 * A2r + p21 * L1r - p11 * L2r;
        Fi[4] += aq1 * Aqi + b11 * A1i + b21 * A2i + p21 * L1i - p11 * L2i;
        Fr[5] += aq2 * Aqr + b12 * A1r + b22 * A2r + p22 * L1r - p12 * L2r;
        Fi[5] += aq2 * Aqi + b12 * A1i + b22 * A2i + p22 * L1i - p12 * L2i;
    }
    const size_t ogl = ((size_t)d * Cs.nC + c) * 6 * nw;     // global output index base
    if (D.max_rotors > 0) rotor_excitation(D, Cs, d, c, i, k, w, beta, sb, cb, zeta, Fr, Fi);
    if (O.F_iner)
        for (int a = 0; a < 6; a++) O.F_iner[ogl + (size_t)a * nw + i] = make_double2(Fr[a], Fi[a]);

    double Br[6] = {0, 0, 0, 0, 0, 0}, Bi[6] = {0, 0, 0, 0, 0, 0};
    if (D.n_bem_head > 0) bem_excitation(D, d, i, k, beta, sb, cb, zeta, Br, Bi);
    if (O.F_BEM)
        for (int a = 0; a < 6; a++) O.F_BEM[ogl + (size_t)a * nw + i] = make_double2(Br[a], Bi[a]);
    double2 *F0 = W.F0 + unit * 6 * nw;
    for (int a = 0; a < 6; a++) {
        const double f2 = Cs.F_2nd ? Cs.F_2nd[ogl + (size_t)a * nw + i] : 0.0;      // raft_model.py:1048
        F0[(size_t)a * nw + i] = make_double2((Br[a] + Fr[a]) + f2, Bi[a] + Fi[a]);
    }
}

// ------------------------------------------------------------------------------------------------
// K2: drag linearisation + impedance solve
// ------------------------------------------------------------------------------------------------
struct SolveParams {
    int n_iter, CS, nwl, mode;          // mode 0: solve loop; 1: single linearisation pass with Xi_in
    double tol, xi_start;
    const double2 *Xi_in;               // [nD][nC][6][nw] (mode 1)
    double2 *Xi_out, *Fdrag_out;        // [nD][nC][6][nw]
    double *Bdrag_out;                  // [nD][nC][36]
    int *status;                        // [nD][nC][4]
};

// shared-memory carve-up (doubles unless noted); sizes depend on max_members / max_nodes / nwl
struct Smem {
    double *mem;        // [Nm][MEM_STRIDE]: q,p1,p2, axq, axp1, axp2, hq,h1,h2
    double *node;       // [7][NsP]: ls, cdq, cd1, cd2, bq, b1, b2
    double *msum;       // [Nm][8]: sum bq, sum b1, sum b1 ls, sum b1 ls^2, sum b2, sum b2 ls, sum b2 ls^2
    double *mat;        // [3][36]: M0, B0 + B_drag, C0
    double *warp_part;  // [nchunk][nwarps][32]
    double *sums;       // [2][nchunk*32 + 2]  (this CTA's partial sums + flags, double buffered)
    double *tot;        // [nchunk*32]
    double *xi;         // [12][nwl]
    int *imem;          // [Nm][3]: node start, node end (local), circ
};

__host__ __device__ inline size_t smem_doubles(int Nm, int NsP, int nchunk, int nwarps, int nwl)
{
    return (size_t)Nm * MEM_STRIDE + 7 * (size_t)NsP + (size_t)Nm * 8 + 108 + (size_t)nchunk * nwarps * 32
           + 2 * ((size_t)nchunk * 32 + 2) + (size_t)nchunk * 32 + 12 * (size_t)nwl;
}

__global__ void __launch_bounds__(SOLVE_THREADS, 2)
k_drag_solve(DesignsDev D, CasesDev Cs, Work W, SolveParams P)
{
    extern __shared__ __align__(16) double smem_raw[];
    cg::cluster_group cluster = cg::this_cluster();
    const int CS = P.CS;
    const int rank = (CS > 1) ? (int)cluster.block_rank() : 0;
    const int unit_l = blockIdx.x / CS;                 // local unit in this chunk
    const int dl = unit_l / Cs.nC, c = unit_l % Cs.nC, d = W.d0 + dl;
    const int nw = D.nw, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nwarps = SOLVE_THREADS / 32;

    const int m0 = D.member_offset[d], Nm = D.member_offset[d + 1] - m0;
    const int nbase = D.mem_node_start[m0];
    const int Ns = D.mem_node_start[m0 + Nm] - nbase;
    const int NsP = D.max_nodes;
    const int nchunk = (D.max_nodes + CHUNK_NODES - 1) / CHUNK_NODES;
    const int nwl = P.nwl;
    const int f_begin = rank * nwl;
    const int nloc = max(0, min(nwl, nw - f_begin));     // frequencies owned by this CTA

    Smem S;
    {
        double *p = smem_raw;
        S.mem = p; p += (size_t)D.max_members * MEM_STRIDE;
        S.node = p; p += 7 * (size_t)NsP;
        S.msum = p; p += (size_t)D.max_members * 8;
        S.mat = p; p += 108;
        S.warp_part = p; p += (size_t)nchunk * nwarps * 32;
        S.sums = p; p += 2 * ((size_t)nchunk * 32 + 2);
        S.tot = p; p += (size_t)nchunk * 32;
        S.xi = p; p += 12 * (size_t)nwl;
        S.imem = reinterpret_cast<int *>(p);
    }
    const int sums_stride = nchunk * 32 + 2;

    // ---- stage design tables (members, nodes, matrices) ----------------------------------------
    const double beta = Cs.beta_deg[c] * (CUDART_PI / 180.0);
    double sb, cb;
    sincos(beta, &sb, &cb);
    for (int m = tid; m < Nm; m += SOLVE_THREADS) {
        const double *fr = D.mem_frame + 9 * (m0 + m);
        const double *arm = D.mem_arm + 3 * (m0 + m);
        double *o = S.mem + m * MEM_STRIDE;
        member_row<true>(o, fr, arm, cb, sb);
        S.imem[3 * m + 0] = D.mem_node_start[m0 + m] - nbase;
        S.imem[3 * m + 1] = D.mem_node_start[m0 + m + 1] - nbase;
        S.imem[3 * m + 2] = D.mem_circ[m0 + m];
    }
    for (int j = tid; j < NsP; j += SOLVE_THREADS) {
        const bool in = j < Ns;
        S.node[0 * NsP + j] = in ? D.node_ls[nbase + j] : 0.0;
        S.node[1 * NsP + j] = in ? D.node_cd_q[nbase + j] : 0.0;
        S.node[2 * NsP + j] = in ? D.node_cd_p1[nbase + j] : 0.0;
        S.node[3 * NsP + j] = in ? D.node_cd_p2[nbase + j] : 0.0;
    }
    for (int t = tid; t < 36; t += SOLVE_THREADS) {
        S.mat[t] = D.M0[(size_t)d * 36 + t];
        S.mat[72 + t] = D.C0[(size_t)d * 36 + t];
    }
    // initial response guess (raft_model.py:999) or the given Xi (mode 1)
    const size_t ogl = ((size_t)d * Cs.nC + c) * 6 * nw;
    for (int t = tid; t < nloc; t += SOLVE_THREADS) {
        for (int a = 0; a < 6; a++) {
            double xr = P.xi_start, xi = 0.0;
            if (P.mode == 1) { const double2 v = P.Xi_in[ogl + (size_t)a * nw + f_begin + t]; xr = v.x; xi = v.y; }
            S.xi[(2 * a) * nwl + t] = xr; S.xi[(2 * a + 1) * nwl + t] = xi;
        }
    }
    __syncthreads();

    const size_t unit = (size_t)dl * Cs.nC + c;
    const double2 *ptab = W.phase_tab + unit * D.max_nodes * nw;
    const double2 *dtab = W.depth_tab + (size_t)dl * D.max_nodes * nw;
    const double2 *F0 = W.F0 + unit * 6 * nw;
    const double *Aw = D.A_w ? D.A_w + (size_t)d * 36 * nw : nullptr;
    const double *Bw = D.B_w ? D.B_w + (size_t)d * 36 * nw : nullptr;

    int passes = 0, converged = 0, flags = 0, par = 0;
    const int max_pass = (P.mode == 1) ? 1 : P.n_iter + 1;

    for (int it = 0; it < max_pass; it++) {
        // ================= pass part 1: sum_w |v_rel . d|^2 per node and direction =================
        for (int ch = 0; ch < nchunk; ch++) {
            double acc[32];
#pragma unroll
            for (int t = 0; t < 32; t++) acc[t] = 0.0;
            const int jc0 = ch * CHUNK_NODES;
            if (jc0 < Ns) {
                for (int t = tid; t < nloc; t += SOLVE_THREADS) {
                    const int i = f_begin + t;
                    const double w = D.w[i];
                    double xr[6], xi[6];
#pragma unroll
                    for (int a = 0; a < 6; a++) { xr[a] = S.xi[(2 * a) * nwl + t]; xi[a] = S.xi[(2 * a + 1) * nwl + t]; }
                    int mcur = -1, mend = 0;
                    double hq = 0, h1 = 0, h2 = 0, dzq = 0, dz1 = 0, dz2 = 0;
                    double mqr = 0, mqi = 0, m1r = 0, m1i = 0, m2r = 0, m2i = 0, t1r = 0, t1i = 0, t2r = 0, t2i = 0;
#pragma unroll
                    for (int jj = 0; jj < CHUNK_NODES; jj++) {
                        const int j = jc0 + jj;
                        if (j < Ns) {
                            if (j >= mend) {        // (uniform) entered a new member: member-level projections of the body velocity
                                do { mcur++; mend = S.imem[3 * mcur + 1]; } while (j >= mend);
                                const double *o = S.mem + mcur * MEM_STRIDE;
                                member_velocity(o, xr, xi, w, mqr, mqi, m1r, m1i, m2r, m2i, t1r, t1i, t2r, t2i);
                                hq = o[18]; h1 = o[19]; h2 = o[20]; dzq = o[2]; dz1 = o[5]; dz2 = o[8];
                            }
                            const double ls = S.node[j];
                            const double2 e = ptab[(size_t)j * nw + i];
                            const double2 cs = dtab[(size_t)j * nw + i];
                            double gr, gi, ar_, ai_;
                            gr = cs.x * hq; gi = cs.y * dzq;
                            ar_ = e.x * gr - e.y * gi + mqr; ai_ = e.x * gi + e.y * gr + mqi;
                            acc[3 * jj + 0] += ar_ * ar_ + ai_ * ai_;
                            gr = cs.x * h1; gi = cs.y * dz1;
                            ar_ = e.x * gr - e.y * gi + m1r + ls * t2r; ai_ = e.x * gi + e.y * gr + m1i + ls * t2i;
                            acc[3 * jj + 1] += ar_ * ar_ + ai_ * ai_;
                            gr = cs.x * h2; gi = cs.y * dz2;
                            ar_ = e.x * gr - e.y * gi + m2r - ls * t1r; ai_ = e.x * gi + e.y * gr + m2i - ls * t1i;
                            acc[3 * jj + 2] += ar_ * ar_ + ai_ * ai_;
                        }
                    }
                }
            }
            const double r = warp_multi_reduce32(acc);
            S.warp_part[((size_t)ch * nwarps + warp) * 32 + lane] = r;
        }
        __syncthreads();
        rms_exchange<SOLVE_THREADS>(cluster, CS, nchunk, par, sums_stride, S.warp_part, S.sums, S.tot);

        // ================= linearised coefficients per node, member sums, B_drag ===================
        for (int j = tid; j < Ns; j += SOLVE_THREADS) {
            const int ch = j / CHUNK_NODES, jj = j - ch * CHUNK_NODES;
            const double sq = S.tot[ch * 32 + 3 * jj], s1 = S.tot[ch * 32 + 3 * jj + 1], s2 = S.tot[ch * 32 + 3 * jj + 2];
            int m = 0;
            while (j >= S.imem[3 * m + 1]) m++;
            double vq, v1, v2;
            drag_rms(sq, s1, s2, S.imem[3 * m + 2] != 0, vq, v1, v2);
            S.node[4 * NsP + j] = S.node[1 * NsP + j] * vq;
            S.node[5 * NsP + j] = S.node[2 * NsP + j] * v1;
            S.node[6 * NsP + j] = S.node[3 * NsP + j] * v2;
        }
        __syncthreads();
        drag_member_sums<SOLVE_THREADS, 3>(Nm, S.imem, S.node, S.node, 4 * NsP, 5 * NsP, 6 * NsP, S.msum);
        __syncthreads();
        if (tid < 36) {
            const double s = drag_bmat_entry(tid, Nm, S.mem, S.msum);
            S.mat[36 + tid] = D.B0[(size_t)d * 36 + tid] + s;
            if (P.Bdrag_out && rank == 0) P.Bdrag_out[((size_t)d * Cs.nC + c) * 36 + tid] = s;
        }
        __syncthreads();

        // ================= pass part 2: drag excitation, impedance, solve, convergence =============
        int conv_local = 1, nan_local = 0;
        for (int t = tid; t < nloc; t += SOLVE_THREADS) {
            const int i = f_begin + t;
            const double w = D.w[i];
            double br[6], bi[6];
#pragma unroll
            for (int a = 0; a < 6; a++) { br[a] = 0.0; bi[a] = 0.0; }
            for (int m = 0; m < Nm; m++) {
                const double *o = S.mem + m * MEM_STRIDE;
                const double hq = o[18], h1 = o[19], h2 = o[20], dzq = o[2], dz1 = o[5], dz2 = o[8];
                double Aqr = 0, Aqi = 0, A1r = 0, A1i = 0, A2r = 0, A2i = 0, L1r = 0, L1i = 0, L2r = 0, L2i = 0;
                const int j1 = S.imem[3 * m + 1];
#pragma unroll 4
                for (int j = S.imem[3 * m]; j < j1; j++) {
                    const double2 e = ptab[(size_t)j * nw + i];
                    const double2 cs = dtab[(size_t)j * nw + i];
                    const double ls = S.node[j], bq = S.node[4 * NsP + j], b1 = S.node[5 * NsP + j], b2 = S.node[6 * NsP + j];
                    double gr, gi, cr, ci;
                    gr = cs.x * hq; gi = cs.y * dzq; cr = e.x * gr - e.y * gi; ci = e.x * gi + e.y * gr;
                    Aqr += bq * cr; Aqi += bq * ci;
                    gr = cs.x * h1; gi = cs.y * dz1; cr = e.x * gr - e.y * gi; ci = e.x * gi + e.y * gr;
                    cr *= b1; ci *= b1; A1r += cr; A1i += ci; L1r += ls * cr; L1i += ls * ci;
                    gr = cs.x * h2; gi = cs.y * dz2; cr = e.x * gr - e.y * gi; ci = e.x * gi + e.y * gr;
                    cr *= b2; ci *= b2; A2r += cr; A2i += ci; L2r += ls * cr; L2i += ls * ci;
                }
                member_force6(o, Aqr, Aqi, A1r, A1i, A2r, A2i, L1r, L1i, L2r, L2i, br, bi);
            }
            if (P.Fdrag_out)
                for (int a = 0; a < 6; a++) P.Fdrag_out[ogl + (size_t)a * nw + i] = make_double2(br[a], bi[a]);
            if (P.mode == 1) continue;

            // F_tot = F_lin + F_drag (raft_model.py:1081); Z = -w^2 M + i w B + C (:1086)
            double ar[6][6], ai[6][6];
#pragma unroll
            for (int a = 0; a < 6; a++) {
                const double2 f0 = F0[(size_t)a * nw + i];
                br[a] += f0.x; bi[a] += f0.y;
            }
            const double w2 = w * w;
            if (Cs.op) {                // the case's operating point, summed with the design's table first (tab_term)
                const double *Ao = op_table(Cs, Cs.op_A_w, d, c, nw), *Bo = op_table(Cs, Cs.op_B_w, d, c, nw);
#pragma unroll
                for (int a = 0; a < 6; a++)
#pragma unroll
                    for (int b = 0; b < 6; b++) {
                        const double M = S.mat[6 * a + b] + tab_term(Aw, Ao, (size_t)(6 * a + b) * nw + i);
                        const double B = S.mat[36 + 6 * a + b] + tab_term(Bw, Bo, (size_t)(6 * a + b) * nw + i);
                        ar[a][b] = S.mat[72 + 6 * a + b] - w2 * M;
                        ai[a][b] = w * B;
                    }
            } else {
#pragma unroll
            for (int a = 0; a < 6; a++)
#pragma unroll
                for (int b = 0; b < 6; b++) {
                    double M = S.mat[6 * a + b], B = S.mat[36 + 6 * a + b];
                    if (Aw) M += Aw[(size_t)(6 * a + b) * nw + i];
                    if (Bw) B += Bw[(size_t)(6 * a + b) * nw + i];
                    ar[a][b] = S.mat[72 + 6 * a + b] - w2 * M;
                    ai[a][b] = w * B;
                }
            }
            const bool ok = solve6(ar, ai, br, bi);
            if (!ok) nan_local |= RAFTK_FLAG_SINGULAR;
            // convergence test (raft_model.py:1103-1104) and relaxation (:1133)
#pragma unroll
            for (int a = 0; a < 6; a++) {
                const double lr = S.xi[(2 * a) * nwl + t], li = S.xi[(2 * a + 1) * nwl + t];
                if (isnan(br[a]) || isnan(bi[a])) nan_local |= RAFTK_FLAG_NAN;
                const double dr = br[a] - lr, di = bi[a] - li;
                const double tc = sqrt(dr * dr + di * di) / (sqrt(br[a] * br[a] + bi[a] * bi[a]) + P.tol);
                if (!(tc < P.tol)) conv_local = 0;
                S.xi[(2 * a) * nwl + t] = 0.2 * lr + 0.8 * br[a];
                S.xi[(2 * a + 1) * nwl + t] = 0.2 * li + 0.8 * bi[a];
                P.Xi_out[ogl + (size_t)a * nw + i] = make_double2(br[a], bi[a]);
            }
        }
        passes++;
        if (P.mode == 1) break;

        // ---- all-reduce of (converged, flags) over the CTA and the cluster ----
        int conv_all, nan_all;
        flags_exchange(cluster, CS, nchunk, par, sums_stride, conv_local, nan_local, S.sums, conv_all, nan_all);
        par ^= 1;
        flags |= nan_all;
        if (nan_all & RAFTK_FLAG_NAN) break;              // raft_model.py:1098-1099 raises here
        if (conv_all) { converged = 1; break; }
    }
    if (P.status && rank == 0 && tid == 0) store_status(P.status + ((size_t)d * Cs.nC + c) * 4, passes, converged, flags, false, 0);
    if (CS > 1) cluster.sync();      // keep shared memory alive until every peer finished reading it
}
