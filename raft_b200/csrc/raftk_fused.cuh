// raftk_fused.cuh -- k_rao_fused: the fused, fully on-chip solver behind raftk_solve_dynamics (included by raftk.cu only).
#pragma once

// ------------------------------------------------------------------------------------------------
// K2f: fused on-chip solver (v2).  One launch does excitation + the whole fixed-point loop; the
// wave-kinematics of the CTA's frequency slice live in SHARED MEMORY for the whole kernel, in a
// compact member-level form, so the iteration loop touches neither L2 nor HBM:
//   per member and frequency   : E0 = zeta w exp(-i k (x0 cos b + y0 sin b)) at the member's first node
//   per distinct first-node z  : A+-(z0) = (C0 +- S0)/2 from the accurate cosh/sinh ratios
//   per "step class" and freq. : W   = exp(-i k (q_x cos b + q_y sin b) step)   (phase factor)
//                                f+- = exp(+-k q_z step)                        (depth factors)
// and nodes are walked along the member with the geometric recurrences E <- E W, A+- <- A+- f+-,
// C = A+ + A-, S = A+ - A-  (the depth functions cosh/sinh(k(z+h))/sinh(kh) split into their growing
// and decaying exponentials, so there is no cancellation in either walking direction; rounding grows
// ~1 ulp per node).  Distinct steps are deduplicated per design (8 classes for VolturnUS-S).
// The node body is branch-free: a member's first node and zero steps use identity rows of the factor tables,
// and the factors of node j+1 are requested while node j is computed (shared-memory latency off the critical path).
// ------------------------------------------------------------------------------------------------
struct FusedParams {
    int n_iter, CS, nwl, maxW, maxH, maxZ;
    double tol, xi_start;
    double2 *Xi_out, *Fdrag_out, *Finer_out, *Fbem_out;
    double2 *Xilast_out;     // [units][6][nw] iterate each pass linearised about (last write = XiLast of the final pass), or NULL
    const double2 *Xi_init;  // [units][6][nw] starting iterate instead of xi_start, or NULL
    double *Bdrag_out, *zeta_out;
    int *status;
    double2 *F0g;            // [units][6][nw] linear excitation kept in global memory (frees 96 B/bin of smem), or NULL
    double *lin_g;           // [units][NCOEF*max_nodes + 36] linearisation hand-over primary -> secondary wave trains, or NULL
    int phase;               // -1: every case is its own primary; 0: run primaries only; 1: run secondaries only
    // multi-GPU exchange fused into the epilogue (raftk_solve_dynamics_gather_dev): every finished unit's Xi / status
    // is also stored into the other ranks' gathered arrays through peer-mapped pointers (NVLink)
    // k_rao_fused2 only: per-design plan blobs (k_fused_plan), member base phases / depth pairs in the workspace
    const double *plan; size_t plan_stride;
    double2 *Eg, *Ag;
    // k_rao_fused2<true> only: per-unit exchange rows [unit][parity][rank][nchunk*32 + 2] and arrival counters [unit]
    double *xrow; unsigned *xcnt;
    int n_peers, peer_rank;
    double2 *peer_Xi[RAFTK_MAX_PEERS];    // [p]: this rank's block inside rank p's gathered array, same indexing as Xi_out
    int *peer_status[RAFTK_MAX_PEERS];    // [p]: likewise for status, or NULL
};

struct FSmem {
    double *mem, *node, *coef, *msum, *mat, *warp_part, *sums, *tot, *xi, *f0, *ckpt, *wkey, *hkey, *zkey, *scr, *trans;
    double2 *ebase, *abase, *wtab, *htab;
    int *imem, *node_w, *node_h, *cnt;
};

// The class of one key (NC = 2: (kx, ky) at keys[2c]; NC = 1: x at keys[c]) among the n classes so far, called by all 32
// lanes of one warp with the same arguments: the FIRST class c with |key_c - key| <= tol in every component, else a new
// class keyed by this key (lane 0 stores it), else -- n == maxn -- class 0 and over = 1.  The lanes compare 32 classes at once.
template <int NC>
__device__ __forceinline__ int warp_step_class(double *keys, int &n, int maxn, double x, double y, double tol, int &over)
{
    const int lane = threadIdx.x & 31;
    for (int b = 0; b < n; b += 32) {
        const int c = b + lane;
        const bool hit = c < n && fabs(keys[NC * c] - x) <= tol && (NC == 1 || fabs(keys[NC * c + NC - 1] - y) <= tol);
        const unsigned m = __ballot_sync(0xffffffffu, hit);
        if (m) return b + __ffs(m) - 1;
    }
    if (n == maxn) { over = 1; return 0; }
    if (lane == 0) { keys[NC * n] = x; if (NC == 2) keys[NC * n + NC - 1] = y; }
    __syncwarp();
    return n++;
}

// Step classes of one design (DESIGN.md section 5), by ONE warp: greedy in node order, each node joins the first class
// whose key is within STEP_RTOL of the node's own key or opens a new one (then members' first-node depths likewise).
// Whether a node opens a class depends on every earlier node's, so nodes are taken one at a time; this is the rule the
// host-side hints count (solver.DesignBatch._step_classes, batch_builder._count_classes, raftk_builder.h count_classes),
// so a hint equal to that count never overflows.  Keys per node: kx[j], ky[j], kz[j] (0 at a member's first node);
// z0[m * z0_stride].  Writes the class keys, node_w / node_h = class * nwl (maxW / maxH * nwl: identity row, no step),
// imem[IMEM_STRIDE m + 4] = z class, cnt = {nW, nH, overflow, nZ}; overflow (a class past maxW / maxH / maxZ) means
// RAFTK_FLAG_PLAN: the unit runs no pass.
__device__ __forceinline__ void step_classes_warp(const double *kx, const double *ky, const double *kz, int Ns, const double *z0,
                                               int z0_stride, int Nm, int maxW, int maxH, int maxZ, int nwl, double *wkey,
                                               double *hkey, double *zkey, int *node_w, int *node_h, int *imem, int *cnt)
{
    const int lane = threadIdx.x & 31;
    int nW = 0, nH = 0, nZ = 0, over = 0;
    for (int j = 0; j < Ns; j++) {
        const double x = kx[j], y = ky[j], z = kz[j];
        int wi = maxW, hi = maxH;
        if (fabs(x) > STEP_ZERO || fabs(y) > STEP_ZERO) wi = warp_step_class<2>(wkey, nW, maxW, x, y, STEP_RTOL * (fabs(x) + fabs(y)), over);
        if (fabs(z) > STEP_ZERO) hi = warp_step_class<1>(hkey, nH, maxH, z, 0.0, STEP_RTOL * fabs(z), over);
        if (lane == 0) { node_w[j] = wi * nwl; node_h[j] = hi * nwl; }
    }
    for (int m = 0; m < Nm; m++) {
        const double z = z0[(size_t)m * z0_stride];
        const int zi = warp_step_class<1>(zkey, nZ, maxZ, z, 0.0, Z0_RTOL * fmax(1.0, fabs(z)), over);
        if (lane == 0) imem[IMEM_STRIDE * m + 4] = zi;
    }
    if (lane == 0) { cnt[0] = nW; cnt[1] = nH; cnt[2] = over; cnt[3] = nZ; }
}

__host__ __device__ inline size_t fused_smem_bytes(int Nm, int NsP, int nchunk, int nwarps, int nwl, int maxW, int maxH, int maxZ, bool f0_smem)
{
    size_t dbl = (size_t)Nm * MEM_STRIDE + 4 * (size_t)NsP + 16 + NCOEF * (size_t)NsP + (size_t)Nm * 8 + 108
                 + (size_t)nchunk * nwarps * 32 + 2 * ((size_t)nchunk * 32 + 2) + (size_t)nchunk * 32 + (size_t)nwarps * 16 * 33
                 + (12 + (f0_smem ? 12 : 0) + 4) * (size_t)nwl + 2 * (size_t)maxW + (size_t)maxH + (size_t)maxZ + 3 * (size_t)NsP
                 + 2 * ((size_t)Nm + maxZ + (maxW + 1) + (maxH + 1)) * nwl;       // +1: identity rows of the factor tables
    size_t ints = (size_t)Nm * IMEM_STRIDE + 4 * (size_t)NsP + 40;
    return dbl * sizeof(double) + ints * sizeof(int) + 32;
}

// projection of the wave velocity on direction d plus a body-velocity term: a = E (C h + i S d_z) + m.
// (A 3-way specialisation on exactly horizontal / vertical directions does not pay: ptxas if-converts it
// into predicated code that issues all variants, so the generic 6-flop form is kept.)
__device__ __forceinline__ void proj_add(double er, double ei, double Cc, double Sc, double h, double dz,
                                         double mr, double mi, double &ar, double &ai)
{
    const double gr = Cc * h, gi = Sc * dz;
    ar = fma(er, gr, fma(-ei, gi, mr));
    ai = fma(er, gi, fma(ei, gr, mi));
}
__device__ __forceinline__ void proj(double er, double ei, double Cc, double Sc, double h, double dz, double &cr, double &ci)
{
    const double gr = Cc * h, gi = Sc * dz;
    cr = fma(er, gr, -ei * gi);
    ci = fma(er, gi, ei * gr);
}

template <int T, bool ROT = false>
__global__ void __launch_bounds__(T, 256 / T)
k_rao_fused(DesignsDev D, CasesDev Cs, FusedParams P)
{
    extern __shared__ __align__(16) double smem_raw[];
    cg::cluster_group cluster = cg::this_cluster();
    const int CS = P.CS;
    const int rank = (CS > 1) ? (int)cluster.block_rank() : 0;
    const int unit = blockIdx.x / CS;
    const int d = unit / Cs.nC, c = unit % Cs.nC;
    const int nw = D.nw, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr int nwarps = T / 32;
    // wave trains: a secondary train reuses the linearisation (per-node coefficients, B_drag) of its primary case
    // (raft_model.py:1200-1236); primaries and secondaries run in two launches (cluster-uniform early exit)
    const int prim = (P.phase >= 0 && Cs.primary) ? Cs.primary[c] : c;
    const bool secondary = prim != c;
    if ((P.phase == 0 && secondary) || (P.phase == 1 && !secondary)) return;

    const int m0 = D.member_offset[d], Nm = D.member_offset[d + 1] - m0;
    const int nbase = D.mem_node_start[m0];
    const int Ns = D.mem_node_start[m0 + Nm] - nbase;
    const int NsP = D.max_nodes, NmP = D.max_members;
    const int nchunk = (D.max_nodes + CHUNK_NODES - 1) / CHUNK_NODES;
    const int nwl = P.nwl;
    const int f_begin = rank * nwl;
    const int nloc = max(0, min(nwl, nw - f_begin));

    FSmem S;
    {
        double *p = smem_raw;
        S.ebase = reinterpret_cast<double2 *>(p); p += 2 * (size_t)NmP * nwl;
        S.abase = reinterpret_cast<double2 *>(p); p += 2 * (size_t)P.maxZ * nwl;
        S.wtab = reinterpret_cast<double2 *>(p); p += 2 * (size_t)(P.maxW + 1) * nwl;
        S.htab = reinterpret_cast<double2 *>(p); p += 2 * (size_t)(P.maxH + 1) * nwl;
        S.mem = p; p += (size_t)NmP * MEM_STRIDE;
        S.node = p; p += 4 * (size_t)NsP + 16;
        S.coef = p; p += NCOEF * (size_t)NsP;
        S.msum = p; p += (size_t)NmP * 8;
        S.mat = p; p += 108;
        S.warp_part = p; p += (size_t)nchunk * nwarps * 32;
        S.sums = p; p += 2 * ((size_t)nchunk * 32 + 2);
        S.tot = p; p += (size_t)nchunk * 32;
        S.xi = p; p += 12 * (size_t)nwl;
        S.f0 = p; p += P.F0g ? 0 : 12 * (size_t)nwl;
        S.ckpt = p; p += 4 * (size_t)nwl;
        S.wkey = p; p += 2 * (size_t)P.maxW;
        S.hkey = p; p += (size_t)P.maxH;
        S.zkey = p; p += (size_t)P.maxZ;
        S.scr = p; p += 3 * (size_t)NsP;
        S.trans = p; p += (size_t)nwarps * 16 * 33;
        S.imem = reinterpret_cast<int *>(p);
        S.node_w = S.imem + (size_t)NmP * IMEM_STRIDE;     // per node: offset (class * nwl) of its step factors,
        S.node_h = S.node_w + NsP + 12;                     // identity row for a member's first node / zero steps
        S.cnt = S.node_h + NsP + 12;        // (+12: the node loop prefetches up to 10 entries ahead)
    }
    const int sums_stride = nchunk * 32 + 2;

    // ---- stage design tables ---------------------------------------------------------------------
    const double beta = Cs.beta_deg[c] * (CUDART_PI / 180.0);
    double sb, cb;
    sincos(beta, &sb, &cb);
    for (int m = tid; m < Nm; m += T) {
        const double *fr = D.mem_frame + 9 * (m0 + m);
        const double *arm = D.mem_arm + 3 * (m0 + m);
        double *o = S.mem + m * MEM_STRIDE;
        member_row<true>(o, fr, arm, cb, sb);
        const int js = D.mem_node_start[m0 + m] - nbase;
        S.imem[IMEM_STRIDE * m + 0] = js;
        S.imem[IMEM_STRIDE * m + 1] = D.mem_node_start[m0 + m + 1] - nbase;
        S.imem[IMEM_STRIDE * m + 2] = D.mem_circ[m0 + m];
        S.imem[IMEM_STRIDE * m + 3] = 0;
        o[21] = D.mem_rA[3 * (m0 + m) + 2] + D.node_ls[nbase + js] * fr[2];    // z of the first submerged node
    }
    for (int j = tid; j < NsP; j += T) {
        const bool in = j < Ns;
        S.node[0 * NsP + j] = in ? D.node_ls[nbase + j] : 0.0;
        S.node[1 * NsP + j] = in ? D.node_cd_q[nbase + j] : 0.0;
        S.node[2 * NsP + j] = in ? D.node_cd_p1[nbase + j] : 0.0;
        S.node[3 * NsP + j] = in ? D.node_cd_p2[nbase + j] : 0.0;
    }
    for (int t = tid; t < 36; t += T) {
        S.mat[t] = D.M0[(size_t)d * 36 + t];
        S.mat[72 + t] = D.C0[(size_t)d * 36 + t];
    }
    __syncthreads();
    // ---- step classes: keys per node in parallel, classes by one warp (step_classes_warp) --------------
    for (int j = tid; j < Ns; j += T) {
        int m = 0;
        while (j >= S.imem[IMEM_STRIDE * m + 1]) m++;
        const double *o = S.mem + m * MEM_STRIDE;
        double kx = 0, ky = 0, kz = 0;
        if (j > S.imem[IMEM_STRIDE * m]) {
            const double step = S.node[j] - S.node[j - 1];
            kx = o[0] * step; ky = o[1] * step; kz = o[2] * step;
        }
        S.scr[j] = kx; S.scr[NsP + j] = ky; S.scr[2 * NsP + j] = kz;
    }
    __syncthreads();
    if (warp == 0)
        step_classes_warp(S.scr, S.scr + NsP, S.scr + 2 * NsP, Ns, S.mem + 21, MEM_STRIDE, Nm, P.maxW, P.maxH, P.maxZ, nwl,
                          S.wkey, S.hkey, S.zkey, S.node_w, S.node_h, S.imem, S.cnt);
    for (int j = Ns + tid; j < NsP + 12; j += T) { S.node_w[j] = P.maxW * nwl; S.node_h[j] = P.maxH * nwl; }   // prefetch padding
    __syncthreads();
    const int nW = S.cnt[0], nH = S.cnt[1], nZ = S.cnt[3];
    const bool plan_overflow = S.cnt[2] != 0;

    // ---- prologue per frequency: sea state, member bases, class factors, excitation F0 -----------
    const size_t ogl = ((size_t)d * Cs.nC + c) * 6 * nw;
    for (int t = tid; t < nloc && !plan_overflow; t += T) {
        const int i = f_begin + t;
        const double w = D.w[i], k = D.k[i];
        const double zeta = sea_state_zeta(Cs, c, i, nw, w, D.dw);
        if (P.zeta_out && d == 0) P.zeta_out[(size_t)c * nw + i] = zeta;
        const double zw = zeta * w;
        const bool deep = k * D.depth > 89.4;
        const double tanh_kh = tanh(k * D.depth);
        for (int x = 0; x < nW; x++) {
            double s_, c_;
            sincos(-(k * (S.wkey[2 * x] * cb + S.wkey[2 * x + 1] * sb)), &s_, &c_);
            S.wtab[x * nwl + t] = make_double2(c_, s_);
        }
        for (int x = 0; x < nH; x++) {
            const double a = k * S.hkey[x];
            S.htab[x * nwl + t] = make_double2(exp(a), exp(-a));
        }
        S.wtab[P.maxW * nwl + t] = make_double2(1.0, 0.0);
        S.htab[P.maxH * nwl + t] = make_double2(1.0, 1.0);
        for (int x = 0; x < nZ; x++) {
            double S_, C_, P_;
            depth_funcs(k, D.depth, S.zkey[x], S_, C_, P_);
            S.abase[x * nwl + t] = make_double2(0.5 * (C_ + S_), 0.5 * (C_ - S_));
        }
        double Fr[6] = {0, 0, 0, 0, 0, 0}, Fi[6] = {0, 0, 0, 0, 0, 0};
        for (int m = 0; m < Nm; m++) {
            const double *o = S.mem + m * MEM_STRIDE;
            const int j0 = S.imem[IMEM_STRIDE * m], j1 = S.imem[IMEM_STRIDE * m + 1];
            const double *rA = D.mem_rA + 3 * (m0 + m);
            const double ls0 = S.node[j0];
            const double x0 = rA[0] + ls0 * o[0], y0 = rA[1] + ls0 * o[1];
            double se, ce;
            sincos(-(k * (cb * x0 + sb * y0)), &se, &ce);
            double er = zw * ce, ei = zw * se;
            S.ebase[m * nwl + t] = make_double2(er, ei);
            const double2 a0 = S.abase[S.imem[IMEM_STRIDE * m + 4] * nwl + t];
            double ap = a0.x, am = a0.y;
            const double hq = o[18], h1 = o[19], h2 = o[20];
            double Aqr = 0, Aqi = 0, A1r = 0, A1i = 0, A2r = 0, A2i = 0, L1r = 0, L1i = 0, L2r = 0, L2i = 0;
            for (int j = j0; j < j1; j++) {
                {   // step factors (identity at the member's first node)
                    const double2 W = S.wtab[S.node_w[j] + t], H = S.htab[S.node_h[j] + t];
                    const double tr = fma(er, W.x, -ei * W.y); ei = fma(er, W.y, ei * W.x); er = tr;
                    ap *= H.x; am *= H.y;
                }
                const int jg = nbase + j;
                const double inq = D.node_in_q[jg], pa = D.node_pa[jg];
                double in1 = D.node_in_p1[jg], in2 = D.node_in_p2[jg], in1i = 0.0, in2i = 0.0;
                if (D.node_in_p1_w) {
                    const double2 v1 = D.node_in_p1_w[(size_t)jg * nw + i], v2 = D.node_in_p2_w[(size_t)jg * nw + i];
                    in1 = v1.x; in1i = v1.y; in2 = v2.x; in2i = v2.y;
                }
                if (inq != 0.0 || in1 != 0.0 || in2 != 0.0 || in1i != 0.0 || in2i != 0.0 || pa != 0.0) {
                    const double ls = S.node[j], Cc = ap + am, Sc = ap - am;
                    double cr, ci;
                    proj(er, ei, Cc, Sc, hq, o[2], cr, ci);
                    double fqr = -w * inq * ci, fqi = w * inq * cr;
                    proj(er, ei, Cc, Sc, h1, o[5], cr, ci);
                    const double f1r = -w * (in1 * ci + in1i * cr), f1i = w * (in1 * cr - in1i * ci);
                    proj(er, ei, Cc, Sc, h2, o[8], cr, ci);
                    const double f2r = -w * (in2 * ci + in2i * cr), f2i = w * (in2 * cr - in2i * ci);
                    if (pa != 0.0 && w != 0.0) {
                        // dynamic pressure: P = cosh(k(z+h))/cosh(kh) = C tanh(kh); deep-water branch of helpers.py:218
                        double Pd = Cc * tanh_kh;
                        if (deep) Pd = Cc + exp(-k * (rA[2] + ls * o[2] + 2.0 * D.depth));
                        const double sc = pa * Pd / w;
                        fqr = fma(sc, er, fqr); fqi = fma(sc, ei, fqi);
                    }
                    Aqr += fqr; Aqi += fqi; A1r += f1r; A1i += f1i; A2r += f2r; A2i += f2i;
                    L1r += ls * f1r; L1i += ls * f1i; L2r += ls * f2r; L2i += ls * f2i;
                }
            }
            member_force6(o, Aqr, Aqi, A1r, A1i, A2r, A2i, L1r, L1i, L2r, L2i, Fr, Fi);
        }
        excitation_sum<ROT>(D, Cs, P, d, c, ogl, nw, i, k, beta, sb, cb, [&] { return zeta; }, Fr, Fi);
#pragma unroll
        for (int a = 0; a < 6; a++) {
            if (P.F0g) P.F0g[ogl + (size_t)a * nw + i] = make_double2(Fr[a], Fi[a]);
            else { S.f0[(2 * a) * nwl + t] = Fr[a]; S.f0[(2 * a + 1) * nwl + t] = Fi[a]; }
            if (P.Xi_init) { const double2 x0 = P.Xi_init[ogl + (size_t)a * nw + i]; S.xi[(2 * a) * nwl + t] = x0.x; S.xi[(2 * a + 1) * nwl + t] = x0.y; }
            else { S.xi[(2 * a) * nwl + t] = P.xi_start; S.xi[(2 * a + 1) * nwl + t] = 0.0; }
        }
    }
    if (plan_overflow) zero_unit_outputs<T>(P.Xi_out, P.Xilast_out, ogl, nw, f_begin, nloc);
    __syncthreads();

    const double *Aw = D.A_w ? D.A_w + (size_t)d * 36 * nw : nullptr;
    const double *Bw = D.B_w ? D.B_w + (size_t)d * 36 * nw : nullptr;
    int passes = 0, converged = 0, flags = plan_overflow ? RAFTK_FLAG_PLAN : 0, par = 0;
    const int max_pass = plan_overflow ? 0 : (secondary ? 1 : P.n_iter + 1);
    const size_t lin_stride = (size_t)NCOEF * NsP + 36;
    if (secondary && !plan_overflow) {          // frozen linearisation of the primary case
        const double *src = P.lin_g + ((size_t)d * Cs.nC + prim) * lin_stride;
        for (int t = tid; t < NCOEF * NsP; t += T) S.coef[t] = src[t];
        for (int t = tid; t < 36; t += T) S.mat[36 + t] = src[NCOEF * NsP + t];
        __syncthreads();
    }

    for (int it = 0; it < max_pass; it++) {
        if (!secondary) {
        // ================= pass part 1: sum_w |v_rel . d|^2 per node and direction =================
        for (int ch = 0; ch < nchunk; ch++) {
            double acc[32];
#pragma unroll
            for (int t = 0; t < 32; t++) acc[t] = 0.0;
            const int jc0 = ch * CHUNK_NODES;
            if (jc0 < Ns) {
                for (int t = tid; t < nloc; t += T) {
                    const double w = D.w[f_begin + t];
                    double xr[6], xi[6];
#pragma unroll
                    for (int a = 0; a < 6; a++) { xr[a] = S.xi[(2 * a) * nwl + t]; xi[a] = S.xi[(2 * a + 1) * nwl + t]; }
                    // walking state: restored from the checkpoint when the chunk starts inside a member
                    double er = S.ckpt[t], ei = S.ckpt[nwl + t], ap = S.ckpt[2 * nwl + t], am = S.ckpt[3 * nwl + t];
                    const double2 *wt_ = S.wtab + t, *ht_ = S.htab + t;
                    int mcur = -1, jj = 0;
                    while (jj < CHUNK_NODES && jc0 + jj < Ns) {
                        // (uniform) member entry: member-level projections of the body velocity, -i w (d . Xi_t + (a x d) . Xi_r)
                        const int jfirst = jc0 + jj;
                        do { mcur++; } while (jfirst >= S.imem[IMEM_STRIDE * mcur + 1]);
                        const int mstart = S.imem[IMEM_STRIDE * mcur], jlast = S.imem[IMEM_STRIDE * mcur + 1] - jc0;
                        const double *o = S.mem + mcur * MEM_STRIDE;
                        double mqr, mqi, m1r, m1i, m2r, m2i, t1r, t1i, t2r, t2i;
                        member_velocity(o, xr, xi, w, mqr, mqi, m1r, m1i, m2r, m2i, t1r, t1i, t2r, t2i);
                        const double hq = o[18], h1 = o[19], h2 = o[20], dzq = o[2], dz1 = o[5], dz2 = o[8];
                        if (jfirst == mstart) {
                            const double2 e0 = S.ebase[mcur * nwl + t], a0 = S.abase[S.imem[IMEM_STRIDE * mcur + 4] * nwl + t];
                            er = e0.x; ei = e0.y; ap = a0.x; am = a0.y;
                        }
                        // node body: branch-free; the step factors / ls of node JJ were loaded one node earlier
                        // (CUR set) and those of node JJ+1 are requested first (NXT set), so the shared-memory
                        // latency overlaps the arithmetic of this node.  Sets alternate with the parity of JJ.
#define P1_NODE(JJ, CW, CH, CL, NW, NH, NL)                                                                        \
    {                                                                                                                \
        const int jn = jc0 + JJ + 1;                                                                                 \
        NW = wt_[S.node_w[jn]]; NH = ht_[S.node_h[jn]]; NL = S.node[jn];                                             \
        { const double tr = fma(er, CW.x, -ei * CW.y); ei = fma(er, CW.y, ei * CW.x); er = tr; }                     \
        ap *= CH.x; am *= CH.y;                                                                                      \
        const double ls = CL, Cc = ap + am, Sc = ap - am;                                                            \
        double ar_, ai_;                                                                                             \
        proj_add(er, ei, Cc, Sc, hq, dzq, mqr, mqi, ar_, ai_);                                                   \
        acc[3 * JJ + 0] = fma(ar_, ar_, fma(ai_, ai_, acc[3 * JJ + 0]));                                             \
        proj_add(er, ei, Cc, Sc, h1, dz1, fma(ls, t2r, m1r), fma(ls, t2i, m1i), ar_, ai_);                       \
        acc[3 * JJ + 1] = fma(ar_, ar_, fma(ai_, ai_, acc[3 * JJ + 1]));                                             \
        proj_add(er, ei, Cc, Sc, h2, dz2, fma(-ls, t1r, m2r), fma(-ls, t1i, m2i), ar_, ai_);                     \
        acc[3 * JJ + 2] = fma(ar_, ar_, fma(ai_, ai_, acc[3 * JJ + 2]));                                             \
    }
                        // Duff-style dispatch: one copy of each node body (static accumulator index), re-entered per member
                        double2 Wa, Ha, Wb, Hb; double La, Lb;
                        if (jj & 1) { Wb = wt_[S.node_w[jfirst]]; Hb = ht_[S.node_h[jfirst]]; Lb = S.node[jfirst]; Wa = Wb; Ha = Hb; La = Lb; }
                        else        { Wa = wt_[S.node_w[jfirst]]; Ha = ht_[S.node_h[jfirst]]; La = S.node[jfirst]; Wb = Wa; Hb = Ha; Lb = La; }
                        switch (jj) {
                        case 0: P1_NODE(0, Wa, Ha, La, Wb, Hb, Lb); jj = 1; if (jlast <= 1) break;
                        case 1: P1_NODE(1, Wb, Hb, Lb, Wa, Ha, La); jj = 2; if (jlast <= 2) break;
                        case 2: P1_NODE(2, Wa, Ha, La, Wb, Hb, Lb); jj = 3; if (jlast <= 3) break;
                        case 3: P1_NODE(3, Wb, Hb, Lb, Wa, Ha, La); jj = 4; if (jlast <= 4) break;
                        case 4: P1_NODE(4, Wa, Ha, La, Wb, Hb, Lb); jj = 5; if (jlast <= 5) break;
                        case 5: P1_NODE(5, Wb, Hb, Lb, Wa, Ha, La); jj = 6; if (jlast <= 6) break;
                        case 6: P1_NODE(6, Wa, Ha, La, Wb, Hb, Lb); jj = 7; if (jlast <= 7) break;
                        case 7: P1_NODE(7, Wb, Hb, Lb, Wa, Ha, La); jj = 8; if (jlast <= 8) break;
                        case 8: P1_NODE(8, Wa, Ha, La, Wb, Hb, Lb); jj = 9; if (jlast <= 9) break;
                        case 9: P1_NODE(9, Wb, Hb, Lb, Wa, Ha, La); jj = 10;
                        }
#undef P1_NODE
                    }
                    S.ckpt[t] = er; S.ckpt[nwl + t] = ei; S.ckpt[2 * nwl + t] = ap; S.ckpt[3 * nwl + t] = am;
                }
            }
            // warp sum of the 30 accumulators through a padded shared-memory transpose (16 values at a time):
            // every lane stores its values, then lane l adds 16 lanes' worth of value (l & 15) -- fixed order.
            {
                double *tr = S.trans + warp * (16 * 33);
                const int row = lane & 15, part = lane >> 4;
#pragma unroll
                for (int half = 0; half < 2; half++) {
#pragma unroll
                    for (int v = 0; v < 16; v++) tr[v * 33 + lane] = acc[half * 16 + v];
                    __syncwarp();
                    double sum = 0.0;
#pragma unroll
                    for (int x = 0; x < 16; x++) sum += tr[row * 33 + part * 16 + x];
                    sum += __shfl_xor_sync(0xffffffffu, sum, 16);
                    if (lane < 16) S.warp_part[(ch * nwarps + warp) * 32 + half * 16 + lane] = sum;
                    __syncwarp();
                }
            }
        }
        __syncthreads();
        rms_exchange<T>(cluster, CS, nchunk, par, sums_stride, S.warp_part, S.sums, S.tot);

        // ================= linearised coefficients per node, member sums, B_drag ===================
        for (int j = tid; j < Ns; j += T) {
            const int ch = j / CHUNK_NODES, jj = j - ch * CHUNK_NODES;
            const double sq = S.tot[ch * 32 + 3 * jj], s1 = S.tot[ch * 32 + 3 * jj + 1], s2 = S.tot[ch * 32 + 3 * jj + 2];
            int m = 0;
            while (j >= S.imem[IMEM_STRIDE * m + 1]) m++;
            double vq, v1, v2;
            drag_rms(sq, s1, s2, S.imem[IMEM_STRIDE * m + 2] != 0, vq, v1, v2);
            const double ls = S.node[j], b1 = S.node[2 * NsP + j] * v1, b2 = S.node[3 * NsP + j] * v2;
            S.coef[0 * NsP + j] = S.node[1 * NsP + j] * vq;
            S.coef[1 * NsP + j] = b1; S.coef[2 * NsP + j] = ls * b1;
            S.coef[3 * NsP + j] = b2; S.coef[4 * NsP + j] = ls * b2;
        }
        __syncthreads();
        drag_member_sums<T, IMEM_STRIDE>(Nm, S.imem, S.node, S.coef, 0, NsP, 3 * NsP, S.msum);
        __syncthreads();
        if (tid < 36) {
            const double s = drag_bmat_entry(tid, Nm, S.mem, S.msum);
            S.mat[36 + tid] = D.B0[(size_t)d * 36 + tid] + s;
            if (P.Bdrag_out && rank == 0) P.Bdrag_out[((size_t)d * Cs.nC + c) * 36 + tid] = s;
        }
        __syncthreads();
        if (P.lin_g && P.phase == 0 && rank == 0) {      // hand the linearisation over to the secondary wave trains
            double *dst = P.lin_g + ((size_t)d * Cs.nC + c) * lin_stride;
            for (int t = tid; t < NCOEF * NsP; t += T) dst[t] = S.coef[t];
            for (int t = tid; t < 36; t += T) dst[NCOEF * NsP + t] = S.mat[36 + t];
        }
        }   // !secondary

        // ================= pass part 2: drag excitation, impedance, solve, convergence =============
        int conv_local = 1, nan_local = 0;
        const double *cq_ = S.coef, *c1_ = S.coef + NsP, *cl1_ = S.coef + 2 * NsP, *c2_ = S.coef + 3 * NsP, *cl2_ = S.coef + 4 * NsP;
        for (int t = tid; t < nloc; t += T) {
            const int i = f_begin + t;
            const double w = D.w[i];
            const double2 *wt_ = S.wtab + t, *ht_ = S.htab + t;
            double br[6], bi[6];
#pragma unroll
            for (int a = 0; a < 6; a++) { br[a] = 0.0; bi[a] = 0.0; }
            for (int m = 0; m < Nm; m++) {
                const double *o = S.mem + m * MEM_STRIDE;
                const double hq = o[18], h1 = o[19], h2 = o[20], dzq = o[2], dz1 = o[5], dz2 = o[8];
                double Aqr = 0, Aqi = 0, A1r = 0, A1i = 0, A2r = 0, A2i = 0, L1r = 0, L1i = 0, L2r = 0, L2i = 0;
                const int j0 = S.imem[IMEM_STRIDE * m], j1 = S.imem[IMEM_STRIDE * m + 1];
                const double2 e0 = S.ebase[m * nwl + t], a0 = S.abase[S.imem[IMEM_STRIDE * m + 4] * nwl + t];
                double er = e0.x, ei = e0.y, ap = a0.x, am = a0.y;
#pragma unroll 2
                for (int j = j0; j < j1; j++) {
                    {
                        const double2 W = wt_[S.node_w[j]], H = ht_[S.node_h[j]];
                        const double tr = fma(er, W.x, -ei * W.y); ei = fma(er, W.y, ei * W.x); er = tr;
                        ap *= H.x; am *= H.y;
                    }
                    const double bq = cq_[j], b1 = c1_[j], lb1 = cl1_[j], b2 = c2_[j], lb2 = cl2_[j];
                    const double Cc = ap + am, Sc = ap - am;
                    double cr, ci;
                    proj(er, ei, Cc, Sc, hq, dzq, cr, ci);
                    Aqr = fma(bq, cr, Aqr); Aqi = fma(bq, ci, Aqi);
                    proj(er, ei, Cc, Sc, h1, dz1, cr, ci);
                    A1r = fma(b1, cr, A1r); A1i = fma(b1, ci, A1i); L1r = fma(lb1, cr, L1r); L1i = fma(lb1, ci, L1i);
                    proj(er, ei, Cc, Sc, h2, dz2, cr, ci);
                    A2r = fma(b2, cr, A2r); A2i = fma(b2, ci, A2i); L2r = fma(lb2, cr, L2r); L2i = fma(lb2, ci, L2i);
                }
                member_force6(o, Aqr, Aqi, A1r, A1i, A2r, A2i, L1r, L1i, L2r, L2i, br, bi);
            }
            if (P.Fdrag_out) {
#pragma unroll
                for (int a = 0; a < 6; a++) P.Fdrag_out[ogl + (size_t)a * nw + i] = make_double2(br[a], bi[a]);
            }
            double ar[6][6], ai[6][6];
            if (P.F0g) {
#pragma unroll
                for (int a = 0; a < 6; a++) { const double2 f = P.F0g[ogl + (size_t)a * nw + i]; br[a] += f.x; bi[a] += f.y; }
            } else {
#pragma unroll
                for (int a = 0; a < 6; a++) { br[a] += S.f0[(2 * a) * nwl + t]; bi[a] += S.f0[(2 * a + 1) * nwl + t]; }
            }
            const double w2 = w * w;
            if (Cs.op) {                   // the case's operating point (per-case aero-servo terms) on top of the design's tables
                const double *Ao = op_table(Cs, Cs.op_A_w, d, c, nw), *Bo = op_table(Cs, Cs.op_B_w, d, c, nw);
                if (Aw) op_impedance<true>(ar, ai, S.mat, S.mat + 36, S.mat + 72, Aw, Bw, Ao, Bo, i, nw, w, w2);
                else op_impedance<false>(ar, ai, S.mat, S.mat + 36, S.mat + 72, nullptr, nullptr, Ao, Bo, i, nw, w, w2);
            } else {
                impedance(ar, ai, S.mat, S.mat + 36, S.mat + 72, Aw, Bw, i, nw, w, w2);
            }
            const bool ok = solve6(ar, ai, br, bi);
            if (!ok) nan_local |= RAFTK_FLAG_SINGULAR;
#pragma unroll
            for (int a = 0; a < 6; a++) {
                const double lr = S.xi[(2 * a) * nwl + t], li = S.xi[(2 * a + 1) * nwl + t];
                if (isnan(br[a]) || isnan(bi[a])) nan_local |= RAFTK_FLAG_NAN;
                const double dr = br[a] - lr, di = bi[a] - li;
                // raft_model.py:1103: |d| / (|x| + tol) < tol  <=>  |d| < tol |x| + tol^2   (no division;
                // same decision up to the last ulp)
                if (!(sqrt(dr * dr + di * di) < fma(P.tol, sqrt(br[a] * br[a] + bi[a] * bi[a]), P.tol * P.tol))) conv_local = 0;
                S.xi[(2 * a) * nwl + t] = 0.2 * lr + 0.8 * br[a];
                S.xi[(2 * a + 1) * nwl + t] = 0.2 * li + 0.8 * bi[a];
                P.Xi_out[ogl + (size_t)a * nw + i] = make_double2(br[a], bi[a]);
                if (P.Xilast_out) P.Xilast_out[ogl + (size_t)a * nw + i] = make_double2(lr, li);
            }
        }
        passes++;
        int conv_all, nan_all;
        flags_exchange(cluster, CS, nchunk, par, sums_stride, conv_local, nan_local, S.sums, conv_all, nan_all);
        par ^= 1;
        flags |= nan_all;
        if (nan_all & RAFTK_FLAG_NAN) break;
        if (conv_all) { converged = 1; break; }
    }
    unit_epilogue<T, 4>(P, d, c, Cs.nC, rank, ogl, nw, f_begin, nloc, passes, converged, flags, secondary, prim);
    if (CS > 1) cluster.sync();
}
