// raftk_rigid.cuh -- the steps the rigid FOWT solvers share around their node walks: member rows, body-velocity projections,
// member-to-6-DOF force sums, the linear excitation's sum, getRMS, B_drag, the unit epilogue and the cluster exchanges.  Used
// by k_drag_solve (raftk_tables.cuh), k_rao_fused (raftk_fused.cuh), k_fused_plan and k_rao_fused2 (raftk_fused2.cuh);
// included by raftk.cu only.  Each helper keeps the expressions and the order of operations of every caller, so the results
// are bit for bit those of the copies it replaced; where the kernels differ (convergence test and relaxation loop, dynamic-
// pressure exponent, node walks, loop unrolling) the difference stays in the kernel or is a parameter.
#pragma once

#define IMEM_STRIDE 6      // ints per member in the fused solvers: node start, node end, circular, (spare), z-class, (spare)
#define NCOEF 5            // per-node linearised coefficients: bq, b1, ls*b1, b2, ls*b2

// Heading projection h_d = d_x cos b + d_y sin b of frame direction d (per case)
__device__ __forceinline__ double heading_proj(double dx, double dy, double cb, double sb) { return dx * cb + dy * sb; }

// Member row (MEM_STRIDE doubles) from the design's frame fr and lever arm: the frame q, p1, p2 at [0, 9), the lever-arm
// products a x q, a x p1, a x p2 at [9, 18) and, with HEADINGS, the heading projections h_q, h_1, h_2 at [18, 21)
template <bool HEADINGS>
__device__ __forceinline__ void member_row(double *o, const double *fr, const double *arm, double cb = 0.0, double sb = 0.0)
{
    for (int t = 0; t < 9; t++) o[t] = fr[t];
    for (int v = 0; v < 3; v++) {
        const double d0_ = fr[3 * v], d1_ = fr[3 * v + 1], d2_ = fr[3 * v + 2];
        o[9 + 3 * v + 0] = arm[1] * d2_ - arm[2] * d1_;
        o[9 + 3 * v + 1] = arm[2] * d0_ - arm[0] * d2_;
        o[9 + 3 * v + 2] = arm[0] * d1_ - arm[1] * d0_;
        if (HEADINGS) o[18 + v] = heading_proj(d0_, d1_, cb, sb);
    }
}

// Member-level projections of the body velocity at frequency w, -i w (d . Xi_t + (a x d) . Xi_r) for d = q, p1, p2 (mq, m1,
// m2), and -i w (d . Xi_r) for d = p1, p2 (t1, t2: the rotation terms that the node's distance ls along the member scales)
__device__ __forceinline__ void member_velocity(const double *o, const double (&xr)[6], const double (&xi)[6], double w,
                                                double &mqr, double &mqi, double &m1r, double &m1i, double &m2r, double &m2i,
                                                double &t1r, double &t1i, double &t2r, double &t2i)
{
    double sr, si;
    sr = o[0] * xr[0] + o[1] * xr[1] + o[2] * xr[2] + o[9] * xr[3] + o[10] * xr[4] + o[11] * xr[5];
    si = o[0] * xi[0] + o[1] * xi[1] + o[2] * xi[2] + o[9] * xi[3] + o[10] * xi[4] + o[11] * xi[5];
    mqr = w * si; mqi = -w * sr;
    sr = o[3] * xr[0] + o[4] * xr[1] + o[5] * xr[2] + o[12] * xr[3] + o[13] * xr[4] + o[14] * xr[5];
    si = o[3] * xi[0] + o[4] * xi[1] + o[5] * xi[2] + o[12] * xi[3] + o[13] * xi[4] + o[14] * xi[5];
    m1r = w * si; m1i = -w * sr;
    sr = o[6] * xr[0] + o[7] * xr[1] + o[8] * xr[2] + o[15] * xr[3] + o[16] * xr[4] + o[17] * xr[5];
    si = o[6] * xi[0] + o[7] * xi[1] + o[8] * xi[2] + o[15] * xi[3] + o[16] * xi[4] + o[17] * xi[5];
    m2r = w * si; m2i = -w * sr;
    sr = o[3] * xr[3] + o[4] * xr[4] + o[5] * xr[5];     // p1 . Xi_r
    si = o[3] * xi[3] + o[4] * xi[4] + o[5] * xi[5];
    t1r = w * si; t1i = -w * sr;
    sr = o[6] * xr[3] + o[7] * xr[4] + o[8] * xr[5];     // p2 . Xi_r
    si = o[6] * xi[3] + o[7] * xi[4] + o[8] * xi[5];
    t2r = w * si; t2i = -w * sr;
}

// One member's factored force sums onto the 6 DOFs, added to (Fr, Fi): Aq, A1, A2 are the sums of the node forces along q,
// p1, p2; L1, L2 the same sums weighted by ls (the moment of a transverse force about the member's reference point)
__device__ __forceinline__ void member_force6(const double *o, double Aqr, double Aqi, double A1r, double A1i, double A2r, double A2i,
                                              double L1r, double L1i, double L2r, double L2i, double (&Fr)[6], double (&Fi)[6])
{
#pragma unroll
    for (int a = 0; a < 3; a++) {
        Fr[a] += o[a] * Aqr + o[3 + a] * A1r + o[6 + a] * A2r;
        Fi[a] += o[a] * Aqi + o[3 + a] * A1i + o[6 + a] * A2i;
        Fr[3 + a] += o[9 + a] * Aqr + o[12 + a] * A1r + o[15 + a] * A2r + o[6 + a] * L1r - o[3 + a] * L2r;
        Fi[3 + a] += o[9 + a] * Aqi + o[12 + a] * A1i + o[15 + a] * A2i + o[6 + a] * L1i - o[3 + a] * L2i;
    }
}

// getRMS (helpers.py:684) of one node from its sums over frequency of |v_rel . d|^2 along q, p1, p2: sqrt(0.5 * sum);
// circular members use the total transverse RMS in both transverse directions
__device__ __forceinline__ void drag_rms(double sq, double s1, double s2, bool circ, double &vq, double &v1, double &v2)
{
    vq = sqrt(0.5 * sq);
    v1 = circ ? sqrt(0.5 * (s1 + s2)) : sqrt(0.5 * s1);
    v2 = circ ? v1 : sqrt(0.5 * s2);
}

// Per-member sums of the node drag coefficients, by the CTA's T threads: msum[8 m + 0..6] = sum bq, sum b1, sum b1 ls,
// sum b1 ls^2, sum b2, sum b2 ls, sum b2 ls^2 over member m's nodes [imem[IS m], imem[IS m + 1]).  Node j's ls is ls_[j], its
// coefficients bq, b1, b2 are col[oq + j], col[o1 + j], col[o2 + j].
template <int T, int IS>
__device__ __forceinline__ void drag_member_sums(int Nm, const int *imem, const double *ls_, const double *col, int oq, int o1, int o2,
                                                 double *msum)
{
    for (int m = threadIdx.x; m < Nm; m += T) {
        double bq = 0, b1 = 0, b1l = 0, b1ll = 0, b2 = 0, b2l = 0, b2ll = 0;
        for (int j = imem[IS * m]; j < imem[IS * m + 1]; j++) {
            const double ls = ls_[j], q_ = col[oq + j], p1_ = col[o1 + j], p2_ = col[o2 + j];
            bq += q_; b1 += p1_; b1l += p1_ * ls; b1ll += p1_ * ls * ls; b2 += p2_; b2l += p2_ * ls; b2ll += p2_ * ls * ls;
        }
        double *o = msum + m * 8;
        o[0] = bq; o[1] = b1; o[2] = b1l; o[3] = b1ll; o[4] = b2; o[5] = b2l; o[6] = b2ll;
    }
}

// Entry e = 6 a + b of B_drag from the member rows and their drag sums (drag_member_sums)
__device__ __forceinline__ double drag_bmat_entry(int e, int Nm, const double *mem, const double *msum)
{
    const int a = e / 6, b = e % 6;
    double s = 0.0;
    for (int m = 0; m < Nm; m++) {
        const double *o = mem + m * MEM_STRIDE, *ms = msum + m * 8;
        // V_q = [q ; a x q]; V_1 = [p1 ; a x p1] + ls [0 ; p2]; V_2 = [p2 ; a x p2] - ls [0 ; p1]
        const double vqa = a < 3 ? o[a] : o[9 + a - 3], vqb = b < 3 ? o[b] : o[9 + b - 3];
        const double v1a = a < 3 ? o[3 + a] : o[12 + a - 3], v1b = b < 3 ? o[3 + b] : o[12 + b - 3];
        const double v2a = a < 3 ? o[6 + a] : o[15 + a - 3], v2b = b < 3 ? o[6 + b] : o[15 + b - 3];
        const double u1a = a < 3 ? 0.0 : o[6 + a - 3], u1b = b < 3 ? 0.0 : o[6 + b - 3];       // +p2
        const double u2a = a < 3 ? 0.0 : -o[3 + a - 3], u2b = b < 3 ? 0.0 : -o[3 + b - 3];     // -p1
        s += ms[0] * vqa * vqb;
        s += ms[1] * v1a * v1b + ms[2] * (v1a * u1b + u1a * v1b) + ms[3] * u1a * u1b;
        s += ms[4] * v2a * v2b + ms[5] * (v2a * u2b + u2a * v2b) + ms[6] * u2a * u2b;
    }
    return s;
}

// The fused solvers' linear excitation of a unit at bin i, in place (P: FusedParams): Fr + i Fi comes in as the strip
// inertial and dynamic-pressure force, which goes to P.Finer_out; the BEM excitation (bem_excitation, raftk_tables.cuh) goes
// to P.Fbem_out (zeros without BEM tables) and is added, and so is the second-order force (raft_model.py:1048, :1212).
// zeta() gives the bin's wave amplitude; only the BEM and rotor terms evaluate it.  ROT: the designs carry submerged rotors,
// whose excitation (rotor_excitation, raftk_tables.cuh) joins the inertial force first; a template flag, so that the solves
// without rotors compile as before.
template <bool ROT, class Params, class Zeta>
__device__ __forceinline__ void excitation_sum(const DesignsDev &D, const CasesDev &Cs, const Params &P, int d, int c, size_t ogl, int nw,
                                               int i, double k, double beta, double sb, double cb, Zeta zeta, double (&Fr)[6], double (&Fi)[6])
{
    if constexpr (ROT) rotor_excitation(D, Cs, d, c, i, k, D.w[i], beta, sb, cb, zeta(), Fr, Fi);
    if (P.Finer_out)
        for (int a = 0; a < 6; a++) P.Finer_out[ogl + (size_t)a * nw + i] = make_double2(Fr[a], Fi[a]);
    if (D.n_bem_head > 0) {
        double Br[6], Bi[6];
        bem_excitation(D, d, i, k, beta, sb, cb, zeta(), Br, Bi);
#pragma unroll
        for (int a = 0; a < 6; a++) {
            if (P.Fbem_out) P.Fbem_out[ogl + (size_t)a * nw + i] = make_double2(Br[a], Bi[a]);
            Fr[a] += Br[a]; Fi[a] += Bi[a];
        }
    } else if (P.Fbem_out) {
        for (int a = 0; a < 6; a++) P.Fbem_out[ogl + (size_t)a * nw + i] = make_double2(0.0, 0.0);
    }
    if (Cs.F_2nd) {
#pragma unroll
        for (int a = 0; a < 6; a++) Fr[a] += Cs.F_2nd[ogl + (size_t)a * nw + i];
    }
}

// A unit whose step classes overflowed runs no pass: zero this CTA's slice of Xi (and Xi_last), so that the outputs never
// hand back whatever the buffers held before
template <int T>
__device__ __forceinline__ void zero_unit_outputs(double2 *Xi_out, double2 *Xilast_out, size_t ogl, int nw, int f_begin, int nloc)
{
    const int tid = threadIdx.x;
    for (int t = tid; t < nloc; t += T)
        for (int a = 0; a < 6; a++) Xi_out[ogl + (size_t)a * nw + f_begin + t] = make_double2(0.0, 0.0);
    if (Xilast_out)
        for (int t = tid; t < 6 * nloc; t += T) Xilast_out[ogl + (size_t)(t / nloc) * nw + f_begin + t % nloc] = make_double2(0.0, 0.0);
}

// Status row of a unit: passes, converged, flags, and primary case + 1 for a secondary wave train (which reports 0 passes,
// converged)
__device__ __forceinline__ void store_status(int *st, int passes, int converged, int flags, bool secondary, int prim)
{
    st[0] = secondary ? 0 : passes; st[1] = secondary ? 1 : converged; st[2] = flags; st[3] = secondary ? prim + 1 : 0;
}

// Unit epilogue of the fused solvers (P: FusedParams): the status row, and with several GPUs the unit's final Xi slice and
// status pushed to every peer's gathered arrays.  Each thread re-reads the Xi values it stored itself in the last pass (L2
// hits); the peer stores are fire-and-forget and overlap the units still iterating.  PEER_UNROLL: the unroll factor of the
// loops over peers (k_rao_fused2 keeps them rolled, its instruction cache holds the pass loop).
template <int T, int PEER_UNROLL, class Params>
__device__ __forceinline__ void unit_epilogue(const Params &P, int d, int c, int nC, int rank, size_t ogl, int nw, int f_begin,
                                              int nloc, int passes, int converged, int flags, bool secondary, int prim)
{
    const int tid = threadIdx.x;
    if (P.status && rank == 0 && tid == 0)
        store_status(P.status + ((size_t)d * nC + c) * 4, passes, converged, flags, secondary, prim);
    if (P.n_peers > 1) {
        for (int t = tid; t < nloc; t += T) {
            const int i = f_begin + t;
#pragma unroll
            for (int a = 0; a < 6; a++) {
                const size_t o_ = ogl + (size_t)a * nw + i;
                const double2 v = P.Xi_out[o_];
#pragma unroll PEER_UNROLL
                for (int p = 0; p < P.n_peers; p++)
                    if (p != P.peer_rank) P.peer_Xi[p][o_] = v;
            }
        }
        if (rank == 0 && tid == 0) {
            const size_t so = ((size_t)d * nC + c) * 4;
#pragma unroll PEER_UNROLL
            for (int p = 0; p < P.n_peers; p++)
                if (p != P.peer_rank && P.peer_status[p]) store_status(P.peer_status[p] + so, passes, converged, flags, secondary, prim);
        }
    }
}

// Per-node RMS sums of one pass, by the CTA's T threads: the warps' partials warp_part [nchunk][T/32][32] are summed into
// this CTA's row sums[par * sums_stride + ...] (double buffered by pass parity), then the rows of the CS CTAs of the unit's
// cluster are summed in rank order into tot [nchunk * 32]
template <int T>
__device__ __forceinline__ void rms_exchange(cg::cluster_group &cluster, int CS, int nchunk, int par, int sums_stride,
                                             const double *warp_part, double *sums, double *tot)
{
    constexpr int nwarps = T / 32;
    const int tid = threadIdx.x;
    for (int t = tid; t < nchunk * 32; t += T) {
        const int ch = t >> 5, l = t & 31;
        double s = 0.0;
        for (int wv = 0; wv < nwarps; wv++) s += warp_part[(ch * nwarps + wv) * 32 + l];
        sums[par * sums_stride + t] = s;
    }
    if (CS > 1) {
        cluster.sync();
        for (int t = tid; t < nchunk * 32; t += T) {
            double s = 0.0;
            for (int r = 0; r < CS; r++) {
                const double *rem = cluster.map_shared_rank(sums, r);
                s += rem[par * sums_stride + t];
            }
            tot[t] = s;
        }
    } else {
        __syncthreads();
        for (int t = tid; t < nchunk * 32; t += T) tot[t] = sums[par * sums_stride + t];
    }
    __syncthreads();
}

// All-reduce of a pass's (converged, flags) over the CTA and the unit's cluster, through the two words after the RMS
// partials in every rank's row of sums (rms_exchange)
__device__ __forceinline__ void flags_exchange(cg::cluster_group &cluster, int CS, int nchunk, int par, int sums_stride, int conv_local,
                                               int nan_local, double *sums, int &conv_flag, int &nan_flag)
{
    int conv_all = __syncthreads_and(conv_local);
    // __syncthreads_or returns a boolean, so reduce the two flag bits separately
    int nan_all = (__syncthreads_or(nan_local & RAFTK_FLAG_NAN) ? RAFTK_FLAG_NAN : 0)
                  | (__syncthreads_or(nan_local & RAFTK_FLAG_SINGULAR) ? RAFTK_FLAG_SINGULAR : 0);
    if (CS > 1) {
        if (threadIdx.x == 0) { sums[par * sums_stride + nchunk * 32] = (double)conv_all; sums[par * sums_stride + nchunk * 32 + 1] = (double)nan_all; }
        cluster.sync();
        int ca = 1, na = 0;
        for (int r = 0; r < CS; r++) {
            const double *rem = cluster.map_shared_rank(sums, r);
            ca &= (int)rem[par * sums_stride + nchunk * 32];
            na |= (int)rem[par * sums_stride + nchunk * 32 + 1];
        }
        conv_all = ca; nan_all = na;
    }
    conv_flag = conv_all; nan_flag = nan_all;
}
