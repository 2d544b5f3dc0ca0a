// raftk.cu -- sm_90a kernels + C ABI for the RAO-solve hot path (see include/raftk.h, DESIGN.md).
//
// Kernels
//   k_depth_table   : depth-decay functions cosh/sinh ratios per (node, frequency)      helpers.py:207-222
//   k_excitation    : sea state -> zeta, node phase table, strip inertial + BEM excitation
//                     raft_fowt.py:1732-1888, raft_member.py:1899-1992, helpers.py:188-236,703-760
//   k_drag_solve    : per (design, case) CTA cluster: drag linearisation (cross-frequency RMS),
//                     B_drag, F_drag, impedance assembly, 6x6 complex LU per frequency, convergence,
//                     relaxation          raft_model.py:1052-1142, raft_fowt.py:1891-1957,
//                                         raft_member.py:1995-2152, helpers.py:149-184,678-684
//   k_system_solve  : dense n x n complex solve per frequency (farm)      raft_model.py:1164-1216
//   k_fp64_peak     : DFMA micro-benchmark for the FP64 roofline denominator
//
// Algebra used by the kernels (DESIGN.md section 4): with member frame (q,p1,p2), node position
// r_j = rA + ls_j q and lever arm a = rA - r_ref, a 3-vector d in {q,p1,p2} at node j acts on the
// 6-DOF body through V_jd = [d ; r_j x d]:
//     V_jq = [q ; a x q],  V_jp1 = [p1 ; a x p1 + ls_j p2],  V_jp2 = [p2 ; a x p2 - ls_j p1]
// (q x p1 = p2, q x p2 = -p1).  Wave velocity projections are c_jd(w) = zeta w E_j (C_j h_d + i S_j d_z)
// with E_j = exp(-i k (x_j cos b + y_j sin b)), h_d = d_x cos b + d_y sin b, and (C_j,S_j) the depth
// functions.  Everything the reference does per (node, frequency) with 3x3 / 6x6 matrices reduces to
// complex scalars per node and a handful of sums per member.
#include <cuda_runtime.h>
#include <cooperative_groups.h>
#include <math_constants.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <mutex>
#include <algorithm>
#include <type_traits>
#include <vector>

#include "../../include/raftk.h"

namespace cg = cooperative_groups;

// ------------------------------------------------------------------------------------------------
// error handling
// ------------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";
static long long g_launches = 0;

static int set_err(int code, const char *fmt, const char *a = "", const char *b = "")
{
    snprintf(g_err, sizeof(g_err), fmt, a, b);
    return code;
}
#define CUDA_TRY(expr)                                                                          \
    do {                                                                                        \
        cudaError_t _e = (expr);                                                                \
        if (_e != cudaSuccess) return set_err(RAFTK_ECUDA, "%s: %s", #expr, cudaGetErrorString(_e)); \
    } while (0)

// ---- per-device opt-in for > 48 KB of dynamic shared memory ------------------------------------------
// cudaFuncSetAttribute applies to the CURRENT device only, so the high-water mark is kept per device
// (a process may drive several GPUs through DeviceSession(device=...)).
#define RAFTK_MAX_DEV 64
static int cur_dev()
{
    int d = 0;
    if (cudaGetDevice(&d) != cudaSuccess) { cudaGetLastError(); return 0; }
    return (d >= 0 && d < RAFTK_MAX_DEV) ? d : 0;
}
struct SmemOptIn {
    std::mutex mu;
    size_t set[RAFTK_MAX_DEV];
    explicit SmemOptIn(size_t floor = 0) { for (auto &v : set) v = floor; }
    template <class K> cudaError_t ensure(K kernel, size_t bytes)
    {
        std::lock_guard<std::mutex> lk(mu);
        const int d = cur_dev();
        if (bytes <= set[d]) return cudaSuccess;
        cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
        if (e == cudaSuccess) set[d] = bytes;
        return e;
    }
};

// ---- optional per-kernel event timing (roofline report) ----------------------------------------------
struct ProfRec { cudaEvent_t a, b; int kind; };
static bool g_prof_on = false;
static std::vector<ProfRec> g_prof;
static std::mutex g_prof_mu;

static void prof_begin_call()
{
    if (!g_prof_on) return;
    std::lock_guard<std::mutex> lk(g_prof_mu);
    for (auto &r : g_prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
    g_prof.clear();
}
struct ProfScope {
    cudaStream_t st; int idx = -1;
    ProfScope(cudaStream_t s, int kind) : st(s)
    {
        if (!g_prof_on) return;
        std::lock_guard<std::mutex> lk(g_prof_mu);
        ProfRec r; r.kind = kind;
        cudaEventCreate(&r.a); cudaEventCreate(&r.b);
        cudaEventRecord(r.a, st);
        g_prof.push_back(r); idx = (int)g_prof.size() - 1;
    }
    ~ProfScope()
    {
        if (idx < 0) return;
        std::lock_guard<std::mutex> lk(g_prof_mu);
        cudaEventRecord(g_prof[idx].b, st);
    }
};
extern "C" void raftk_profile_enable(int on) { g_prof_on = on != 0; }
extern "C" int raftk_profile_read(double ms[3], int launches[3])
{
    std::lock_guard<std::mutex> lk(g_prof_mu);
    for (int t = 0; t < 3; t++) { ms[t] = 0.0; launches[t] = 0; }
    for (auto &r : g_prof) {
        if (cudaEventSynchronize(r.b) != cudaSuccess) return RAFTK_ECUDA;
        float f = 0.f;
        if (cudaEventElapsedTime(&f, r.a, r.b) != cudaSuccess) return RAFTK_ECUDA;
        ms[r.kind] += f; launches[r.kind]++;
    }
    return RAFTK_OK;
}

extern "C" int raftk_version(void) { return RAFTK_VERSION; }
extern "C" const char *raftk_last_error(void) { return g_err; }
extern "C" long long raftk_launch_count(void) { return g_launches; }

// ---- record of the kernel variant the last call launched (raftk_last_dispatch) ------------------------------------------
// Written at the launch sites, per host thread.  disp_reset() at every entry point; disp_launch() next to each launch.
static thread_local raftk_dispatch g_disp = {};
static void disp_reset() { memset(&g_disp, 0, sizeof(g_disp)); }
static void disp_launch(int family, int kernel, int threads, int cluster_size = 0, int bins_per_cta = 0)
{
    disp_reset();
    g_disp.family = family; g_disp.kernel = kernel; g_disp.threads_per_cta = threads;
    g_disp.cluster_size = cluster_size; g_disp.bins_per_cta = bins_per_cta;
}
extern "C" int raftk_last_dispatch(raftk_dispatch *out)
{
    if (!out) return set_err(RAFTK_EINVAL, "raftk_last_dispatch: null output");
    *out = g_disp;
    return RAFTK_OK;
}

#include "raftk_common.cuh"
#include "raftk_tables.cuh"
#include "raftk_fused.cuh"
#include "raftk_fused2.cuh"
#include "raftk_qtf.cuh"
#include "raftk_slender.cuh"
#include "raftk_general.cuh"
#include "raftk_misc.cuh"
#include "raftk_builder.h"

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
static DesignsDev to_dev(const raftk_designs *d, int max_nodes, int max_members)
{
    DesignsDev D;
    D.nD = d->n_designs; D.nw = d->nw; D.max_nodes = max_nodes; D.max_members = max_members; D.n_bem_head = d->n_bem_head;
    D.depth = d->depth; D.rho = d->rho; D.g = d->g; D.dw = d->dw;
    D.w = d->w; D.k = d->k; D.member_offset = d->member_offset;
    D.mem_frame = d->mem_frame; D.mem_rA = d->mem_rA; D.mem_arm = d->mem_arm;
    D.mem_node_start = d->mem_node_start; D.mem_circ = d->mem_circ;
    D.node_ls = d->node_ls; D.node_cd_q = d->node_cd_q; D.node_cd_p1 = d->node_cd_p1; D.node_cd_p2 = d->node_cd_p2;
    D.node_in_q = d->node_in_q; D.node_in_p1 = d->node_in_p1; D.node_in_p2 = d->node_in_p2; D.node_pa = d->node_pa;
    D.node_in_p1_w = reinterpret_cast<const double2 *>(d->node_in_p1_w);
    D.node_in_p2_w = reinterpret_cast<const double2 *>(d->node_in_p2_w);
    D.M0 = d->M0; D.B0 = d->B0; D.C0 = d->C0; D.A_w = d->A_w; D.B_w = d->B_w;
    D.bem_headings = d->bem_headings; D.X_BEM = d->X_BEM; D.bem_xyh = d->bem_xyh;
    return D;
}

static CasesDev to_dev(const raftk_cases *c)
{
    CasesDev C;
    C.nC = c->n_cases; C.Hs = c->Hs; C.Tp = c->Tp; C.gamma = c->gamma; C.beta_deg = c->beta_deg;
    C.zeta_in = c->zeta; C.spec = c->spec; C.primary = c->primary; C.F_2nd = c->F_2nd;
    return C;
}

static size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

static size_t chunk_bytes(int nDc, int nC, int max_nodes, int nw)
{
    size_t b = 0;
    b += align_up((size_t)nDc * max_nodes * nw * sizeof(double2), 256);
    b += align_up((size_t)nDc * nC * max_nodes * nw * sizeof(double2), 256);
    b += align_up((size_t)nDc * nC * 6 * nw * sizeof(double2), 256);
    b += align_up((size_t)nC * nw * sizeof(double), 256);
    return b;
}

extern "C" size_t raftk_workspace_bytes(const raftk_designs *d, int32_t n_cases)
{
    if (!d || d->n_designs <= 0) return 0;
    const size_t cap = (size_t)8 << 30;       // plan at most 8 GiB; larger batches run in design chunks
    const int maxn = d->max_nodes > 0 ? d->max_nodes : 1;
    const size_t full = chunk_bytes(d->n_designs, n_cases, maxn, d->nw);
    const size_t one = chunk_bytes(1, n_cases, maxn, d->nw);
    return full <= cap ? full : std::max(cap, one);
}

static int validate(const raftk_designs *d, const raftk_cases *c)
{
    if (!d || !c) return set_err(RAFTK_EINVAL, "null designs/cases");
    if (d->n_designs <= 0 || d->nw <= 0 || c->n_cases <= 0) return set_err(RAFTK_EINVAL, "empty batch (n_designs, nw, n_cases must be > 0)");
    if (d->max_nodes <= 0 || d->max_members <= 0) return set_err(RAFTK_EINVAL, "max_nodes/max_members must be > 0");
    if (d->max_members > 512 || d->max_nodes > 4096) return set_err(RAFTK_EINVAL, "design too large for the shared-memory tables");
    if ((d->node_in_p1_w == nullptr) != (d->node_in_p2_w == nullptr)) return set_err(RAFTK_EINVAL, "node_in_p1_w / node_in_p2_w must both be given or both NULL");
    return 0;
}

// ---- second-order forces from the designs' QTF table -------------------------------------------------
static int validate_qtf(const raftk_designs *d, const raftk_cases *c)
{
    if (!d || !c) return set_err(RAFTK_EINVAL, "null designs/cases");
    if (d->n_designs <= 0 || d->nw <= 0 || c->n_cases <= 0) return set_err(RAFTK_EINVAL, "empty batch (n_designs, nw, n_cases must be > 0)");
    if (d->n_qtf_w < 2 || d->n_qtf_head < 1 || !d->qtf || !d->qtf_w || !d->qtf_heads)
        return set_err(RAFTK_EINVAL, "designs carry no QTF table (n_qtf_w >= 2, n_qtf_head >= 1, qtf, qtf_w, qtf_heads)");
    if (d->qtf_shared < 0 || d->qtf_shared > 2) return set_err(RAFTK_EINVAL, "qtf_shared must be 0, 1 or 2");
    if ((size_t)d->nw * 20 > 227 * 1024) return set_err(RAFTK_EINVAL, "nw too large for the second-order force kernel's shared-memory tables");
    return 0;
}

// The second-order force launches for the table, grid and output rows in P (P.F2 required) and the sea states of c: the
// rigid path (designs' table, run_qtf) and the generalised-DOF path (one FOWT's table) both come here.
static int launch_qtf(const QtfParams &P, const raftk_cases *c, cudaStream_t st)
{
    CasesDev C = to_dev(c);
    const size_t smem = (size_t)P.nw * 20;
    static SmemOptIn opt_plain(48 * 1024), opt_mix(48 * 1024), opt_tiles(48 * 1024);
    CUDA_TRY(opt_plain.ensure(k_qtf_force<false>, smem));
    CUDA_TRY(opt_mix.ensure(k_qtf_force<true>, smem));
    if (P.shared != 1 && P.nD > 65535) return set_err(RAFTK_EINVAL, "second-order force: more than 65535 designs per call");
    if (c->n_cases > 65535) return set_err(RAFTK_EINVAL, "second-order force: more than 65535 cases per call");
    // tile variant (registers hold the table-cell corners, systolic diagonal accumulators) when its shared-memory
    // tables fit and the frequency rows fit k_qtf_finish's register staging; RAFTK_QTF_DIAG=1 forces the diagonal kernel
    const int ncell = P.n2 - 1;
    const size_t tsmem = (size_t)P.nw * 68 + (size_t)ncell * 8 + 16;
    const bool tiles = !getenv("RAFTK_QTF_DIAG") && tsmem <= 226 * 1024 && P.nw <= 4096;
    if (tiles) {
        CUDA_TRY(opt_tiles.ensure(k_qtf_tiles, tsmem));
        QtfTileParams TP;
        TP.q = P; TP.ncell = ncell;
        const size_t rows = (size_t)((P.shared == 1) ? 1 : P.nD) * c->n_cases * 6 * P.nw;
        CUDA_TRY(cudaMemsetAsync(P.F2, 0, rows * sizeof(double), st));
        dim3 gt(QT_GROUPS, c->n_cases, P.shared == 1 ? 1 : P.nD);
        k_qtf_tiles<<<gt, QT_THREADS, tsmem, st>>>(C, TP);
        dim3 gf(6, c->n_cases, P.shared == 1 ? 1 : P.nD);
        k_qtf_finish<<<gf, 256, 0, st>>>(C, P);
        g_launches += 2;
        disp_launch(RAFTK_FAMILY_QTF, RAFTK_KERNEL_QTF_TILES, QT_THREADS);
        CUDA_TRY(cudaGetLastError());
        return RAFTK_OK;
    }
    const int ntasks = P.nw / 2 + 1, per_cta = (QTF_THREADS / 32) * QTF_TASKS_PER_WARP;
    dim3 grid((ntasks + per_cta - 1) / per_cta, c->n_cases, P.shared == 1 ? 1 : P.nD);
    if (P.nh > 1) k_qtf_force<true><<<grid, QTF_THREADS, smem, st>>>(C, P);
    else k_qtf_force<false><<<grid, QTF_THREADS, smem, st>>>(C, P);
    g_launches++;
    disp_launch(RAFTK_FAMILY_QTF, P.nh > 1 ? RAFTK_KERNEL_QTF_DIAG_MIX : RAFTK_KERNEL_QTF_DIAG, QTF_THREADS);
    CUDA_TRY(cudaGetLastError());
    return RAFTK_OK;
}

static int run_qtf(const raftk_designs *d, const raftk_cases *c, double *F2, double *F2mean, cudaStream_t st)
{
    int rc = validate_qtf(d, c);
    if (rc) return rc;
    if (!F2) return set_err(RAFTK_EINVAL, "second-order force needs the F_2nd buffer");
    QtfParams P;
    P.nD = d->n_designs; P.shared = d->qtf_shared;
    P.n2 = d->n_qtf_w; P.nh = d->n_qtf_head; P.nw = d->nw; P.dw = d->dw;
    P.w = d->w; P.qw = d->qtf_w; P.qh = d->qtf_heads;
    P.qtf = reinterpret_cast<const double2 *>(d->qtf);
    P.F2 = F2; P.F2mean = F2mean;
    return launch_qtf(P, c, st);
}

extern "C" int raftk_second_order_force_dev(const raftk_designs *d, const raftk_cases *c, const raftk_outputs *out, void *stream)
{
    disp_reset();
    if (!out || !out->F_2nd) return set_err(RAFTK_EINVAL, "outputs.F_2nd is required");
    return run_qtf(d, c, out->F_2nd, out->F_2nd_mean, (cudaStream_t)stream);
}

// ---- the rigid solve's plan --------------------------------------------------------------------------------------------
// One decision for every entry point: which kernel solves (k_rao_fused2, k_rao_fused<T> or k_drag_solve on the v1 tables
// path), at what cluster size, and how the workspace is laid out.  The size queries, the host entry points and the launches
// all read the plan made here.

static int sm_count()                 // 132 (an H100 SXM) when no device answers, so that the size queries work without one
{
    int dev = 0, sms = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) {
        cudaGetLastError();
        return 132;
    }
    return sms;
}

// ctas CTAs of `threads` threads with smem bytes of dynamic shared memory on st, in thread-block clusters of cs CTAs; at is
// the cluster attribute cfg points to
static void cluster_config(cudaLaunchConfig_t &cfg, cudaLaunchAttribute &at, size_t ctas, int threads, size_t smem, int cs, cudaStream_t st)
{
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3((unsigned)ctas, 1, 1);
    cfg.blockDim = dim3(threads, 1, 1);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    at.id = cudaLaunchAttributeClusterDimension;
    at.val.clusterDim.x = cs; at.val.clusterDim.y = 1; at.val.clusterDim.z = 1;
    cfg.attrs = &at; cfg.numAttrs = 1;
}

enum SolveKind { SOLVE_V1, SOLVE_FUSED, SOLVE_FUSED2 };
struct SolvePlan {
    SolveKind kind;
    int CS, nwl, T, nchunk, maxW, maxH, maxZ;    // cluster size, bins and threads per CTA, node chunks, step-class maxima
    size_t smem;
    bool f0_global;                              // k_rao_fused<T>: F0 in the workspace instead of shared memory
    // Workspace of the fused kernels: F0 [units][6][nw] at 0, the wave-train hand-over [units][NCOEF*max_nodes + 36] from
    // o_lin to lin_end; k_rao_fused2 adds Eg, Ag, the plan blobs (blob doubles per design) and, with xslots, the grid
    // variant's exchange rows and arrival counters.  bytes: what the plan needs (v1: the tables' whole budget).
    size_t o_lin, lin_end, o_E, o_A, o_plan, blob, o_xrow, o_xcnt, bytes;
    bool xslots;
    int per;                                     // v1: designs per chunk of tables
};
static const size_t WS_UNBOUNDED = SIZE_MAX;     // plan to size a workspace: it will hold whatever the plan needs

// Plan a solve of d x n_cases against wbytes of workspace.  requested_cs: the caller's cluster size when it is 1, 2, 4 or 8,
// else the planner picks one.  v1_only: the tables path (excitation, linearisation), as RAFTK_FORCE_V1 does for the solve.
static SolvePlan plan_solve(const raftk_designs *d, int n_cases, int requested_cs, size_t wbytes, bool v1_only = false)
{
    const int nw = d->nw;
    const size_t units = (size_t)d->n_designs * n_cases;
    const int sms = sm_count();
    // k_rao_fused2 takes a requested cluster size as given; the one-bin kernels halve it while a CTA would get < 32 bins
    const int req = (requested_cs == 1 || requested_cs == 2 || requested_cs == 4 || requested_cs == 8) ? requested_cs : 0;
    int req_halved = req;
    while (req_halved > 1 && nw / req_halved < 32) req_halved >>= 1;

    SolvePlan base;
    memset(&base, 0, sizeof(base));
    base.nchunk = (d->max_nodes + CHUNK_NODES - 1) / CHUNK_NODES;
    base.maxW = d->max_w_classes > 0 ? d->max_w_classes : d->max_nodes;
    base.maxH = d->max_h_classes > 0 ? d->max_h_classes : d->max_nodes;
    base.maxZ = d->max_z_classes > 0 ? std::min(d->max_z_classes, d->max_members) : d->max_members;
    const size_t f0 = units * 6 * nw * sizeof(double2);
    base.o_lin = align_up(f0, 256);
    base.lin_end = base.o_lin + units * ((size_t)NCOEF * d->max_nodes + 36) * sizeof(double);

    if (!v1_only && !getenv("RAFTK_FORCE_V1") && d->max_nodes > 0 && d->max_members > 0) {
        SolvePlan p = base;
        p.kind = SOLVE_FUSED2; p.T = F2_T;
        p.CS = req;
        if (!p.CS) for (p.CS = 1; p.CS < 8 && (nw + p.CS - 1) / p.CS > 2 * F2_T; p.CS <<= 1) {}
        p.nwl = (nw + p.CS - 1) / p.CS;
        // two bins per thread pay when most threads own two: 192 < bins per CTA <= 256; otherwise the one-bin kernel runs
        if (p.nwl <= 2 * F2_T && p.nwl > (3 * F2_T) / 2) {
            p.smem = fused2_smem_bytes(d->max_members, d->max_nodes, p.nchunk, p.nwl, p.maxW, p.maxH, p.maxZ);
            p.blob = (size_t)plan_layout(d->max_members, d->max_nodes, p.maxW, p.maxH, p.maxZ).total;
            size_t o = align_up(p.lin_end, 256);
            p.o_E = o; o += align_up(units * (size_t)d->max_members * nw * sizeof(double2), 256);
            p.o_A = o; o += align_up(units * (size_t)p.maxZ * nw * sizeof(double2), 256);
            p.o_plan = o; o += align_up((size_t)d->n_designs * p.blob * sizeof(double), 256);
            // exchange rows and arrival counters of the grid variant (k_rao_fused2<true>).  It needs all units x CS CTAs
            // resident at once, at most 2 per SM (255 registers x 128 threads), so with CS >= 2 only batches of at most one
            // unit per SM qualify; the rows are sized for the largest cluster (8) so that the workspace does not depend on
            // cluster_size.
            p.xslots = units <= (size_t)sms;
            if (p.xslots) {
                p.o_xrow = o; o += align_up(units * 2 * 8 * ((size_t)p.nchunk * 32 + 2) * sizeof(double), 256);
                p.o_xcnt = o; o += align_up(units * sizeof(unsigned), 256);
            }
            p.bytes = o;
            if (p.smem <= (size_t)113 * 1024 && wbytes >= p.bytes) return p;           // two CTAs per SM
        }
        // k_rao_fused<T> at cluster size cs.  255 registers cap residency at 256 threads per SM (at 168 registers for 3 CTAs
        // the LU spills); shared memory must allow 2 CTAs of 128 threads or 1 of 256.  F0 lives in shared memory when it
        // fits, else in the caller's workspace.
        auto fused = [&](int cs) {
            p = base;
            p.kind = SOLVE_FUSED;
            p.CS = cs;
            p.nwl = (nw + cs - 1) / cs;
            p.T = p.nwl > 128 ? 256 : 128;
            p.bytes = align_up(p.lin_end, 256);
            const size_t limit = (p.T == 128) ? (size_t)112 * 1024 : (size_t)226 * 1024;
            p.smem = fused_smem_bytes(d->max_members, d->max_nodes, p.nchunk, p.T / 32, p.nwl, p.maxW, p.maxH, p.maxZ, true);
            if (p.smem > limit && wbytes >= f0) {
                p.f0_global = true;
                p.smem = fused_smem_bytes(d->max_members, d->max_nodes, p.nchunk, p.T / 32, p.nwl, p.maxW, p.maxH, p.maxZ, false);
            }
            return p.smem <= limit && p.nwl <= 2 * p.T;
        };
        if (req_halved) {
            if (fused(req_halved)) return p;
        } else if (units >= (size_t)4 * sms) {     // plenty of units: smallest cluster whose slice fits on chip
            for (int cs = 1; cs <= 8; cs <<= 1) if (fused(cs) && p.nwl <= p.T) return p;
            for (int cs = 1; cs <= 8; cs <<= 1) if (fused(cs)) return p;
        } else {                                   // few units: largest cluster that keeps >= 128 bins per CTA
            for (int cs = 8; cs >= 1; cs >>= 1) if ((cs == 1 || nw / cs >= 128) && fused(cs)) return p;
        }
    }

    // v1: the tables take the whole workspace, in chunks of at most 65535 designs
    SolvePlan p = base;
    p.kind = SOLVE_V1;
    p.T = SOLVE_THREADS;
    p.bytes = wbytes == WS_UNBOUNDED ? raftk_workspace_bytes(d, n_cases) : wbytes;
    p.per = d->n_designs;
    while (p.per > 1 && (chunk_bytes(p.per, n_cases, d->max_nodes, nw) > p.bytes || p.per > 65535)) p.per = (p.per + 1) / 2;
    p.CS = req_halved;
    if (!p.CS)     // fill ~2 CTAs per SM, keep >= 128 frequencies per CTA, and keep 12*nwl doubles of state <= 48 KB
        for (p.CS = 1; p.CS < 8 && ((size_t)p.per * n_cases * p.CS < (size_t)2 * sms || nw / p.CS > 512) && nw / (p.CS * 2) >= 128; p.CS <<= 1) {}
    p.nwl = (nw + p.CS - 1) / p.CS;
    p.smem = smem_doubles(d->max_members, d->max_nodes, p.nchunk, SOLVE_THREADS / 32, p.nwl) * sizeof(double)
             + (size_t)d->max_members * 3 * sizeof(int) + 16;
    return p;
}

// ---- fused launchers ---------------------------------------------------------------------------------------------------

// Parameters both fused kernels take: zeroed, then the options, the outputs, Xi_init and, with peers, this rank's block in
// every rank's gathered arrays (each finished unit's Xi and status are stored there too).
static FusedParams fused_params(const raftk_designs *d, const raftk_cases *c, const raftk_solve_opts *o, const raftk_outputs *out,
                                const SolvePlan &pl, const raftk_peers *peers)
{
    FusedParams P;
    memset(&P, 0, sizeof(P));
    P.n_iter = o->n_iter; P.CS = pl.CS; P.nwl = pl.nwl; P.maxW = pl.maxW; P.maxH = pl.maxH; P.maxZ = pl.maxZ;
    P.tol = o->tol; P.xi_start = o->xi_start;
    P.Xi_out = reinterpret_cast<double2 *>(out->Xi);
    P.Fdrag_out = reinterpret_cast<double2 *>(out->F_drag);
    P.Finer_out = reinterpret_cast<double2 *>(out->F_iner);
    P.Fbem_out = reinterpret_cast<double2 *>(out->F_BEM);
    P.Bdrag_out = out->B_drag; P.zeta_out = out->zeta; P.status = out->status;
    P.Xilast_out = reinterpret_cast<double2 *>(out->Xi_last);
    P.Xi_init = reinterpret_cast<const double2 *>(c->Xi_init);
    P.phase = -1;
    if (peers && peers->n_ranks > 1) {
        P.n_peers = peers->n_ranks; P.peer_rank = peers->rank;
        const size_t units_per_rank = peers->block_elems / ((size_t)6 * d->nw);
        for (int p = 0; p < peers->n_ranks; p++) {
            P.peer_Xi[p] = reinterpret_cast<double2 *>(peers->gathered[p]) + (size_t)peers->rank * peers->block_elems;
            P.peer_status[p] = peers->status[p] ? peers->status[p] + (size_t)peers->rank * units_per_rank * 4 : nullptr;
        }
    }
    return P;
}

template <int T>
static int fused_launch(const DesignsDev &D, const CasesDev &C, const FusedParams &P, const SolvePlan &pl, int units, cudaStream_t st)
{
    static SmemOptIn opt;
    CUDA_TRY(opt.ensure(k_rao_fused<T>, pl.smem));
    cudaLaunchConfig_t cfg;
    cudaLaunchAttribute at;
    cluster_config(cfg, at, (size_t)units * pl.CS, T, pl.smem, pl.CS, st);
    {
        ProfScope ps(st, 2);
        CUDA_TRY(cudaLaunchKernelEx(&cfg, k_rao_fused<T>, D, C, P));
    }
    g_launches++;
    disp_launch(RAFTK_FAMILY_SOLVE, T == 128 ? RAFTK_KERNEL_FUSED128 : RAFTK_KERNEL_FUSED256, T, pl.CS, pl.nwl);
    g_disp.f0_global = P.F0g != nullptr;
    g_disp.trains = P.phase >= 0;
    CUDA_TRY(cudaGetLastError());
    return RAFTK_OK;
}

static int run_fused(const raftk_designs *d, const raftk_cases *c, const raftk_solve_opts *o, const raftk_outputs *out,
                     const SolvePlan &pl, void *workspace, size_t wbytes, cudaStream_t st, const raftk_peers *peers)
{
    prof_begin_call();
    DesignsDev D = to_dev(d, d->max_nodes, d->max_members);
    CasesDev C = to_dev(c);
    FusedParams P = fused_params(d, c, o, out, pl, peers);
    P.F0g = pl.f0_global ? reinterpret_cast<double2 *>(workspace) : nullptr;
    const int units = d->n_designs * c->n_cases;
    if (c->primary) {                                  // wave trains: primaries first, then the trains that follow them
        if (!workspace || wbytes < pl.lin_end) return set_err(RAFTK_ENOMEM, "wave-train cases need raftk_solve_workspace_bytes() of workspace");
        P.lin_g = reinterpret_cast<double *>(static_cast<char *>(workspace) + pl.o_lin);
        for (int phase = 0; phase < 2; phase++) {
            P.phase = phase;
            const int rc = (pl.T == 128) ? fused_launch<128>(D, C, P, pl, units, st) : fused_launch<256>(D, C, P, pl, units, st);
            if (rc) return rc;
        }
        return RAFTK_OK;
    }
    if (pl.T == 128) return fused_launch<128>(D, C, P, pl, units, st);
    return fused_launch<256>(D, C, P, pl, units, st);
}

// Grid or cluster exchange for k_rao_fused2 (RAFTK_FUSED2_XCHG=cluster|grid overrides, read per call, for A/B runs and
// tests).  The grid variant runs when a unit spans several CTAs, every CTA of the launch can be resident at once, and the
// hardware cannot place every unit's cluster at once (cudaOccupancyMaxActiveClusters < units): then the clusters that do not
// fit would start only when the first units finish.  The occupancy queries are cached per device and launch shape.
static SmemOptIn g_f2_opt_cluster, g_f2_opt_grid;
struct F2Occ { int dev, units, CS; size_t smem; int clusters, resident; };
static std::mutex g_f2_occ_mu;
static std::vector<F2Occ> g_f2_occ;

static int f2_occupancy(const SolvePlan &pl, int units, int &clusters, int &resident)
{
    const int dev = cur_dev();
    {
        std::lock_guard<std::mutex> lk(g_f2_occ_mu);
        for (const F2Occ &e : g_f2_occ)
            if (e.dev == dev && e.units == units && e.CS == pl.CS && e.smem == pl.smem) { clusters = e.clusters; resident = e.resident; return RAFTK_OK; }
    }
    CUDA_TRY(g_f2_opt_cluster.ensure(k_rao_fused2<false>, pl.smem));
    CUDA_TRY(g_f2_opt_grid.ensure(k_rao_fused2<true>, pl.smem));
    cudaLaunchConfig_t cfg;
    cudaLaunchAttribute at;
    cluster_config(cfg, at, (size_t)units * pl.CS, F2_T, pl.smem, pl.CS, 0);
    int per_sm = 0;
    CUDA_TRY(cudaOccupancyMaxActiveClusters(&clusters, k_rao_fused2<false>, &cfg));
    CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_rao_fused2<true>, F2_T, pl.smem));
    resident = per_sm * sm_count();
    std::lock_guard<std::mutex> lk(g_f2_occ_mu);
    g_f2_occ.push_back(F2Occ{dev, units, pl.CS, pl.smem, clusters, resident});
    return RAFTK_OK;
}

static int f2_pick_grid(const SolvePlan &pl, int units, bool &grid)
{
    grid = false;
    const char *x = getenv("RAFTK_FUSED2_XCHG");
    const bool force_c = x && !strcmp(x, "cluster"), force_g = x && !strcmp(x, "grid");
    if (x && *x && !force_c && !force_g) return set_err(RAFTK_EINVAL, "RAFTK_FUSED2_XCHG must be 'cluster' or 'grid', not '%s'", x);
    if (pl.CS <= 1 || force_c) return RAFTK_OK;                 // one CTA per unit: nothing to exchange
    int clusters = 0, resident = 0;
    if (int rc = f2_occupancy(pl, units, clusters, resident)) return rc;
    const bool fits = pl.xslots && (size_t)units * pl.CS <= (size_t)resident;
    if (force_g && !fits) return set_err(RAFTK_EINVAL, "RAFTK_FUSED2_XCHG=grid: the launch's CTAs cannot all be resident at once");
    grid = fits && (force_g || clusters < units);
    return RAFTK_OK;
}

static int run_fused2(const raftk_designs *d, const raftk_cases *c, const raftk_solve_opts *o, const raftk_outputs *out,
                      const SolvePlan &pl, void *workspace, cudaStream_t st, const raftk_peers *peers)
{
    prof_begin_call();
    DesignsDev D = to_dev(d, d->max_nodes, d->max_members);
    CasesDev C = to_dev(c);
    char *ws = static_cast<char *>(workspace);
    FusedParams P = fused_params(d, c, o, out, pl, peers);
    P.F0g = reinterpret_cast<double2 *>(ws);
    P.Eg = reinterpret_cast<double2 *>(ws + pl.o_E);
    P.Ag = reinterpret_cast<double2 *>(ws + pl.o_A);
    double *plan = reinterpret_cast<double *>(ws + pl.o_plan);
    P.plan = plan; P.plan_stride = pl.blob;
    if (!(o->flags & RAFTK_SOLVE_REUSE_PLAN)) {
        ProfScope ps(st, 0);
        const size_t psm = (3 * (size_t)d->max_nodes + d->max_members) * sizeof(double) + 2 * (size_t)d->max_members * sizeof(int);
        k_fused_plan<<<d->n_designs, 128, psm, st>>>(D, plan, pl.blob, pl.maxW, pl.maxH, pl.maxZ, pl.nwl);
        g_launches++;
    }
    const int units = d->n_designs * c->n_cases;
    bool grid = false;
    if (int rc = f2_pick_grid(pl, units, grid)) return rc;
    CUDA_TRY(grid ? g_f2_opt_grid.ensure(k_rao_fused2<true>, pl.smem) : g_f2_opt_cluster.ensure(k_rao_fused2<false>, pl.smem));
    cudaLaunchConfig_t cfg;
    cudaLaunchAttribute at;
    cluster_config(cfg, at, (size_t)units * pl.CS, F2_T, pl.smem, pl.CS, st);
    if (grid) {                    // all CTAs resident at once, or the launch fails: the exchange waits cannot deadlock
        at.id = cudaLaunchAttributeCooperative;
        at.val.cooperative = 1;
        P.xrow = reinterpret_cast<double *>(ws + pl.o_xrow);
        P.xcnt = reinterpret_cast<unsigned *>(ws + pl.o_xcnt);
    }
    const int nphase = c->primary ? 2 : 1;
    if (c->primary) P.lin_g = reinterpret_cast<double *>(ws + pl.o_lin);
    for (int phase = 0; phase < nphase; phase++) {
        P.phase = c->primary ? phase : -1;
        {
            ProfScope ps(st, 2);
            if (grid) {
                CUDA_TRY(cudaMemsetAsync(P.xcnt, 0, (size_t)units * sizeof(unsigned), st));      // counters count up from 0 per launch
                CUDA_TRY(cudaLaunchKernelEx(&cfg, k_rao_fused2<true>, D, C, P));
            } else {
                CUDA_TRY(cudaLaunchKernelEx(&cfg, k_rao_fused2<false>, D, C, P));
            }
        }
        g_launches++;
    }
    disp_launch(RAFTK_FAMILY_SOLVE, grid ? RAFTK_KERNEL_FUSED2_GRID : RAFTK_KERNEL_FUSED2_CLUSTER, F2_T, pl.CS, pl.nwl);
    g_disp.trains = c->primary != nullptr;
    CUDA_TRY(cudaGetLastError());
    return RAFTK_OK;
}

#ifdef RAFTK_F2_WAVE_TRACE
// diagnostic build only: see g_f2_trace (raftk_fused2.cuh) and tools/fused2_waves.py
extern "C" int raftk_f2_trace_read(unsigned long long *host, int n_cta)
{
    if (n_cta < 0 || n_cta > F2_TRACE_MAX) return set_err(RAFTK_EINVAL, "n_cta must be in [0, F2_TRACE_MAX]");
    CUDA_TRY(cudaMemcpyFromSymbol(host, g_f2_trace, (size_t)n_cta * 3 * sizeof(unsigned long long)));
    return RAFTK_OK;
}
// out: max co-resident clusters of the plan's cluster size, co-resident CTAs of the grid variant, grid variant picked (0/1),
// cluster size, dynamic shared memory bytes
extern "C" int raftk_f2_occupancy(const raftk_designs *d, int n_cases, int cluster_size, int out[5])
{
    const SolvePlan pl = plan_solve(d, n_cases, cluster_size, WS_UNBOUNDED);
    if (pl.kind != SOLVE_FUSED2) return set_err(RAFTK_EINVAL, "not a k_rao_fused2 shape");
    const int units = d->n_designs * n_cases;
    int clusters = 0, resident = 0;
    bool grid = false;
    if (int rc = f2_occupancy(pl, units, clusters, resident)) return rc;
    if (int rc = f2_pick_grid(pl, units, grid)) return rc;
    out[0] = clusters; out[1] = resident; out[2] = grid ? 1 : 0; out[3] = pl.CS; out[4] = (int)pl.smem;
    return RAFTK_OK;
}
#endif

// ---- v1 tables path ----------------------------------------------------------------------------------------------------
// Depth and phase tables and F0 in the workspace (k_depth_table, k_excitation), then k_drag_solve linearises (mode 1) or
// solves (mode 0); mode 2 stops after the excitation.  Linearisation reads the tables a preceding excitation left.  The
// designs run in chunks of pl.per.
static int run_tables(const raftk_designs *d, const raftk_cases *c, const raftk_solve_opts *o, const raftk_outputs *out,
                      const double *Xi_in, int mode /*0 solve, 1 linearise, 2 excitation only*/, const SolvePlan &pl,
                      void *workspace, size_t wbytes, cudaStream_t st)
{
    if (c->primary && mode != 2) return set_err(RAFTK_EINVAL, "cases.primary is only supported by raftk_solve_dynamics_*");
    const int nD = d->n_designs, nC = c->n_cases, nw = d->nw, per = pl.per;
    const bool excitation = mode != 1;
    if (excitation) prof_begin_call();
    DesignsDev D = to_dev(d, d->max_nodes, d->max_members);
    CasesDev C = to_dev(c);
    if (!workspace || wbytes < chunk_bytes(1, nC, d->max_nodes, nw)) return set_err(RAFTK_ENOMEM, "workspace smaller than one design's tables");
    if (mode == 1 && per < nD)
        return set_err(RAFTK_ENOMEM, "linearization needs the whole batch's tables resident in the workspace");
    if (mode != 2) {
        if (pl.smem > 227 * 1024) return set_err(RAFTK_EINVAL, "shared-memory plan exceeds 227 KB (nw per CTA too large)");
        static SmemOptIn opt;
        CUDA_TRY(opt.ensure(k_drag_solve, pl.smem));
    }

    for (int d0 = 0; d0 < nD; d0 += per) {
        const int nDc = std::min(per, nD - d0);
        Work W;
        W.d0 = d0; W.nDc = nDc;
        char *p = static_cast<char *>(workspace);
        W.depth_tab = reinterpret_cast<double2 *>(p); p += align_up((size_t)nDc * d->max_nodes * nw * sizeof(double2), 256);
        W.phase_tab = reinterpret_cast<double2 *>(p); p += align_up((size_t)nDc * nC * d->max_nodes * nw * sizeof(double2), 256);
        W.F0 = reinterpret_cast<double2 *>(p); p += align_up((size_t)nDc * nC * 6 * nw * sizeof(double2), 256);
        W.zeta = reinterpret_cast<double *>(p);

        if (excitation) {
            dim3 g0((nw + 127) / 128, nDc, 1);
            {
                ProfScope ps(st, 0);
                k_depth_table<<<g0, 128, 0, st>>>(D, W);
            }
            g_launches++;
            ExcOut EO;
            EO.F_iner = reinterpret_cast<double2 *>(out->F_iner);
            EO.F_BEM = reinterpret_cast<double2 *>(out->F_BEM);
            EO.zeta = out->zeta;
            dim3 g1((nw + 127) / 128, nC, nDc);
            {
                ProfScope ps(st, 1);
                k_excitation<<<g1, 128, 0, st>>>(D, C, W, EO);
            }
            g_launches++;
        }
        if (mode != 2) {
            SolveParams P;
            P.n_iter = o ? o->n_iter : 0; P.CS = pl.CS; P.nwl = pl.nwl; P.mode = mode;
            P.tol = o ? o->tol : 0.01; P.xi_start = o ? o->xi_start : 0.0;
            P.Xi_in = reinterpret_cast<const double2 *>(Xi_in);
            P.Xi_out = reinterpret_cast<double2 *>(out->Xi);
            P.Fdrag_out = reinterpret_cast<double2 *>(out->F_drag);
            P.Bdrag_out = out->B_drag;
            P.status = out->status;
            cudaLaunchConfig_t cfg;
            cudaLaunchAttribute at;
            cluster_config(cfg, at, (size_t)nDc * nC * pl.CS, SOLVE_THREADS, pl.smem, pl.CS, st);
            {
                ProfScope ps(st, 2);
                CUDA_TRY(cudaLaunchKernelEx(&cfg, k_drag_solve, D, C, W, P));
            }
            g_launches++;
        }
        if (d0 == 0) {
            if (mode != 2) disp_launch(RAFTK_FAMILY_SOLVE, RAFTK_KERNEL_V1, SOLVE_THREADS, pl.CS, pl.nwl);
            else disp_launch(RAFTK_FAMILY_SOLVE, RAFTK_KERNEL_V1, 128);
        }
        g_disp.chunks++;
        CUDA_TRY(cudaGetLastError());
    }
    return RAFTK_OK;
}

// excitation (mode 2) or linearisation (mode 1) over the caller's workspace
static int tables(const raftk_designs *d, const raftk_cases *c, const double *Xi_in, const raftk_outputs *out, int mode,
                  void *workspace, size_t wbytes, cudaStream_t st)
{
    if (int rc = validate(d, c)) return rc;
    return run_tables(d, c, nullptr, out, Xi_in, mode, plan_solve(d, c->n_cases, 0, wbytes, true), workspace, wbytes, st);
}

// ---- the rigid solve: launch a plan --------------------------------------------------------------------------------------
static int launch_solve(const raftk_designs *d, const raftk_cases *c, const raftk_solve_opts *o, const raftk_outputs *out,
                        const SolvePlan &pl, void *workspace, size_t wbytes, cudaStream_t st, const raftk_peers *peers)
{
    if (pl.kind == SOLVE_FUSED2) return run_fused2(d, c, o, out, pl, workspace, st, peers);
    if (pl.kind == SOLVE_FUSED) return run_fused(d, c, o, out, pl, workspace, wbytes, st, peers);
    if (peers && peers->n_ranks > 1) return set_err(RAFTK_EINVAL, "the fused exchange needs the fused solver; the design's frequency slice does not fit on chip");
    if (c->primary) return set_err(RAFTK_EINVAL, "wave-train cases (cases.primary) need the fused solver; the design's frequency slice does not fit on chip");
    if (c->Xi_init || out->Xi_last) return set_err(RAFTK_EINVAL, "cases.Xi_init / outputs.Xi_last need the fused solver; the design's frequency slice does not fit on chip");
    return run_tables(d, c, o, out, nullptr, 0, pl, workspace, wbytes, st);
}

// the rigid solve over the caller's workspace: planned against it, then launched
static int solve(const raftk_designs *d, const raftk_cases *c, const raftk_solve_opts *o, const raftk_outputs *out,
                 void *workspace, size_t wbytes, cudaStream_t st, const raftk_peers *peers = nullptr)
{
    if (int rc = validate(d, c)) return rc;
    const SolvePlan pl = plan_solve(d, c->n_cases, o->cluster_size, workspace ? wbytes : 0);
    return launch_solve(d, c, o, out, pl, workspace, wbytes, st, peers);
}

extern "C" size_t raftk_solve_workspace_bytes(const raftk_designs *d, int32_t n_cases)
{
    if (!d || d->n_designs <= 0 || n_cases <= 0) return 0;
    return plan_solve(d, n_cases, 0, WS_UNBOUNDED).bytes;
}

extern "C" int raftk_hydro_excitation_dev(const raftk_designs *d, const raftk_cases *c, const raftk_outputs *out,
                                          void *workspace, size_t workspace_bytes, void *stream)
{
    disp_reset();
    if (!out) return set_err(RAFTK_EINVAL, "null outputs");
    if (d && c && chunk_bytes(d->n_designs, c->n_cases, d->max_nodes, d->nw) > workspace_bytes)
        return set_err(RAFTK_ENOMEM, "excitation needs the whole batch's tables in the workspace");
    return tables(d, c, nullptr, out, 2, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int raftk_hydro_linearization_dev(const raftk_designs *d, const raftk_cases *c, const double *Xi_in,
                                             const raftk_outputs *out, void *workspace, size_t workspace_bytes, void *stream)
{
    disp_reset();
    if (!out || !Xi_in) return set_err(RAFTK_EINVAL, "null outputs / Xi_in");
    return tables(d, c, Xi_in, out, 1, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int raftk_solve_dynamics_dev(const raftk_designs *d, const raftk_cases *c, const raftk_solve_opts *o,
                                        const raftk_outputs *out, void *workspace, size_t workspace_bytes, void *stream)
{
    disp_reset();
    if (!out || !out->Xi || !out->status || !o) return set_err(RAFTK_EINVAL, "Xi, status and opts are required");
    if (d && c && d->n_qtf_w > 0 && !c->F_2nd) {          // potSecOrder 2: the solve computes the force itself (raft_model.py:1035-1038)
        if (!out->F_2nd) return set_err(RAFTK_EINVAL, "designs carry a QTF: pass outputs.F_2nd as the buffer, or cases.F_2nd precomputed");
        int rc = run_qtf(d, c, out->F_2nd, out->F_2nd_mean, (cudaStream_t)stream);
        if (rc) return rc;
        raftk_cases cc = *c;
        cc.F_2nd = out->F_2nd;
        return solve(d, &cc, o, out, workspace, workspace_bytes, (cudaStream_t)stream);
    }
    return solve(d, c, o, out, workspace, workspace_bytes, (cudaStream_t)stream);
}

// ---- multi-GPU exchange fused into the solve (peer stores over NVLink) ------------------------------------------
extern "C" int raftk_peer_alloc(size_t bytes, void **dev_ptr, unsigned char handle[64])
{
    if (!dev_ptr || !handle || bytes == 0) return set_err(RAFTK_EINVAL, "peer_alloc: null argument / zero size");
    void *p = nullptr;
    CUDA_TRY(cudaMalloc(&p, bytes));
    cudaError_t e = cudaMemset(p, 0, bytes);
    cudaIpcMemHandle_t h;
    if (e == cudaSuccess) e = cudaIpcGetMemHandle(&h, p);
    if (e != cudaSuccess) { cudaFree(p); return set_err(RAFTK_ECUDA, "peer_alloc: %s", cudaGetErrorString(e)); }
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handle size");
    memcpy(handle, &h, 64);
    *dev_ptr = p;
    return RAFTK_OK;
}
extern "C" int raftk_peer_free(void *dev_ptr)
{
    if (dev_ptr) CUDA_TRY(cudaFree(dev_ptr));
    return RAFTK_OK;
}
extern "C" int raftk_peer_open(const unsigned char handle[64], void **dev_ptr)
{
    if (!dev_ptr || !handle) return set_err(RAFTK_EINVAL, "peer_open: null argument");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, 64);
    CUDA_TRY(cudaIpcOpenMemHandle(dev_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return RAFTK_OK;
}
extern "C" int raftk_peer_close(void *dev_ptr)
{
    if (dev_ptr) CUDA_TRY(cudaIpcCloseMemHandle(dev_ptr));
    return RAFTK_OK;
}

static int validate_peers(const raftk_peers *p)
{
    if (!p) return set_err(RAFTK_EINVAL, "null peers");
    if (p->n_ranks < 1 || p->n_ranks > RAFTK_MAX_PEERS || p->rank < 0 || p->rank >= p->n_ranks)
        return set_err(RAFTK_EINVAL, "peers: 1 <= n_ranks <= RAFTK_MAX_PEERS and 0 <= rank < n_ranks");
    for (int r = 0; r < p->n_ranks; r++)
        if (!p->gathered[r] || !p->flags[r]) return set_err(RAFTK_EINVAL, "peers: gathered / flags pointer missing for a rank");
    return 0;
}

extern "C" int raftk_solve_dynamics_gather_dev(const raftk_designs *d, const raftk_cases *c, const raftk_solve_opts *o,
                                               const raftk_outputs *out, const raftk_peers *peers, void *workspace,
                                               size_t workspace_bytes, void *stream)
{
    disp_reset();
    if (!out || !out->Xi || !out->status || !o) return set_err(RAFTK_EINVAL, "Xi, status and opts are required");
    int rc = validate_peers(peers);
    if (rc) return rc;
    if (!d || !c) return set_err(RAFTK_EINVAL, "null designs/cases");
    if ((size_t)d->n_designs * c->n_cases * 6 * d->nw > peers->block_elems)
        return set_err(RAFTK_EINVAL, "peers.block_elems is smaller than this rank's response block");
    if (out->Xi != peers->gathered[peers->rank] + 2 * (size_t)peers->rank * peers->block_elems)
        return set_err(RAFTK_EINVAL, "outputs.Xi must be this rank's block of its own gathered array");
    if (d->n_qtf_w > 0 && !c->F_2nd) return set_err(RAFTK_EINVAL, "gather solve: pass cases.F_2nd precomputed (raftk_second_order_force_dev)");
    return solve(d, c, o, out, workspace, workspace_bytes, (cudaStream_t)stream, peers);
}

extern "C" int raftk_peer_barrier_dev(const raftk_peers *peers, int32_t *timeout_flag, void *stream)
{
    int rc = validate_peers(peers);
    if (rc) return rc;
    if (peers->epoch == 0) return set_err(RAFTK_EINVAL, "peers.epoch must be > 0");
    PeerFlags F;
    F.n = peers->n_ranks; F.rank = peers->rank; F.epoch = peers->epoch;
    for (int p = 0; p < RAFTK_MAX_PEERS; p++) F.flags[p] = p < peers->n_ranks ? peers->flags[p] : nullptr;
    k_peer_barrier<<<1, 32, 0, (cudaStream_t)stream>>>(F, timeout_flag);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RAFTK_OK;
}

// ---- farm system solve ----------------------------------------------------------------------------
// Which dense solver takes a system.  The shared-memory kernels (k_system_solve, k_farm_response) keep every system whose
// augmented matrix fits in the device's opt-in shared memory next to the kernel's static shared memory; everything larger
// goes to the global-memory LU (lu_global).  Without a device the rule uses an H100's limits and the static sizes of the
// sm_90a build, so that the workspace query answers the same on a machine without a GPU.
static size_t dev_attr(cudaDeviceAttr a, size_t fallback)
{
    int dev = 0, v = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&v, a, dev) != cudaSuccess) { cudaGetLastError(); return fallback; }
    return (size_t)v;
}
static size_t smem_optin() { return dev_attr(cudaDevAttrMaxSharedMemoryPerBlockOptin, 227 * 1024); }
static size_t smem_per_sm() { return dev_attr(cudaDevAttrMaxSharedMemoryPerMultiprocessor, 228 * 1024); }
template <class K> static size_t static_smem(K kernel, size_t fallback)
{
    cudaFuncAttributes fa;
    if (cudaFuncGetAttributes(&fa, kernel) != cudaSuccess) { cudaGetLastError(); return fallback; }
    return fa.sharedSizeBytes;
}
// static shared memory of the sm_90a build (cudaFuncGetAttributes), used when no device answers
#define SMEM_STATIC_SYS 32
#define SMEM_STATIC_FARM_BLOCK 32
#define SMEM_STATIC_GLU 176
static bool smem_fits(size_t bytes, size_t static_bytes) { return bytes + static_bytes <= smem_optin(); }

// Panel width and CTAs per SM of the global-memory LU: the widest panel (16, 8, ..., 1 columns; n x pw double2 of shared
// memory) with which two CTAs share an SM, else the widest with which one CTA fits.  pw = 0: no panel fits (n > ~14 000).
struct GluPlan { int pw = 0, per_sm = 0; size_t smem = 0; };
static GluPlan glu_plan(int n)
{
    GluPlan g;
    const size_t st = static_smem(k_system_solve_global, SMEM_STATIC_GLU), per_sm = smem_per_sm(), optin = smem_optin();
    for (int ctas = 2; ctas >= 1 && !g.pw; ctas--)
        for (int pw = GLU_PWMAX; pw >= 1; pw >>= 1) {
            const size_t b = (size_t)n * pw * sizeof(double2);
            if (b + st <= optin && ctas * (b + st + 1024) <= per_sm) { g.pw = pw; g.per_sm = ctas; g.smem = b; break; }
        }
    return g;
}

static int launch_system_global(int n, int nw, int nrhs, double *Z, double *F, int32_t *info, cudaStream_t st)
{
    const GluPlan g = glu_plan(n);
    if (!g.pw) return set_err(RAFTK_EINVAL, "system solve: n too large for one panel column in shared memory");
    static SmemOptIn opt(0);                          // static + dynamic shared memory may pass 48 KB below 48 KB of panel
    CUDA_TRY(opt.ensure(k_system_solve_global, g.smem));
    const int grid = std::min(nw, g.per_sm * sm_count());
    k_system_solve_global<<<grid, GLU_T, g.smem, st>>>(n, nw, nrhs, g.pw, reinterpret_cast<double2 *>(Z), reinterpret_cast<double2 *>(F), info);
    g_launches++;
    disp_launch(RAFTK_FAMILY_SYSTEM, RAFTK_KERNEL_SYS_GLOBAL, GLU_T);
    CUDA_TRY(cudaGetLastError());
    return RAFTK_OK;
}

extern "C" int raftk_system_solve_dev(int32_t n, int32_t nw, int32_t nrhs, double *Z, double *F, int32_t *info, void *stream)
{
    disp_reset();
    if (n <= 0 || nw <= 0 || nrhs <= 0 || !Z || !F) return set_err(RAFTK_EINVAL, "bad system-solve arguments");
    const size_t smem = (size_t)n * (n + nrhs) * sizeof(double2);
    if (!smem_fits(smem, static_smem(k_system_solve, SMEM_STATIC_SYS))) return launch_system_global(n, nw, nrhs, Z, F, info, (cudaStream_t)stream);
    static SmemOptIn opt(48 * 1024);
    CUDA_TRY(opt.ensure(k_system_solve, smem));
    k_system_solve<<<nw, 128, smem, (cudaStream_t)stream>>>(n, nrhs, reinterpret_cast<double2 *>(Z), reinterpret_cast<double2 *>(F), info);
    g_launches++;
    disp_launch(RAFTK_FAMILY_SYSTEM, n > 24 ? RAFTK_KERNEL_SYS_BLOCKED : RAFTK_KERNEL_SYS_UNBLOCKED, 128);   // k_system_solve's switch
    CUDA_TRY(cudaGetLastError());
    return RAFTK_OK;
}

// true when the shared-memory farm kernels take a farm of N FOWTs (6N <= 24: warp per system; else one CTA per system with
// the [6N][6N+1] system in shared memory); false sends it to k_farm_response_global
static bool farm_on_chip(int N)
{
    const int n = 6 * N;
    return n <= 24 || smem_fits((size_t)n * (n + 1) * sizeof(double2), static_smem(k_farm_response<false>, SMEM_STATIC_FARM_BLOCK));
}

// workspace of k_farm_response_global: one [6N][6N+1] slab per resident CTA, no more slabs than (case, frequency) systems
static size_t farm_slab_bytes(int N) { return (size_t)6 * N * (6 * N + 1) * sizeof(double2); }
static size_t farm_ws_bytes(const raftk_designs *d, const raftk_cases *c, const raftk_farm *f)
{
    if (!d || !c || !f || f->n_fowt < 1 || d->nw < 1 || c->n_cases < 1 || farm_on_chip(f->n_fowt)) return 0;
    const GluPlan g = glu_plan(6 * f->n_fowt);
    const long long slabs = std::min<long long>((long long)c->n_cases * d->nw, (long long)std::max(g.per_sm, 1) * sm_count());
    return (size_t)slabs * farm_slab_bytes(f->n_fowt);
}

extern "C" size_t raftk_farm_workspace_bytes(const raftk_designs *d, const raftk_cases *c, const raftk_farm *f)
{
    return farm_ws_bytes(d, c, f);
}

static int farm_launch(const raftk_designs *d, const raftk_cases *c, const raftk_outputs *solved, const raftk_farm *f, void *ws,
                       size_t ws_bytes, cudaStream_t st)
{
    if (!d || !c || !solved || !f) return set_err(RAFTK_EINVAL, "farm response: null argument");
    if (f->n_fowt != d->n_designs || f->n_fowt < 1) return set_err(RAFTK_EINVAL, "farm response: farm.n_fowt must equal designs.n_designs");
    if (!solved->B_drag || !solved->F_drag || !solved->F_iner || !f->Xi_sys)
        return set_err(RAFTK_EINVAL, "farm response needs B_drag, F_drag, F_iner of the per-FOWT solve and farm.Xi_sys");
    if (d->n_bem_head > 0 && !solved->F_BEM) return set_err(RAFTK_EINVAL, "farm response: the designs carry BEM excitation, F_BEM is required");
    const int n = 6 * f->n_fowt;
    if (!farm_on_chip(f->n_fowt)) {
        // persistent CTAs over the (case, frequency) systems, each CTA on its own slab of the caller's workspace
        const GluPlan g = glu_plan(n);
        if (!g.pw) return set_err(RAFTK_EINVAL, "farm response: 6N too large for one panel column in shared memory");
        const size_t slab = farm_slab_bytes(f->n_fowt);
        if (!ws || ws_bytes < slab)
            return set_err(RAFTK_EINVAL, "farm response: a farm this size needs a workspace of at least one [6N][6N+1] slab "
                                         "(raftk_farm_workspace_bytes, raftk_farm_response_ws_dev)");
        const long long nsys = (long long)c->n_cases * d->nw;
        const int grid = (int)std::min<long long>(std::min<long long>(nsys, (long long)(ws_bytes / slab)), (long long)g.per_sm * sm_count());
        static SmemOptIn opt_g(0);
        CUDA_TRY(opt_g.ensure(k_farm_response_global, g.smem));
        DesignsDev D = to_dev(d, d->max_nodes, d->max_members);
        CasesDev C = to_dev(c);
        FarmParams P;
        P.N = f->n_fowt; P.nC = c->n_cases; P.nw = d->nw;
        P.B_drag = solved->B_drag;
        P.F_drag = reinterpret_cast<const double2 *>(solved->F_drag);
        P.F_iner = reinterpret_cast<const double2 *>(solved->F_iner);
        P.F_BEM = d->n_bem_head > 0 ? reinterpret_cast<const double2 *>(solved->F_BEM) : nullptr;
        P.M_arr = f->M_arr; P.B_arr = f->B_arr; P.C_arr = f->C_arr;
        P.Xi = reinterpret_cast<double2 *>(f->Xi_sys); P.info = f->info;
        {
            ProfScope ps(st, 1);
            k_farm_response_global<<<grid, GLU_T, g.smem, st>>>(D, C, P, static_cast<double2 *>(ws), g.pw);
            disp_launch(RAFTK_FAMILY_FARM, RAFTK_KERNEL_FARM_GLOBAL, GLU_T);
        }
        g_launches++;
        CUDA_TRY(cudaGetLastError());
        return RAFTK_OK;
    }
    const bool warp = n <= 24;                          // one warp per (frequency, case), wpc systems per CTA; blocked LU above
    const size_t sys_bytes = (size_t)n * (n + 1) * sizeof(double2);
    const int wpc = warp ? (int)std::max<size_t>(1, std::min<size_t>(FARM_WPC, (100 * 1024) / sys_bytes)) : 1;
    const size_t smem = (size_t)wpc * sys_bytes;
    if (c->n_cases > 65535) return set_err(RAFTK_EINVAL, "farm response: more than 65535 cases per call");
    static SmemOptIn opt_w(48 * 1024), opt_b(48 * 1024);
    if (warp) CUDA_TRY(opt_w.ensure(k_farm_response<true>, smem));
    else CUDA_TRY(opt_b.ensure(k_farm_response<false>, smem));
    DesignsDev D = to_dev(d, d->max_nodes, d->max_members);
    CasesDev C = to_dev(c);
    FarmParams P;
    P.N = f->n_fowt; P.nC = c->n_cases; P.nw = d->nw;
    P.B_drag = solved->B_drag;
    P.F_drag = reinterpret_cast<const double2 *>(solved->F_drag);
    P.F_iner = reinterpret_cast<const double2 *>(solved->F_iner);
    P.F_BEM = d->n_bem_head > 0 ? reinterpret_cast<const double2 *>(solved->F_BEM) : nullptr;
    P.M_arr = f->M_arr; P.B_arr = f->B_arr; P.C_arr = f->C_arr;
    P.Xi = reinterpret_cast<double2 *>(f->Xi_sys); P.info = f->info;
    {
        ProfScope ps(st, 1);
        // 6N = 12 (the shipped two-FOWT farm): rows in registers, one lane per row, two systems per warp (k_farm_rows);
        // RAFTK_FARM_SMEM=1 keeps the shared-memory warp kernel (A/B).  At 6N = 18 / 24 the register rows need 188 / 238
        // registers, so those stay on the warp kernel.
        const bool rows = n == 12 && !getenv("RAFTK_FARM_SMEM");
        if (rows) k_farm_rows<12><<<dim3((d->nw + 7) / 8, c->n_cases), 128, 0, st>>>(D, C, P);
        else if (warp) k_farm_response<true><<<dim3((d->nw + wpc - 1) / wpc, c->n_cases), 32 * wpc, smem, st>>>(D, C, P);
        else k_farm_response<false><<<dim3(d->nw, c->n_cases), 256, smem, st>>>(D, C, P);
        if (rows) disp_launch(RAFTK_FAMILY_FARM, RAFTK_KERNEL_FARM_ROWS12, 128);
        else if (warp) disp_launch(RAFTK_FAMILY_FARM, RAFTK_KERNEL_FARM_WARP, 32 * wpc);
        else disp_launch(RAFTK_FAMILY_FARM, RAFTK_KERNEL_FARM_BLOCK, 256);
    }
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RAFTK_OK;
}

extern "C" int raftk_farm_response_dev(const raftk_designs *d, const raftk_cases *c, const raftk_outputs *solved, const raftk_farm *f,
                                       void *stream)
{
    disp_reset();
    return farm_launch(d, c, solved, f, nullptr, 0, (cudaStream_t)stream);
}

extern "C" int raftk_farm_response_ws_dev(const raftk_designs *d, const raftk_cases *c, const raftk_outputs *solved, const raftk_farm *f,
                                          void *workspace, size_t workspace_bytes, void *stream)
{
    disp_reset();
    return farm_launch(d, c, solved, f, workspace, workspace_bytes, (cudaStream_t)stream);
}


// ---- native node-table builder for design families (pure host code, raftk_builder.h) ---------------------------------
static int set_err_i(int code, const char *fmt, int a = 0, int b = 0)
{
    snprintf(g_err, sizeof(g_err), fmt, a, b);
    return code;
}

static int family_run(const raftk_family *f, raftk_family_tables *t, int32_t *n_mem_total, int32_t *n_node_total)
{
    if (!f || f->n_designs <= 0 || f->n_members <= 0 || !f->members) return set_err(RAFTK_EINVAL, "family: empty family");
    for (int m = 0; m < f->n_members; m++) {
        const raftk_family_member &M = f->members[m];
        if (M.n_stations < 2) return set_err_i(RAFTK_EINVAL, "family: member %d: at least two stations entries must be provided", m);
        if (!M.stations || !M.rA || !M.rB || !M.d || !M.Cd_q || !M.Cd_p1 || !M.Cd_p2 || !M.Cd_End || !M.Ca_p1 || !M.Ca_p2 || !M.Ca_End)
            return set_err_i(RAFTK_EINVAL, "family: member %d: null array", m);
        if (!(M.dls_max > 0.0)) return set_err_i(RAFTK_EINVAL, "family: member %d: dls_max must be positive", m);
    }
    std::vector<rkb::MemberOut> mem(f->n_members);
    int64_t nm = 0, nn = 0;
    int max_nodes = 0, max_members = 0, mw = 0, mh = 0, mz = 0;
    if (t) t->member_offset[0] = 0, t->mem_node_start[0] = 0;
    for (int d = 0; d < f->n_designs; d++) {
        double A[36];
        for (int i = 0; i < 36; i++) A[i] = 0.0;
        int kept = 0, nodes = 0;
        for (int m = 0; m < f->n_members; m++) {
            const int rc = rkb::build_member(f->members[m], d, f->rho, f->g, f->Rp, f->r0, mem[m], A, t == nullptr);
            if (rc == -1) return set_err_i(RAFTK_EINVAL, "RAFT Members cannot start or end on the waterplane (design %d, member %d)", d, m);
            if (rc) return set_err_i(RAFTK_EINVAL, "family: the station list of member %d is not in ascending order", m);
            if (!mem[m].nodes.empty()) { kept++; nodes += (int)mem[m].nodes.size(); }
        }
        if (t) {
            for (int m = 0; m < f->n_members; m++) {
                const rkb::MemberOut &M = mem[m];
                if (M.nodes.empty()) continue;
                for (int a = 0; a < 3; a++) {
                    t->mem_frame[9 * nm + a] = M.q[a]; t->mem_frame[9 * nm + 3 + a] = M.p1[a]; t->mem_frame[9 * nm + 6 + a] = M.p2[a];
                    t->mem_rA[3 * nm + a] = M.rA[a]; t->mem_arm[3 * nm + a] = M.rA[a] - f->r0[a];
                }
                t->mem_circ[nm] = M.circ;
                for (const rkb::Node &N : M.nodes) {
                    t->node_ls[nn] = N.ls; t->node_cd_q[nn] = N.cd_q; t->node_cd_p1[nn] = N.cd_p1; t->node_cd_p2[nn] = N.cd_p2;
                    t->node_in_q[nn] = N.in_q; t->node_in_p1[nn] = N.in_p1; t->node_in_p2[nn] = N.in_p2; t->node_pa[nn] = N.pa;
                    nn++;
                }
                nm++;
                t->mem_node_start[nm] = (int32_t)nn;
            }
            t->member_offset[d + 1] = (int32_t)nm;
            for (int i = 0; i < 36; i++) t->A_morison[36 * (size_t)d + i] = A[i];
            int nW, nH, nZ;
            rkb::count_classes(mem, nW, nH, nZ);
            mw = std::max(mw, nW); mh = std::max(mh, nH); mz = std::max(mz, nZ);
        } else { nm += kept; nn += nodes; }
        max_nodes = std::max(max_nodes, nodes); max_members = std::max(max_members, kept);
        if (nn > 2000000000LL) return set_err(RAFTK_EINVAL, "family: more than 2^31 nodes");
    }
    if (n_mem_total) *n_mem_total = (int32_t)nm;
    if (n_node_total) *n_node_total = (int32_t)nn;
    if (t) {
        t->max_nodes = std::max(1, max_nodes); t->max_members = std::max(1, max_members);
        t->max_w_classes = std::max(1, mw); t->max_h_classes = std::max(1, mh); t->max_z_classes = std::max(1, mz);
    }
    return RAFTK_OK;
}

extern "C" int raftk_family_sizes(const raftk_family *f, int32_t *n_members_total, int32_t *n_nodes_total)
{
    if (!n_members_total || !n_nodes_total) return set_err(RAFTK_EINVAL, "family sizes: null output");
    return family_run(f, nullptr, n_members_total, n_nodes_total);
}

extern "C" int raftk_build_family_host(const raftk_family *f, raftk_family_tables *t)
{
    if (!t || !t->member_offset || !t->mem_node_start || !t->mem_circ || !t->mem_frame || !t->mem_rA || !t->mem_arm || !t->node_ls ||
        !t->node_cd_q || !t->node_cd_p1 || !t->node_cd_p2 || !t->node_in_q || !t->node_in_p1 || !t->node_in_p2 || !t->node_pa || !t->A_morison)
        return set_err(RAFTK_EINVAL, "family tables: null array");
    return family_run(f, t, nullptr, nullptr);
}

// ---- host-pointer front ends -------------------------------------------------------------------------
// A *_host call stages through one Staging: it declares its inputs, device-only buffers and outputs, commits once (which
// sizes the device arena from that same list and uploads the inputs), runs its *_dev twin and finishes (downloads, one
// synchronise).  The arena is grow-only, one per device: no cudaMalloc / cudaFree on the call path once its high-water mark
// has been reached (SURVEY.md 8b: no hidden allocation per call).
//
// Small inputs (grid, member/node tables, case table: ~30 arrays of a few KB) are packed into one pinned block and sent with
// a single copy to the head of the arena; only large arrays (frequency tables, big sweeps) are copied one by one.  This trims
// ~100 us of per-copy launch overhead per call.
static const size_t PIN_BYTES = (size_t)256 << 10, PIN_MAX = (size_t)64 << 10;   // a typical call packs ~30 KB
struct Arena { char *base = nullptr; size_t cap = 0; };
static Arena g_arena[RAFTK_MAX_DEV];       // one per device: the *_host paths run on whichever device is current
static char *g_pin = nullptr;              // pinned, PIN_BYTES, one per process
static std::mutex g_stage_mu;              // the arenas and the pinned block

class Staging {
    struct Buf { const void *from; void *to; size_t bytes; const void **slot; size_t off; bool pinned; };
    std::lock_guard<std::mutex> lk_;
    const char *who_;
    std::vector<Buf> bufs_;
    char *base_ = nullptr;
    bool pending_ = false;                 // copies enqueued that finish() has not waited for
    cudaError_t e_ = cudaSuccess;
    void note(cudaError_t r) { if (r != cudaSuccess && e_ == cudaSuccess) e_ = r; }

public:
    explicit Staging(const char *who) : lk_(g_stage_mu), who_(who) { bufs_.reserve(64); }
    ~Staging() { if (pending_) cudaStreamSynchronize(0); }     // an early return: the next call reuses the pinned block
    // n elements on the device, uploaded from `from` by commit() and downloaded to `to` by finish() when those are given;
    // *slot receives the device address, NULL when n is 0
    template <class T> void buf(T *&slot, size_t n, const std::remove_const_t<T> *from = nullptr, std::remove_const_t<T> *to = nullptr)
    {
        bufs_.push_back({from, to, n * sizeof(T), (const void **)&slot, 0, false});
    }
    template <class T> void in(T *&slot, const std::remove_const_t<T> *h, size_t n) { buf(slot, h ? n : 0, h); }   // NULL h: NULL slot
    template <class T> void out(T *&slot, size_t n, std::remove_const_t<T> *h) { buf(slot, n, nullptr, h); }      // NULL h: no download

    int commit()
    {
        if (!g_pin && cudaHostAlloc(&g_pin, PIN_BYTES, cudaHostAllocPortable) != cudaSuccess) { cudaGetLastError(); g_pin = nullptr; }
        size_t pin = 0;                    // the head of the arena mirrors the pinned block
        for (Buf &b : bufs_)
            if (b.from && b.bytes && b.bytes <= PIN_MAX && g_pin && pin + align_up(b.bytes, 256) <= PIN_BYTES) {
                b.off = pin; b.pinned = true; pin += align_up(b.bytes, 256);
            }
        size_t total = pin;
        for (Buf &b : bufs_)
            if (!b.pinned) { b.off = total; total += align_up(b.bytes, 256); }
        Arena &A = g_arena[cur_dev()];
        if (total > A.cap) {
            if (A.base) cudaFree(A.base);
            A.base = nullptr; A.cap = 0;
            if (cudaMalloc(&A.base, total) != cudaSuccess) { cudaGetLastError(); A.base = nullptr; return set_err(RAFTK_ENOMEM, "%s: device arena allocation failed", who_); }
            A.cap = total;
        }
        base_ = A.base;
        pending_ = true;
        for (Buf &b : bufs_) {
            *b.slot = b.bytes ? base_ + b.off : nullptr;
            if (!b.from || !b.bytes) continue;
            if (b.pinned) memcpy(g_pin + b.off, b.from, b.bytes);
            else note(cudaMemcpyAsync(base_ + b.off, b.from, b.bytes, cudaMemcpyHostToDevice, 0));
        }
        if (pin) note(cudaMemcpyAsync(base_, g_pin, pin, cudaMemcpyHostToDevice, 0));
        return e_ == cudaSuccess ? RAFTK_OK : set_err(RAFTK_ECUDA, "%s: H2D copy: %s", who_, cudaGetErrorString(e_));
    }

    int finish()
    {
        for (const Buf &b : bufs_)
            if (b.to && b.bytes) note(cudaMemcpyAsync(b.to, base_ + b.off, b.bytes, cudaMemcpyDeviceToHost, 0));
        const cudaError_t se = cudaStreamSynchronize(0);
        pending_ = false;
        if (se != cudaSuccess) e_ = se;
        return e_ == cudaSuccess ? RAFTK_OK : set_err(RAFTK_ECUDA, "%s: %s", who_, cudaGetErrorString(e_));
    }
};

// the design and case tables of a host call (dd, cc: copies of *d, *c whose pointers commit() turns into device addresses)
static void stage_designs_cases(Staging &S, const raftk_designs *d, const raftk_cases *c, raftk_designs &dd, raftk_cases &cc)
{
    const size_t nD = d->n_designs, nw = d->nw, nC = c->n_cases, Nm = d->n_members_total, Ns = d->n_nodes_total;
    const size_t nR = nD * nC * 6 * nw * 2;             // doubles of one complex [nD,nC,6,nw] array
    S.in(dd.w, d->w, nw); S.in(dd.k, d->k, nw);
    S.in(dd.member_offset, d->member_offset, nD + 1);
    S.in(dd.mem_frame, d->mem_frame, Nm * 9); S.in(dd.mem_rA, d->mem_rA, Nm * 3); S.in(dd.mem_arm, d->mem_arm, Nm * 3);
    S.in(dd.mem_node_start, d->mem_node_start, Nm + 1); S.in(dd.mem_circ, d->mem_circ, Nm);
    S.in(dd.node_ls, d->node_ls, Ns); S.in(dd.node_cd_q, d->node_cd_q, Ns);
    S.in(dd.node_cd_p1, d->node_cd_p1, Ns); S.in(dd.node_cd_p2, d->node_cd_p2, Ns);
    S.in(dd.node_in_q, d->node_in_q, Ns); S.in(dd.node_in_p1, d->node_in_p1, Ns);
    S.in(dd.node_in_p2, d->node_in_p2, Ns); S.in(dd.node_pa, d->node_pa, Ns);
    S.in(dd.node_in_p1_w, d->node_in_p1_w, Ns * nw * 2); S.in(dd.node_in_p2_w, d->node_in_p2_w, Ns * nw * 2);
    S.in(dd.M0, d->M0, nD * 36); S.in(dd.B0, d->B0, nD * 36); S.in(dd.C0, d->C0, nD * 36);
    S.in(dd.A_w, d->A_w, nD * 36 * nw); S.in(dd.B_w, d->B_w, nD * 36 * nw);
    if (d->n_bem_head > 0) {
        S.in(dd.bem_headings, d->bem_headings, (size_t)d->n_bem_head);
        S.in(dd.X_BEM, d->X_BEM, nD * d->n_bem_head * 6 * nw * 2);
        S.in(dd.bem_xyh, d->bem_xyh, nD * 3);
    }
    S.in(cc.Hs, c->Hs, nC); S.in(cc.Tp, c->Tp, nC); S.in(cc.gamma, c->gamma, nC);
    S.in(cc.beta_deg, c->beta_deg, nC); S.in(cc.spec, c->spec, nC);
    S.in(cc.zeta, c->zeta, nC * nw);
    S.in(cc.primary, c->primary, nC);
    S.in(cc.F_2nd, c->F_2nd, nR / 2);
    S.in(cc.Xi_init, c->Xi_init, nR);
    if (d->n_qtf_w > 0) {
        S.in(dd.qtf_w, d->qtf_w, (size_t)d->n_qtf_w);
        S.in(dd.qtf_heads, d->qtf_heads, (size_t)d->n_qtf_head);
        S.in(dd.qtf, d->qtf, (d->qtf_shared == 1 ? 1 : (d->qtf_shared == 2 ? nD * nC : nD)) * (size_t)d->n_qtf_w * d->n_qtf_w * d->n_qtf_head * 12);
    }
}

static int host_run(const char *who, const raftk_designs *d, const raftk_cases *c, const raftk_solve_opts *o, const raftk_outputs *out,
                    const double *Xi_in, int mode, const raftk_farm *farm = nullptr)
{
    disp_reset();
    int rc = validate(d, c);
    if (rc) return rc;
    if (!out) return set_err(RAFTK_EINVAL, "null outputs");
    Staging S(who);
    const size_t nD = d->n_designs, nw = d->nw, nC = c->n_cases;
    const size_t nR = nD * nC * 6 * nw * 2;             // doubles of one complex [nD,nC,6,nw] array
    raftk_designs dd = *d;
    raftk_cases cc = *c;
    stage_designs_cases(S, d, c, dd, cc);
    const double *Xi_in_d = nullptr;
    S.in(Xi_in_d, Xi_in, nR);
    raftk_farm fd;
    memset(&fd, 0, sizeof(fd));
    if (farm) {                                           // array-level matrices: staged with the other small inputs
        fd = *farm;
        S.in(fd.M_arr, farm->M_arr, 36 * nD * nD); S.in(fd.B_arr, farm->B_arr, 36 * nD * nD); S.in(fd.C_arr, farm->C_arr, 36 * nD * nD);
    }
    // the solve is planned once, at the caller's cluster size, and launched with the workspace that plan needs; excitation
    // and linearisation need the whole batch's tables in one chunk
    const SolvePlan pl = mode == 0 ? plan_solve(d, (int)nC, o->cluster_size, WS_UNBOUNDED) : SolvePlan{};
    const size_t wb = mode == 0 ? pl.bytes : chunk_bytes((int)nD, (int)nC, d->max_nodes, (int)nw);
    // Page-locked output buffers (raftk_host_alloc / cudaHostAlloc / cudaHostRegister): the solve kernel stores every finished
    // unit's Xi and status word straight into host memory through the unified address space -- the same epilogue that feeds
    // peer GPUs, with the host as the "peer" -- so the device-to-host transfer overlaps the units still iterating instead of
    // following the kernel as a separate copy.  RAFTK_NO_DIRECT_D2H=1 keeps the copy (A/B).
    double *xi_direct = nullptr;
    int32_t *st_direct = nullptr;
    if (mode == 0 && out->Xi && !getenv("RAFTK_NO_DIRECT_D2H")) {
        cudaPointerAttributes pa;
        const bool pinned_xi = cudaPointerGetAttributes(&pa, out->Xi) == cudaSuccess && pa.type == cudaMemoryTypeHost && pa.devicePointer != nullptr;
        if (!pinned_xi) cudaGetLastError();
        if (pl.kind != SOLVE_V1 && pinned_xi) {
            xi_direct = static_cast<double *>(pa.devicePointer);          // block of "rank 0" inside the host array = its start
            cudaPointerAttributes ps;
            if (out->status && cudaPointerGetAttributes(&ps, out->status) == cudaSuccess && ps.type == cudaMemoryTypeHost && ps.devicePointer)
                st_direct = static_cast<int32_t *>(ps.devicePointer);
            else cudaGetLastError();
        }
    }
    raftk_outputs od;
    memset(&od, 0, sizeof(od));
    S.out(od.Xi, out->Xi ? nR : 0, xi_direct ? nullptr : out->Xi);
    S.out(od.status, out->status ? nD * nC * 4 : 0, st_direct ? nullptr : out->status);
    // the system response reads the per-FOWT loads on the device: those buffers exist even when the caller does not want them back
    S.out(od.B_drag, out->B_drag || farm ? nD * nC * 36 : 0, out->B_drag);
    S.out(od.F_drag, out->F_drag || farm ? nR : 0, out->F_drag);
    S.out(od.F_iner, out->F_iner || farm ? nR : 0, out->F_iner);
    S.out(od.F_BEM, out->F_BEM || (farm && d->n_bem_head > 0) ? nR : 0, out->F_BEM);
    S.out(od.zeta, out->zeta ? nC * nw : 0, out->zeta);
    const bool qtf_solve = (mode == 0 && d->n_qtf_w > 0 && !c->F_2nd);   // potSecOrder 2: compute the force on the device first
    if (qtf_solve) { S.out(od.F_2nd, nR / 2, out->F_2nd); S.out(od.F_2nd_mean, nD * nC * 6, out->F_2nd_mean); }
    S.out(od.Xi_last, out->Xi_last ? nR : 0, out->Xi_last);
    char *ws, *fws = nullptr;
    S.buf(ws, wb);
    const size_t fwb = farm ? farm_ws_bytes(d, c, farm) : 0;                  // slabs of the global-memory system kernel (0 on chip)
    if (farm) { S.out(fd.Xi_sys, nR, farm->Xi_sys); S.out(fd.info, farm->info ? nC * nw : 0, farm->info); S.buf(fws, fwb); }
    if ((rc = S.commit())) return rc;
    if (qtf_solve) {
        if ((rc = run_qtf(&dd, &cc, od.F_2nd, od.F_2nd_mean, 0))) return rc;
        cc.F_2nd = od.F_2nd;
    }
    raftk_peers hostpeer;
    if (xi_direct) {
        memset(&hostpeer, 0, sizeof(hostpeer));
        hostpeer.n_ranks = 2; hostpeer.rank = 0; hostpeer.epoch = 1; hostpeer.block_elems = nR / 2;
        hostpeer.gathered[0] = od.Xi; hostpeer.gathered[1] = xi_direct; hostpeer.status[1] = st_direct;
    }
    if (mode == 0) rc = launch_solve(&dd, &cc, o, &od, pl, ws, wb, 0, xi_direct ? &hostpeer : nullptr);
    else {
        rc = tables(&dd, &cc, nullptr, &od, 2, ws, wb, 0);
        if (!rc && mode == 1) rc = tables(&dd, &cc, Xi_in_d, &od, 1, ws, wb, 0);
    }
    if (rc) return rc;
    if (farm && (rc = farm_launch(&dd, &cc, &od, &fd, fws, fwb, 0))) return rc;
    g_disp.direct_d2h = xi_direct != nullptr;
    return S.finish();
}

extern "C" int raftk_hydro_excitation_host(const raftk_designs *d, const raftk_cases *c, const raftk_outputs *out)
{
    return host_run("raftk_hydro_excitation_host", d, c, nullptr, out, nullptr, 2);
}
extern "C" int raftk_hydro_linearization_host(const raftk_designs *d, const raftk_cases *c, const double *Xi_in, const raftk_outputs *out)
{
    if (!Xi_in) return set_err(RAFTK_EINVAL, "null Xi_in");
    return host_run("raftk_hydro_linearization_host", d, c, nullptr, out, Xi_in, 1);
}
extern "C" int raftk_solve_dynamics_host(const raftk_designs *d, const raftk_cases *c, const raftk_solve_opts *o, const raftk_outputs *out)
{
    if (!out || !out->Xi || !out->status || !o) return set_err(RAFTK_EINVAL, "Xi, status and opts are required");
    return host_run("raftk_solve_dynamics_host", d, c, o, out, nullptr, 0);
}

extern "C" int raftk_solve_dynamics_farm_host(const raftk_designs *d, const raftk_cases *c, const raftk_solve_opts *o,
                                              const raftk_outputs *out, const raftk_farm *f)
{
    if (!out || !out->Xi || !out->status || !o) return set_err(RAFTK_EINVAL, "Xi, status and opts are required");
    if (!f || !f->Xi_sys) return set_err(RAFTK_EINVAL, "farm.Xi_sys is required");
    if (d && f->n_fowt != d->n_designs) return set_err(RAFTK_EINVAL, "farm response: farm.n_fowt must equal designs.n_designs");
    return host_run("raftk_solve_dynamics_farm_host", d, c, o, out, nullptr, 0, f);
}

extern "C" int raftk_second_order_force_host(const raftk_designs *d, const raftk_cases *c, const raftk_outputs *out)
{
    disp_reset();
    if (!out || !out->F_2nd) return set_err(RAFTK_EINVAL, "outputs.F_2nd is required");
    int rc = validate_qtf(d, c);
    if (rc) return rc;
    const size_t nD = d->n_designs, nw = d->nw, nC = c->n_cases, n2 = d->n_qtf_w, nh = d->n_qtf_head, nF = nD * nC * 6 * nw;
    Staging S("raftk_second_order_force_host");
    raftk_designs dd = *d;
    S.in(dd.w, d->w, nw); S.in(dd.qtf_w, d->qtf_w, n2); S.in(dd.qtf_heads, d->qtf_heads, nh);
    S.in(dd.qtf, d->qtf, (d->qtf_shared == 1 ? 1 : (d->qtf_shared == 2 ? nD * nC : nD)) * n2 * n2 * nh * 12);
    raftk_cases cc = *c;
    S.in(cc.Hs, c->Hs, nC); S.in(cc.Tp, c->Tp, nC); S.in(cc.gamma, c->gamma, nC); S.in(cc.beta_deg, c->beta_deg, nC);
    S.in(cc.spec, c->spec, nC); S.in(cc.zeta, c->zeta, nC * nw);
    cc.primary = nullptr; cc.F_2nd = nullptr;
    double *F2, *F2mean;
    S.out(F2, nF, out->F_2nd); S.out(F2mean, nF / nw, out->F_2nd_mean);
    if ((rc = S.commit()) || (rc = run_qtf(&dd, &cc, F2, F2mean, 0))) return rc;
    return S.finish();
}

// ---- generalised degrees of freedom (flexible members) ---------------------------------------------------------------
struct GenLayout { size_t u, f6, Fi, Fd, XL, Bm, Bd, Z, pv, fl, fb6, FB, F2, F2m, total; };
static GenLayout gen_layout(const raftk_general *g, const raftk_general_fd *fd, const raftk_general_qtf *q, size_t nC)
{
    const size_t n = g->n_dof, nw = g->nw, Ns = std::max(g->n_nodes, 1);
    const size_t nbem = (fd && fd->n_bem_head > 0) ? 1 : 0, nq = q ? 1 : 0;
    GenLayout L; size_t t = 0;
    auto take = [&](size_t b) { size_t o = t; t += align_up(b, 256); return o; };
    L.u = take(nC * Ns * 3 * nw * 16); L.f6 = take(nC * Ns * 6 * nw * 16);
    L.Fi = take(nC * n * nw * 16); L.Fd = take(nC * n * nw * 16); L.XL = take(nC * n * nw * 16);
    L.Bm = take(nC * Ns * 9 * 8); L.Bd = take(nC * n * n * 8);
    L.Z = take(nC * nw * n * (n + 1) * 16); L.pv = take(nC * nw * n * 4); L.fl = take(nC * 16);
    L.fb6 = take(nbem * nC * 6 * nw * 16); L.FB = take(nbem * nC * n * nw * 16);     // BEM force (full DOFs 0-5, reduced DOFs)
    L.F2 = take(nq * nC * 6 * nw * 8); L.F2m = take(nq * nC * 6 * 8);                 // second-order force and mean drift
    L.total = t;
    return L;
}

// raftk_general_qtf checks (include/raftk.h); qw, qh: host copies of qtf_w and qtf_heads, read only once the counts and
// pointers have passed
static int validate_gen_qtf(const raftk_general *g, const raftk_general_qtf *q, const double *qw, const double *qh)
{
    if (q->n_qtf_w < 2 || q->n_qtf_head < 1 || !q->qtf || !q->qtf_w || !q->qtf_heads)
        return set_err(RAFTK_EINVAL, "general solve: qtf needs n_qtf_w >= 2, n_qtf_head >= 1, qtf, qtf_w and qtf_heads");
    if (g->n_dof < 6) return set_err(RAFTK_EINVAL, "general solve: a QTF table needs n_dof >= 6 (it loads reduced DOFs 0-5)");
    if ((size_t)g->nw * 20 > 227 * 1024) return set_err(RAFTK_EINVAL, "general solve: nw too large for the second-order force kernel's shared-memory tables");
    if (!qw || !qh) return 0;
    for (int t = 1; t < q->n_qtf_w; t++)
        if (!(qw[t] > qw[t - 1])) return set_err(RAFTK_EINVAL, "general solve: qtf.qtf_w must be strictly increasing");
    for (int t = 1; t < q->n_qtf_head; t++)
        if (!(qh[t] > qh[t - 1])) return set_err(RAFTK_EINVAL, "general solve: qtf.qtf_heads must be strictly increasing");
    return 0;
}

// raftk_general_fd checks on host copies of fd_idx and bem_headings (include/raftk.h)
static int validate_gen_fd(const raftk_general *g, const raftk_general_fd *fd, const int32_t *idx, const double *hd)
{
    if (fd->n_fd < 0 || fd->n_fd > g->n_dof) return set_err(RAFTK_EINVAL, "general solve: fd.n_fd must be in [0, n_dof]");
    if (fd->n_bem_head < 0) return set_err(RAFTK_EINVAL, "general solve: fd.n_bem_head must be >= 0");
    if (fd->n_fd > 0 && (!fd->fd_idx || !fd->A_w || !fd->B_w))
        return set_err(RAFTK_EINVAL, "general solve: fd.n_fd > 0 needs fd_idx, A_w and B_w");
    if (fd->n_bem_head > 0 && (!fd->bem_headings || !fd->X_BEM || !fd->T0))
        return set_err(RAFTK_EINVAL, "general solve: fd.n_bem_head > 0 needs bem_headings, X_BEM and T0");
    for (int t = 0; t < fd->n_fd; t++) {
        if (idx[t] < 0 || idx[t] >= g->n_dof) return set_err(RAFTK_EINVAL, "general solve: fd.fd_idx entry out of range [0, n_dof)");
        if (t > 0 && idx[t] <= idx[t - 1]) return set_err(RAFTK_EINVAL, "general solve: fd.fd_idx must be strictly increasing (no repeats)");
    }
    for (int t = 0; t < fd->n_bem_head; t++) {
        if (!(hd[t] >= 0.0 && hd[t] < 360.0)) return set_err(RAFTK_EINVAL, "general solve: fd.bem_headings must lie in [0, 360) deg");
        if (t > 0 && hd[t] < hd[t - 1]) return set_err(RAFTK_EINVAL, "general solve: fd.bem_headings must be non-decreasing");
    }
    return 0;
}

extern "C" size_t raftk_general_qtf_workspace_bytes(const raftk_general *g, const raftk_general_fd *fd, const raftk_general_qtf *qtf,
                                                    int32_t n_cases)
{
    if (!g || n_cases <= 0 || g->n_dof <= 0 || g->nw <= 0) return 0;
    return gen_layout(g, fd, qtf, (size_t)n_cases).total;
}

extern "C" size_t raftk_general_fd_workspace_bytes(const raftk_general *g, const raftk_general_fd *fd, int32_t n_cases)
{
    return raftk_general_qtf_workspace_bytes(g, fd, nullptr, n_cases);
}

extern "C" size_t raftk_general_workspace_bytes(const raftk_general *g, int32_t n_cases)
{
    return raftk_general_fd_workspace_bytes(g, nullptr, n_cases);
}

extern "C" int raftk_general_solve_dynamics_qtf_dev(const raftk_general *g, const raftk_general_fd *fd, const raftk_general_qtf *qtf,
                                                    const raftk_cases *c, const raftk_solve_opts *o, double *Xi, int32_t *status,
                                                    double *F_BEM, double *F_2nd, double *F_2nd_mean, void *workspace,
                                                    size_t workspace_bytes, void *stream)
{
    disp_reset();
    if (!g || !c || !o || !Xi || !status) return set_err(RAFTK_EINVAL, "general solve: null argument");
    if (g->n_dof <= 0 || g->n_dof > 256 || g->nw <= 0 || g->n_nodes < 0 || c->n_cases <= 0 || c->n_cases > 65535)
        return set_err(RAFTK_EINVAL, "general solve: 0 < n_dof <= 256, nw > 0, 0 < n_cases <= 65535");
    if (c->F_2nd || c->Xi_init) return set_err(RAFTK_EINVAL, "general solve: F_2nd / Xi_init are not supported");
    cudaStream_t st = (cudaStream_t)stream;
    if (qtf) {                                         // the frequency and heading vectors are read back for the checks
        if (int rc = validate_gen_qtf(g, qtf, nullptr, nullptr)) return rc;
        std::vector<double> qw(qtf->n_qtf_w), qh(qtf->n_qtf_head);
        CUDA_TRY(cudaMemcpyAsync(qw.data(), qtf->qtf_w, qw.size() * 8, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(qh.data(), qtf->qtf_heads, qh.size() * 8, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaStreamSynchronize(st));
        if (int rc = validate_gen_qtf(g, qtf, qw.data(), qh.data())) return rc;
    }
    if (fd) {                                          // the index and heading tables are read back for the checks
        if (fd->n_fd < 0 || fd->n_fd > g->n_dof || fd->n_bem_head < 0 || (fd->n_fd > 0 && !fd->fd_idx) || (fd->n_bem_head > 0 && !fd->bem_headings))
            return validate_gen_fd(g, fd, nullptr, nullptr);
        std::vector<int32_t> idx(fd->n_fd);
        std::vector<double> hd(fd->n_bem_head);
        if (fd->n_fd > 0) CUDA_TRY(cudaMemcpyAsync(idx.data(), fd->fd_idx, idx.size() * 4, cudaMemcpyDeviceToHost, st));
        if (fd->n_bem_head > 0) CUDA_TRY(cudaMemcpyAsync(hd.data(), fd->bem_headings, hd.size() * 8, cudaMemcpyDeviceToHost, st));
        if (fd->n_fd > 0 || fd->n_bem_head > 0) CUDA_TRY(cudaStreamSynchronize(st));
        if (int rc = validate_gen_fd(g, fd, idx.data(), hd.data())) return rc;
    }
    const size_t nC = c->n_cases;
    const GenLayout L = gen_layout(g, fd, qtf, nC);
    if (!workspace || workspace_bytes < L.total) return set_err(RAFTK_ENOMEM, "general solve: workspace too small");
    const bool bem = fd && fd->n_bem_head > 0;
    GenDev D;
    D.n = g->n_dof; D.nw = g->nw; D.Ns = g->n_nodes; D.depth = g->depth; D.dw = g->dw; D.rho = g->rho;
    D.w = g->w; D.k = g->k; D.node_r = g->node_r; D.node_frame = g->node_frame; D.node_circ = g->node_circ;
    D.node_Imat = g->node_Imat; D.node_Imat_w = reinterpret_cast<const double2 *>(g->node_Imat_w);
    D.node_a_i = g->node_a_i; D.node_cd = g->node_cd; D.Tn = g->Tn; D.rr = g->rr; D.M = g->M; D.B = g->B; D.C = g->C;
    GenFdDev Fx;
    Fx.n_fd = fd ? fd->n_fd : 0; Fx.n_bem_head = bem ? fd->n_bem_head : 0;
    Fx.fd_idx = fd ? fd->fd_idx : nullptr; Fx.A_w = fd ? fd->A_w : nullptr; Fx.B_w = fd ? fd->B_w : nullptr;
    Fx.bem_headings = bem ? fd->bem_headings : nullptr; Fx.X_BEM = bem ? reinterpret_cast<const double2 *>(fd->X_BEM) : nullptr;
    Fx.T0 = bem ? fd->T0 : nullptr;
    Fx.x_ref = fd ? fd->x_ref : 0.0; Fx.y_ref = fd ? fd->y_ref : 0.0; Fx.hadj = fd ? fd->heading_adjust : 0.0;
    char *b = static_cast<char *>(workspace);
    GenWork W;
    W.u = reinterpret_cast<double2 *>(b + L.u); W.f6 = reinterpret_cast<double2 *>(b + L.f6);
    W.F_iner = reinterpret_cast<double2 *>(b + L.Fi); W.F_drag = reinterpret_cast<double2 *>(b + L.Fd);
    W.XiLast = reinterpret_cast<double2 *>(b + L.XL); W.Bmat = reinterpret_cast<double *>(b + L.Bm);
    W.B_drag = reinterpret_cast<double *>(b + L.Bd); W.Z = reinterpret_cast<double2 *>(b + L.Z); W.flags = reinterpret_cast<int *>(b + L.fl);
    W.piv = reinterpret_cast<int *>(b + L.pv);
    Fx.fb6 = bem ? reinterpret_cast<double2 *>(b + L.fb6) : nullptr;
    double2 *Fbem = bem ? (F_BEM ? reinterpret_cast<double2 *>(F_BEM) : reinterpret_cast<double2 *>(b + L.FB)) : nullptr;
    Fx.F_BEM = Fbem;
    const int *prim = c->primary;
    CasesDev C = to_dev(c);
    double2 *X = reinterpret_cast<double2 *>(Xi);
    const unsigned fb = (unsigned)((g->nw + 127) / 128);
    // blocked LU (panel + row block in shared memory); RAFTK_GEN_UNBLOCKED=1 keeps the first, column-at-a-time kernel for A/B runs
    const size_t lu_smem = ((size_t)g->n_dof * GB + (size_t)GB * (g->n_dof + 1)) * sizeof(double2);
    const bool blocked = !getenv("RAFTK_GEN_UNBLOCKED") && lu_smem <= 110 * 1024;
    const bool fdz = Fx.n_fd > 0;                      // impedance with the frequency-dependent terms on their support
    if (blocked) {
        static SmemOptIn opt(48 * 1024), opt_fd(48 * 1024);
        CUDA_TRY(fdz ? opt_fd.ensure(k_gen_solve_blocked<true>, lu_smem) : opt.ensure(k_gen_solve_blocked<false>, lu_smem));
    }
    if (F_BEM && !bem) CUDA_TRY(cudaMemsetAsync(F_BEM, 0, nC * g->n_dof * g->nw * 16, st));
    double *F2 = nullptr;
    if (qtf) {                                         // second-order force of every case and train (k_qtf_*), before the loop
        QtfParams QP;
        QP.nD = 1; QP.shared = 0;
        QP.n2 = qtf->n_qtf_w; QP.nh = qtf->n_qtf_head; QP.nw = g->nw; QP.dw = g->dw;
        QP.w = g->w; QP.qw = qtf->qtf_w; QP.qh = qtf->qtf_heads;
        QP.qtf = reinterpret_cast<const double2 *>(qtf->qtf);
        QP.F2 = F2 = F_2nd ? F_2nd : reinterpret_cast<double *>(b + L.F2);
        QP.F2mean = F_2nd_mean ? F_2nd_mean : reinterpret_cast<double *>(b + L.F2m);
        if (int rc = launch_qtf(QP, c, st)) return rc;
    }
    prof_begin_call();
    k_gen_init<<<(unsigned)nC, 256, 0, st>>>(D, W, o->xi_start, prim);
    if (g->n_nodes > 0) k_gen_wave<<<dim3(fb, g->n_nodes, (unsigned)nC), 128, 0, st>>>(D, C, W);
    if (bem) {                                         // F_BEM = T0^T f_BEM, then F_iner = F_BEM + sum_j Tn_j^T f6_j
        k_gen_bem<<<dim3(fb, (unsigned)nC), 128, 0, st>>>(D, C, Fx);
        k_gen_project<true, false><<<dim3(fb, g->n_dof, (unsigned)nC), 128, 0, st>>>(D, W, Fbem, 0, nullptr, Fx);
        g_launches += 2;
    }
    if (bem) k_gen_project<false, true><<<dim3(fb, g->n_dof, (unsigned)nC), 128, 0, st>>>(D, W, W.F_iner, 0, nullptr, Fx);
    else k_gen_project<false, false><<<dim3(fb, g->n_dof, (unsigned)nC), 128, 0, st>>>(D, W, W.F_iner, 0, nullptr, Fx);
    g_launches += 3;
    if (F2) {                                          // (F_BEM + F_iner) + F_2nd on reduced DOFs 0-5
        k_gen_add_2nd<<<dim3(fb, 6, (unsigned)nC), 128, 0, st>>>(D, W, F2);
        g_launches++;
    }
    for (int pass = 0; pass < o->n_iter + 1; pass++) {
        if (g->n_nodes > 0) k_gen_node_pass<false><<<dim3(g->n_nodes, (unsigned)nC), 128, 0, st>>>(D, W, nullptr);
        k_gen_bdrag<<<dim3(g->n_dof, (unsigned)nC), 128, 0, st>>>(D, W);
        k_gen_project<false, false><<<dim3(fb, g->n_dof, (unsigned)nC), 128, 0, st>>>(D, W, W.F_drag, 1, nullptr, Fx);
        if (blocked) {
            ProfScope ps(st, 2);
            if (fdz) k_gen_solve_blocked<true><<<dim3(g->nw, (unsigned)nC), GT, lu_smem, st>>>(D, W, X, o->tol, Fx);
            else k_gen_solve_blocked<false><<<dim3(g->nw, (unsigned)nC), GT, lu_smem, st>>>(D, W, X, o->tol, Fx);
        } else {
            ProfScope ps(st, 2);
            if (fdz) k_gen_solve<true><<<dim3(g->nw, (unsigned)nC), 256, 0, st>>>(D, W, X, o->tol, Fx);
            else k_gen_solve<false><<<dim3(g->nw, (unsigned)nC), 256, 0, st>>>(D, W, X, o->tol, Fx);
        }
        k_gen_relax<<<(unsigned)nC, 256, 0, st>>>(D, W, X);
        g_launches += 5;
    }
    if (prim) {                                        // secondary trains: the primary's last Bmat and LU factors
        if (g->n_nodes > 0) k_gen_node_pass<true><<<dim3(g->n_nodes, (unsigned)nC), 128, 0, st>>>(D, W, prim);
        k_gen_project<false, false><<<dim3(fb, g->n_dof, (unsigned)nC), 128, 0, st>>>(D, W, W.F_drag, 0, prim, Fx);
        k_gen_train_solve<<<dim3(g->nw, (unsigned)nC), 128, 0, st>>>(D, W, prim, X);
        g_launches += 3;
    }
    disp_launch(RAFTK_FAMILY_GENERAL, blocked ? RAFTK_KERNEL_GEN_BLOCKED : RAFTK_KERNEL_GEN_UNBLOCKED, blocked ? GT : 256);
    g_disp.trains = prim != nullptr;
    k_gen_status<<<(unsigned)((nC + 127) / 128), 128, 0, st>>>((int)nC, W.flags, prim, status);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RAFTK_OK;
}

extern "C" int raftk_general_solve_dynamics_fd_dev(const raftk_general *g, const raftk_general_fd *fd, const raftk_cases *c,
                                                   const raftk_solve_opts *o, double *Xi, int32_t *status, double *F_BEM,
                                                   void *workspace, size_t workspace_bytes, void *stream)
{
    return raftk_general_solve_dynamics_qtf_dev(g, fd, nullptr, c, o, Xi, status, F_BEM, nullptr, nullptr, workspace, workspace_bytes, stream);
}

extern "C" int raftk_general_solve_dynamics_dev(const raftk_general *g, const raftk_cases *c, const raftk_solve_opts *o, double *Xi,
                                                int32_t *status, void *workspace, size_t workspace_bytes, void *stream)
{
    return raftk_general_solve_dynamics_fd_dev(g, nullptr, c, o, Xi, status, nullptr, workspace, workspace_bytes, stream);
}

extern "C" int raftk_general_solve_dynamics_qtf_host(const raftk_general *g, const raftk_general_fd *fd, const raftk_general_qtf *qtf,
                                                     const raftk_cases *c, const raftk_solve_opts *o, double *Xi, int32_t *status,
                                                     double *F_BEM, double *F_2nd, double *F_2nd_mean)
{
    disp_reset();
    if (!g || !c || !o || !Xi || !status) return set_err(RAFTK_EINVAL, "general solve: null argument");
    if (g->n_dof <= 0 || g->nw <= 0 || c->n_cases <= 0) return set_err(RAFTK_EINVAL, "general solve: empty problem");
    const size_t n = g->n_dof, nw = g->nw, Ns = g->n_nodes, nC = c->n_cases;
    if (c->primary)
        for (size_t i = 0; i < nC; i++) {
            const int p = c->primary[i];
            if (p < 0 || (size_t)p >= nC || c->primary[p] != p) return set_err(RAFTK_EINVAL, "general solve: cases.primary must map every case to a primary case");
        }
    if (fd)
        if (int rc = validate_gen_fd(g, fd, fd->fd_idx, fd->bem_headings)) return rc;
    if (qtf) {
        if (int rc = validate_gen_qtf(g, qtf, nullptr, nullptr)) return rc;
        if (int rc = validate_gen_qtf(g, qtf, qtf->qtf_w, qtf->qtf_heads)) return rc;
    }
    Staging S(qtf ? "raftk_general_solve_dynamics_qtf_host" : "raftk_general_solve_dynamics_fd_host");
    raftk_general gg = *g;
    S.in(gg.w, g->w, nw); S.in(gg.k, g->k, nw);
    S.in(gg.node_r, g->node_r, Ns * 3); S.in(gg.node_frame, g->node_frame, Ns * 9);
    S.in(gg.node_circ, g->node_circ, Ns); S.in(gg.node_Imat, g->node_Imat, Ns * 9);
    S.in(gg.node_Imat_w, g->node_Imat_w, Ns * 9 * nw * 2); S.in(gg.node_a_i, g->node_a_i, Ns);
    S.in(gg.node_cd, g->node_cd, Ns * 4); S.in(gg.Tn, g->Tn, Ns * 6 * n); S.in(gg.rr, g->rr, Ns * 3);
    S.in(gg.M, g->M, n * n); S.in(gg.B, g->B, n * n); S.in(gg.C, g->C, n * n);
    raftk_cases cc = *c;
    S.in(cc.Hs, c->Hs, nC); S.in(cc.Tp, c->Tp, nC); S.in(cc.gamma, c->gamma, nC);
    S.in(cc.beta_deg, c->beta_deg, nC); S.in(cc.spec, c->spec, nC); S.in(cc.zeta, c->zeta, nC * nw);
    S.in(cc.primary, c->primary, nC);
    raftk_general_fd ff = fd ? *fd : raftk_general_fd{};
    if (fd) {
        const size_t nf = fd->n_fd, nh = fd->n_bem_head;             // validate_gen_fd: both >= 0
        S.in(ff.fd_idx, fd->fd_idx, nf); S.in(ff.A_w, fd->A_w, nf * nf * nw); S.in(ff.B_w, fd->B_w, nf * nf * nw);
        S.in(ff.bem_headings, fd->bem_headings, nh); S.in(ff.X_BEM, fd->X_BEM, nh * 6 * nw * 2); S.in(ff.T0, fd->T0, nh ? 6 * n : 0);
    }
    raftk_general_qtf qq = qtf ? *qtf : raftk_general_qtf{};
    if (qtf) {                                                    // validate_gen_qtf: both counts >= 1
        const size_t n2 = qtf->n_qtf_w, nh = qtf->n_qtf_head;
        S.in(qq.qtf_w, qtf->qtf_w, n2); S.in(qq.qtf_heads, qtf->qtf_heads, nh); S.in(qq.qtf, qtf->qtf, n2 * n2 * nh * 12);
    }
    double *dXi, *dF_BEM, *dF2, *dF2m;
    int32_t *dStatus;
    char *ws;
    const size_t wb = raftk_general_qtf_workspace_bytes(g, fd, qtf, (int32_t)nC);
    S.out(dXi, nC * n * nw * 2, Xi); S.out(dStatus, nC * 4, status); S.out(dF_BEM, F_BEM ? nC * n * nw * 2 : 0, F_BEM);
    S.out(dF2, qtf && F_2nd ? nC * 6 * nw : 0, F_2nd); S.out(dF2m, qtf && F_2nd_mean ? nC * 6 : 0, F_2nd_mean);
    S.buf(ws, wb);
    int rc = S.commit();
    if (rc || (rc = raftk_general_solve_dynamics_qtf_dev(&gg, fd ? &ff : nullptr, qtf ? &qq : nullptr, &cc, o, dXi, dStatus, dF_BEM, dF2, dF2m,
                                                         ws, wb, nullptr))) return rc;
    return S.finish();
}

extern "C" int raftk_general_solve_dynamics_fd_host(const raftk_general *g, const raftk_general_fd *fd, const raftk_cases *c,
                                                    const raftk_solve_opts *o, double *Xi, int32_t *status, double *F_BEM)
{
    return raftk_general_solve_dynamics_qtf_host(g, fd, nullptr, c, o, Xi, status, F_BEM, nullptr, nullptr);
}

extern "C" int raftk_general_solve_dynamics_host(const raftk_general *g, const raftk_cases *c, const raftk_solve_opts *o, double *Xi,
                                                 int32_t *status)
{
    return raftk_general_solve_dynamics_fd_host(g, nullptr, c, o, Xi, status, nullptr);
}

// ---- slender-body QTF ----------------------------------------------------------------------------------
static int validate_slender(const raftk_slender *s, int32_t n_cases)
{
    if (!s || n_cases <= 0 || s->nw <= 0 || s->n_members <= 0 || s->n_nodes < 0 || s->n_seg < 0)
        return set_err(RAFTK_EINVAL, "bad slender-body QTF arguments (n_cases, nw, n_members must be > 0)");
    if (n_cases > 65535) return set_err(RAFTK_EINVAL, "slender-body QTF: more than 65535 cases per call");
    return 0;
}

static SlenderDev slender_dev(const raftk_slender *s)
{
    SlenderDev D;
    D.n_nodes = s->n_nodes; D.n_members = s->n_members; D.n_seg = s->n_seg; D.nw = s->nw;
    D.depth = s->depth; D.rho = s->rho; D.g = s->g;
    D.mem_q = s->mem_q; D.mem_p1 = s->mem_p1; D.mem_p2 = s->mem_p2; D.mem_mcf = s->mem_mcf; D.mem_wl = s->mem_wl;
    D.mem_r_int = s->mem_r_int; D.mem_a_wl = s->mem_a_wl; D.mem_rwl = s->mem_rwl; D.mem_R_wl = s->mem_R_wl;
    D.mem_node_start = s->mem_node_start; D.node_r = s->node_r; D.node_v_side = s->node_v_side;
    D.node_Ca_p1 = s->node_Ca_p1; D.node_Ca_p2 = s->node_Ca_p2; D.node_Ca_End = s->node_Ca_End; D.node_v_end = s->node_v_end; D.node_a_i = s->node_a_i;
    D.seg_mem = s->seg_mem; D.seg_z1 = s->seg_z1; D.seg_z2 = s->seg_z2; D.seg_R = s->seg_R; D.seg_rmid = s->seg_rmid;
    D.M_struc = s->M_struc; D.w = s->w; D.k = s->k;
    return D;
}

// QTFs of `units` units (L.u0 ..) into qtf [units][nw][nw][6]: tables, pairs, Hermitian fill
static int slender_launch(const SlenderDev &D, const SlenderLaunch &L, int units, const double *beta_rad, const cx *X, cx *Tn, cx *Tm, cx *Th,
                          cx *Q, cudaStream_t st)
{
    k_slender_tables<<<dim3(L.maxN + 2 * L.maxM + L.maxS, units), SL_THREADS, 0, st>>>(D, L, beta_rad, X, Tn, Tm, Th);
    const unsigned npairs = (unsigned)((size_t)D.nw * (D.nw + 1) / 2);
    k_slender_pairs<<<dim3(npairs, units), SL_THREADS, 0, st>>>(D, L, beta_rad, X, Tn, Tm, Th, Q);
    k_slender_fill<<<dim3(D.nw, units), 64, 0, st>>>(D.nw, Q);
    g_launches += 3;
    CUDA_TRY(cudaGetLastError());
    return RAFTK_OK;
}

extern "C" size_t raftk_qtf_slender_workspace_bytes(const raftk_slender *s, int32_t n_cases)
{
    if (!s || n_cases <= 0) return 0;
    return align_up((size_t)n_cases * std::max(s->n_nodes, 1) * s->nw * SL_NODE_C * sizeof(cx), 256)
           + align_up((size_t)n_cases * s->n_members * s->nw * SL_MEM_C * sizeof(cx), 256)
           + align_up((size_t)(s->n_members + s->n_seg) * s->nw * SL_HANK * sizeof(cx), 256);
}

extern "C" int raftk_qtf_slender_dev(const raftk_slender *s, int32_t n_cases, const double *beta_rad, const double *Xi_rao, double *qtf,
                                     void *workspace, size_t workspace_bytes, void *stream)
{
    int rc = validate_slender(s, n_cases);
    if (rc) return rc;
    if (!beta_rad || !Xi_rao || !qtf) return set_err(RAFTK_EINVAL, "slender-body QTF: null beta / Xi_rao / qtf");
    if (!workspace || workspace_bytes < raftk_qtf_slender_workspace_bytes(s, n_cases)) return set_err(RAFTK_ENOMEM, "slender-body QTF: workspace too small");
    SlenderLaunch L;
    L.node_off = L.mem_off = L.seg_off = nullptr;
    L.nC = n_cases; L.u0 = 0; L.d0 = 0; L.maxN = s->n_nodes; L.maxM = s->n_members; L.maxS = s->n_seg;
    char *ws = static_cast<char *>(workspace);
    cx *Tn = reinterpret_cast<cx *>(ws);
    cx *Tm = reinterpret_cast<cx *>(ws + align_up((size_t)n_cases * std::max(s->n_nodes, 1) * s->nw * SL_NODE_C * sizeof(cx), 256));
    cx *Th = reinterpret_cast<cx *>(reinterpret_cast<char *>(Tm) + align_up((size_t)n_cases * s->n_members * s->nw * SL_MEM_C * sizeof(cx), 256));
    return slender_launch(slender_dev(s), L, n_cases, beta_rad, reinterpret_cast<const cx *>(Xi_rao), Tn, Tm, Th, reinterpret_cast<cx *>(qtf),
                          (cudaStream_t)stream);
}

extern "C" int raftk_qtf_slender_host(const raftk_slender *s, int32_t n_cases, const double *beta_rad, const double *Xi_rao, double *qtf)
{
    int rc = validate_slender(s, n_cases);
    if (rc) return rc;
    if (!beta_rad || !Xi_rao || !qtf) return set_err(RAFTK_EINVAL, "slender-body QTF: null beta / Xi_rao / qtf");
    const size_t Nm = s->n_members, Ns = s->n_nodes, Ng = s->n_seg, nw = s->nw, nC = n_cases;
    Staging S("raftk_qtf_slender_host");
    raftk_slender dd = *s;
    S.in(dd.w, s->w, nw); S.in(dd.k, s->k, nw);
    S.in(dd.mem_q, s->mem_q, Nm * 3); S.in(dd.mem_p1, s->mem_p1, Nm * 3); S.in(dd.mem_p2, s->mem_p2, Nm * 3);
    S.in(dd.mem_mcf, s->mem_mcf, Nm); S.in(dd.mem_wl, s->mem_wl, Nm);
    S.in(dd.mem_r_int, s->mem_r_int, Nm * 3); S.in(dd.mem_a_wl, s->mem_a_wl, Nm);
    S.in(dd.mem_rwl, s->mem_rwl, Nm * 3); S.in(dd.mem_R_wl, s->mem_R_wl, Nm);
    S.in(dd.mem_node_start, s->mem_node_start, Nm + 1);
    S.in(dd.node_r, s->node_r, Ns * 3); S.in(dd.node_v_side, s->node_v_side, Ns);
    S.in(dd.node_Ca_p1, s->node_Ca_p1, Ns); S.in(dd.node_Ca_p2, s->node_Ca_p2, Ns);
    S.in(dd.node_Ca_End, s->node_Ca_End, Ns); S.in(dd.node_v_end, s->node_v_end, Ns);
    S.in(dd.node_a_i, s->node_a_i, Ns);
    S.in(dd.seg_mem, s->seg_mem, Ng); S.in(dd.seg_z1, s->seg_z1, Ng); S.in(dd.seg_z2, s->seg_z2, Ng);
    S.in(dd.seg_R, s->seg_R, Ng); S.in(dd.seg_rmid, s->seg_rmid, Ng * 3);
    S.in(dd.M_struc, s->M_struc, 36);
    const double *dBeta, *dXi;
    double *dQ;
    char *ws;
    const size_t wb = raftk_qtf_slender_workspace_bytes(s, n_cases);
    S.in(dBeta, beta_rad, nC); S.in(dXi, Xi_rao, nC * 6 * nw * 2); S.out(dQ, nC * nw * nw * 6 * 2, qtf);
    S.buf(ws, wb);
    if ((rc = S.commit()) || (rc = raftk_qtf_slender_dev(&dd, n_cases, dBeta, dXi, dQ, ws, wb, nullptr))) return rc;
    return S.finish();
}

// ---- potSecOrder 1: loop A -> RAOs -> slender-body QTF -> second-order force -> loop B, one call -------------------------
// Workspace: the solve's plan at its head, then loop A's outputs (the merge falls back to them), the RAOs, the second-order
// force, and one chunk of QTF tables: per unit Tn, Tm and the QTF, plus the Hankel rows of the designs a chunk spans.
struct SlenderWs { size_t solve, Xi, st, Xl, Bd, Fd, Fi, Fb, zeta, F2, rao, beta, Tn, Tm, Th, Q, total; int chunk; };

static SlenderWs slender_ws(const raftk_designs *d, const raftk_slender_batch *s, int nC, int qtf_chunk)
{
    SlenderWs L;
    const size_t units = (size_t)d->n_designs * nC, nw = d->nw, nw2 = s->cols.nw, R = units * 6 * nw * sizeof(cx);
    L.chunk = (qtf_chunk <= 0 || (size_t)qtf_chunk > units) ? (int)units : qtf_chunk;
    const size_t K = L.chunk, span = std::min((size_t)d->n_designs, (K - 1) / nC + 2);
    size_t o = 0;
    auto take = [&](size_t bytes) { const size_t at = o; o += align_up(bytes, 256); return at; };
    L.solve = take(plan_solve(d, nC, 0, WS_UNBOUNDED).bytes);
    L.Xi = take(R); L.st = take(units * 4 * sizeof(int32_t)); L.Xl = take(R);
    L.Bd = take(units * 36 * sizeof(double)); L.Fd = take(R); L.Fi = take(R); L.Fb = take(R);
    L.zeta = take((size_t)nC * nw * sizeof(double));
    L.F2 = take(units * 6 * nw * sizeof(double));
    L.rao = take(units * 6 * nw2 * sizeof(cx));
    L.beta = take((size_t)nC * sizeof(double));
    L.Tn = take(K * std::max(s->max_nodes, 1) * nw2 * SL_NODE_C * sizeof(cx));
    L.Tm = take(K * s->max_members * nw2 * SL_MEM_C * sizeof(cx));
    L.Th = take(span * (s->max_members + s->max_seg) * nw2 * SL_HANK * sizeof(cx));
    L.Q = take(K * nw2 * nw2 * 6 * sizeof(cx));
    L.total = o;
    return L;
}

static int validate_slender_flow(const raftk_designs *d, const raftk_slender_batch *s, const raftk_cases *c, int qtf_chunk)
{
    if (int rc = validate(d, c)) return rc;
    if (!s || s->n_designs != d->n_designs) return set_err(RAFTK_EINVAL, "slender flow: the slender tables must have one design per design of the batch");
    if (!s->node_offset || !s->member_offset || !s->seg_offset || s->cols.nw <= 0 || s->max_members <= 0 || s->max_nodes < 0 || s->max_seg < 0)
        return set_err(RAFTK_EINVAL, "slender flow: offsets, nw > 0 and max_members > 0 are required");
    if (c->primary) return set_err(RAFTK_EINVAL, "slender flow: potSecOrder 1 takes one wave train per case");
    if (c->F_2nd || c->Xi_init) return set_err(RAFTK_EINVAL, "slender flow: cases.F_2nd / Xi_init are the flow's own");
    if (d->n_qtf_w > 0) return set_err(RAFTK_EINVAL, "slender flow: the designs must not carry an external QTF table");
    if ((size_t)d->nw * 20 > 227 * 1024) return set_err(RAFTK_EINVAL, "nw too large for the second-order force kernel's shared-memory tables");
    const size_t units = (size_t)d->n_designs * c->n_cases;
    const size_t K = (qtf_chunk <= 0 || (size_t)qtf_chunk > units) ? units : (size_t)qtf_chunk;
    if (units > INT32_MAX || K > 65535) return set_err(RAFTK_EINVAL, "slender flow: more than 65535 units per QTF chunk (set qtf_chunk)");
    return 0;
}

extern "C" size_t raftk_solve_dynamics_slender_workspace_bytes(const raftk_designs *d, const raftk_slender_batch *s, int32_t n_cases, int32_t qtf_chunk)
{
    if (!d || !s || d->n_designs <= 0 || n_cases <= 0 || s->cols.nw <= 0) return 0;
    return slender_ws(d, s, n_cases, qtf_chunk).total;
}

extern "C" int raftk_solve_dynamics_slender_dev(const raftk_designs *d, const raftk_slender_batch *s, const raftk_cases *c,
                                                const raftk_solve_opts *o, const raftk_outputs *out, const raftk_slender_outputs *so,
                                                void *workspace, size_t workspace_bytes, void *stream)
{
    disp_reset();
    if (!out || !out->Xi || !out->status || !o) return set_err(RAFTK_EINVAL, "Xi, status and opts are required");
    if (o->n_iter < 1) return set_err(RAFTK_EINVAL, "slender flow: potSecOrder 1 needs n_iter >= 1");
    const int qtf_chunk = so ? so->qtf_chunk : 0;
    if (int rc = validate_slender_flow(d, s, c, qtf_chunk)) return rc;
    const int nD = d->n_designs, nC = c->n_cases, nw = d->nw, nw2 = s->cols.nw, units = nD * nC;
    const SlenderWs L = slender_ws(d, s, nC, qtf_chunk);
    if (!workspace || workspace_bytes < L.total) return set_err(RAFTK_ENOMEM, "slender flow: workspace smaller than raftk_solve_dynamics_slender_workspace_bytes()");
    cudaStream_t st = (cudaStream_t)stream;
    char *ws = static_cast<char *>(workspace);
    const size_t solve_bytes = L.Xi - L.solve;
    // loop A: the plain solve, outputs in the workspace
    raftk_outputs oA;
    memset(&oA, 0, sizeof(oA));
    oA.Xi = reinterpret_cast<double *>(ws + L.Xi); oA.status = reinterpret_cast<int32_t *>(ws + L.st);
    oA.Xi_last = reinterpret_cast<double *>(ws + L.Xl); oA.zeta = reinterpret_cast<double *>(ws + L.zeta);
    if (out->B_drag) oA.B_drag = reinterpret_cast<double *>(ws + L.Bd);
    if (out->F_drag) oA.F_drag = reinterpret_cast<double *>(ws + L.Fd);
    if (out->F_iner) oA.F_iner = reinterpret_cast<double *>(ws + L.Fi);
    if (out->F_BEM) oA.F_BEM = reinterpret_cast<double *>(ws + L.Fb);
    if (int rc = solve(d, c, o, &oA, ws + L.solve, solve_bytes, st)) return rc;
    // RAOs of the converged units on the second-order grid
    cx *rao = reinterpret_cast<cx *>(so && so->Xi_rao ? so->Xi_rao : reinterpret_cast<double *>(ws + L.rao));
    double *beta = reinterpret_cast<double *>(ws + L.beta);
    k_slender_rao<<<units, 64, 0, st>>>(nC, nw, nw2, d->w, s->cols.w, reinterpret_cast<const cx *>(oA.Xi), oA.zeta, oA.status, c->beta_deg, beta, rao);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    // QTF and second-order force, one chunk of units at a time
    double *F2 = out->F_2nd ? out->F_2nd : reinterpret_cast<double *>(ws + L.F2);
    const SlenderDev D = slender_dev(&s->cols);
    const size_t slab = (size_t)nw2 * nw2 * 6;
    for (int u0 = 0; u0 < units; u0 += L.chunk) {
        const int K = std::min(L.chunk, units - u0);
        SlenderLaunch SL;
        SL.node_off = s->node_offset; SL.mem_off = s->member_offset; SL.seg_off = s->seg_offset;
        SL.nC = nC; SL.u0 = u0; SL.d0 = u0 / nC; SL.maxN = s->max_nodes; SL.maxM = s->max_members; SL.maxS = s->max_seg;
        cx *Q = so && so->qtf ? reinterpret_cast<cx *>(so->qtf) + (size_t)u0 * slab : reinterpret_cast<cx *>(ws + L.Q);
        if (int rc = slender_launch(D, SL, K, beta, rao + (size_t)u0 * 6 * nw2, reinterpret_cast<cx *>(ws + L.Tn), reinterpret_cast<cx *>(ws + L.Tm),
                                    reinterpret_cast<cx *>(ws + L.Th), Q, st)) return rc;
        // the force of the chunk's units, one table per (design, case): whole designs in one launch, a design's partial case
        // range in one of its own
        for (int u = u0; u < u0 + K;) {
            const int c0 = u % nC;
            const int nd = (c0 == 0 && u + nC <= u0 + K) ? (u0 + K - u) / nC : 1;
            const int nc = std::min(nC - c0, u0 + K - u);
            raftk_cases cp;
            memset(&cp, 0, sizeof(cp));
            cp.n_cases = nc; cp.Hs = c->Hs + c0; cp.Tp = c->Tp + c0; cp.gamma = c->gamma + c0; cp.beta_deg = c->beta_deg + c0; cp.spec = c->spec + c0;
            cp.zeta = c->zeta ? c->zeta + (size_t)c0 * nw : nullptr;
            QtfParams P;
            P.nD = nd; P.shared = 2; P.n2 = nw2; P.nh = 1; P.nw = nw; P.dw = d->dw;
            P.w = d->w; P.qw = s->cols.w; P.qh = s->cols.w;                 // one heading: never read
            P.qtf = reinterpret_cast<const double2 *>(Q + (size_t)(u - u0) * slab);
            P.F2 = F2 + (size_t)u * 6 * nw;
            P.F2mean = out->F_2nd_mean ? out->F_2nd_mean + (size_t)u * 6 : nullptr;
            if (int rc = launch_qtf(P, &cp, st)) return rc;
            u += nd * nc;
        }
    }
    // loop B: continues from loop A's last iterate with the force added, n_iter - 1 more passes, into the caller's outputs
    raftk_cases cB = *c;
    cB.F_2nd = F2; cB.Xi_init = oA.Xi_last;
    raftk_solve_opts oB = *o;
    oB.n_iter = o->n_iter - 1; oB.flags |= RAFTK_SOLVE_REUSE_PLAN;        // loop A left the plan in the same workspace
    raftk_outputs ob = *out;
    ob.zeta = nullptr; ob.F_2nd = nullptr; ob.F_2nd_mean = nullptr;
    if (int rc = solve(d, &cB, &oB, &ob, ws + L.solve, solve_bytes, st)) return rc;
    SlenderMerge M;
    M.nC = nC; M.nw = nw; M.nw2 = nw2;
    M.stA = oA.status;
    M.XiA = reinterpret_cast<const cx *>(oA.Xi); M.XlA = reinterpret_cast<const cx *>(oA.Xi_last);
    M.FdA = reinterpret_cast<const cx *>(oA.F_drag); M.FiA = reinterpret_cast<const cx *>(oA.F_iner); M.FbA = reinterpret_cast<const cx *>(oA.F_BEM);
    M.BdA = oA.B_drag; M.zetaA = oA.zeta;
    M.st = out->status;
    M.Xi = reinterpret_cast<cx *>(out->Xi); M.Xl = reinterpret_cast<cx *>(out->Xi_last);
    M.Fd = reinterpret_cast<cx *>(out->F_drag); M.Fi = reinterpret_cast<cx *>(out->F_iner); M.Fb = reinterpret_cast<cx *>(out->F_BEM);
    M.qtf = so && so->qtf ? reinterpret_cast<cx *>(so->qtf) : nullptr;
    M.Bd = out->B_drag; M.zeta = out->zeta; M.F2 = out->F_2nd; M.F2m = out->F_2nd_mean;
    k_slender_merge<<<units, 256, 0, st>>>(M);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RAFTK_OK;
}

extern "C" int raftk_solve_dynamics_slender_host(const raftk_designs *d, const raftk_slender_batch *s, const raftk_cases *c,
                                                 const raftk_solve_opts *o, const raftk_outputs *out, const raftk_slender_outputs *so)
{
    disp_reset();
    if (!out || !out->Xi || !out->status || !o) return set_err(RAFTK_EINVAL, "Xi, status and opts are required");
    if (o->n_iter < 1) return set_err(RAFTK_EINVAL, "slender flow: potSecOrder 1 needs n_iter >= 1");
    const int qtf_chunk = so ? so->qtf_chunk : 0;
    if (int rc = validate_slender_flow(d, s, c, qtf_chunk)) return rc;
    Staging S("raftk_solve_dynamics_slender_host");
    raftk_designs dd = *d;
    raftk_cases cc = *c;
    stage_designs_cases(S, d, c, dd, cc);
    const size_t nD = d->n_designs, nw = d->nw, nC = c->n_cases, nR = nD * nC * 6 * nw * 2, nw2 = s->cols.nw;
    const size_t Nm = s->cols.n_members, Ns = s->cols.n_nodes, Ng = s->cols.n_seg;
    raftk_slender_batch sb = *s;
    raftk_slender &sc = sb.cols;
    const raftk_slender &h = s->cols;
    S.in(sb.node_offset, s->node_offset, nD + 1); S.in(sb.member_offset, s->member_offset, nD + 1); S.in(sb.seg_offset, s->seg_offset, nD + 1);
    S.in(sc.w, h.w, nw2); S.in(sc.k, h.k, nw2);
    S.in(sc.mem_q, h.mem_q, Nm * 3); S.in(sc.mem_p1, h.mem_p1, Nm * 3); S.in(sc.mem_p2, h.mem_p2, Nm * 3);
    S.in(sc.mem_mcf, h.mem_mcf, Nm); S.in(sc.mem_wl, h.mem_wl, Nm);
    S.in(sc.mem_r_int, h.mem_r_int, Nm * 3); S.in(sc.mem_a_wl, h.mem_a_wl, Nm);
    S.in(sc.mem_rwl, h.mem_rwl, Nm * 3); S.in(sc.mem_R_wl, h.mem_R_wl, Nm);
    S.in(sc.mem_node_start, h.mem_node_start, Nm + nD);
    S.in(sc.node_r, h.node_r, Ns * 3); S.in(sc.node_v_side, h.node_v_side, Ns);
    S.in(sc.node_Ca_p1, h.node_Ca_p1, Ns); S.in(sc.node_Ca_p2, h.node_Ca_p2, Ns);
    S.in(sc.node_Ca_End, h.node_Ca_End, Ns); S.in(sc.node_v_end, h.node_v_end, Ns);
    S.in(sc.node_a_i, h.node_a_i, Ns);
    S.in(sc.seg_mem, h.seg_mem, Ng); S.in(sc.seg_z1, h.seg_z1, Ng); S.in(sc.seg_z2, h.seg_z2, Ng);
    S.in(sc.seg_R, h.seg_R, Ng); S.in(sc.seg_rmid, h.seg_rmid, Ng * 3);
    S.in(sc.M_struc, h.M_struc, nD * 36);
    raftk_outputs od;
    memset(&od, 0, sizeof(od));
    S.out(od.Xi, nR, out->Xi);
    S.out(od.status, nD * nC * 4, out->status);
    S.out(od.B_drag, out->B_drag ? nD * nC * 36 : 0, out->B_drag);
    S.out(od.F_drag, out->F_drag ? nR : 0, out->F_drag);
    S.out(od.F_iner, out->F_iner ? nR : 0, out->F_iner);
    S.out(od.F_BEM, out->F_BEM ? nR : 0, out->F_BEM);
    S.out(od.zeta, out->zeta ? nC * nw : 0, out->zeta);
    S.out(od.F_2nd, out->F_2nd ? nR / 2 : 0, out->F_2nd);
    S.out(od.F_2nd_mean, out->F_2nd_mean ? nD * nC * 6 : 0, out->F_2nd_mean);
    S.out(od.Xi_last, out->Xi_last ? nR : 0, out->Xi_last);
    raftk_slender_outputs sd;
    memset(&sd, 0, sizeof(sd));
    sd.qtf_chunk = qtf_chunk;
    if (so) {
        S.out(sd.qtf, so->qtf ? nD * nC * nw2 * nw2 * 12 : 0, so->qtf);
        S.out(sd.Xi_rao, so->Xi_rao ? nD * nC * 6 * nw2 * 2 : 0, so->Xi_rao);
    }
    char *ws;
    const size_t wb = slender_ws(d, s, (int)nC, qtf_chunk).total;
    S.buf(ws, wb);
    int rc;
    if ((rc = S.commit()) || (rc = raftk_solve_dynamics_slender_dev(&dd, &sb, &cc, o, &od, &sd, ws, wb, nullptr))) return rc;
    return S.finish();
}

extern "C" int raftk_system_solve_host(int32_t n, int32_t nw, int32_t nrhs, double *Z, double *F, int32_t *info)
{
    disp_reset();
    if (n <= 0 || nw <= 0 || nrhs <= 0 || !Z || !F) return set_err(RAFTK_EINVAL, "bad system-solve arguments");
    Staging S("raftk_system_solve_host");
    double *dZ, *dF;
    int32_t *dInfo;
    S.in(dZ, Z, (size_t)nw * n * n * 2); S.buf(dF, (size_t)nw * n * nrhs * 2, F, F); S.out(dInfo, nw, info);
    int rc = S.commit();
    if (rc || (rc = raftk_system_solve_dev(n, nw, nrhs, dZ, dF, dInfo, nullptr))) return rc;
    return S.finish();
}

extern "C" int raftk_response_stats_dev(int32_t n_units, int32_t nw, double dw, int32_t rot_deg, const double *Xi,
                                        double *sd, double *psd, void *stream)
{
    if (n_units <= 0 || nw <= 0 || !Xi || !sd || !(dw > 0.0)) return set_err(RAFTK_EINVAL, "bad response-stats arguments");
    k_response_stats<<<(unsigned)n_units * 6u, 128, 0, (cudaStream_t)stream>>>(nw, dw, rot_deg, reinterpret_cast<const double2 *>(Xi), sd, psd);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RAFTK_OK;
}

extern "C" int raftk_response_stats_host(int32_t n_units, int32_t nw, double dw, int32_t rot_deg, const double *Xi,
                                         double *sd, double *psd)
{
    if (n_units <= 0 || nw <= 0 || !Xi || !sd || !(dw > 0.0)) return set_err(RAFTK_EINVAL, "bad response-stats arguments");
    Staging S("raftk_response_stats_host");
    const double *dXi;
    double *dSd, *dPsd;
    S.in(dXi, Xi, (size_t)n_units * 6 * nw * 2); S.out(dSd, (size_t)n_units * 6, sd); S.out(dPsd, psd ? (size_t)n_units * 6 * nw : 0, psd);
    int rc = S.commit();
    if (rc || (rc = raftk_response_stats_dev(n_units, nw, dw, rot_deg, dXi, dSd, dPsd, nullptr))) return rc;
    return S.finish();
}

extern "C" int raftk_channel_stats_dev(int32_t n_designs, int32_t n_cases, int32_t n_ch, int32_t nw, double dw, const double *coef,
                                       const double *Xi, double *sd, double *psd, double *amp, void *stream)
{
    if (n_designs <= 0 || n_cases <= 0 || n_ch <= 0 || nw <= 0 || !coef || !Xi || !sd || !(dw > 0.0))
        return set_err(RAFTK_EINVAL, "bad channel-stats arguments");
    const size_t rows = (size_t)n_designs * n_cases * n_ch;
    if (rows > 2147483647u) return set_err(RAFTK_EINVAL, "channel-stats: too many (design, case, channel) rows");
    k_channel_stats<<<(unsigned)rows, 128, 0, (cudaStream_t)stream>>>(n_cases, n_ch, nw, dw, reinterpret_cast<const double2 *>(coef),
                                                                    reinterpret_cast<const double2 *>(Xi), sd, psd, reinterpret_cast<double2 *>(amp));
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RAFTK_OK;
}

extern "C" int raftk_channel_stats_host(int32_t n_designs, int32_t n_cases, int32_t n_ch, int32_t nw, double dw, const double *coef,
                                        const double *Xi, double *sd, double *psd, double *amp)
{
    if (n_designs <= 0 || n_cases <= 0 || n_ch <= 0 || nw <= 0 || !coef || !Xi || !sd || !(dw > 0.0))
        return set_err(RAFTK_EINVAL, "bad channel-stats arguments");
    const size_t rows = (size_t)n_designs * n_cases * n_ch;
    Staging S("raftk_channel_stats_host");
    const double *dCoef, *dXi;
    double *dSd, *dPsd, *dAmp;
    S.in(dCoef, coef, (size_t)n_designs * n_ch * 6 * nw * 2); S.in(dXi, Xi, (size_t)n_designs * n_cases * 6 * nw * 2);
    S.out(dSd, rows, sd); S.out(dPsd, psd ? rows * nw : 0, psd); S.out(dAmp, amp ? rows * nw * 2 : 0, amp);
    int rc = S.commit();
    if (rc || (rc = raftk_channel_stats_dev(n_designs, n_cases, n_ch, nw, dw, dCoef, dXi, dSd, dPsd, dAmp, nullptr))) return rc;
    return S.finish();
}

// k_general_channel_stats applies w^0, w^1 or w^2; wpow: a host copy
static int validate_wpow(int32_t n_ch, const int32_t *wpow)
{
    for (int32_t t = 0; t < n_ch; t++)
        if (wpow[t] < 0 || wpow[t] > 2) return set_err(RAFTK_EINVAL, "general channel-stats: wpow must be 0, 1 or 2");
    return 0;
}

static int launch_general_channel_stats(int32_t n_units, int32_t n_dof, int32_t n_ch, int32_t nw, double dw, const double *w, const double *R,
                                        const int32_t *wpow, const double *Xi, double *sd, double *psd, double *amp, cudaStream_t stream)
{
    const size_t rows = (size_t)n_units * n_ch;
    if (rows > 2147483647u) return set_err(RAFTK_EINVAL, "general channel-stats: too many (unit, channel) rows");
    k_general_channel_stats<<<(unsigned)rows, 128, 0, stream>>>(n_dof, n_ch, nw, dw, w, R, wpow, reinterpret_cast<const double2 *>(Xi),
                                                              sd, psd, reinterpret_cast<double2 *>(amp));
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RAFTK_OK;
}

extern "C" int raftk_general_channel_stats_dev(int32_t n_units, int32_t n_dof, int32_t n_ch, int32_t nw, double dw, const double *w,
                                               const double *R, const int32_t *wpow, const double *Xi, double *sd, double *psd, double *amp,
                                               void *stream)
{
    if (n_units <= 0 || n_dof <= 0 || n_ch <= 0 || nw <= 0 || !w || !R || !wpow || !Xi || !sd || !(dw > 0.0))
        return set_err(RAFTK_EINVAL, "bad general channel-stats arguments");
    cudaStream_t st = (cudaStream_t)stream;            // the powers are read back for the check
    std::vector<int32_t> p(n_ch);
    CUDA_TRY(cudaMemcpyAsync(p.data(), wpow, p.size() * 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (int rc = validate_wpow(n_ch, p.data())) return rc;
    return launch_general_channel_stats(n_units, n_dof, n_ch, nw, dw, w, R, wpow, Xi, sd, psd, amp, st);
}

extern "C" int raftk_general_channel_stats_host(int32_t n_units, int32_t n_dof, int32_t n_ch, int32_t nw, double dw, const double *w,
                                                const double *R, const int32_t *wpow, const double *Xi, double *sd, double *psd, double *amp)
{
    if (n_units <= 0 || n_dof <= 0 || n_ch <= 0 || nw <= 0 || !w || !R || !wpow || !Xi || !sd || !(dw > 0.0))
        return set_err(RAFTK_EINVAL, "bad general channel-stats arguments");
    if (int rc = validate_wpow(n_ch, wpow)) return rc;
    const size_t rows = (size_t)n_units * n_ch;
    Staging S("raftk_general_channel_stats_host");
    const double *dW, *dR, *dXi;
    const int32_t *dWpow;
    double *dSd, *dPsd, *dAmp;
    S.in(dW, w, nw); S.in(dR, R, (size_t)n_ch * n_dof); S.in(dWpow, wpow, n_ch); S.in(dXi, Xi, (size_t)n_units * n_dof * nw * 2);
    S.out(dSd, rows, sd); S.out(dPsd, psd ? rows * nw : 0, psd); S.out(dAmp, amp ? rows * nw * 2 : 0, amp);
    int rc = S.commit();
    if (rc || (rc = launch_general_channel_stats(n_units, n_dof, n_ch, nw, dw, dW, dR, dWpow, dXi, dSd, dPsd, dAmp, nullptr))) return rc;
    return S.finish();
}

extern "C" void *raftk_host_alloc(size_t bytes)
{
    void *p = nullptr;
    if (cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return p;
}
extern "C" void raftk_host_free(void *p) { if (p) cudaFreeHost(p); }

extern "C" double raftk_fp64_peak_gflops(int iters)
{
    const int blocks = sm_count() * 8, threads = 256;
    double *out = nullptr;
    if (cudaMalloc(&out, (size_t)blocks * threads * 8) != cudaSuccess) return -1.0;
    cudaEvent_t a, b;
    cudaEventCreate(&a); cudaEventCreate(&b);
    k_fp64_peak<<<blocks, threads>>>(out, 1000);
    cudaDeviceSynchronize();
    cudaEventRecord(a);
    k_fp64_peak<<<blocks, threads>>>(out, iters);
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    g_launches += 2;
    float ms = 0;
    cudaEventElapsedTime(&ms, a, b);
    cudaEventDestroy(a); cudaEventDestroy(b); cudaFree(out);
    const double flops = 2.0 * 8.0 * (double)iters * blocks * threads;
    return flops / (ms * 1e-3) * 1e-9;
}
