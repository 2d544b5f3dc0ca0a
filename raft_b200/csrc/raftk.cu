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
#include <cmath>
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
    if (family == RAFTK_FAMILY_FARM) g_disp.farm_classes = 1 << kernel;
}
extern "C" int raftk_last_dispatch(raftk_dispatch *out)
{
    if (!out) return set_err(RAFTK_EINVAL, "raftk_last_dispatch: null output");
    *out = g_disp;
    return RAFTK_OK;
}

#include "raftk_common.cuh"
#include "raftk_rigid.cuh"
#include "raftk_tables.cuh"
#include "raftk_fused.cuh"
#include "raftk_fused2.cuh"
#include "raftk_qtf.cuh"
#include "raftk_slender.cuh"
#include "raftk_lu.cuh"
#include "raftk_general.cuh"
#include "raftk_misc.cuh"
#include "raftk_rotor.cuh"
#include "raftk_fatigue.cuh"
#include "raftk_stress.cuh"
#include "raftk_eigen.cuh"
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
    D.max_rotors = d->max_rotors; D.rot_count = d->rot_count; D.rot_r3 = d->rot_r3; D.rot_G = d->rot_G;
    return D;
}

static CasesDev to_dev(const raftk_cases *c)
{
    CasesDev C;
    C.nC = c->n_cases; C.Hs = c->Hs; C.Tp = c->Tp; C.gamma = c->gamma; C.beta_deg = c->beta_deg;
    C.zeta_in = c->zeta; C.spec = c->spec; C.primary = c->primary; C.F_2nd = c->F_2nd;
    C.op = c->op; C.n_op = c->n_op; C.op_shared = c->op_shared; C.op_A_w = c->op_A_w; C.op_B_w = c->op_B_w;
    return C;
}

// cases.op (operating points): the counts and tables, then -- when host copies are given -- every case's index and the
// wave trains' agreement with their primaries.  Nothing is checked without op.
static int validate_op(const raftk_cases *c, const int32_t *op_h, const int32_t *prim_h)
{
    if (!c || !c->op) return 0;
    if (c->n_op < 1) return set_err(RAFTK_EINVAL, "cases.op: n_op must be >= 1");
    if (c->op_shared != 0 && c->op_shared != 1) return set_err(RAFTK_EINVAL, "cases.op_shared must be 0 or 1");
    if (!c->op_A_w || !c->op_B_w) return set_err(RAFTK_EINVAL, "cases.op needs op_A_w and op_B_w");
    if (!op_h) return 0;
    char m[160];
    for (int i = 0; i < c->n_cases; i++)
        if (op_h[i] < 0 || op_h[i] >= c->n_op) {
            snprintf(m, sizeof(m), "cases.op[%d] = %d is outside [0, n_op = %d)", i, op_h[i], c->n_op);
            return set_err(RAFTK_EINVAL, "%s", m);
        }
    if (prim_h)
        for (int i = 0; i < c->n_cases; i++) {
            const int p = prim_h[i];
            if (p >= 0 && p < c->n_cases && op_h[p] != op_h[i]) {
                snprintf(m, sizeof(m), "cases.op: secondary train %d names operating point %d, its primary %d names %d", i, op_h[i], p, op_h[p]);
                return set_err(RAFTK_EINVAL, "%s", m);
            }
        }
    return 0;
}

// validate_op for a *_dev entry: op and primary are device memory, which these entries do not read back (they run without a
// host synchronisation); their values are the caller's to check (solver.CaseTable does, and the host entries do)
static int validate_op_dev(const raftk_cases *c) { return validate_op(c, nullptr, nullptr); }

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

// The solve options every fixed-point loop takes.  tol is 0 or at least RAFTK_TOL_MIN (include/raftk.h): below that the
// kernels' forms of the convergence test |d| / (|x| + tol) < tol (squared in the fused solvers, sqrt(d.d) in v1 and the
// generalised-DOF solve) underflow and no longer decide as the reference does.
static int validate_opts(const raftk_solve_opts *o)
{
    if (!o) return set_err(RAFTK_EINVAL, "null solve options");
    if (!(o->tol == 0.0 || o->tol >= RAFTK_TOL_MIN)) {
        char got[32];
        snprintf(got, sizeof got, "%g", o->tol);
        return set_err(RAFTK_EINVAL, "solve options: tol must be 0 or at least 1e-70 (RAFTK_TOL_MIN), got %s", got);
    }
    return 0;
}

static int validate(const raftk_designs *d, const raftk_cases *c)
{
    if (!d || !c) return set_err(RAFTK_EINVAL, "null designs/cases");
    if (d->n_designs <= 0 || d->nw <= 0 || c->n_cases <= 0) return set_err(RAFTK_EINVAL, "empty batch (n_designs, nw, n_cases must be > 0)");
    if (d->max_nodes <= 0 || d->max_members <= 0) return set_err(RAFTK_EINVAL, "max_nodes/max_members must be > 0");
    if (d->max_members > 512 || d->max_nodes > 4096) return set_err(RAFTK_EINVAL, "design too large for the shared-memory tables");
    if ((d->node_in_p1_w == nullptr) != (d->node_in_p2_w == nullptr)) return set_err(RAFTK_EINVAL, "node_in_p1_w / node_in_p2_w must both be given or both NULL");
    if (d->max_rotors < 0) return set_err(RAFTK_EINVAL, "designs.max_rotors must be >= 0");
    if (d->max_rotors > 0 && (!d->rot_count || !d->rot_r3 || !d->rot_G))
        return set_err(RAFTK_EINVAL, "designs.max_rotors > 0 needs rot_count, rot_r3 and rot_G");
    return 0;
}

// The submerged-rotor table of a host call: every design's count in [0, max_rotors], every hub below the waterline (the
// reference adds the term only there, raft_fowt.py:1861) and every G finite; with a cases.primary map, every train group
// contiguous with its primary first, which is how the kernels find a group's last train (rotor_excitation).
static int validate_rotors_host(const raftk_designs *d, const raftk_cases *c)
{
    char m[160];
    if (d->max_rotors > 0 && c->primary)
        for (int i = 0; i < c->n_cases; i++) {
            const int p = c->primary[i];
            if (!(p == i || (i > 0 && p < i && c->primary[i - 1] == p))) {
                snprintf(m, sizeof(m), "cases.primary: with submerged rotors every train group must be contiguous with its primary "
                         "first (case %d names primary %d)", i, p);
                return set_err(RAFTK_EINVAL, "%s", m);
            }
        }
    for (int i = 0; i < d->n_designs && d->max_rotors > 0; i++) {
        const int n = d->rot_count[i];
        if (n < 0 || n > d->max_rotors) {
            snprintf(m, sizeof(m), "designs.rot_count[%d] = %d is outside [0, max_rotors = %d]", i, n, d->max_rotors);
            return set_err(RAFTK_EINVAL, "%s", m);
        }
        for (int r = 0; r < n; r++) {
            const size_t e = (size_t)i * d->max_rotors + r;
            if (!(d->rot_r3[3 * e + 2] < 0.0)) {
                snprintf(m, sizeof(m), "designs.rot_r3: rotor %d of design %d is not submerged (z = %g)", r, i, d->rot_r3[3 * e + 2]);
                return set_err(RAFTK_EINVAL, "%s", m);
            }
            for (int t = 0; t < 18; t++)
                if (!std::isfinite(d->rot_G[18 * e + t])) {
                    snprintf(m, sizeof(m), "designs.rot_G: rotor %d of design %d has a non-finite entry", r, i);
                    return set_err(RAFTK_EINVAL, "%s", m);
                }
        }
    }
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
// Designs whose node walk the fused kernels cannot carry exactly (d->walk_exact == 0, DESIGN.md section 4) go to v1.
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

    if (!v1_only && !getenv("RAFTK_FORCE_V1") && d->walk_exact && d->max_nodes > 0 && d->max_members > 0) {
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

template <int T, bool ROT>
static int fused_launch(const DesignsDev &D, const CasesDev &C, const FusedParams &P, const SolvePlan &pl, int units, cudaStream_t st)
{
    static SmemOptIn opt;
    CUDA_TRY(opt.ensure(k_rao_fused<T, ROT>, pl.smem));
    cudaLaunchConfig_t cfg;
    cudaLaunchAttribute at;
    cluster_config(cfg, at, (size_t)units * pl.CS, T, pl.smem, pl.CS, st);
    {
        ProfScope ps(st, 2);
        CUDA_TRY(cudaLaunchKernelEx(&cfg, k_rao_fused<T, ROT>, D, C, P));
    }
    g_launches++;
    disp_launch(RAFTK_FAMILY_SOLVE, T == 128 ? RAFTK_KERNEL_FUSED128 : RAFTK_KERNEL_FUSED256, T, pl.CS, pl.nwl);
    g_disp.f0_global = P.F0g != nullptr;
    g_disp.trains = P.phase >= 0;
    CUDA_TRY(cudaGetLastError());
    return RAFTK_OK;
}

// k_rao_fused at the plan's CTA size, in the instantiation with the submerged-rotor term when the designs carry rotors
static int fused_launch(const DesignsDev &D, const CasesDev &C, const FusedParams &P, const SolvePlan &pl, int units, cudaStream_t st)
{
    const bool rot = D.max_rotors > 0;
    if (pl.T == 128) return rot ? fused_launch<128, true>(D, C, P, pl, units, st) : fused_launch<128, false>(D, C, P, pl, units, st);
    return rot ? fused_launch<256, true>(D, C, P, pl, units, st) : fused_launch<256, false>(D, C, P, pl, units, st);
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
            if (int rc = fused_launch(D, C, P, pl, units, st)) return rc;
        }
        return RAFTK_OK;
    }
    return fused_launch(D, C, P, pl, units, st);
}

// Grid or cluster exchange for k_rao_fused2 (RAFTK_FUSED2_XCHG=cluster|grid overrides, read per call, for A/B runs and
// tests).  The grid variant runs when a unit spans several CTAs, every CTA of the launch can be resident at once, and the
// hardware cannot place every unit's cluster at once (cudaOccupancyMaxActiveClusters < units): then the clusters that do not
// fit would start only when the first units finish.  The occupancy queries are cached per device and launch shape.
static SmemOptIn g_f2_opt_var[8];

// k_rao_fused2's instantiation number var: bit 0 GRID, bit 1 OP, bit 2 ROT
using F2Kernel = void (*)(DesignsDev, CasesDev, FusedParams);
static F2Kernel f2_kernel(int var)
{
    static const F2Kernel k[8] = {k_rao_fused2<false>, k_rao_fused2<true>, k_rao_fused2<false, true>, k_rao_fused2<true, true>,
                                  k_rao_fused2<false, false, true>, k_rao_fused2<true, false, true>, k_rao_fused2<false, true, true>,
                                  k_rao_fused2<true, true, true>};
    return k[var];
}
static cudaError_t f2_opt_in(int var, size_t smem) { return g_f2_opt_var[var].ensure(f2_kernel(var), smem); }
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
    CUDA_TRY(f2_opt_in(0, pl.smem));
    CUDA_TRY(f2_opt_in(1, pl.smem));
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
    // the instantiations with operating points and with submerged rotors (same registers and occupancy)
    const int var = (grid ? 1 : 0) | (c->op ? 2 : 0) | (d->max_rotors > 0 ? 4 : 0);
    CUDA_TRY(f2_opt_in(var, pl.smem));
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
            if (grid) CUDA_TRY(cudaMemsetAsync(P.xcnt, 0, (size_t)units * sizeof(unsigned), st));      // counters count up from 0 per launch
            CUDA_TRY(cudaLaunchKernelEx(&cfg, f2_kernel(var), D, C, P));
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
    const char *why = d->walk_exact ? "the design's frequency slice does not fit on chip"
                                     : "its node walk is inexact on this design and grid (designs.walk_exact = 0)";
    if (peers && peers->n_ranks > 1) return set_err(RAFTK_EINVAL, "the fused exchange needs the fused solver; %s", why);
    if (c->primary) return set_err(RAFTK_EINVAL, "wave-train cases (cases.primary) need the fused solver; %s", why);
    if (c->Xi_init || out->Xi_last) return set_err(RAFTK_EINVAL, "cases.Xi_init / outputs.Xi_last need the fused solver; %s", why);
    const int rc = run_tables(d, c, o, out, nullptr, 0, pl, workspace, wbytes, st);
    g_disp.inexact_walk = !d->walk_exact;
    return rc;
}

// the rigid solve over the caller's workspace: planned against it, then launched
static int solve(const raftk_designs *d, const raftk_cases *c, const raftk_solve_opts *o, const raftk_outputs *out,
                 void *workspace, size_t wbytes, cudaStream_t st, const raftk_peers *peers = nullptr)
{
    if (int rc = validate(d, c)) return rc;
    if (int rc = validate_opts(o)) return rc;
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
    if (int rc = validate_op_dev(c)) return rc;
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
    if ((rc = validate_op_dev(c))) return rc;
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
// goes to the global-memory kernels (lu_blocked with a staged panel).  Without a device the rule uses an H100's limits and the static sizes of the
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

// ---- farm system response: single farms, uniform and ragged batches --------------------------------------------------------
// Every farm goes to one of four kernel classes by its N alone, and a call launches each class it needs once, over that class's
// farms, in this order.  A uniform batch (a single farm is a batch of one) is one run of F farms of one N, whose kernels derive
// every offset from the farm index.  A ragged batch (raftk_farm_ragged) groups its farms by class (farms of a class in batch
// order); each farm's first design, N, offsets and panel width are in a descriptor copied to the head of the workspace, where
// the class's launch finds its run.
enum { FC_ROWS, FC_WARP, FC_BLOCK, FC_GLOBAL, FC_N };
static const int fc_kernel[FC_N] = {RAFTK_KERNEL_FARM_ROWS12, RAFTK_KERNEL_FARM_WARP, RAFTK_KERNEL_FARM_BLOCK, RAFTK_KERNEL_FARM_GLOBAL};

// The class of a farm of N FOWTs.  6N <= 24: one warp per (frequency, case), except 6N = 12 (the shipped two-FOWT farm), whose
// rows live in registers, one lane per row, two systems per warp (k_farm_rows; RAFTK_FARM_SMEM=1 keeps the shared-memory warp
// kernel, for A/B).  At 6N = 18 / 24 the register rows would need 188 / 238 registers, so those stay on the warp kernel.
// Above 24, one CTA per system while its [6N][6N+1] fits in shared memory, else k_farm_response_global.
static int farm_class(int N)
{
    const int n = 6 * N;
    if (n > 24 && !smem_fits((size_t)n * (n + 1) * sizeof(double2), static_smem(k_farm_response<false>, SMEM_STATIC_FARM_BLOCK)))
        return FC_GLOBAL;
    if (n == 12 && !getenv("RAFTK_FARM_SMEM")) return FC_ROWS;
    return n <= 24 ? FC_WARP : FC_BLOCK;
}

// What a call launches and the workspace it needs, from a raftk_farm_batch or a raftk_farm_ragged (farm_plan)
struct FarmPlan {
    bool rag = false;                   // a ragged batch: the descriptor table heads the workspace
    const char *who = "farm response";  // the refusals' prefix
    int N = 0, F = 0;                   // uniform: farms of N FOWTs; F farms in all
    std::vector<FarmDesc> fd;           // ragged: grouped by class
    int first[FC_N + 1] = {};           // class k is farms [first[k], first[k + 1]) of the launch order
    int nmax[FC_N] = {};                // largest N of each class
    size_t table = 0;                   // bytes of the descriptor table at the head of the workspace (256-aligned)
    size_t slab = 0;                    // double2 elements of one k_farm_response_global slab (the class's largest N)
    size_t pan_smem = 0;                // k_farm_response_global's panel: the largest n * pw of its farms
    int pw = 0;                         // uniform: that panel's width (ragged farms carry their own)
    int per_sm = 0;                     // its CTAs per SM: the fewest any of its farms' glu_plan allows
    long long gsys = 0;                 // (farm, case, bin) systems of that class
    size_t bytes = 0;                   // the full workspace: table + min(gsys, resident CTAs) slabs
    const double *M_arr = nullptr, *B_arr = nullptr, *C_arr = nullptr;
    size_t n_arr = 0, arr_stride = 0;   // doubles of each array-matrix set; uniform: between two farms' sets (0: shared)
    double *Xi_sys = nullptr;
    int32_t *info = nullptr;
};

// the global class's slabs after the table: one [6N][6N+1] of its largest N per resident CTA, no more than its systems
static void farm_plan_slabs(const raftk_designs *d, const raftk_cases *c, FarmPlan &R)
{
    const int nk = R.first[FC_GLOBAL + 1] - R.first[FC_GLOBAL], N = R.nmax[FC_GLOBAL];
    R.bytes = R.table;
    if (!nk) return;
    R.slab = (size_t)6 * N * (6 * N + 1);
    R.gsys = (long long)nk * c->n_cases * d->nw;
    R.bytes += (size_t)std::max<long long>(0, std::min<long long>(R.gsys, (long long)R.per_sm * sm_count())) * R.slab * sizeof(double2);
}

// A uniform batch: one class run of F farms of N, no descriptor table, its slab and panel from glu_plan(6N).  It refuses
// nothing (its grid limits are farm_run's), so the workspace queries never touch the last-error string.
static void farm_plan(const raftk_designs *d, const raftk_cases *c, const raftk_farm_batch *f, FarmPlan &R)
{
    const int k = farm_class(f->n_fowt);
    R.N = f->n_fowt; R.F = std::max(f->n_farms, 0);
    for (int j = k + 1; j <= FC_N; j++) R.first[j] = R.F;
    R.nmax[k] = R.N;
    if (k == FC_GLOBAL) {
        const GluPlan g = glu_plan(6 * R.N);
        R.pw = g.pw; R.pan_smem = g.smem; R.per_sm = std::max(g.per_sm, 1);
    }
    farm_plan_slabs(d, c, R);
    R.n_arr = (f->arr_shared ? 1 : (size_t)R.F) * 36 * R.N * R.N;
    R.arr_stride = f->arr_shared ? 0 : (size_t)36 * R.N * R.N;
    R.M_arr = f->M_arr; R.B_arr = f->B_arr; R.C_arr = f->C_arr;
    R.Xi_sys = f->Xi_sys; R.info = f->info;
}

// A ragged batch: its CSR arrays checked, each farm's descriptor in its class's run
static int farm_plan(const raftk_designs *d, const raftk_cases *c, const raftk_farm_ragged *f, FarmPlan &R)
{
    if (!d || !c || !f) return set_err(RAFTK_EINVAL, "ragged farm batch: null argument");
    auto bad_farm = [](const char *fmt, int k) { char b[16]; snprintf(b, sizeof(b), "%d", k); return set_err(RAFTK_EINVAL, fmt, b); };
    const int F = f->n_farms;
    if (F < 1) return set_err(RAFTK_EINVAL, "ragged farm batch: n_farms must be >= 1");
    if (!f->farm_fowt0) return set_err(RAFTK_EINVAL, "ragged farm batch: farm_fowt0 is required");
    if (f->farm_fowt0[0] != 0) return set_err(RAFTK_EINVAL, "ragged farm batch: farm_fowt0[0] must be 0");
    for (int k = 0; k < F; k++)
        if (f->farm_fowt0[k + 1] <= f->farm_fowt0[k])
            return bad_farm("ragged farm batch: farm_fowt0 must be strictly increasing (farm %s is empty)", k);
    if (f->farm_fowt0[F] != d->n_designs) return set_err(RAFTK_EINVAL, "ragged farm batch: farm_fowt0[n_farms] must equal designs.n_designs");
    if (f->arr_shared != 0 && f->arr_shared != 1) return set_err(RAFTK_EINVAL, "ragged farm batch: arr_shared must be 0 or 1");
    const bool mats = f->M_arr || f->B_arr || f->C_arr;
    for (int k = 0; k < F; k++) {
        const long long N = f->farm_fowt0[k + 1] - f->farm_fowt0[k];
        if (f->arr_shared && N != f->farm_fowt0[1])
            return bad_farm("ragged farm batch: arr_shared = 1 needs every farm to have the same N (farm %s differs)", k);
        if (!f->arr_shared && mats) {
            if (!f->arr_offset) return set_err(RAFTK_EINVAL, "ragged farm batch: arr_offset is required with per-farm array matrices");
            if (f->arr_offset[0] != 0 || f->arr_offset[k + 1] - f->arr_offset[k] != 36 * N * N)
                return bad_farm("ragged farm batch: arr_offset must start at 0 and step by 36 N^2 (farm %s does not)", k);
        }
    }
    if (c->n_cases < 1 || d->nw < 1) return set_err(RAFTK_EINVAL, "ragged farm batch: no cases or no frequency bins");
    R.rag = true; R.who = "ragged farm batch"; R.F = F;
    std::vector<int> cls(F);
    int count[FC_N] = {};
    for (int k = 0; k < F; k++) {
        const int N = f->farm_fowt0[k + 1] - f->farm_fowt0[k];
        cls[k] = farm_class(N);
        count[cls[k]]++;
        R.nmax[cls[k]] = std::max(R.nmax[cls[k]], N);
    }
    for (int k = 0; k < FC_N; k++) R.first[k + 1] = R.first[k] + count[k];
    if (R.first[FC_GLOBAL] > 0) {      // the grids of the on-chip classes are (frequency groups, case, farm of the class)
        if (c->n_cases > 65535) return set_err(RAFTK_EINVAL, "ragged farm batch: more than 65535 cases per call with farms solved on chip (6N <= 120)");
        for (int k = 0; k < FC_GLOBAL; k++)
            if (count[k] > 65535) return set_err(RAFTK_EINVAL, "ragged farm batch: more than 65535 farms of one on-chip kernel class per call");
    }
    R.fd.resize(F);
    int next[FC_N];
    for (int k = 0; k < FC_N; k++) next[k] = R.first[k];
    R.per_sm = 2;
    for (int k = 0; k < F; k++) {
        FarmDesc &e = R.fd[next[cls[k]]++];
        e.d0 = f->farm_fowt0[k]; e.N = f->farm_fowt0[k + 1] - f->farm_fowt0[k]; e.pw = 0; e._pad = 0;
        e.xo = (size_t)6 * c->n_cases * d->nw * e.d0;
        e.io = (size_t)k * c->n_cases * d->nw;
        e.ao = (!f->arr_shared && mats) ? (size_t)f->arr_offset[k] : 0;
        if (cls[k] == FC_GLOBAL) {
            const GluPlan g = glu_plan(6 * e.N);
            if (!g.pw) return bad_farm("ragged farm batch: farm %s: 6N too large for one panel column in shared memory", k);
            e.pw = g.pw;
            R.pan_smem = std::max(R.pan_smem, g.smem);
            R.per_sm = std::min(R.per_sm, g.per_sm);
        }
    }
    // the global class walks its systems in descriptor order, dealt round-robin over the resident CTAs: largest farms first,
    // so that no CTA is left with two of the largest systems while others finish small ones (a farm's bits do not depend on it)
    std::stable_sort(R.fd.begin() + R.first[FC_GLOBAL], R.fd.begin() + R.first[FC_GLOBAL + 1],
                     [](const FarmDesc &a, const FarmDesc &b) { return a.N > b.N; });
    R.table = align_up((size_t)F * sizeof(FarmDesc), 256);
    farm_plan_slabs(d, c, R);
    const size_t N0 = (size_t)f->farm_fowt0[1];
    R.n_arr = f->arr_shared ? 36 * N0 * N0 : (f->arr_offset ? (size_t)f->arr_offset[F] : 0);
    R.M_arr = f->M_arr; R.B_arr = f->B_arr; R.C_arr = f->C_arr;
    R.Xi_sys = f->Xi_sys; R.info = f->info;
    return RAFTK_OK;
}

// one farm is a batch of one: its matrices are the shared set
static raftk_farm_batch farm_as_batch(const raftk_farm *f)
{
    raftk_farm_batch b;
    memset(&b, 0, sizeof(b));
    b.n_farms = 1; b.n_fowt = f->n_fowt; b.arr_shared = 1;
    b.M_arr = f->M_arr; b.B_arr = f->B_arr; b.C_arr = f->C_arr;
    b.Xi_sys = f->Xi_sys; b.info = f->info;
    return b;
}

extern "C" size_t raftk_farm_workspace_bytes(const raftk_designs *d, const raftk_cases *c, const raftk_farm *f)
{
    if (!f) return 0;
    const raftk_farm_batch b = farm_as_batch(f);
    return raftk_farm_batch_workspace_bytes(d, c, &b);
}

extern "C" size_t raftk_farm_batch_workspace_bytes(const raftk_designs *d, const raftk_cases *c, const raftk_farm_batch *f)
{
    if (!d || !c || !f) return 0;
    FarmPlan R;
    farm_plan(d, c, f, R);
    return R.bytes;
}

extern "C" size_t raftk_farm_ragged_workspace_bytes(const raftk_designs *d, const raftk_cases *c, const raftk_farm_ragged *f)
{
    FarmPlan R;
    return farm_plan(d, c, f, R) ? 0 : R.bytes;
}

// the launch of class k's run of farms: grid, shared memory and its opt-in (per instantiation), and the dispatch record
template <bool OP, bool RAG>
static int farm_launch_class(int k, const FarmPlan &R, const FarmArg<RAG> &P, const DesignsDev &D, const CasesDev &C, void *ws,
                             size_t ws_bytes, cudaStream_t st)
{
    static SmemOptIn opt_w(48 * 1024), opt_b(48 * 1024), opt_g(0);
    const int n = 6 * R.nmax[k], nw = P.nw;              // shared memory for the class's largest N
    const size_t sys_bytes = (size_t)n * (n + 1) * sizeof(double2);
    const unsigned gy = P.nC, gz = P.nF;
    int threads = GLU_T;
    {
        ProfScope ps(st, 1);
        if (k == FC_ROWS) {
            threads = 128;
            k_farm_rows<12, OP, RAG><<<dim3((nw + 7) / 8, gy, gz), threads, 0, st>>>(D, C, P);
        } else if (k == FC_WARP) {                        // one warp per (frequency, case), wpc systems per CTA
            const int wpc = (int)std::max<size_t>(1, std::min<size_t>(FARM_WPC, (100 * 1024) / sys_bytes));
            threads = 32 * wpc;
            CUDA_TRY(opt_w.ensure(k_farm_response<true, OP, RAG>, wpc * sys_bytes));
            k_farm_response<true, OP, RAG><<<dim3((nw + wpc - 1) / wpc, gy, gz), threads, wpc * sys_bytes, st>>>(D, C, P);
        } else if (k == FC_BLOCK) {
            threads = 256;
            CUDA_TRY(opt_b.ensure(k_farm_response<false, OP, RAG>, sys_bytes));
            k_farm_response<false, OP, RAG><<<dim3(nw, gy, gz), threads, sys_bytes, st>>>(D, C, P);
        } else {                                          // persistent CTAs, each on its own slab of the workspace after the table
            CUDA_TRY(opt_g.ensure(k_farm_response_global<OP, RAG>, R.pan_smem));
            double2 *slabs = reinterpret_cast<double2 *>(static_cast<char *>(ws) + R.table);
            const long long fit = (long long)((ws_bytes - R.table) / (R.slab * sizeof(double2)));
            const int grid = (int)std::min<long long>(std::min<long long>(R.gsys, fit), (long long)R.per_sm * sm_count());
            k_farm_response_global<OP, RAG><<<grid, GLU_T, R.pan_smem, st>>>(D, C, P, slabs, R.pw);
        }
        disp_launch(RAFTK_FAMILY_FARM, fc_kernel[k], threads);
    }
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RAFTK_OK;
}

// The farm response of a plan: each non-empty class run launched in class order.  The dispatch record names the last launch,
// and farm_classes every class that ran.
static int farm_run(const raftk_designs *d, const raftk_cases *c, const raftk_outputs *solved, const FarmPlan &R, void *ws,
                    size_t ws_bytes, cudaStream_t st)
{
    if (!solved->B_drag || !solved->F_drag || !solved->F_iner)
        return set_err(RAFTK_EINVAL, "%s needs B_drag, F_drag, F_iner of the per-FOWT solve", R.who);
    if (d->n_bem_head > 0 && !solved->F_BEM) return set_err(RAFTK_EINVAL, "%s: the designs carry BEM excitation, F_BEM is required", R.who);
    if (R.rag) {
        if (!ws || ws_bytes < R.table + R.slab * sizeof(double2))
            return set_err(RAFTK_EINVAL, "ragged farm batch: the workspace must hold the farm descriptor table%s (raftk_farm_ragged_workspace_bytes)",
                           R.slab ? " and one [6N][6N+1] slab of the largest farm solved in global memory" : "");
    } else if (!R.slab) {               // the grid is (frequency groups, case, farm): its y and z extents end at 65535
        if (c->n_cases > 65535) return set_err(RAFTK_EINVAL, "farm response: more than 65535 cases per call");
        if (R.F > 65535) return set_err(RAFTK_EINVAL, "farm response: more than 65535 farms per call with the system in shared memory (6N <= 120)");
    } else {
        if (!R.pw) return set_err(RAFTK_EINVAL, "farm response: 6N too large for one panel column in shared memory");
        if (!ws || ws_bytes < R.slab * sizeof(double2))
            return set_err(RAFTK_EINVAL, "farm response: a farm this size needs a workspace of at least one [6N][6N+1] slab "
                                         "(raftk_farm_workspace_bytes, raftk_farm_response_ws_dev)");
    }
    FarmRagParams P{};
    P.N = R.N; P.nC = c->n_cases; P.nw = d->nw;
    P.arr_stride = R.arr_stride;
    P.B_drag = solved->B_drag;
    P.F_drag = reinterpret_cast<const double2 *>(solved->F_drag);
    P.F_iner = reinterpret_cast<const double2 *>(solved->F_iner);
    P.F_BEM = d->n_bem_head > 0 ? reinterpret_cast<const double2 *>(solved->F_BEM) : nullptr;
    P.M_arr = R.M_arr; P.B_arr = R.B_arr; P.C_arr = R.C_arr;
    P.Xi = reinterpret_cast<double2 *>(R.Xi_sys); P.info = R.info;
    P.slab = R.slab;
    FarmDesc *dfd = static_cast<FarmDesc *>(ws);
    if (R.rag) CUDA_TRY(cudaMemcpyAsync(dfd, R.fd.data(), R.fd.size() * sizeof(FarmDesc), cudaMemcpyHostToDevice, st));
    DesignsDev D = to_dev(d, d->max_nodes, d->max_members);
    CasesDev C = to_dev(c);
    int mask = 0;
    for (int k = 0; k < FC_N; k++) {
        if (R.first[k + 1] == R.first[k]) continue;
        P.nF = R.first[k + 1] - R.first[k];
        if (R.rag) P.fd = dfd + R.first[k];
        const FarmParams &U = P;
        const int rc = R.rag ? (c->op ? farm_launch_class<true, true>(k, R, P, D, C, ws, ws_bytes, st)
                                      : farm_launch_class<false, true>(k, R, P, D, C, ws, ws_bytes, st))
                             : (c->op ? farm_launch_class<true, false>(k, R, U, D, C, ws, ws_bytes, st)
                                      : farm_launch_class<false, false>(k, R, U, D, C, ws, ws_bytes, st));
        if (rc) return rc;
        mask |= 1 << fc_kernel[k];
    }
    g_disp.farm_classes = mask;
    return RAFTK_OK;
}

// the shape of a farm batch against its designs (everything the host entry can refuse before it stages anything)
static int farm_batch_shape(const raftk_designs *d, const raftk_farm_batch *f)
{
    if (f->n_farms < 1 || f->n_fowt < 1) return set_err(RAFTK_EINVAL, "farm batch: n_farms and n_fowt must be >= 1");
    if ((long long)f->n_farms * f->n_fowt != d->n_designs)
        return set_err(RAFTK_EINVAL, "farm batch: n_farms * n_fowt must equal designs.n_designs");
    if (f->arr_shared != 0 && f->arr_shared != 1) return set_err(RAFTK_EINVAL, "farm batch: arr_shared must be 0 or 1");
    if (!f->Xi_sys) return set_err(RAFTK_EINVAL, "farm batch: Xi_sys is required");
    return RAFTK_OK;
}

static int farm_launch(const raftk_designs *d, const raftk_cases *c, const raftk_outputs *solved, const raftk_farm_batch *f, void *ws,
                       size_t ws_bytes, cudaStream_t st)
{
    if (!d || !c || !solved || !f) return set_err(RAFTK_EINVAL, "farm response: null argument");
    if (int rc = farm_batch_shape(d, f)) return rc;
    FarmPlan R;
    farm_plan(d, c, f, R);
    return farm_run(d, c, solved, R, ws, ws_bytes, st);
}

static int farm_ragged_launch(const raftk_designs *d, const raftk_cases *c, const raftk_outputs *solved, const raftk_farm_ragged *f,
                              void *ws, size_t ws_bytes, cudaStream_t st)
{
    if (!solved) return set_err(RAFTK_EINVAL, "ragged farm batch: null argument");
    FarmPlan R;
    if (int rc = farm_plan(d, c, f, R)) return rc;
    if (!f->Xi_sys) return set_err(RAFTK_EINVAL, "ragged farm batch: Xi_sys is required");
    return farm_run(d, c, solved, R, ws, ws_bytes, st);
}

// the single-farm entries: farm.n_fowt names the whole batch of designs
static int farm_launch_one(const raftk_designs *d, const raftk_cases *c, const raftk_outputs *solved, const raftk_farm *f, void *ws,
                           size_t ws_bytes, cudaStream_t st)
{
    if (!d || !c || !solved || !f) return set_err(RAFTK_EINVAL, "farm response: null argument");
    if (f->n_fowt != d->n_designs || f->n_fowt < 1) return set_err(RAFTK_EINVAL, "farm response: farm.n_fowt must equal designs.n_designs");
    if (!f->Xi_sys) return set_err(RAFTK_EINVAL, "farm response needs farm.Xi_sys");
    const raftk_farm_batch b = farm_as_batch(f);
    return farm_launch(d, c, solved, &b, ws, ws_bytes, st);
}

extern "C" int raftk_farm_response_dev(const raftk_designs *d, const raftk_cases *c, const raftk_outputs *solved, const raftk_farm *f,
                                       void *stream)
{
    disp_reset();
    if (int rc = validate_op_dev(c)) return rc;
    return farm_launch_one(d, c, solved, f, nullptr, 0, (cudaStream_t)stream);
}

extern "C" int raftk_farm_response_ws_dev(const raftk_designs *d, const raftk_cases *c, const raftk_outputs *solved, const raftk_farm *f,
                                          void *workspace, size_t workspace_bytes, void *stream)
{
    disp_reset();
    if (int rc = validate_op_dev(c)) return rc;
    return farm_launch_one(d, c, solved, f, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int raftk_farm_batch_response_ws_dev(const raftk_designs *d, const raftk_cases *c, const raftk_outputs *solved,
                                                const raftk_farm_batch *f, void *workspace, size_t workspace_bytes, void *stream)
{
    disp_reset();
    if (int rc = validate_op_dev(c)) return rc;
    return farm_launch(d, c, solved, f, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int raftk_farm_ragged_response_ws_dev(const raftk_designs *d, const raftk_cases *c, const raftk_outputs *solved,
                                                 const raftk_farm_ragged *f, void *workspace, size_t workspace_bytes, void *stream)
{
    disp_reset();
    if (int rc = validate_op_dev(c)) return rc;
    return farm_ragged_launch(d, c, solved, f, workspace, workspace_bytes, (cudaStream_t)stream);
}

// After a rank's solve: k_farm_publish copies its farms' Xi_sys, info and per-FOWT status rows (three contiguous runs, its
// n_farms farms from farm_row0 and its d->n_designs FOWTs from fowt_row0, of the n_farms_total) to the same offsets of the other
// ranks' copies, and the status rows to its own.
static int farm_publish(const raftk_designs *d, const raftk_cases *c, const raftk_outputs *solved, const double *Xi_sys,
                        const int32_t *info, int n_farms, const raftk_peers *peers, long long farm_row0, long long fowt_row0,
                        long long n_farms_total, cudaStream_t st)
{
    const size_t per = (size_t)6 * c->n_cases * d->nw, info_farm = (size_t)c->n_cases * d->nw;   // one FOWT's Xi_sys, one farm's info
    FarmFlatPeer P{};
    P.n_peers = peers->n_ranks;
    P.nx = per * d->n_designs; P.ni = (size_t)n_farms * info_farm; P.ns = (size_t)d->n_designs * c->n_cases * 4;
    P.Xi = reinterpret_cast<const double2 *>(Xi_sys); P.info = info; P.status = solved->status;
    for (int r = 0; r < peers->n_ranks; r++) {
        const bool other = r != peers->rank;
        P.X[r] = other ? reinterpret_cast<double2 *>(peers->gathered[r]) + per * fowt_row0 : nullptr;
        P.I[r] = other ? peers->status[r] + farm_row0 * info_farm : nullptr;
        P.S[r] = peers->status[r] + n_farms_total * info_farm + fowt_row0 * c->n_cases * 4;
    }
    k_farm_publish<<<dim3((unsigned)std::min<size_t>((P.nx + 255) / 256, 1024), (unsigned)P.n_peers), 256, 0, st>>>(P);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RAFTK_OK;
}

extern "C" int raftk_farm_batch_response_gather_dev(const raftk_designs *d, const raftk_cases *c, const raftk_outputs *solved,
                                                    const raftk_farm_batch *f, const raftk_peers *peers, int32_t farm_row0,
                                                    void *workspace, size_t workspace_bytes, void *stream)
{
    disp_reset();
    if (int rc = validate_peers(peers)) return rc;
    if (!d || !c || !solved || !f) return set_err(RAFTK_EINVAL, "farm gather: null argument");
    if (int rc = farm_batch_shape(d, f)) return rc;
    if (!f->info || !solved->status) return set_err(RAFTK_EINVAL, "farm gather: farm_batch.info and the per-FOWT status are required");
    for (int r = 0; r < peers->n_ranks; r++)
        if (!peers->status[r]) return set_err(RAFTK_EINVAL, "farm gather: a rank's gathered info and status (peers.status) is missing");
    const size_t per_farm = (size_t)c->n_cases * 6 * f->n_fowt * d->nw;          // complex elements of one farm's Xi_sys
    if (c->n_cases < 1 || d->nw < 1 || peers->block_elems == 0 || peers->block_elems % per_farm)
        return set_err(RAFTK_EINVAL, "farm gather: peers.block_elems must be F_max * nC * 6N * nw with F_max >= 1");
    const long long F_max = (long long)(peers->block_elems / per_farm);
    if (f->n_farms > F_max) return set_err(RAFTK_EINVAL, "farm gather: farm_batch.n_farms exceeds F_max, the farms of a rank block");
    if (farm_row0 != (long long)peers->rank * F_max)                              // a rank writes its own block, no other rank's
        return set_err(RAFTK_EINVAL, "farm gather: farm_row0 must be rank * F_max, the first farm slot of this rank's block");
    const size_t info_farm = (size_t)c->n_cases * d->nw;
    if (f->Xi_sys != peers->gathered[peers->rank] + 2 * (size_t)farm_row0 * per_farm ||
        f->info != peers->status[peers->rank] + (size_t)farm_row0 * info_farm)
        return set_err(RAFTK_EINVAL, "farm gather: farm_batch.Xi_sys and info must be this rank's farms in its own gathered copy");
    if (int rc = validate_op_dev(c)) return rc;
    if (int rc = farm_launch(d, c, solved, f, workspace, workspace_bytes, (cudaStream_t)stream)) return rc;
    return farm_publish(d, c, solved, f->Xi_sys, f->info, f->n_farms, peers, farm_row0, (long long)farm_row0 * f->n_fowt,
                        peers->n_ranks * F_max, (cudaStream_t)stream);
}

extern "C" int raftk_farm_ragged_response_gather_dev(const raftk_designs *d, const raftk_cases *c, const raftk_outputs *solved,
                                                     const raftk_farm_ragged *f, const raftk_peers *peers, int32_t farm_row0,
                                                     int32_t fowt_row0, int32_t n_farms_total, void *workspace, size_t workspace_bytes,
                                                     void *stream)
{
    disp_reset();
    if (int rc = validate_peers(peers)) return rc;
    if (!d || !c || !solved || !f) return set_err(RAFTK_EINVAL, "ragged farm gather: null argument");
    if (!f->info || !solved->status) return set_err(RAFTK_EINVAL, "ragged farm gather: farm.info and the per-FOWT status are required");
    for (int r = 0; r < peers->n_ranks; r++)
        if (!peers->status[r]) return set_err(RAFTK_EINVAL, "ragged farm gather: a rank's gathered info and status (peers.status) is missing");
    if (farm_row0 < 0 || fowt_row0 < 0 || (long long)farm_row0 + f->n_farms > n_farms_total)
        return set_err(RAFTK_EINVAL, "ragged farm gather: farms [farm_row0, farm_row0 + n_farms) must lie in [0, n_farms_total)");
    const size_t per = (size_t)6 * c->n_cases * d->nw;                        // complex elements of one FOWT's rows of Xi_sys
    if (c->n_cases < 1 || d->nw < 1 || per * ((size_t)fowt_row0 + d->n_designs) > (size_t)peers->n_ranks * peers->block_elems)
        return set_err(RAFTK_EINVAL, "ragged farm gather: the gathered copies (n_ranks * peers.block_elems) do not hold this rank's farms");
    const size_t info_farm = (size_t)c->n_cases * d->nw;
    if (f->Xi_sys != peers->gathered[peers->rank] + 2 * per * fowt_row0 || f->info != peers->status[peers->rank] + (size_t)farm_row0 * info_farm)
        return set_err(RAFTK_EINVAL, "ragged farm gather: farm.Xi_sys and info must be this rank's farms in its own gathered copy");
    if (int rc = validate_op_dev(c)) return rc;
    if (int rc = farm_ragged_launch(d, c, solved, f, workspace, workspace_bytes, (cudaStream_t)stream)) return rc;
    return farm_publish(d, c, solved, f->Xi_sys, f->info, f->n_farms, peers, farm_row0, fowt_row0, n_farms_total, (cudaStream_t)stream);
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
    if (d->max_rotors > 0) {
        S.in(dd.rot_count, d->rot_count, nD);
        S.in(dd.rot_r3, d->rot_r3, nD * d->max_rotors * 3);
        S.in(dd.rot_G, d->rot_G, nD * d->max_rotors * 18);
    }
    S.in(cc.Hs, c->Hs, nC); S.in(cc.Tp, c->Tp, nC); S.in(cc.gamma, c->gamma, nC);
    S.in(cc.beta_deg, c->beta_deg, nC); S.in(cc.spec, c->spec, nC);
    S.in(cc.zeta, c->zeta, nC * nw);
    S.in(cc.primary, c->primary, nC);
    S.in(cc.F_2nd, c->F_2nd, nR / 2);
    S.in(cc.Xi_init, c->Xi_init, nR);
    if (c->op) {
        S.in(cc.op, c->op, nC);
        const size_t nT = (c->op_shared ? 1 : nD) * (size_t)c->n_op * 36 * nw;
        S.in(cc.op_A_w, c->op_A_w, nT); S.in(cc.op_B_w, c->op_B_w, nT);
    }
    if (d->n_qtf_w > 0) {
        S.in(dd.qtf_w, d->qtf_w, (size_t)d->n_qtf_w);
        S.in(dd.qtf_heads, d->qtf_heads, (size_t)d->n_qtf_head);
        S.in(dd.qtf, d->qtf, (d->qtf_shared == 1 ? 1 : (d->qtf_shared == 2 ? nD * nC : nD)) * (size_t)d->n_qtf_w * d->n_qtf_w * d->n_qtf_head * 12);
    }
}

static int host_run(const char *who, const raftk_designs *d, const raftk_cases *c, const raftk_solve_opts *o, const raftk_outputs *out,
                    const double *Xi_in, int mode, const raftk_farm_batch *farm = nullptr, const raftk_farm_ragged *rag = nullptr)
{
    disp_reset();
    int rc = validate(d, c);
    if (rc || (rc = validate_rotors_host(d, c))) return rc;
    if (mode == 0 && (rc = validate_opts(o))) return rc;
    if (!out) return set_err(RAFTK_EINVAL, "null outputs");
    raftk_cases cin = *c;
    if (mode != 0) cin.op = nullptr;                      // excitation and linearisation assemble no impedance
    else if ((rc = validate_op(c, c->op, c->primary))) return rc;
    c = &cin;
    FarmPlan fp;
    const bool farms = farm || rag;
    if (farm) farm_plan(d, c, farm, fp);
    if (rag && (rc = farm_plan(d, c, rag, fp))) return rc;
    Staging S(who);
    const size_t nD = d->n_designs, nw = d->nw, nC = c->n_cases;
    const size_t nR = nD * nC * 6 * nw * 2;             // doubles of one complex [nD,nC,6,nw] array
    raftk_designs dd = *d;
    raftk_cases cc = *c;
    stage_designs_cases(S, d, c, dd, cc);
    const double *Xi_in_d = nullptr;
    S.in(Xi_in_d, Xi_in, nR);
    if (farms) {                                          // array-level matrices (one set, or one per farm): staged with the other small inputs
        S.in(fp.M_arr, fp.M_arr, fp.n_arr); S.in(fp.B_arr, fp.B_arr, fp.n_arr); S.in(fp.C_arr, fp.C_arr, fp.n_arr);
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
    S.out(od.B_drag, out->B_drag || farms ? nD * nC * 36 : 0, out->B_drag);
    S.out(od.F_drag, out->F_drag || farms ? nR : 0, out->F_drag);
    S.out(od.F_iner, out->F_iner || farms ? nR : 0, out->F_iner);
    S.out(od.F_BEM, out->F_BEM || (farms && d->n_bem_head > 0) ? nR : 0, out->F_BEM);
    S.out(od.zeta, out->zeta ? nC * nw : 0, out->zeta);
    const bool qtf_solve = (mode == 0 && d->n_qtf_w > 0 && !c->F_2nd);   // potSecOrder 2: compute the force on the device first
    if (qtf_solve) { S.out(od.F_2nd, nR / 2, out->F_2nd); S.out(od.F_2nd_mean, nD * nC * 6, out->F_2nd_mean); }
    S.out(od.Xi_last, out->Xi_last ? nR : 0, out->Xi_last);
    char *ws, *fws = nullptr;
    S.buf(ws, wb);
    if (farms) { S.out(fp.Xi_sys, nR, fp.Xi_sys); S.out(fp.info, fp.info ? fp.F * nC * nw : 0, fp.info); S.buf(fws, fp.bytes); }
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
    if (farms && (rc = farm_run(&dd, &cc, &od, fp, fws, fp.bytes, 0))) return rc;
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
    if (d && (f->n_fowt != d->n_designs || f->n_fowt < 1)) return set_err(RAFTK_EINVAL, "farm response: farm.n_fowt must equal designs.n_designs");
    const raftk_farm_batch b = farm_as_batch(f);
    return host_run("raftk_solve_dynamics_farm_host", d, c, o, out, nullptr, 0, &b);
}

extern "C" int raftk_solve_dynamics_farm_batch_host(const raftk_designs *d, const raftk_cases *c, const raftk_solve_opts *o,
                                                    const raftk_outputs *out, const raftk_farm_batch *f)
{
    if (!out || !out->Xi || !out->status || !o) return set_err(RAFTK_EINVAL, "Xi, status and opts are required");
    if (!d || !f) return set_err(RAFTK_EINVAL, "farm batch: null argument");
    if (int rc = farm_batch_shape(d, f)) return rc;
    return host_run("raftk_solve_dynamics_farm_batch_host", d, c, o, out, nullptr, 0, f);
}

extern "C" int raftk_solve_dynamics_farm_ragged_host(const raftk_designs *d, const raftk_cases *c, const raftk_solve_opts *o,
                                                     const raftk_outputs *out, const raftk_farm_ragged *f)
{
    disp_reset();
    if (!out || !out->Xi || !out->status || !o) return set_err(RAFTK_EINVAL, "Xi, status and opts are required");
    FarmPlan R;
    if (int rc = farm_plan(d, c, f, R)) return rc;
    if (!f->Xi_sys) return set_err(RAFTK_EINVAL, "ragged farm batch: Xi_sys is required");
    return host_run("raftk_solve_dynamics_farm_ragged_host", d, c, o, out, nullptr, 0, nullptr, f);
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
    cc.primary = nullptr; cc.F_2nd = nullptr; cc.op = nullptr;
    double *F2, *F2mean;
    S.out(F2, nF, out->F_2nd); S.out(F2mean, nF / nw, out->F_2nd_mean);
    if ((rc = S.commit()) || (rc = run_qtf(&dd, &cc, F2, F2mean, 0))) return rc;
    return S.finish();
}

// ---- generalised degrees of freedom (flexible members) ---------------------------------------------------------------
struct GenLayout { size_t u, f6, Fi, Fd, XL, Bm, Bd, Z, pv, fl, fb6, FB, F2, F2m, total; };
// nC units of Ns_rows node rows each (one design: its n_nodes; a design batch: its largest design's count)
static GenLayout gen_layout(const raftk_general *g, const raftk_general_fd *fd, const raftk_general_qtf *q, size_t nC, int Ns_rows)
{
    const size_t n = g->n_dof, nw = g->nw, Ns = std::max(Ns_rows, 1);
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

// raftk_general_fd checks (include/raftk.h); idx, hd: host copies of fd_idx and bem_headings, read only once the counts and
// pointers have passed (both NULL: those checks alone)
static int validate_gen_fd(const raftk_general *g, const raftk_general_fd *fd, const int32_t *idx, const double *hd)
{
    if (fd->n_fd < 0 || fd->n_fd > g->n_dof) return set_err(RAFTK_EINVAL, "general solve: fd.n_fd must be in [0, n_dof]");
    if (fd->n_bem_head < 0) return set_err(RAFTK_EINVAL, "general solve: fd.n_bem_head must be >= 0");
    if (fd->n_fd > 0 && (!fd->fd_idx || !fd->A_w || !fd->B_w))
        return set_err(RAFTK_EINVAL, "general solve: fd.n_fd > 0 needs fd_idx, A_w and B_w");
    if (fd->n_bem_head > 0 && (!fd->bem_headings || !fd->X_BEM || !fd->T0))
        return set_err(RAFTK_EINVAL, "general solve: fd.n_bem_head > 0 needs bem_headings, X_BEM and T0");
    if (!idx && !hd) return 0;
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

// cases.op on the generalised-DOF path: the tables live on the support of fd, so an fd with n_fd >= 1 is required; then
// validate_op's counts and tables and, with host copies op_h / prim_h, every index and the trains' agreement with their primaries
static int validate_gen_op(const raftk_general_fd *fd, const raftk_cases *c, const int32_t *op_h, const int32_t *prim_h)
{
    if (!c->op) return 0;
    if (!fd || fd->n_fd < 1)
        return set_err(RAFTK_EINVAL, "general solve: cases.op (per-case operating points) without fd.n_fd >= 1 is not supported for "
                                     "generalised-DOF FOWTs: the tables are given on the support of fd_idx");
    return validate_op(c, op_h, prim_h);
}

// the elements of one operating-point table of a call: [nD or 1][n_op][n_fd][n_fd][nw] doubles
static size_t gen_op_elems(const raftk_general_fd *fd, const raftk_cases *c, size_t nD, size_t nw)
{
    const size_t nf = fd->n_fd;
    return (c->op_shared ? 1 : nD) * (size_t)c->n_op * nf * nf * nw;
}

extern "C" size_t raftk_general_qtf_workspace_bytes(const raftk_general *g, const raftk_general_fd *fd, const raftk_general_qtf *qtf,
                                                    int32_t n_cases)
{
    if (!g || n_cases <= 0 || g->n_dof <= 0 || g->nw <= 0) return 0;
    return gen_layout(g, fd, qtf, (size_t)n_cases, g->n_nodes).total;
}

extern "C" size_t raftk_general_fd_workspace_bytes(const raftk_general *g, const raftk_general_fd *fd, int32_t n_cases)
{
    return raftk_general_qtf_workspace_bytes(g, fd, nullptr, n_cases);
}

extern "C" size_t raftk_general_workspace_bytes(const raftk_general *g, int32_t n_cases)
{
    return raftk_general_fd_workspace_bytes(g, nullptr, n_cases);
}

// A design batch as the launch sequence sees it.  nD = 1 with node_off = NULL is one design: the single-design entries run as
// that batch.  Units are (design, case) pairs, design-major: unit d * n_cases + c.
struct GenBatch {
    int nD = 1, max_nodes = 0, qtf_shared = 0;
    const int32_t *node_off = nullptr;                 // device [nD+1], or NULL (one design)
    const int32_t *hnode_off = nullptr;                // host copy of node_off (the chunks' node grids), or NULL
    const double *x_ref = nullptr, *y_ref = nullptr, *hadj = nullptr;      // device [nD], or NULL: fd's scalars
};

static GenBatch gen_single(const raftk_general *g)
{
    GenBatch B;
    B.max_nodes = g->n_nodes;
    return B;
}

// cases c0 .. c0+m-1 of a case table
static raftk_cases gen_case_view(const raftk_cases *c, size_t c0, size_t m, size_t nw)
{
    raftk_cases cc = *c;
    cc.n_cases = (int32_t)m;
    cc.Hs = c->Hs ? c->Hs + c0 : nullptr; cc.Tp = c->Tp ? c->Tp + c0 : nullptr;
    cc.gamma = c->gamma ? c->gamma + c0 : nullptr; cc.beta_deg = c->beta_deg ? c->beta_deg + c0 : nullptr;
    cc.spec = c->spec ? c->spec + c0 : nullptr; cc.zeta = c->zeta ? c->zeta + c0 * nw : nullptr;
    cc.primary = c->primary ? c->primary + c0 : nullptr;
    cc.op = c->op ? c->op + c0 : nullptr;
    return cc;
}

// the launch sequence of units u0 .. u0+m-1 (m <= 65535) of batch Bt over the case table c, in a workspace of
// gen_layout(g, fd, qtf, m, Bt.max_nodes).total bytes.  prim: the chunk's primary map as chunk-local units, or NULL; Xi, status,
// F_BEM, F_2nd, F_2nd_mean: advanced to unit u0.  prof_reset: start a new profile record (a chunked call keeps one record)
static int gen_launch(const raftk_general *g, const GenBatch &Bt, const raftk_general_fd *fd, const raftk_general_qtf *qtf, const raftk_cases *c,
                      size_t u0, size_t m, const int *prim, const raftk_solve_opts *o, double *Xi, int32_t *status, double *F_BEM,
                      double *F_2nd, double *F_2nd_mean, void *workspace, cudaStream_t st, bool prof_reset)
{
    const size_t nC = m, nCt = c->n_cases;
    const GenLayout L = gen_layout(g, fd, qtf, nC, Bt.max_nodes);
    const bool bem = fd && fd->n_bem_head > 0;
    int Ns_grid = Bt.max_nodes;                        // node grids: the chunk's largest design
    if (Bt.hnode_off) {
        Ns_grid = 0;
        for (size_t d = u0 / nCt; d <= (u0 + m - 1) / nCt; d++) Ns_grid = std::max(Ns_grid, Bt.hnode_off[d + 1] - Bt.hnode_off[d]);
    }
    GenDev D;
    D.n = g->n_dof; D.nw = g->nw; D.Ns = Bt.max_nodes; D.depth = g->depth; D.dw = g->dw; D.rho = g->rho;
    D.u0 = (int)u0; D.nCt = (int)nCt; D.node_off = Bt.node_off;
    D.w = g->w; D.k = g->k; D.node_r = g->node_r; D.node_frame = g->node_frame; D.node_circ = g->node_circ;
    D.node_Imat = g->node_Imat; D.node_Imat_w = reinterpret_cast<const double2 *>(g->node_Imat_w);
    D.node_a_i = g->node_a_i; D.node_cd = g->node_cd; D.Tn = g->Tn; D.rr = g->rr; D.M = g->M; D.B = g->B; D.C = g->C;
    GenFdDev Fx;
    Fx.n_fd = fd ? fd->n_fd : 0; Fx.n_bem_head = bem ? fd->n_bem_head : 0;
    Fx.fd_idx = fd ? fd->fd_idx : nullptr; Fx.A_w = fd ? fd->A_w : nullptr; Fx.B_w = fd ? fd->B_w : nullptr;
    Fx.bem_headings = bem ? fd->bem_headings : nullptr; Fx.X_BEM = bem ? reinterpret_cast<const double2 *>(fd->X_BEM) : nullptr;
    Fx.T0 = bem ? fd->T0 : nullptr;
    Fx.x_ref = fd ? fd->x_ref : 0.0; Fx.y_ref = fd ? fd->y_ref : 0.0; Fx.hadj = fd ? fd->heading_adjust : 0.0;
    Fx.x_ref_d = Bt.x_ref; Fx.y_ref_d = Bt.y_ref; Fx.hadj_d = Bt.hadj;
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
    CasesDev C = to_dev(c);
    double2 *X = reinterpret_cast<double2 *>(Xi);
    const unsigned fb = (unsigned)((g->nw + 127) / 128);
    // the blocked LU's panel and row block in shared memory (n_dof <= 256: at most 65.7 KB)
    const size_t lu_smem = ((size_t)g->n_dof * GB + (size_t)GB * (g->n_dof + 1)) * sizeof(double2);
    const bool fdz = Fx.n_fd > 0;                      // impedance with the frequency-dependent terms on their support
    const bool op = c->op != nullptr;                  // plus every case's operating point there (validate_gen_op: n_fd >= 1)
    GenFdOpDev Fo;
    static_cast<GenFdDev &>(Fo) = Fx;
    Fo.op = c->op; Fo.n_op = c->n_op; Fo.op_shared = c->op_shared; Fo.op_A_w = c->op_A_w; Fo.op_B_w = c->op_B_w;
    {
        static SmemOptIn opt(48 * 1024), opt_fd(48 * 1024), opt_op(48 * 1024);
        CUDA_TRY(op ? opt_op.ensure(k_gen_solve_blocked<true, true>, lu_smem)
                    : fdz ? opt_fd.ensure(k_gen_solve_blocked<true>, lu_smem) : opt.ensure(k_gen_solve_blocked<false>, lu_smem));
    }
    if (F_BEM && !bem) CUDA_TRY(cudaMemsetAsync(F_BEM, 0, nC * g->n_dof * g->nw * 16, st));
    double *F2 = nullptr;
    if (qtf) {                                         // second-order force of every case and train (k_qtf_*), before the loop
        F2 = F_2nd ? F_2nd : reinterpret_cast<double *>(b + L.F2);
        double *F2m = F_2nd_mean ? F_2nd_mean : reinterpret_cast<double *>(b + L.F2m);
        const size_t nw = g->nw, tab = (size_t)qtf->n_qtf_w * qtf->n_qtf_w * qtf->n_qtf_head * 12;
        // one launch per run of units with a rectangular (design, case) layout: a partial design, or whole designs
        for (size_t a = u0; a < u0 + m;) {
            const size_t d = a / nCt, ca = a % nCt, left = u0 + m - a;
            const size_t nd = (ca == 0 && left >= nCt) ? left / nCt : 1, ce = (ca == 0 && left >= nCt) ? nCt : std::min(nCt, ca + left);
            QtfParams QP;
            QP.nD = (int)nd; QP.shared = Bt.qtf_shared;
            QP.n2 = qtf->n_qtf_w; QP.nh = qtf->n_qtf_head; QP.nw = g->nw; QP.dw = g->dw;
            QP.w = g->w; QP.qw = qtf->qtf_w; QP.qh = qtf->qtf_heads;
            QP.qtf = reinterpret_cast<const double2 *>(qtf->qtf + (Bt.qtf_shared ? 0 : d * tab));
            QP.F2 = F2 + (a - u0) * 6 * nw;
            QP.F2mean = F2m + (a - u0) * 6;
            const raftk_cases cs = gen_case_view(c, ca, ce - ca, nw);
            if (int rc = launch_qtf(QP, &cs, st)) return rc;
            a += nd * (ce - ca);
        }
    }
    if (prof_reset) prof_begin_call();
    k_gen_init<<<(unsigned)nC, 256, 0, st>>>(D, W, o->xi_start, prim);
    if (Ns_grid > 0) k_gen_wave<<<dim3(fb, Ns_grid, (unsigned)nC), 128, 0, st>>>(D, C, W);
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
        if (Ns_grid > 0) k_gen_node_pass<false><<<dim3(Ns_grid, (unsigned)nC), 128, 0, st>>>(D, W, nullptr);
        k_gen_bdrag<<<dim3(g->n_dof, (unsigned)nC), 128, 0, st>>>(D, W);
        k_gen_project<false, false><<<dim3(fb, g->n_dof, (unsigned)nC), 128, 0, st>>>(D, W, W.F_drag, 1, nullptr, Fx);
        {
            ProfScope ps(st, 2);
            if (op) k_gen_solve_blocked<true, true><<<dim3(g->nw, (unsigned)nC), GT, lu_smem, st>>>(D, W, X, o->tol, Fo);
            else if (fdz) k_gen_solve_blocked<true><<<dim3(g->nw, (unsigned)nC), GT, lu_smem, st>>>(D, W, X, o->tol, Fx);
            else k_gen_solve_blocked<false><<<dim3(g->nw, (unsigned)nC), GT, lu_smem, st>>>(D, W, X, o->tol, Fx);
        }
        k_gen_relax<<<(unsigned)nC, 256, 0, st>>>(D, W, X);
        g_launches += 5;
    }
    if (prim) {                                        // secondary trains: the primary's last Bmat and LU factors
        if (Ns_grid > 0) k_gen_node_pass<true><<<dim3(Ns_grid, (unsigned)nC), 128, 0, st>>>(D, W, prim);
        k_gen_project<false, false><<<dim3(fb, g->n_dof, (unsigned)nC), 128, 0, st>>>(D, W, W.F_drag, 0, prim, Fx);
        k_gen_train_solve<<<dim3(g->nw, (unsigned)nC), 128, 0, st>>>(D, W, prim, X);
        g_launches += 3;
    }
    disp_launch(RAFTK_FAMILY_GENERAL, RAFTK_KERNEL_GEN_BLOCKED, GT);
    g_disp.trains = prim != nullptr;
    k_gen_status<<<(unsigned)((nC + 127) / 128), 128, 0, st>>>((int)nC, W.flags, prim, status);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RAFTK_OK;
}

// ---- generalised DOFs, streamed: the units in chunks of whole train groups through one bounded workspace ---------------
static size_t gen_chunk_cap(int64_t n_units, int32_t max_chunk)
{
    return (max_chunk <= 0 || max_chunk >= n_units) ? (size_t)n_units : (size_t)max_chunk;
}

// gen_layout of the largest chunk, plus the chunk-local primary map [K] at the end when the units run in more than one chunk or
// span more than one design
static size_t gen_run_bytes(const raftk_general *g, const GenBatch &Bt, const raftk_general_fd *fd, const raftk_general_qtf *qtf, int64_t n_units,
                            int32_t max_chunk, size_t *prim_off)
{
    const size_t K = gen_chunk_cap(n_units, max_chunk);
    const size_t base = gen_layout(g, fd, qtf, K, Bt.max_nodes).total;
    if (prim_off) *prim_off = base;
    return (K < (size_t)n_units || Bt.nD > 1) ? base + align_up(K * 4, 256) : base;
}

extern "C" size_t raftk_general_stream_workspace_bytes(const raftk_general *g, const raftk_general_fd *fd, const raftk_general_qtf *qtf,
                                                       int32_t n_cases, int32_t max_chunk_cases)
{
    if (!g || n_cases <= 0 || g->n_dof <= 0 || g->nw <= 0) return 0;
    return gen_run_bytes(g, gen_single(g), fd, qtf, n_cases, max_chunk_cases, nullptr);
}

// Chunk starts (and the end) of the units of nD designs over a case table: whole train groups, greedily packed into chunks of
// at most K units; a chunk may cross design boundaries.  prim: host copy of cases.primary or NULL (every case a group of its
// own).  A group is the set of cases sharing one primary; it must be contiguous in the table (packer.pack_case_trains lays
// tables out so) and no larger than K.  batch: the batch entry's wording (max_chunk_units).
static int gen_plan_chunks(const int32_t *prim, size_t nC, size_t nD, size_t K, bool batch, std::vector<size_t> &starts)
{
    starts.clear();
    std::vector<size_t> gs;                            // group starts within the case table
    if (prim) {
        std::vector<size_t> first(nC, SIZE_MAX), last(nC, 0), count(nC, 0);
        for (size_t i = 0; i < nC; i++) {
            const int p = prim[i];
            if (p < 0 || (size_t)p >= nC || prim[p] != p) return set_err(RAFTK_EINVAL, "general solve: cases.primary must map every case to a primary case");
            first[p] = std::min(first[p], i); last[p] = i; count[p]++;
        }
        for (size_t p = 0; p < nC; p++)
            if (count[p] && last[p] - first[p] + 1 != count[p])
                return set_err(RAFTK_EINVAL, "general stream: the train groups of cases.primary interleave (a group must be contiguous in the table)");
        for (size_t i = 0; i < nC; i++)
            if (i == 0 || prim[i] != prim[i - 1]) gs.push_back(i);
    } else {
        for (size_t i = 0; i < nC; i++) gs.push_back(i);
    }
    gs.push_back(nC);
    for (size_t t = 0; t + 1 < gs.size(); t++)
        if (gs[t + 1] - gs[t] > K)
            return set_err(RAFTK_EINVAL, batch ? "general batch: a train group has more cases than max_chunk_units"
                                               : "general stream: a train group has more cases than max_chunk_cases");
    starts.push_back(0);
    for (size_t d = 0; d < nD; d++)
        for (size_t t = 0; t + 1 < gs.size(); t++)
            if (d * nC + gs[t + 1] - starts.back() > K) starts.push_back(d * nC + gs[t]);
    starts.push_back(nD * nC);
    return 0;
}

// the chunk loop on device pointers; hprim: host copy of c->primary (NULL without trains)
static int gen_run(const raftk_general *g, const GenBatch &Bt, const raftk_general_fd *fd, const raftk_general_qtf *qtf, const raftk_cases *c,
                   const int32_t *hprim, const raftk_solve_opts *o, double *Xi, int32_t *status, double *F_BEM, double *F_2nd,
                   double *F_2nd_mean, void *workspace, size_t workspace_bytes, int32_t max_chunk, bool batch, cudaStream_t st)
{
    const size_t nC = c->n_cases, nU = (size_t)Bt.nD * nC, K = gen_chunk_cap((int64_t)nU, max_chunk);
    if (K > 65535)
        return set_err(RAFTK_EINVAL, batch ? "general batch: a chunk takes at most 65535 units (max_chunk_units)"
                                           : "general stream: a chunk takes at most 65535 cases (max_chunk_cases)");
    std::vector<size_t> starts;
    if (int rc = gen_plan_chunks(hprim, nC, Bt.nD, K, batch, starts)) return rc;
    size_t prim_off = 0;
    const size_t need = gen_run_bytes(g, Bt, fd, qtf, (int64_t)nU, max_chunk, &prim_off);
    if (!workspace || workspace_bytes < need)
        return set_err(RAFTK_EINVAL, batch ? "general batch: workspace smaller than raftk_general_batch_workspace_bytes()"
                                           : "general stream: workspace smaller than raftk_general_stream_workspace_bytes()");
    int *local = reinterpret_cast<int *>(static_cast<char *>(workspace) + prim_off);
    const size_t n = g->n_dof, nw = g->nw, nch = starts.size() - 1;
    for (size_t k = 0; k < nch; k++) {
        const size_t u0 = starts[k], m = starts[k + 1] - u0;
        const int *prim = c->primary;
        if (c->primary && (nch > 1 || Bt.nD > 1)) {    // table primaries -> chunk-local units
            k_gen_chunk_primary<<<(unsigned)((m + 127) / 128), 128, 0, st>>>((int)m, (int)u0, (int)nC, c->primary, local);
            g_launches++;
            prim = local;
        }
        if (int rc = gen_launch(g, Bt, fd, qtf, c, u0, m, prim, o, Xi + u0 * n * nw * 2, status + u0 * 4, F_BEM ? F_BEM + u0 * n * nw * 2 : nullptr,
                                F_2nd ? F_2nd + u0 * 6 * nw : nullptr, F_2nd_mean ? F_2nd_mean + u0 * 6 : nullptr, workspace, st, k == 0))
            return rc;
        if (c->primary && (u0 % nC != 0 || u0 % nC + m > nC)) {      // status word 3 of the secondaries: the primary's case + 1
            k_gen_status_rebase<<<(unsigned)((m + 127) / 128), 128, 0, st>>>((int)m, (int)u0, (int)nC, status + u0 * 4);
            g_launches++;
        }
    }
    g_disp.chunks = (int32_t)nch;
    CUDA_TRY(cudaGetLastError());
    return RAFTK_OK;
}

// ---- generalised DOFs, design batches: designs sharing n_dof, the frequency grid, depth and rho ------------------------
static GenBatch gen_batch_of(const raftk_general_batch *b)
{
    GenBatch B;
    B.nD = b->n_designs; B.max_nodes = b->max_nodes; B.qtf_shared = b->qtf_shared;
    B.node_off = b->node_offset; B.x_ref = b->x_ref; B.y_ref = b->y_ref; B.hadj = b->heading_adjust;
    return B;
}

extern "C" size_t raftk_general_batch_workspace_bytes(const raftk_general *g, const raftk_general_batch *b, const raftk_general_fd *fd,
                                                      const raftk_general_qtf *qtf, int32_t n_cases, int32_t max_chunk_units)
{
    if (!g || !b || n_cases <= 0 || b->n_designs <= 0 || b->max_nodes < 0 || g->n_dof <= 0 || g->nw <= 0) return 0;
    const int64_t nU = (int64_t)b->n_designs * n_cases;
    if (nU > INT32_MAX) return 0;
    return gen_run_bytes(g, gen_batch_of(b), fd, qtf, nU, max_chunk_units, nullptr);
}

// ---- generalised DOFs, the entry points: one-shot, streamed and design batches through one set of checks, one staging
// list and one launch path -------------------------------------------------------------------------------------------
enum GenMode { GEN_ONE_SHOT, GEN_STREAM, GEN_BATCH };

// One call as its entry received it.  b is NULL on the single-design entries, which run as gen_single()'s batch; nD and
// qtf_shared size the per-design tables (1 and 0 there).
struct GenCall {
    const raftk_general *g; const raftk_general_batch *b; const raftk_general_fd *fd; const raftk_general_qtf *qtf; const raftk_cases *c;
    int nD, qtf_shared;
};

static GenCall gen_call(const raftk_general *g, const raftk_general_batch *b, const raftk_general_fd *fd, const raftk_general_qtf *qtf,
                        const raftk_cases *c)
{
    return {g, b, fd, qtf, c, b ? b->n_designs : 1, b ? b->qtf_shared : 0};
}

// Host copies of the tables the checks and the chunk plan read; NULL: not in the call, or not read back
struct GenTables { const int32_t *off, *idx; const double *hd, *qw, *qh; const int32_t *op, *prim; };

// The checks that need no table contents, before anything is read back or staged.  The wording follows the entry family:
// the one-shot entries take at most one launch grid of cases, the stream and batch entries a chunk cap max_chunk.
static int gen_check_counts(const GenCall &k, GenMode mode, const raftk_solve_opts *o, const double *Xi, const int32_t *status,
                            int32_t max_chunk)
{
    const raftk_general *g = k.g;
    const raftk_cases *c = k.c;
    const bool one = mode == GEN_ONE_SHOT, batch = mode == GEN_BATCH;
    if (!g || !c || !o || !Xi || !status || (batch && (!k.b || !k.b->node_offset)))
        return set_err(RAFTK_EINVAL, batch ? "general batch: null argument" : "general solve: null argument");
    if (int rc = validate_opts(o)) return rc;
    if (batch && (k.nD <= 0 || k.b->max_nodes < 0)) return set_err(RAFTK_EINVAL, "general batch: n_designs > 0 and max_nodes >= 0");
    if (g->n_dof <= 0 || g->n_dof > 256 || g->nw <= 0 || g->n_nodes < 0 || c->n_cases <= 0 || (one && c->n_cases > 65535))
        return set_err(RAFTK_EINVAL, one ? "general solve: 0 < n_dof <= 256, nw > 0, 0 < n_cases <= 65535"
                                         : "general solve: 0 < n_dof <= 256, nw > 0, n_cases > 0");
    const int64_t nU = (int64_t)k.nD * c->n_cases;
    if (nU > INT32_MAX) return set_err(RAFTK_EINVAL, "general batch: n_designs * n_cases must stay below 2^31");
    if (c->F_2nd || c->Xi_init) return set_err(RAFTK_EINVAL, "general solve: F_2nd / Xi_init are not supported");
    if (int rc = validate_gen_op(k.fd, c, nullptr, nullptr)) return rc;
    if (!one && max_chunk < 0)
        return set_err(RAFTK_EINVAL, batch ? "general batch: max_chunk_units must be >= 0 (0: all units)"
                                           : "general stream: max_chunk_cases must be >= 0 (0: all cases)");
    if (!one && gen_chunk_cap(nU, max_chunk) > 65535)
        return set_err(RAFTK_EINVAL, batch ? "general batch: a chunk takes at most 65535 units (max_chunk_units)"
                                           : "general stream: a chunk takes at most 65535 cases (max_chunk_cases)");
    if (k.qtf_shared < 0 || k.qtf_shared > 1) return set_err(RAFTK_EINVAL, "general batch: qtf_shared must be 0 or 1");
    if (k.qtf)
        if (int rc = validate_gen_qtf(g, k.qtf, nullptr, nullptr)) return rc;
    return k.fd ? validate_gen_fd(g, k.fd, nullptr, nullptr) : 0;
}

// The checks on table contents, on host copies t of a call that passed gen_check_counts: node_offset, every design's fd_idx
// and bem_headings rows, the QTF grid, cases.op and, when t holds it, that every case maps to a case that is its own primary.
// The chunk plan's own rule (each train group contiguous in the table) stays with gen_plan_chunks.
static int gen_check_tables(const GenCall &k, const GenTables &t)
{
    const raftk_general *g = k.g;
    const int nD = k.nD, nC = k.c->n_cases;
    if (const int32_t *off = t.off) {                  // (a design batch)
        if (off[0] != 0) return set_err(RAFTK_EINVAL, "general batch: node_offset must start at 0");
        for (int d = 0; d < nD; d++) {
            if (off[d + 1] < off[d]) return set_err(RAFTK_EINVAL, "general batch: node_offset must be non-decreasing");
            if (off[d + 1] - off[d] > k.b->max_nodes) return set_err(RAFTK_EINVAL, "general batch: a design has more nodes than max_nodes");
        }
        if (off[nD] != g->n_nodes) return set_err(RAFTK_EINVAL, "general batch: node_offset[n_designs] must equal n_nodes");
    }
    if (k.fd)
        for (int d = 0; d < nD; d++)
            if (int rc = validate_gen_fd(g, k.fd, t.idx + (size_t)d * k.fd->n_fd, t.hd + (size_t)d * k.fd->n_bem_head)) return rc;
    if (k.qtf)
        if (int rc = validate_gen_qtf(g, k.qtf, t.qw, t.qh)) return rc;
    if (int rc = validate_gen_op(k.fd, k.c, t.op, t.prim)) return rc;
    if (t.prim)
        for (int i = 0; i < nC; i++) {
            const int p = t.prim[i];
            if (p < 0 || p >= nC || t.prim[p] != p) return set_err(RAFTK_EINVAL, "general solve: cases.primary must map every case to a primary case");
        }
    return 0;
}

// The tables a *_dev call's checks read, copied back with one wait (none when there is nothing to read).  cases.primary is read
// when the chunk plan needs it (primary) or cases.op is checked against it.
struct GenReadback { std::vector<int32_t> off, idx, op, prim; std::vector<double> hd, qw, qh; GenTables t{}; };

static int gen_read_back(const GenCall &k, bool primary, cudaStream_t st, GenReadback &r)
{
    const raftk_general_fd *fd = k.fd;
    const raftk_general_qtf *q = k.qtf;
    const raftk_cases *c = k.c;
    const size_t nD = k.nD, nC = c->n_cases;
    cudaError_t e = cudaSuccess;
    auto back = [&](auto &v, const auto *d, size_t n) -> decltype(d) {
        if (!d || !n) return nullptr;
        v.resize(n);
        if (e == cudaSuccess) e = cudaMemcpyAsync(v.data(), d, n * sizeof(v[0]), cudaMemcpyDeviceToHost, st);
        return v.data();
    };
    r.t.off = back(r.off, k.b ? k.b->node_offset : nullptr, nD + 1);
    r.t.idx = back(r.idx, fd ? fd->fd_idx : nullptr, fd ? nD * fd->n_fd : 0);
    r.t.hd = back(r.hd, fd ? fd->bem_headings : nullptr, fd ? nD * fd->n_bem_head : 0);
    r.t.qw = back(r.qw, q ? q->qtf_w : nullptr, q ? q->n_qtf_w : 0);
    r.t.qh = back(r.qh, q ? q->qtf_heads : nullptr, q ? q->n_qtf_head : 0);
    r.t.op = back(r.op, c->op, nC);
    r.t.prim = back(r.prim, primary || c->op ? c->primary : nullptr, nC);
    if (e == cudaSuccess && (r.t.off || r.t.idx || r.t.hd || r.t.qw || r.t.op || r.t.prim)) e = cudaStreamSynchronize(st);
    return e == cudaSuccess ? 0 : set_err(RAFTK_ECUDA, "general solve: reading the tables back: %s", cudaGetErrorString(e));
}

// workspace bytes of a checked call
static size_t gen_ws_bytes(GenMode mode, const GenCall &k, int32_t max_chunk)
{
    if (mode == GEN_ONE_SHOT) return gen_layout(k.g, k.fd, k.qtf, k.c->n_cases, k.g->n_nodes).total;
    return gen_run_bytes(k.g, k.b ? gen_batch_of(k.b) : gen_single(k.g), k.fd, k.qtf, (int64_t)k.nD * k.c->n_cases, max_chunk, nullptr);
}

// A checked call on device pointers: the one-shot launch sequence, or the chunk loop.  t: host copies of node_offset and
// cases.primary for the chunks' node grids and plan.
static int gen_go(GenMode mode, const GenCall &k, const GenTables &t, const raftk_solve_opts *o, double *Xi, int32_t *status, double *F_BEM,
                  double *F_2nd, double *F_2nd_mean, void *workspace, size_t workspace_bytes, int32_t max_chunk, cudaStream_t st)
{
    if (mode == GEN_ONE_SHOT) {
        if (!workspace || workspace_bytes < gen_ws_bytes(mode, k, 0)) return set_err(RAFTK_ENOMEM, "general solve: workspace too small");
        return gen_launch(k.g, gen_single(k.g), k.fd, k.qtf, k.c, 0, k.c->n_cases, k.c->primary, o, Xi, status, F_BEM, F_2nd, F_2nd_mean,
                          workspace, st, true);
    }
    GenBatch Bt = k.b ? gen_batch_of(k.b) : gen_single(k.g);
    Bt.hnode_off = t.off;
    return gen_run(k.g, Bt, k.fd, k.qtf, k.c, t.prim, o, Xi, status, F_BEM, F_2nd, F_2nd_mean, workspace, workspace_bytes, max_chunk,
                   mode == GEN_BATCH, st);
}

static int gen_dev(GenMode mode, const GenCall &k, const raftk_solve_opts *o, double *Xi, int32_t *status, double *F_BEM, double *F_2nd,
                   double *F_2nd_mean, void *workspace, size_t workspace_bytes, int32_t max_chunk, void *stream)
{
    disp_reset();
    cudaStream_t st = (cudaStream_t)stream;
    GenReadback r;
    if (int rc = gen_check_counts(k, mode, o, Xi, status, max_chunk)) return rc;
    if (int rc = gen_read_back(k, mode != GEN_ONE_SHOT, st, r)) return rc;
    if (int rc = gen_check_tables(k, r.t)) return rc;
    return gen_go(mode, k, r.t, o, Xi, status, F_BEM, F_2nd, F_2nd_mean, workspace, workspace_bytes, max_chunk, st);
}

// The device side of a *_host call: copies of its structs, whose pointers Staging::commit() turns into device addresses, the
// five outputs and the workspace
struct GenStaged {
    raftk_general g; raftk_general_batch b; raftk_general_fd fd; raftk_general_qtf qtf; raftk_cases c; GenCall k;
    double *Xi, *F_BEM, *F_2nd, *F_2nd_mean; int32_t *status; char *ws;
};

// every input of call k (the per-design tables nD deep, the QTF table qtf_shared-deep), the outputs the caller asked for and
// wb bytes of workspace
static void gen_stage(Staging &S, const GenCall &k, double *Xi, int32_t *status, double *F_BEM, double *F_2nd, double *F_2nd_mean,
                      size_t wb, GenStaged &D)
{
    const raftk_general *g = k.g;
    const raftk_general_fd *fd = k.fd;
    const raftk_general_qtf *q = k.qtf;
    const raftk_cases *c = k.c;
    const size_t nD = k.nD, n = g->n_dof, nw = g->nw, Ns = g->n_nodes, nC = c->n_cases, nU = nD * nC;
    D.g = *g;
    S.in(D.g.w, g->w, nw); S.in(D.g.k, g->k, nw);
    S.in(D.g.node_r, g->node_r, Ns * 3); S.in(D.g.node_frame, g->node_frame, Ns * 9);
    S.in(D.g.node_circ, g->node_circ, Ns); S.in(D.g.node_Imat, g->node_Imat, Ns * 9);
    S.in(D.g.node_Imat_w, g->node_Imat_w, Ns * 9 * nw * 2); S.in(D.g.node_a_i, g->node_a_i, Ns);
    S.in(D.g.node_cd, g->node_cd, Ns * 4); S.in(D.g.Tn, g->Tn, Ns * 6 * n); S.in(D.g.rr, g->rr, Ns * 3);
    S.in(D.g.M, g->M, nD * n * n); S.in(D.g.B, g->B, nD * n * n); S.in(D.g.C, g->C, nD * n * n);
    if (k.b) {
        D.b = *k.b;
        S.in(D.b.node_offset, k.b->node_offset, nD + 1);
        S.in(D.b.x_ref, k.b->x_ref, nD); S.in(D.b.y_ref, k.b->y_ref, nD); S.in(D.b.heading_adjust, k.b->heading_adjust, nD);
    }
    D.c = *c;
    S.in(D.c.Hs, c->Hs, nC); S.in(D.c.Tp, c->Tp, nC); S.in(D.c.gamma, c->gamma, nC);
    S.in(D.c.beta_deg, c->beta_deg, nC); S.in(D.c.spec, c->spec, nC); S.in(D.c.zeta, c->zeta, nC * nw);
    S.in(D.c.primary, c->primary, nC);
    if (c->op) { S.in(D.c.op, c->op, nC); S.in(D.c.op_A_w, c->op_A_w, gen_op_elems(fd, c, nD, nw)); S.in(D.c.op_B_w, c->op_B_w, gen_op_elems(fd, c, nD, nw)); }
    if (fd) {                                          // validate_gen_fd: both counts >= 0
        const size_t nf = fd->n_fd, nh = fd->n_bem_head;
        D.fd = *fd;
        S.in(D.fd.fd_idx, fd->fd_idx, nD * nf); S.in(D.fd.A_w, fd->A_w, nD * nf * nf * nw); S.in(D.fd.B_w, fd->B_w, nD * nf * nf * nw);
        S.in(D.fd.bem_headings, fd->bem_headings, nD * nh); S.in(D.fd.X_BEM, fd->X_BEM, nD * nh * 6 * nw * 2);
        S.in(D.fd.T0, fd->T0, nh ? nD * 6 * n : 0);
    }
    if (q) {                                           // validate_gen_qtf: both counts >= 1
        const size_t n2 = q->n_qtf_w, nh = q->n_qtf_head;
        D.qtf = *q;
        S.in(D.qtf.qtf_w, q->qtf_w, n2); S.in(D.qtf.qtf_heads, q->qtf_heads, nh);
        S.in(D.qtf.qtf, q->qtf, (k.qtf_shared ? 1 : nD) * n2 * n2 * nh * 12);
    }
    S.out(D.Xi, nU * n * nw * 2, Xi); S.out(D.status, nU * 4, status); S.out(D.F_BEM, F_BEM ? nU * n * nw * 2 : 0, F_BEM);
    S.out(D.F_2nd, q && F_2nd ? nU * 6 * nw : 0, F_2nd); S.out(D.F_2nd_mean, q && F_2nd_mean ? nU * 6 : 0, F_2nd_mean);
    S.buf(D.ws, wb);
    D.k = {&D.g, k.b ? &D.b : nullptr, fd ? &D.fd : nullptr, q ? &D.qtf : nullptr, &D.c, k.nD, k.qtf_shared};
}

// Every check on the caller's arrays (the stream and batch entries' chunk plan included) before any CUDA call, then one
// staging, the launch path and one download
static int gen_host(const char *who, GenMode mode, const GenCall &k, const raftk_solve_opts *o, double *Xi, int32_t *status, double *F_BEM,
                    double *F_2nd, double *F_2nd_mean, int32_t max_chunk)
{
    disp_reset();
    if (int rc = gen_check_counts(k, mode, o, Xi, status, max_chunk)) return rc;
    const GenTables t = {k.b ? k.b->node_offset : nullptr, k.fd ? k.fd->fd_idx : nullptr, k.fd ? k.fd->bem_headings : nullptr,
                         k.qtf ? k.qtf->qtf_w : nullptr, k.qtf ? k.qtf->qtf_heads : nullptr, k.c->op, k.c->primary};
    if (int rc = gen_check_tables(k, t)) return rc;
    std::vector<size_t> starts;                        // the chunk plan's checks, before anything is staged
    const size_t nC = k.c->n_cases;
    if (mode != GEN_ONE_SHOT)
        if (int rc = gen_plan_chunks(t.prim, nC, k.nD, gen_chunk_cap((int64_t)k.nD * nC, max_chunk), mode == GEN_BATCH, starts)) return rc;
    Staging S(who);
    GenStaged D;
    const size_t wb = gen_ws_bytes(mode, k, max_chunk);
    gen_stage(S, k, Xi, status, F_BEM, F_2nd, F_2nd_mean, wb, D);
    int rc = S.commit();
    if (rc || (rc = gen_go(mode, D.k, t, o, D.Xi, D.status, D.F_BEM, D.F_2nd, D.F_2nd_mean, D.ws, wb, max_chunk, nullptr))) return rc;
    return S.finish();
}

extern "C" int raftk_general_solve_dynamics_qtf_dev(const raftk_general *g, const raftk_general_fd *fd, const raftk_general_qtf *qtf,
                                                    const raftk_cases *c, const raftk_solve_opts *o, double *Xi, int32_t *status,
                                                    double *F_BEM, double *F_2nd, double *F_2nd_mean, void *workspace,
                                                    size_t workspace_bytes, void *stream)
{
    return gen_dev(GEN_ONE_SHOT, gen_call(g, nullptr, fd, qtf, c), o, Xi, status, F_BEM, F_2nd, F_2nd_mean, workspace, workspace_bytes, 0,
                   stream);
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
    return gen_host(qtf ? "raftk_general_solve_dynamics_qtf_host" : "raftk_general_solve_dynamics_fd_host", GEN_ONE_SHOT,
                    gen_call(g, nullptr, fd, qtf, c), o, Xi, status, F_BEM, F_2nd, F_2nd_mean, 0);
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

extern "C" int raftk_general_solve_dynamics_stream_dev(const raftk_general *g, const raftk_general_fd *fd, const raftk_general_qtf *qtf,
                                                       const raftk_cases *c, const raftk_solve_opts *o, double *Xi, int32_t *status,
                                                       double *F_BEM, double *F_2nd, double *F_2nd_mean, void *workspace,
                                                       size_t workspace_bytes, int32_t max_chunk_cases, void *stream)
{
    return gen_dev(GEN_STREAM, gen_call(g, nullptr, fd, qtf, c), o, Xi, status, F_BEM, F_2nd, F_2nd_mean, workspace, workspace_bytes,
                   max_chunk_cases, stream);
}

extern "C" int raftk_general_solve_dynamics_stream_host(const raftk_general *g, const raftk_general_fd *fd, const raftk_general_qtf *qtf,
                                                        const raftk_cases *c, const raftk_solve_opts *o, double *Xi, int32_t *status,
                                                        double *F_BEM, double *F_2nd, double *F_2nd_mean, int32_t max_chunk_cases)
{
    return gen_host("raftk_general_solve_dynamics_stream_host", GEN_STREAM, gen_call(g, nullptr, fd, qtf, c), o, Xi, status, F_BEM, F_2nd,
                    F_2nd_mean, max_chunk_cases);
}

extern "C" int raftk_general_batch_solve_dynamics_dev(const raftk_general *g, const raftk_general_batch *b, const raftk_general_fd *fd,
                                                      const raftk_general_qtf *qtf, const raftk_cases *c, const raftk_solve_opts *o,
                                                      double *Xi, int32_t *status, double *F_BEM, double *F_2nd, double *F_2nd_mean,
                                                      void *workspace, size_t workspace_bytes, int32_t max_chunk_units, void *stream)
{
    return gen_dev(GEN_BATCH, gen_call(g, b, fd, qtf, c), o, Xi, status, F_BEM, F_2nd, F_2nd_mean, workspace, workspace_bytes,
                   max_chunk_units, stream);
}

extern "C" int raftk_general_batch_solve_dynamics_host(const raftk_general *g, const raftk_general_batch *b, const raftk_general_fd *fd,
                                                       const raftk_general_qtf *qtf, const raftk_cases *c, const raftk_solve_opts *o,
                                                       double *Xi, int32_t *status, double *F_BEM, double *F_2nd, double *F_2nd_mean,
                                                       int32_t max_chunk_units)
{
    return gen_host("raftk_general_batch_solve_dynamics_host", GEN_BATCH, gen_call(g, b, fd, qtf, c), o, Xi, status, F_BEM, F_2nd,
                    F_2nd_mean, max_chunk_units);
}

// Peer publication of a streamed shard (raftk_general_publish_dev): rows [row0, row0 + n_rows) of every rank's gathered array
__global__ void __launch_bounds__(256) k_gen_publish(GenPublish P, const double2 *Xi, const int *status)
{
    const int p = blockIdx.y;
    const size_t stride = (size_t)gridDim.x * 256, t0 = (size_t)blockIdx.x * 256 + threadIdx.x;
    double2 *dst = P.X[p];
    for (size_t t = t0; t < P.elems; t += stride) dst[t] = Xi[t];
    if (int *sd = P.S[p])
        for (size_t t = t0; t < (size_t)P.rows * 4; t += stride) {
            const int v = status[t];
            sd[t] = ((t & 3) == 3 && v != 0) ? v + P.primary_base : v;
        }
}

extern "C" int raftk_general_publish_dev(const raftk_peers *peers, const double *Xi, const int32_t *status, int32_t row0, int32_t n_rows,
                                         int32_t n_dof, int32_t nw, int32_t primary_base, void *stream)
{
    disp_reset();
    if (int rc = validate_peers(peers)) return rc;
    if (!Xi || row0 < 0 || n_rows < 0 || n_dof <= 0 || nw <= 0)
        return set_err(RAFTK_EINVAL, "general publish: Xi is required, row0 >= 0, n_rows >= 0, n_dof > 0, nw > 0");
    const size_t row = (size_t)n_dof * nw;
    if (((size_t)row0 + n_rows) * row > (size_t)peers->n_ranks * peers->block_elems)
        return set_err(RAFTK_EINVAL, "general publish: rows past the gathered array (n_ranks * block_elems complex elements)");
    if (status)
        for (int r = 0; r < peers->n_ranks; r++)
            if (!peers->status[r]) return set_err(RAFTK_EINVAL, "general publish: status given but a rank's gathered status is missing");
    if (n_rows == 0) return RAFTK_OK;
    GenPublish P;
    P.elems = (size_t)n_rows * row; P.rows = n_rows; P.primary_base = primary_base;
    for (int r = 0; r < RAFTK_MAX_PEERS; r++) {
        const bool on = r < peers->n_ranks;
        P.X[r] = on ? reinterpret_cast<double2 *>(peers->gathered[r]) + (size_t)row0 * row : nullptr;
        P.S[r] = on && status ? peers->status[r] + (size_t)row0 * 4 : nullptr;
    }
    const unsigned bx = (unsigned)std::min<size_t>((P.elems + 255) / 256, 1024);
    k_gen_publish<<<dim3(bx, (unsigned)peers->n_ranks), 256, 0, (cudaStream_t)stream>>>(P, reinterpret_cast<const double2 *>(Xi), status);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RAFTK_OK;
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

// the slender-body columns of nD designs: one design's tables, or a batch's concatenated ones, where every design has its own
// member-local mem_node_start row (its n_members + 1 entries) and its own M_struc
static void stage_slender(Staging &S, const raftk_slender &from, raftk_slender &to, size_t nD)
{
    const size_t Nm = from.n_members, Ns = from.n_nodes, Ng = from.n_seg, nw = from.nw;
    S.in(to.w, from.w, nw); S.in(to.k, from.k, nw);
    S.in(to.mem_q, from.mem_q, Nm * 3); S.in(to.mem_p1, from.mem_p1, Nm * 3); S.in(to.mem_p2, from.mem_p2, Nm * 3);
    S.in(to.mem_mcf, from.mem_mcf, Nm); S.in(to.mem_wl, from.mem_wl, Nm);
    S.in(to.mem_r_int, from.mem_r_int, Nm * 3); S.in(to.mem_a_wl, from.mem_a_wl, Nm);
    S.in(to.mem_rwl, from.mem_rwl, Nm * 3); S.in(to.mem_R_wl, from.mem_R_wl, Nm);
    S.in(to.mem_node_start, from.mem_node_start, Nm + nD);
    S.in(to.node_r, from.node_r, Ns * 3); S.in(to.node_v_side, from.node_v_side, Ns);
    S.in(to.node_Ca_p1, from.node_Ca_p1, Ns); S.in(to.node_Ca_p2, from.node_Ca_p2, Ns);
    S.in(to.node_Ca_End, from.node_Ca_End, Ns); S.in(to.node_v_end, from.node_v_end, Ns);
    S.in(to.node_a_i, from.node_a_i, Ns);
    S.in(to.seg_mem, from.seg_mem, Ng); S.in(to.seg_z1, from.seg_z1, Ng); S.in(to.seg_z2, from.seg_z2, Ng);
    S.in(to.seg_R, from.seg_R, Ng); S.in(to.seg_rmid, from.seg_rmid, Ng * 3);
    S.in(to.M_struc, from.M_struc, nD * 36);
}

extern "C" int raftk_qtf_slender_host(const raftk_slender *s, int32_t n_cases, const double *beta_rad, const double *Xi_rao, double *qtf)
{
    int rc = validate_slender(s, n_cases);
    if (rc) return rc;
    if (!beta_rad || !Xi_rao || !qtf) return set_err(RAFTK_EINVAL, "slender-body QTF: null beta / Xi_rao / qtf");
    const size_t nw = s->nw, nC = n_cases;
    Staging S("raftk_qtf_slender_host");
    raftk_slender dd = *s;
    stage_slender(S, *s, dd, 1);
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
    if (int rc = validate_op_dev(c)) return rc;
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
    if (int rc = validate_rotors_host(d, c)) return rc;
    if (int rc = validate_op(c, c->op, nullptr)) return rc;
    Staging S("raftk_solve_dynamics_slender_host");
    raftk_designs dd = *d;
    raftk_cases cc = *c;
    stage_designs_cases(S, d, c, dd, cc);
    const size_t nD = d->n_designs, nw = d->nw, nC = c->n_cases, nR = nD * nC * 6 * nw * 2, nw2 = s->cols.nw;
    raftk_slender_batch sb = *s;
    S.in(sb.node_offset, s->node_offset, nD + 1); S.in(sb.member_offset, s->member_offset, nD + 1); S.in(sb.seg_offset, s->seg_offset, nD + 1);
    stage_slender(S, s->cols, sb.cols, nD);
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

// ---- argument checks shared by the post-solve reductions -------------------------------------------------------------------
// `who` is the entry's prefix of its refusals ("fatigue", "stress ring", "rotor-stats", ...).

// The channel kernels apply w^0, w^1 or w^2; wpow: a host copy of n powers, or NULL (every power 0)
static int check_wpow(const char *who, const int32_t *wpow, int32_t n)
{
    for (int32_t t = 0; wpow && t < n; t++)
        if (wpow[t] < 0 || wpow[t] > 2) return set_err(RAFTK_EINVAL, "%s: wpow must be 0, 1 or 2", who);
    return RAFTK_OK;
}

// case c reads rows case_row0[c] .. case_row0[c + 1] - 1 of every unit
static int check_case_rows(const char *who, const int32_t *case_row0, int32_t n_cases, int32_t n_rows)
{
    if (case_row0[0] != 0 || case_row0[n_cases] != n_rows)
        return set_err(RAFTK_EINVAL, "%s: case_row0 must start at 0 and end at n_rows", who);
    for (int32_t c = 0; c < n_cases; c++)
        if (case_row0[c + 1] <= case_row0[c]) return set_err(RAFTK_EINVAL, "%s: every case needs at least one row", who);
    return RAFTK_OK;
}

// the case probabilities of a lifetime sum, or NULL (every case 1)
static int check_weights(const char *who, const double *weights, int32_t n_cases)
{
    if (!weights) return RAFTK_OK;
    double s = 0.0;
    for (int32_t c = 0; c < n_cases; c++) {
        if (!(std::isfinite(weights[c]) && weights[c] >= 0.0)) return set_err(RAFTK_EINVAL, "%s: weights must be finite and >= 0", who);
        s += weights[c];
    }
    if (!(s > 0.0)) return set_err(RAFTK_EINVAL, "%s: the weights must not all be 0", who);
    return RAFTK_OK;
}

// a _dev entry's workspace: at least `need` bytes (what `sizer` returns), 32-byte aligned for the kernels' double4 reads
static int check_workspace(const char *who, const char *sizer, const void *ws, size_t bytes, size_t need)
{
    if (!ws || bytes < need) return set_err(RAFTK_EINVAL, "%s: the workspace is too small (%s)", who, sizer);
    if ((uintptr_t)ws % 32) return set_err(RAFTK_EINVAL, "%s: the workspace must be 32-byte aligned", who);
    return RAFTK_OK;
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
    if (int rc = check_wpow("general channel-stats", p.data(), n_ch)) return rc;
    return launch_general_channel_stats(n_units, n_dof, n_ch, nw, dw, w, R, wpow, Xi, sd, psd, amp, st);
}

extern "C" int raftk_general_channel_stats_host(int32_t n_units, int32_t n_dof, int32_t n_ch, int32_t nw, double dw, const double *w,
                                                const double *R, const int32_t *wpow, const double *Xi, double *sd, double *psd, double *amp)
{
    if (n_units <= 0 || n_dof <= 0 || n_ch <= 0 || nw <= 0 || !w || !R || !wpow || !Xi || !sd || !(dw > 0.0))
        return set_err(RAFTK_EINVAL, "bad general channel-stats arguments");
    if (int rc = check_wpow("general channel-stats", wpow, n_ch)) return rc;
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

// ---- channels of farm batches (raftk_farm_channel_stats_*) -----------------------------------------------------------------
static size_t farm_ch_scratch(int32_t n_farms, int32_t n_rows, int32_t nw, const raftk_farm_channels *ch)
{
    return (size_t)n_farms * n_rows * ch->n_ch * nw * sizeof(double);
}

static int farm_ch_check(int32_t n_farms, int32_t n_rows, int32_t n_dof, int32_t nw, const double *w, const double *Xi_sys,
                         const raftk_farm_channels *ch)
{
    if (!ch) return set_err(RAFTK_EINVAL, "farm channel-stats: null argument");
    if (n_farms < 1 || n_rows < 1 || n_dof < 1 || nw < 1 || ch->n_ch < 1)
        return set_err(RAFTK_EINVAL, "farm channel-stats: n_farms, n_rows, n_dof, nw and n_ch must be >= 1");
    if (ch->n_ch > RAFTK_FARM_CH_MAX) return set_err_i(RAFTK_EINVAL, "farm channel-stats: at most %d channels per call", RAFTK_FARM_CH_MAX);
    if (ch->R_shared != 0 && ch->R_shared != 1) return set_err(RAFTK_EINVAL, "farm channel-stats: R_shared must be 0 or 1");
    if (!ch->R || !Xi_sys || !ch->std) return set_err(RAFTK_EINVAL, "farm channel-stats: R, Xi_sys and std are required");
    if (!(ch->dw > 0.0)) return set_err(RAFTK_EINVAL, "farm channel-stats: dw must be > 0");
    if (int rc = check_wpow("farm channel-stats", ch->wpow, ch->n_ch)) return rc;
    const bool powers = ch->wpow && std::any_of(ch->wpow, ch->wpow + ch->n_ch, [](int32_t p) { return p != 0; });
    if (powers && !w) return set_err(RAFTK_EINVAL, "farm channel-stats: w is required when a channel has wpow 1 or 2");
    const size_t units = (size_t)n_farms * n_rows;
    if (units * nw > 2147483647u || units * ch->n_ch > 2147483647u)
        return set_err(RAFTK_EINVAL, "farm channel-stats: too many (farm, row, bin) or (farm, row, channel) rows");
    return RAFTK_OK;
}

// Bins per CTA: as many as the opt-in shared memory holds (n x 16 bytes each), fewer when the batch alone would leave SMs
// idle; 0 when not even one bin fits (Xi_sys is then read from L2).  tile_w > 0 caps it; RAFTK_FARM_TILE_L2 forces L2.
static int farm_ch_tile(int32_t n_units, int32_t n_dof, int32_t nw, int32_t tile_w)
{
    if (tile_w == RAFTK_FARM_TILE_L2) return 0;
    const int tmax = (int)std::min<size_t>((size_t)nw, smem_optin() / ((size_t)n_dof * sizeof(double2)));
    if (tmax < 1) return 0;
    if (tile_w > 0) return std::min(tmax, (int)tile_w);
    const long long want = (2LL * sm_count() + n_units - 1) / n_units;                      // tiles per (farm, row)
    const int split = (int)std::max<long long>(32, (nw + want - 1) / want);
    return std::min(tmax, split);
}

extern "C" size_t raftk_farm_channel_stats_workspace_bytes(int32_t n_farms, int32_t n_rows, int32_t nw, const raftk_farm_channels *ch)
{
    if (!ch || n_farms < 1 || n_rows < 1 || nw < 1 || ch->n_ch < 1 || ch->psd) return 0;
    return farm_ch_scratch(n_farms, n_rows, nw, ch);
}

extern "C" int raftk_farm_channel_stats_dev(int32_t n_farms, int32_t n_rows, int32_t n_dof, int32_t nw, const double *w,
                                            const double *Xi_sys, const raftk_farm_channels *ch, void *workspace,
                                            size_t workspace_bytes, void *stream)
{
    if (int rc = farm_ch_check(n_farms, n_rows, n_dof, nw, w, Xi_sys, ch)) return rc;
    if (!ch->psd && (!workspace || workspace_bytes < farm_ch_scratch(n_farms, n_rows, nw, ch)))
        return set_err(RAFTK_EINVAL, "farm channel-stats: without psd the workspace must hold |Y|^2 (raftk_farm_channel_stats_workspace_bytes)");
    const cudaStream_t st = (cudaStream_t)stream;
    const int32_t units = n_farms * n_rows;
    FarmChParams P = {};
    P.n = n_dof; P.nch = ch->n_ch; P.nw = nw; P.n_rows = n_rows;
    P.r_stride = ch->R_shared ? 0 : (size_t)ch->n_ch * n_dof;
    P.w = w; P.R = ch->R; P.Xi = reinterpret_cast<const double2 *>(Xi_sys);
    P.a2 = ch->psd ? ch->psd : static_cast<double *>(workspace);
    P.amp = reinterpret_cast<double2 *>(ch->amp);
    for (int32_t t = 0; ch->wpow && t < ch->n_ch; t++) P.wbits[t >> 4] |= (unsigned)ch->wpow[t] << ((t & 15) * 2);
    const int tile = farm_ch_tile(units, n_dof, nw, ch->tile_w);
    P.tile = tile ? tile : std::min<int32_t>(nw, 64);
    P.n_tiles = (nw + P.tile - 1) / P.tile;
    const long long grid = (long long)units * P.n_tiles;
    if (grid > 2147483647LL) return set_err(RAFTK_EINVAL, "farm channel-stats: too many (farm, row, bin tile) blocks");
    if (tile) {
        const size_t smem = (size_t)n_dof * tile * sizeof(double2);
        static SmemOptIn opt(48 * 1024);
        CUDA_TRY(opt.ensure(k_farm_channels<true>, smem));
        k_farm_channels<true><<<(unsigned)grid, FARM_CH_T, smem, st>>>(P);
    } else {
        k_farm_channels<false><<<(unsigned)grid, FARM_CH_T, 0, st>>>(P);
    }
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    k_farm_channel_reduce<<<(unsigned)(units * ch->n_ch), 128, 0, st>>>(nw, ch->dw, P.a2, ch->std, ch->psd);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RAFTK_OK;
}

extern "C" int raftk_farm_channel_stats_host(int32_t n_farms, int32_t n_rows, int32_t n_dof, int32_t nw, const double *w,
                                             const double *Xi_sys, const raftk_farm_channels *ch)
{
    if (int rc = farm_ch_check(n_farms, n_rows, n_dof, nw, w, Xi_sys, ch)) return rc;
    const size_t units = (size_t)n_farms * n_rows, rows = units * ch->n_ch, nch = ch->n_ch;
    const size_t wb = raftk_farm_channel_stats_workspace_bytes(n_farms, n_rows, nw, ch);
    raftk_farm_channels d = *ch;
    const double *dW, *dXi;
    char *ws;
    Staging S("raftk_farm_channel_stats_host");
    S.in(dW, w, nw); S.in(d.R, ch->R, (ch->R_shared ? 1 : (size_t)n_farms) * nch * n_dof); S.in(dXi, Xi_sys, units * n_dof * nw * 2);
    S.out(d.std, rows, ch->std); S.out(d.psd, ch->psd ? rows * nw : 0, ch->psd); S.out(d.amp, ch->amp ? rows * nw * 2 : 0, ch->amp);
    S.buf(ws, wb);
    int rc;
    if ((rc = S.commit()) || (rc = raftk_farm_channel_stats_dev(n_farms, n_rows, n_dof, nw, dW, dXi, &d, ws, wb, nullptr))) return rc;
    return S.finish();
}

// ---- channels of ragged farm batches (raftk_farm_ragged_channel_stats_*) ---------------------------------------------------
struct RagChPlan {
    std::vector<FarmChDesc> fd;
    int n_max = 0, n_ch = 0;
    size_t table = 0, n_r = 0, n_xi = 0;   // descriptor bytes (256-aligned); doubles of the packed R; complex elements of Xi_sys
};
static int ragch_plan(int32_t n_farms, int32_t n_rows, int32_t nw, const int32_t *farm_fowt0, const int32_t *ch0, const double *w,
                      const double *Xi_sys, const raftk_farm_channels *ch, RagChPlan &R)
{
    if (!ch || !farm_fowt0 || !ch0) return set_err(RAFTK_EINVAL, "ragged farm channel-stats: null argument");
    if (n_farms < 1 || n_rows < 1 || nw < 1) return set_err(RAFTK_EINVAL, "ragged farm channel-stats: n_farms, n_rows and nw must be >= 1");
    if (farm_fowt0[0] != 0 || ch0[0] != 0) return set_err(RAFTK_EINVAL, "ragged farm channel-stats: farm_fowt0[0] and ch0[0] must be 0");
    for (int k = 0; k < n_farms; k++)
        if (farm_fowt0[k + 1] <= farm_fowt0[k] || ch0[k + 1] <= ch0[k])
            return set_err(RAFTK_EINVAL, "ragged farm channel-stats: farm_fowt0 and ch0 must be strictly increasing (a farm without FOWTs or channels)");
    if (ch->n_ch != ch0[n_farms]) return set_err(RAFTK_EINVAL, "ragged farm channel-stats: channels.n_ch must equal ch0[n_farms]");
    if (ch->R_shared != 0) return set_err(RAFTK_EINVAL, "ragged farm channel-stats: R_shared must be 0 (R_f is per farm)");
    int nmax = 0;
    for (int k = 0; k < n_farms; k++) nmax = std::max(nmax, 6 * (farm_fowt0[k + 1] - farm_fowt0[k]));
    if (int rc = farm_ch_check(n_farms, n_rows, nmax, nw, w, Xi_sys, ch)) return rc;
    R.fd.resize(n_farms);
    size_t ro = 0;
    for (int k = 0; k < n_farms; k++) {
        FarmChDesc &e = R.fd[k];
        e.n = 6 * (farm_fowt0[k + 1] - farm_fowt0[k]); e.nch = ch0[k + 1] - ch0[k]; e.ch0 = ch0[k]; e._pad = 0;
        e.xo = (size_t)6 * n_rows * nw * farm_fowt0[k]; e.ro = ro;
        ro += (size_t)e.nch * e.n;
    }
    R.n_max = nmax; R.n_ch = ch->n_ch; R.n_r = ro; R.n_xi = (size_t)6 * n_rows * nw * farm_fowt0[n_farms];
    R.table = align_up((size_t)n_farms * sizeof(FarmChDesc), 256);
    return RAFTK_OK;
}

extern "C" size_t raftk_farm_ragged_channel_stats_workspace_bytes(int32_t n_farms, int32_t n_rows, int32_t nw, const int32_t *farm_fowt0,
                                                                  const int32_t *ch0, const raftk_farm_channels *ch)
{
    RagChPlan R;
    static const double one = 1.0;                                             // (w and Xi_sys are not read by the query)
    if (ragch_plan(n_farms, n_rows, nw, farm_fowt0, ch0, &one, &one, ch, R)) return 0;
    return R.table + (ch->psd ? 0 : (size_t)n_rows * ch->n_ch * nw * sizeof(double));
}

extern "C" int raftk_farm_ragged_channel_stats_dev(int32_t n_farms, int32_t n_rows, int32_t nw, const int32_t *farm_fowt0,
                                                   const int32_t *ch0, const double *w, const double *Xi_sys,
                                                   const raftk_farm_channels *ch, void *workspace, size_t workspace_bytes, void *stream)
{
    RagChPlan R;
    if (int rc = ragch_plan(n_farms, n_rows, nw, farm_fowt0, ch0, w, Xi_sys, ch, R)) return rc;
    const size_t scratch = ch->psd ? 0 : (size_t)n_rows * ch->n_ch * nw * sizeof(double);
    if (!workspace || workspace_bytes < R.table + scratch)
        return set_err(RAFTK_EINVAL, "ragged farm channel-stats: the workspace must hold the farm descriptors and, without psd, |Y|^2 "
                                     "(raftk_farm_ragged_channel_stats_workspace_bytes)");
    const cudaStream_t st = (cudaStream_t)stream;
    FarmChDesc *dfd = static_cast<FarmChDesc *>(workspace);
    CUDA_TRY(cudaMemcpyAsync(dfd, R.fd.data(), R.fd.size() * sizeof(FarmChDesc), cudaMemcpyHostToDevice, st));
    const int32_t units = n_farms * n_rows;
    FarmChRagParams P = {};
    P.n = R.n_max; P.nch = ch->n_ch; P.nw = nw; P.n_rows = n_rows;
    P.w = w; P.R = ch->R; P.Xi = reinterpret_cast<const double2 *>(Xi_sys);
    P.a2 = ch->psd ? ch->psd : reinterpret_cast<double *>(static_cast<char *>(workspace) + R.table);
    P.amp = reinterpret_cast<double2 *>(ch->amp);
    P.fd = dfd;
    for (int32_t t = 0; ch->wpow && t < ch->n_ch; t++) P.wbits[t >> 4] |= (unsigned)ch->wpow[t] << ((t & 15) * 2);
    const int tile = farm_ch_tile(units, R.n_max, nw, ch->tile_w);            // one tile width for every farm: the largest n's
    P.tile = tile ? tile : std::min<int32_t>(nw, 64);
    P.n_tiles = (nw + P.tile - 1) / P.tile;
    const long long grid = (long long)units * P.n_tiles;
    if (grid > 2147483647LL) return set_err(RAFTK_EINVAL, "ragged farm channel-stats: too many (farm, row, bin tile) blocks");
    if (tile) {
        const size_t smem = (size_t)R.n_max * tile * sizeof(double2);
        static SmemOptIn opt(48 * 1024);
        CUDA_TRY(opt.ensure(k_farm_channels_ragged<true>, smem));
        k_farm_channels_ragged<true><<<(unsigned)grid, FARM_CH_T, smem, st>>>(P);
    } else {
        k_farm_channels_ragged<false><<<(unsigned)grid, FARM_CH_T, 0, st>>>(P);
    }
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    // the output rows are farm after farm, [n_rows, n_ch_f] each: n_rows * n_ch rows in all, reduced as the uniform batch's
    k_farm_channel_reduce<<<(unsigned)((size_t)n_rows * ch->n_ch), 128, 0, st>>>(nw, ch->dw, P.a2, ch->std, ch->psd);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RAFTK_OK;
}

extern "C" int raftk_farm_ragged_channel_stats_host(int32_t n_farms, int32_t n_rows, int32_t nw, const int32_t *farm_fowt0,
                                                    const int32_t *ch0, const double *w, const double *Xi_sys,
                                                    const raftk_farm_channels *ch)
{
    RagChPlan R;
    if (int rc = ragch_plan(n_farms, n_rows, nw, farm_fowt0, ch0, w, Xi_sys, ch, R)) return rc;
    const size_t rows = (size_t)n_rows * ch->n_ch;
    const size_t wb = raftk_farm_ragged_channel_stats_workspace_bytes(n_farms, n_rows, nw, farm_fowt0, ch0, ch);
    raftk_farm_channels d = *ch;
    const double *dW, *dXi;
    char *ws;
    Staging S("raftk_farm_ragged_channel_stats_host");
    S.in(dW, w, nw); S.in(d.R, ch->R, R.n_r); S.in(dXi, Xi_sys, R.n_xi * 2);
    S.out(d.std, rows, ch->std); S.out(d.psd, ch->psd ? rows * nw : 0, ch->psd); S.out(d.amp, ch->amp ? rows * nw * 2 : 0, ch->amp);
    S.buf(ws, wb);
    int rc;
    if ((rc = S.commit()) || (rc = raftk_farm_ragged_channel_stats_dev(n_farms, n_rows, nw, farm_fowt0, ch0, dW, dXi, &d, ws, wb, nullptr)))
        return rc;
    return S.finish();
}

// ---- rotor speed, generator torque and blade pitch (raftk_rotor_stats_*) ---------------------------------------------------
static int rotor_check(int32_t n_units, int32_t n_rows, int32_t n_dof, int32_t nw, const double *w, const double *Xi,
                       const raftk_rotor_outputs *ro)
{
    if (!ro) return set_err(RAFTK_EINVAL, "rotor-stats: null argument");
    if (n_units < 1 || n_rows < 1 || n_dof < 1 || nw < 1 || ro->n_cases < 1 || ro->n_rot < 1 || ro->n_r < 1)
        return set_err(RAFTK_EINVAL, "rotor-stats: n_units, n_rows, n_dof, nw, n_cases, n_rot and n_r must be >= 1");
    if (ro->R_shared != 0 && ro->R_shared != 1) return set_err(RAFTK_EINVAL, "rotor-stats: R_shared must be 0 or 1");
    if (ro->tf_shared != 0 && ro->tf_shared != 1) return set_err(RAFTK_EINVAL, "rotor-stats: tf_shared must be 0 or 1");
    if (!w || !Xi || !ro->R || !ro->C || !ro->V_w || !ro->gains || !ro->std || !ro->col0 || !ro->case_row0)
        return set_err(RAFTK_EINVAL, "rotor-stats: w, Xi, R, C, V_w, gains, std, col0 and case_row0 are required");
    if (!(ro->dw > 0.0)) return set_err(RAFTK_EINVAL, "rotor-stats: dw must be > 0");
    if (ro->n_r > n_dof) return set_err(RAFTK_EINVAL, "rotor-stats: n_r must be <= n_dof");
    for (int32_t k = 0; k < ro->n_rot; k++)
        if (ro->col0[k] < 0 || ro->col0[k] > n_dof - ro->n_r)
            return set_err(RAFTK_EINVAL, "rotor-stats: every col0 must satisfy 0 <= col0 and col0 + n_r <= n_dof");
    if (int rc = check_case_rows("rotor-stats", ro->case_row0, ro->n_cases, n_rows)) return rc;
    if ((size_t)n_units * ro->n_cases * ro->n_rot > 2147483647u)
        return set_err(RAFTK_EINVAL, "rotor-stats: too many (unit, case, rotor) blocks");
    return RAFTK_OK;
}

extern "C" int raftk_rotor_stats_dev(int32_t n_units, int32_t n_rows, int32_t n_dof, int32_t nw, const double *w, const double *Xi,
                                     const raftk_rotor_outputs *ro, void *stream)
{
    if (int rc = rotor_check(n_units, n_rows, n_dof, nw, w, Xi, ro)) return rc;
    const cudaStream_t st = (cudaStream_t)stream;
    RotorParams P = {};
    P.n_rows = n_rows; P.n_dof = n_dof; P.nw = nw; P.n_r = ro->n_r;
    P.n_cases = ro->n_cases; P.n_rot = ro->n_rot;
    P.r_stride = ro->R_shared ? 0 : (size_t)ro->n_rot * ro->n_r;
    P.tf_stride = ro->tf_shared ? 0 : (size_t)ro->n_cases * ro->n_rot;
    P.dw = ro->dw;
    P.w = w; P.R = ro->R; P.gains = ro->gains;
    P.Xi = reinterpret_cast<const double2 *>(Xi);
    P.C = reinterpret_cast<const double2 *>(ro->C);
    P.Vw = reinterpret_cast<const double2 *>(ro->V_w);
    P.sd = ro->std; P.psd = ro->psd;
    // chunks of cases and rotors only bound the launch parameters: every CTA computes the same thing in any chunk
    for (int32_t c0 = 0; c0 < ro->n_cases; c0 += ROTOR_CHUNK) {
        P.c0 = c0; P.nc = std::min<int32_t>(ROTOR_CHUNK, ro->n_cases - c0);
        for (int j = 0; j <= P.nc; j++) P.row0[j] = ro->case_row0[c0 + j];
        for (int32_t k0 = 0; k0 < ro->n_rot; k0 += ROTOR_CHUNK) {
            P.k0 = k0; P.nk = std::min<int32_t>(ROTOR_CHUNK, ro->n_rot - k0);
            for (int j = 0; j < P.nk; j++) P.col0[j] = ro->col0[k0 + j];
            k_rotor_stats<<<(unsigned)((size_t)n_units * P.nc * P.nk), ROTOR_T, 0, st>>>(P);
            g_launches++;
            CUDA_TRY(cudaGetLastError());
        }
    }
    return RAFTK_OK;
}

extern "C" int raftk_rotor_stats_host(int32_t n_units, int32_t n_rows, int32_t n_dof, int32_t nw, const double *w, const double *Xi,
                                      const raftk_rotor_outputs *ro)
{
    if (int rc = rotor_check(n_units, n_rows, n_dof, nw, w, Xi, ro)) return rc;
    for (int32_t i = 0; i < nw; i++)
        if (!(w[i] > 0.0)) return set_err(RAFTK_EINVAL, "rotor-stats: every w must be > 0 (the wind row divides by w)");
    const size_t tf = (ro->tf_shared ? 1 : (size_t)n_units) * ro->n_cases * ro->n_rot;
    const size_t rows = (size_t)n_units * ro->n_cases * ro->n_rot * 3;
    raftk_rotor_outputs d = *ro;
    const double *dW, *dXi;
    Staging S("raftk_rotor_stats_host");
    S.in(dW, w, nw); S.in(dXi, Xi, (size_t)n_units * n_rows * n_dof * nw * 2);
    S.in(d.R, ro->R, (ro->R_shared ? 1 : (size_t)n_units) * ro->n_rot * ro->n_r);
    S.in(d.C, ro->C, tf * nw * 2); S.in(d.V_w, ro->V_w, tf * nw * 2); S.in(d.gains, ro->gains, tf * 4);
    S.out(d.std, rows, ro->std); S.out(d.psd, ro->psd ? rows * nw : 0, ro->psd);
    int rc;
    if ((rc = S.commit()) || (rc = raftk_rotor_stats_dev(n_units, n_rows, n_dof, nw, dW, dXi, &d, nullptr))) return rc;
    return S.finish();
}

// ---- spectral moments shared by fatigue and the stress ring: channel form, bin tiles, launches ------------------------------
// The channels of k_fatigue_moments and k_stress_moments: real rows R, one set for every unit (R_shared 1) or one per unit,
// or complex per-bin coefficients coef, one set (RAFTK_FATIGUE_COEF_SHARED), one per unit (_UNIT) or one per (unit, row)
// (_ROW); method: the DEL closed form
static int check_channel_form(const char *who, const void *R, int32_t R_shared, const void *coef, int32_t coef_mode, int32_t method)
{
    if (!R == !coef) return set_err(RAFTK_EINVAL, "%s: give exactly one of R (real rows) and coef (complex coefficients)", who);
    if (R && R_shared != 0 && R_shared != 1) return set_err(RAFTK_EINVAL, "%s: R_shared must be 0 or 1", who);
    if (coef && (coef_mode < RAFTK_FATIGUE_COEF_SHARED || coef_mode > RAFTK_FATIGUE_COEF_ROW))
        return set_err(RAFTK_EINVAL, "%s: unknown coef_mode", who);
    if (method != RAFTK_FATIGUE_DIRLIK && method != RAFTK_FATIGUE_NARROWBAND_METHOD) return set_err(RAFTK_EINVAL, "%s: unknown method", who);
    return RAFTK_OK;
}

// The strides of a checked channel form, `per` doubles of R (or coefficients per bin) for one unit: between two units' R, two
// units' and two rows' coefficients (0: shared); and the doubles of R and coef that raftk_*_host stages
struct ChannelForm { size_t r_stride, cf_ustride, cf_rstride, n_R, n_coef; };
static ChannelForm channel_form(int32_t R_shared, const void *coef, int32_t coef_mode, size_t per, int32_t n_units, int32_t n_rows,
                                int32_t nw)
{
    const size_t cf = per * nw;
    ChannelForm f;
    f.r_stride = R_shared ? 0 : per;
    f.cf_ustride = coef_mode == RAFTK_FATIGUE_COEF_UNIT ? cf : (coef_mode == RAFTK_FATIGUE_COEF_ROW ? cf * n_rows : 0);
    f.cf_rstride = coef_mode == RAFTK_FATIGUE_COEF_ROW ? cf : 0;
    f.n_R = (R_shared ? 1 : (size_t)n_units) * per;
    f.n_coef = coef ? (coef_mode == RAFTK_FATIGUE_COEF_SHARED ? 1 : (size_t)n_units) * (coef_mode == RAFTK_FATIGUE_COEF_ROW ? n_rows : 1) * cf * 2
                    : 0;
    return f;
}

static int moment_chunks(int32_t nw) { return (nw + FAT_CHUNK - 1) / FAT_CHUNK; }

// Bins per CTA of the moment kernels, whole FAT_CHUNK chunks: at most what the opt-in shared memory holds (n x 16 bytes per bin)
// and 256, fewer when the batch alone would leave SMs idle; 0 when not even one chunk fits (Xi is then read from L2).  tile_w > 0
// caps it.
static int moment_tile(size_t n_rows_total, int32_t n_dof, int32_t nw, int32_t tile_w)
{
    if (tile_w == RAFTK_FARM_TILE_L2) return 0;
    const int round_nw = moment_chunks(nw) * FAT_CHUNK;
    const int tmax = (int)std::min<size_t>((size_t)round_nw, smem_optin() / ((size_t)n_dof * sizeof(double2))) / FAT_CHUNK * FAT_CHUNK;
    if (tmax < FAT_CHUNK) return 0;
    if (tile_w > 0) return std::max(FAT_CHUNK, std::min(tmax, (int)tile_w / FAT_CHUNK * FAT_CHUNK));
    const long long want = (2LL * sm_count() + (long long)n_rows_total - 1) / (long long)n_rows_total;   // tiles per (unit, row)
    const int split = (int)((nw + want - 1) / want + FAT_CHUNK - 1) / FAT_CHUNK * FAT_CHUNK;
    return std::min(std::min(tmax, 256), std::max(FAT_CHUNK, split));
}

// Sets P's bin tiling (n_chunks, tile, n_tiles) for `rows` (unit, row) pairs and launches the moment kernel k[SMEM][COEF]: the
// Xi tile in shared memory when moment_tile gives one, else from L2.  The opt-in is per function, so each instantiation of this
// template (one per moment kernel) keeps one SmemOptIn per shared-memory kernel.
template <class Prm>
static int launch_moments(void (*const (&k)[2][2])(Prm), int threads, Prm &P, size_t rows, int32_t n_dof, int32_t nw, int32_t tile_w,
                          bool coef, cudaStream_t st)
{
    static SmemOptIn opt[2] = {SmemOptIn(48 * 1024), SmemOptIn(48 * 1024)};
    const int tile = moment_tile(rows, n_dof, nw, tile_w);
    P.n_chunks = moment_chunks(nw);
    P.tile = tile ? tile : std::min<int32_t>(P.n_chunks * FAT_CHUNK, 256);
    P.n_tiles = (nw + P.tile - 1) / P.tile;
    const unsigned grid = (unsigned)(rows * P.n_tiles);
    if (tile) {
        const size_t smem = (size_t)n_dof * tile * sizeof(double2);
        CUDA_TRY(opt[coef].ensure(k[1][coef], smem));
        k[1][coef]<<<grid, threads, smem, st>>>(P);
    } else {
        k[0][coef]<<<grid, threads, 0, st>>>(P);
    }
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RAFTK_OK;
}

// DEL_life [U, nk] from the log(p_c d_c) table wd [U, n_cases, nk] (nk channels, or (ring, angle) pairs) through
// k_fatigue_life; column k's exponent is m[k * m_stride]
static int launch_life(int32_t n_units, int32_t n_cases, int32_t nk, const double *weights, double f_eq, const double *m, int m_stride,
                       const double *wd, double *DEL_life, cudaStream_t st)
{
    FatLifeParams L = {};
    double W = 0.0;
    for (int32_t c = 0; c < n_cases; c++) W += weights ? weights[c] : 1.0;
    L.n_cases = n_cases; L.nch = nk; L.log_fw = std::log(f_eq * W); L.wd = wd; L.DEL_life = DEL_life;
    for (int32_t k0 = 0; k0 < nk; k0 += FAT_LAUNCH_CHUNK) {
        L.k0 = k0; L.nk = std::min<int32_t>(FAT_LAUNCH_CHUNK, nk - k0);
        for (int j = 0; j < L.nk; j++) L.m[j] = m[(size_t)(k0 + j) * m_stride];
        const size_t nt = (size_t)n_units * L.nk;
        k_fatigue_life<<<(unsigned)((nt + FAT_FIN_T - 1) / FAT_FIN_T), FAT_FIN_T, 0, st>>>(L, nt);
        g_launches++;
        CUDA_TRY(cudaGetLastError());
    }
    return RAFTK_OK;
}

// ---- fatigue damage-equivalent loads (raftk_fatigue_*) --------------------------------------------------------------------
static size_t fat_part_elems(int32_t n_units, int32_t n_rows, int32_t nw, int32_t n_ch)
{
    return (size_t)n_units * n_rows * moment_chunks(nw) * n_ch * 4;
}

static int fat_check(int32_t n_units, int32_t n_rows, int32_t n_dof, int32_t nw, const double *w, const double *Xi, const raftk_fatigue *fa)
{
    if (!fa) return set_err(RAFTK_EINVAL, "fatigue: null argument");
    if (n_units < 1 || n_rows < 1 || n_dof < 1 || nw < 1 || fa->n_cases < 1 || fa->n_ch < 1)
        return set_err(RAFTK_EINVAL, "fatigue: n_units, n_rows, n_dof, nw, n_cases and n_ch must be >= 1");
    if (fa->n_ch > RAFTK_FATIGUE_CH_MAX) return set_err_i(RAFTK_EINVAL, "fatigue: at most %d channels per call", RAFTK_FATIGUE_CH_MAX);
    if (int rc = check_channel_form("fatigue", fa->R, fa->R_shared, fa->coef, fa->coef_mode, fa->method)) return rc;
    if (!w || !Xi || !fa->m || !fa->case_row0 || !fa->DEL || !fa->info)
        return set_err(RAFTK_EINVAL, "fatigue: w, Xi, m, case_row0, DEL and info are required");
    if (int rc = check_wpow("fatigue", fa->R ? fa->wpow : nullptr, fa->n_ch)) return rc;
    if (int rc = check_case_rows("fatigue", fa->case_row0, fa->n_cases, n_rows)) return rc;
    for (int32_t t = 0; t < fa->n_ch; t++)
        if (!(std::isfinite(fa->m[t]) && fa->m[t] > 0.0)) return set_err(RAFTK_EINVAL, "fatigue: every m must be finite and > 0");
    if (!(std::isfinite(fa->f_eq) && fa->f_eq > 0.0)) return set_err(RAFTK_EINVAL, "fatigue: f_eq must be finite and > 0");
    if (int rc = check_weights("fatigue", fa->weights, fa->n_cases)) return rc;
    if ((size_t)n_units * n_rows * moment_chunks(nw) > 2147483647u || (size_t)n_units * fa->n_ch > 2147483647u)
        return set_err(RAFTK_EINVAL, "fatigue: too many (unit, row, bin tile) blocks");
    return RAFTK_OK;
}

static size_t fat_ws(int32_t n_units, int32_t n_rows, int32_t nw, const raftk_fatigue *fa)
{
    return (fat_part_elems(n_units, n_rows, nw, fa->n_ch) + (fa->DEL_life ? (size_t)n_units * fa->n_cases * fa->n_ch : 0)) * sizeof(double);
}

extern "C" size_t raftk_fatigue_workspace_bytes(int32_t n_units, int32_t n_rows, int32_t nw, const raftk_fatigue *fa)
{
    if (!fa || n_units < 1 || n_rows < 1 || nw < 1 || fa->n_cases < 1 || fa->n_ch < 1) return 0;
    return fat_ws(n_units, n_rows, nw, fa);
}

extern "C" int raftk_fatigue_dev(int32_t n_units, int32_t n_rows, int32_t n_dof, int32_t nw, const double *w, const double *Xi,
                                 const raftk_fatigue *fa, void *workspace, size_t workspace_bytes, void *stream)
{
    if (int rc = fat_check(n_units, n_rows, n_dof, nw, w, Xi, fa)) return rc;
    if (int rc = check_workspace("fatigue", "raftk_fatigue_workspace_bytes", workspace, workspace_bytes, fat_ws(n_units, n_rows, nw, fa)))
        return rc;
    const cudaStream_t st = (cudaStream_t)stream;
    double *part = static_cast<double *>(workspace);
    double *wd = fa->DEL_life ? part + fat_part_elems(n_units, n_rows, nw, fa->n_ch) : nullptr;
    const ChannelForm cf = channel_form(fa->R_shared, fa->coef, fa->coef_mode, (size_t)fa->n_ch * n_dof, n_units, n_rows, nw);
    FatMomParams P = {};
    P.n = n_dof; P.nch = fa->n_ch; P.nw = nw; P.n_rows = n_rows;
    P.w = w; P.R = fa->R; P.Xi = reinterpret_cast<const double2 *>(Xi); P.part = part;
    P.coef = reinterpret_cast<const double2 *>(fa->coef);
    P.r_stride = cf.r_stride; P.cf_ustride = cf.cf_ustride; P.cf_rstride = cf.cf_rstride;
    for (int32_t t = 0; fa->R && fa->wpow && t < fa->n_ch; t++) P.wbits[t >> 4] |= (unsigned)fa->wpow[t] << ((t & 15) * 2);
    static void (*const mom[2][2])(FatMomParams) = {{k_fatigue_moments<false, false>, k_fatigue_moments<false, true>},
                                                    {k_fatigue_moments<true, false>, k_fatigue_moments<true, true>}};
    if (int rc = launch_moments(mom, FAT_T, P, (size_t)n_units * n_rows, n_dof, nw, fa->tile_w, fa->coef != nullptr, st)) return rc;
    // chunks of cases and channels only bound the launch parameters: every thread computes the same thing in any chunk
    FatFinParams F = {};
    F.n_rows = n_rows; F.n_cases = fa->n_cases; F.nch = fa->n_ch; F.n_chunks = P.n_chunks; F.method = fa->method;
    F.f_eq = fa->f_eq; F.part = part; F.moments = fa->moments; F.DEL = fa->DEL; F.wd = wd; F.info = fa->info;
    for (int32_t c0 = 0; c0 < fa->n_cases; c0 += FAT_LAUNCH_CHUNK) {
        F.c0 = c0; F.nc = std::min<int32_t>(FAT_LAUNCH_CHUNK, fa->n_cases - c0);
        for (int j = 0; j <= F.nc; j++) F.row0[j] = fa->case_row0[c0 + j];
        for (int j = 0; j < F.nc; j++) F.p[j] = fa->weights ? fa->weights[c0 + j] : 1.0;
        for (int32_t k0 = 0; k0 < fa->n_ch; k0 += FAT_LAUNCH_CHUNK) {
            F.k0 = k0; F.nk = std::min<int32_t>(FAT_LAUNCH_CHUNK, fa->n_ch - k0);
            for (int j = 0; j < F.nk; j++) F.m[j] = fa->m[k0 + j];
            const size_t nt = (size_t)n_units * F.nc * F.nk;
            k_fatigue_finish<<<(unsigned)((nt + FAT_FIN_T - 1) / FAT_FIN_T), FAT_FIN_T, 0, st>>>(F, nt);
            g_launches++;
            CUDA_TRY(cudaGetLastError());
        }
    }
    return fa->DEL_life ? launch_life(n_units, fa->n_cases, fa->n_ch, fa->weights, fa->f_eq, fa->m, 1, wd, fa->DEL_life, st) : RAFTK_OK;
}

extern "C" int raftk_fatigue_host(int32_t n_units, int32_t n_rows, int32_t n_dof, int32_t nw, const double *w, const double *Xi,
                                  const raftk_fatigue *fa)
{
    if (int rc = fat_check(n_units, n_rows, n_dof, nw, w, Xi, fa)) return rc;
    const size_t out = (size_t)n_units * fa->n_cases * fa->n_ch, nch = fa->n_ch;
    const size_t wb = fat_ws(n_units, n_rows, nw, fa);
    const ChannelForm cf = channel_form(fa->R_shared, fa->coef, fa->coef_mode, nch * n_dof, n_units, n_rows, nw);
    raftk_fatigue d = *fa;
    const double *dW, *dXi;
    char *ws;
    Staging S("raftk_fatigue_host");
    S.in(dW, w, nw); S.in(dXi, Xi, (size_t)n_units * n_rows * n_dof * nw * 2);
    S.in(d.R, fa->R, cf.n_R); S.in(d.coef, fa->coef, cf.n_coef);
    S.out(d.moments, fa->moments ? out * 4 : 0, fa->moments); S.out(d.DEL, out, fa->DEL); S.out(d.info, out, fa->info);
    S.out(d.DEL_life, fa->DEL_life ? (size_t)n_units * nch : 0, fa->DEL_life);
    S.buf(ws, wb);
    int rc;
    if ((rc = S.commit()) || (rc = raftk_fatigue_dev(n_units, n_rows, n_dof, nw, dW, dXi, &d, ws, wb, nullptr))) return rc;
    return S.finish();
}

// ---- tower-base axial stress around the circumference (raftk_stress_ring_*) -------------------------------------------------
static size_t str_part_elems(int32_t n_units, int32_t n_rows, int32_t nw, int32_t n_rings)
{
    return (size_t)n_units * n_rows * moment_chunks(nw) * n_rings * STR_NS;
}

static size_t str_ws(int32_t n_units, int32_t n_rows, int32_t nw, const raftk_stress_ring *sr)
{
    return (str_part_elems(n_units, n_rows, nw, sr->n_rings)
            + (sr->DEL_life ? (size_t)n_units * sr->n_cases * sr->n_rings * sr->n_angles : 0)) * sizeof(double);
}

static int str_check(int32_t n_units, int32_t n_rows, int32_t n_dof, int32_t nw, const double *w, const double *Xi, const raftk_stress_ring *sr)
{
    if (!sr) return set_err(RAFTK_EINVAL, "stress ring: null argument");
    if (n_units < 1 || n_rows < 1 || n_dof < 1 || nw < 1 || sr->n_cases < 1 || sr->n_rings < 1 || sr->n_r < 1 || sr->n_angles < 1)
        return set_err(RAFTK_EINVAL, "stress ring: n_units, n_rows, n_dof, nw, n_cases, n_rings, n_r and n_angles must be >= 1");
    if (sr->n_ch != 1 && sr->n_ch != 2) return set_err(RAFTK_EINVAL, "stress ring: n_ch must be 1 (fore-aft) or 2 (fore-aft, side-side)");
    if (sr->n_rings > RAFTK_STRESS_RING_MAX) return set_err_i(RAFTK_EINVAL, "stress ring: at most %d rings per call", RAFTK_STRESS_RING_MAX);
    if (sr->n_angles > RAFTK_STRESS_ANGLE_MAX) return set_err_i(RAFTK_EINVAL, "stress ring: at most %d angles per call", RAFTK_STRESS_ANGLE_MAX);
    if (sr->n_r > n_dof) return set_err(RAFTK_EINVAL, "stress ring: n_r must not exceed n_dof");
    for (int32_t k = 0; sr->col0 && k < sr->n_rings; k++)
        if (sr->col0[k] < 0 || sr->col0[k] > n_dof - sr->n_r) return set_err_i(RAFTK_EINVAL, "stress ring: col0 of ring %d outside [0, n_dof - n_r]", k);
    if (int rc = check_channel_form("stress ring", sr->R, sr->R_shared, sr->coef, sr->coef_mode, sr->method)) return rc;
    if (!w || !Xi || !sr->angles || !sr->case_row0 || !sr->std || !sr->avg || !sr->max || !sr->min)
        return set_err(RAFTK_EINVAL, "stress ring: w, Xi, angles, case_row0, std, avg, max and min are required");
    if (int rc = check_wpow("stress ring", sr->R ? sr->wpow : nullptr, sr->n_rings * sr->n_ch)) return rc;
    for (int32_t a = 0; a < sr->n_angles; a++)
        if (!std::isfinite(sr->angles[a])) return set_err(RAFTK_EINVAL, "stress ring: every angle must be finite");
    if (!(std::isfinite(sr->d) && sr->d > 0.0) || !(std::isfinite(sr->t) && sr->t > 0.0))
        return set_err(RAFTK_EINVAL, "stress ring: d and t must be finite and > 0");
    if (!(sr->m == 0.0 || (std::isfinite(sr->m) && sr->m > 0.0))) return set_err(RAFTK_EINVAL, "stress ring: m must be 0 (no DEL) or finite and > 0");
    if (sr->m > 0.0 && (!sr->DEL || !sr->info)) return set_err(RAFTK_EINVAL, "stress ring: DEL and info are required with m > 0");
    if (sr->DEL_life && !(sr->m > 0.0)) return set_err(RAFTK_EINVAL, "stress ring: DEL_life needs m > 0");
    if (sr->hot_life && !sr->DEL_life) return set_err(RAFTK_EINVAL, "stress ring: hot_life needs DEL_life");
    if (sr->psd && !(std::isfinite(sr->dw) && sr->dw > 0.0)) return set_err(RAFTK_EINVAL, "stress ring: psd needs a finite dw > 0");
    if (!(std::isfinite(sr->f_eq) && sr->f_eq > 0.0)) return set_err(RAFTK_EINVAL, "stress ring: f_eq must be finite and > 0");
    if (int rc = check_case_rows("stress ring", sr->case_row0, sr->n_cases, n_rows)) return rc;
    if (int rc = check_weights("stress ring", sr->weights, sr->n_cases)) return rc;
    if ((size_t)n_units * n_rows * moment_chunks(nw) > 2147483647u || (size_t)n_units * sr->n_rings * sr->n_angles > 2147483647u)
        return set_err(RAFTK_EINVAL, "stress ring: too many (unit, row, bin tile) blocks");
    return RAFTK_OK;
}

extern "C" size_t raftk_stress_ring_workspace_bytes(int32_t n_units, int32_t n_rows, int32_t nw, const raftk_stress_ring *sr)
{
    if (!sr || n_units < 1 || n_rows < 1 || nw < 1 || sr->n_cases < 1 || sr->n_rings < 1 || sr->n_angles < 1) return 0;
    return str_ws(n_units, n_rows, nw, sr);
}

extern "C" int raftk_stress_ring_dev(int32_t n_units, int32_t n_rows, int32_t n_dof, int32_t nw, const double *w, const double *Xi,
                                     const raftk_stress_ring *sr, void *workspace, size_t workspace_bytes, void *stream)
{
    if (int rc = str_check(n_units, n_rows, n_dof, nw, w, Xi, sr)) return rc;
    if (int rc = check_workspace("stress ring", "raftk_stress_ring_workspace_bytes", workspace, workspace_bytes, str_ws(n_units, n_rows, nw, sr)))
        return rc;
    const cudaStream_t st = (cudaStream_t)stream;
    double *part = static_cast<double *>(workspace);
    double *wd = sr->DEL_life ? part + str_part_elems(n_units, n_rows, nw, sr->n_rings) : nullptr;
    const ChannelForm cf = channel_form(sr->R_shared, sr->coef, sr->coef_mode, (size_t)sr->n_rings * sr->n_ch * sr->n_r, n_units, n_rows, nw);
    StrParams P = {};
    P.n = n_dof; P.n_r = sr->n_r; P.nw = nw; P.n_rows = n_rows; P.n_rings = sr->n_rings; P.n_ch = sr->n_ch;
    P.w = w; P.R = sr->R; P.Xi = reinterpret_cast<const double2 *>(Xi); P.part = part;
    P.coef = reinterpret_cast<const double2 *>(sr->coef);
    P.r_stride = cf.r_stride; P.cf_ustride = cf.cf_ustride; P.cf_rstride = cf.cf_rstride;
    for (int32_t k = 0; k < sr->n_rings; k++) P.col0[k] = sr->col0 ? sr->col0[k] : 0;
    for (int32_t t = 0; sr->R && sr->wpow && t < sr->n_rings * sr->n_ch; t++) {
        const int k = t / sr->n_ch, j = t - k * sr->n_ch;
        P.wbits[k >> 3] |= (unsigned)sr->wpow[t] << ((k & 7) * 4 + 2 * j);
    }
    const double Izz = 3.141592653589793 / 8.0 * sr->t * sr->d * sr->d * sr->d;
    P.c = 0.5 * sr->d / Izz / 1e6; P.c2 = P.c * P.c;
    P.n_cases = sr->n_cases; P.n_angles = sr->n_angles; P.method = sr->method;
    P.f_eq = sr->f_eq; P.m = sr->m; P.dw = sr->dw; P.mean = sr->mean;
    P.std = sr->std; P.avg = sr->avg; P.mx = sr->max; P.mn = sr->min; P.DEL = sr->DEL; P.info = sr->info; P.wd = wd;
    P.psd = sr->psd;
    for (int32_t a = 0; a < sr->n_angles; a++) P.angle[a] = sr->angles[a];
    const bool coef = sr->coef != nullptr;
    static void (*const mom[2][2])(StrParams) = {{k_stress_moments<false, false>, k_stress_moments<false, true>},
                                                 {k_stress_moments<true, false>, k_stress_moments<true, true>}};
    if (int rc = launch_moments(mom, STR_T, P, (size_t)n_units * n_rows, n_dof, nw, sr->tile_w, coef, st)) return rc;
    // chunks of cases only bound the launch parameters: every thread computes the same thing in any chunk
    for (int32_t c0 = 0; c0 < sr->n_cases; c0 += STR_LAUNCH_CASES) {
        P.c0 = c0; P.nc = std::min<int32_t>(STR_LAUNCH_CASES, sr->n_cases - c0);
        for (int j = 0; j <= P.nc; j++) P.row0[j] = sr->case_row0[c0 + j];
        for (int j = 0; j < P.nc; j++) P.p[j] = sr->weights ? sr->weights[c0 + j] : 1.0;
        const size_t nt = (size_t)n_units * P.nc * sr->n_rings * sr->n_angles;
        k_stress_finish<<<(unsigned)((nt + STR_FIN_T - 1) / STR_FIN_T), STR_FIN_T, 0, st>>>(P, nt);
        g_launches++;
        CUDA_TRY(cudaGetLastError());
        if (sr->hot) {
            P.hot = sr->hot;
            const size_t nh = (size_t)n_units * P.nc * sr->n_rings;
            k_stress_hot<<<(unsigned)((nh + STR_FIN_T - 1) / STR_FIN_T), STR_FIN_T, 0, st>>>(P, nh);
            g_launches++;
            CUDA_TRY(cudaGetLastError());
        }
        if (sr->psd) {
            const size_t np_ = (size_t)n_units * P.nc * sr->n_rings * nw;
            const unsigned gp = (unsigned)((np_ + STR_FIN_T - 1) / STR_FIN_T);
            if (coef) k_stress_psd<true><<<gp, STR_FIN_T, 0, st>>>(P, np_);
            else k_stress_psd<false><<<gp, STR_FIN_T, 0, st>>>(P, np_);
            g_launches++;
            CUDA_TRY(cudaGetLastError());
        }
    }
    if (sr->DEL_life) {
        // per (ring, angle) the lifetime sum of k_fatigue_life, the (ring, angle) pairs taking the place of its channels
        if (int rc = launch_life(n_units, sr->n_cases, sr->n_rings * sr->n_angles, sr->weights, sr->f_eq, &sr->m, 0, wd, sr->DEL_life, st))
            return rc;
        if (sr->hot_life) {
            P.hot = sr->hot_life;
            const size_t nh = (size_t)n_units * sr->n_rings;
            k_stress_hot_life<<<(unsigned)((nh + STR_FIN_T - 1) / STR_FIN_T), STR_FIN_T, 0, st>>>(P, sr->DEL_life, nh);
            g_launches++;
            CUDA_TRY(cudaGetLastError());
        }
    }
    return RAFTK_OK;
}

extern "C" int raftk_stress_ring_host(int32_t n_units, int32_t n_rows, int32_t n_dof, int32_t nw, const double *w, const double *Xi,
                                      const raftk_stress_ring *sr)
{
    if (int rc = str_check(n_units, n_rows, n_dof, nw, w, Xi, sr)) return rc;
    const size_t ring = (size_t)sr->n_rings, na = sr->n_angles;
    const size_t out = (size_t)n_units * sr->n_cases * ring * na, ucr = (size_t)n_units * sr->n_cases * ring;
    const size_t wb = str_ws(n_units, n_rows, nw, sr);
    const ChannelForm cf = channel_form(sr->R_shared, sr->coef, sr->coef_mode, ring * sr->n_ch * sr->n_r, n_units, n_rows, nw);
    raftk_stress_ring d = *sr;
    const double *dW, *dXi;
    char *ws;
    Staging S("raftk_stress_ring_host");
    S.in(dW, w, nw); S.in(dXi, Xi, (size_t)n_units * n_rows * n_dof * nw * 2);
    S.in(d.R, sr->R, cf.n_R); S.in(d.coef, sr->coef, cf.n_coef);
    S.in(d.mean, sr->mean, ucr * sr->n_ch);
    S.out(d.std, out, sr->std); S.out(d.avg, out, sr->avg); S.out(d.max, out, sr->max); S.out(d.min, out, sr->min);
    S.out(d.DEL, sr->DEL ? out : 0, sr->DEL); S.out(d.info, sr->info ? out : 0, sr->info);
    S.out(d.hot, sr->hot ? ucr * 6 : 0, sr->hot);
    S.out(d.DEL_life, sr->DEL_life ? (size_t)n_units * ring * na : 0, sr->DEL_life);
    S.out(d.hot_life, sr->hot_life ? (size_t)n_units * ring * 2 : 0, sr->hot_life);
    S.out(d.psd, sr->psd ? out * nw : 0, sr->psd);
    S.buf(ws, wb);
    int rc;
    if ((rc = S.commit()) || (rc = raftk_stress_ring_dev(n_units, n_rows, n_dof, nw, dW, dXi, &d, ws, wb, nullptr))) return rc;
    return S.finish();
}

// ---- natural frequencies and mode shapes (raftk_eigen_*) ------------------------------------------------------------------
// Which kernel takes n, its dynamic shared memory, its workspace slab and how many of its CTAs an SM holds.  kernel 0: n too
// large for the per-system vectors in shared memory.  Without a device the rule answers for an H100.
struct EigPlan { int kernel = 0, per_sm = 0; size_t smem = 0, slab = 0; };
static EigPlan eig_plan(int n)
{
    EigPlan p;
    const size_t mat = (size_t)n * eig_ld(n) * sizeof(double);
    if (n <= EIG_SMALL_NMAX) {
        p.kernel = RAFTK_KERNEL_EIG_SMALL;
        p.smem = EIG_SMALL_T * (3 * mat + eig_vec_doubles(n) * sizeof(double) + eig_vec_ints(n) * sizeof(int));
        return p;
    }
    const size_t vec = ((size_t)eig_vec_doubles(n) + (eig_vec_ints(n) + 1) / 2) * sizeof(double), optin = smem_optin();
    if (vec + mat <= optin) { p.kernel = RAFTK_KERNEL_EIG_CTA_SMEM; p.smem = vec + mat; p.slab = align_up(2 * mat, 256); }
    else if (vec <= optin) { p.kernel = RAFTK_KERNEL_EIG_CTA_SLAB; p.smem = vec; p.slab = align_up(3 * mat, 256); }
    else return p;
    p.per_sm = (int)std::max<size_t>(1, std::min<size_t>(2048 / EIG_CTA_T, smem_per_sm() / (p.smem + 1024)));
    return p;
}
static long long eig_ctas(const raftk_eigen *e, const EigPlan &p) { return std::min<long long>(e->n_systems, (long long)p.per_sm * sm_count()); }

static int eig_check(const raftk_eigen *e)
{
    if (!e) return set_err(RAFTK_EINVAL, "eigen: null argument");
    if (e->n < 1 || e->n_systems < 1) return set_err(RAFTK_EINVAL, "eigen: n and n_systems must be >= 1");
    if (e->sort != RAFTK_EIG_SORT_DOF && e->sort != RAFTK_EIG_SORT_ASCENDING)
        return set_err(RAFTK_EINVAL, "eigen: sort must be RAFTK_EIG_SORT_DOF or RAFTK_EIG_SORT_ASCENDING");
    if (!e->M || !e->C || !e->lam || !e->info) return set_err(RAFTK_EINVAL, "eigen: M, C, lam and info are required");
    if (!eig_plan(e->n).kernel) return set_err(RAFTK_EINVAL, "eigen: n too large for the per-system vectors in shared memory");
    return RAFTK_OK;
}

extern "C" size_t raftk_eigen_workspace_bytes(const raftk_eigen *e)
{
    if (!e || e->n < 1 || e->n_systems < 1) return 0;
    const EigPlan p = eig_plan(e->n);
    if (p.kernel == 0 || p.kernel == RAFTK_KERNEL_EIG_SMALL) return 0;
    return (size_t)eig_ctas(e, p) * p.slab;
}

extern "C" int raftk_eigen_dev(const raftk_eigen *e, void *workspace, size_t workspace_bytes, void *stream)
{
    disp_reset();
    int rc = eig_check(e);
    if (rc) return rc;
    const EigPlan p = eig_plan(e->n);
    const cudaStream_t st = (cudaStream_t)stream;
    if (p.kernel == RAFTK_KERNEL_EIG_SMALL) {
        static SmemOptIn opt(48 * 1024);
        CUDA_TRY(opt.ensure(k_eig_small, p.smem));
        k_eig_small<<<(e->n_systems + EIG_SMALL_T - 1) / EIG_SMALL_T, EIG_SMALL_T, p.smem, st>>>(*e);
        g_launches++;
        disp_launch(RAFTK_FAMILY_EIGEN, p.kernel, EIG_SMALL_T);
        CUDA_TRY(cudaGetLastError());
        return RAFTK_OK;
    }
    const long long slabs = workspace ? (long long)(workspace_bytes / p.slab) : 0;
    if (slabs < 1) return set_err(RAFTK_EINVAL, "eigen: the workspace holds less than one slab (raftk_eigen_workspace_bytes)");
    const int grid = (int)std::min<long long>(slabs, eig_ctas(e, p));
    double *ws = static_cast<double *>(workspace);
    const size_t slab_doubles = p.slab / sizeof(double);
    if (p.kernel == RAFTK_KERNEL_EIG_CTA_SMEM) {
        static SmemOptIn opt(48 * 1024);
        CUDA_TRY(opt.ensure(k_eig_cta<true>, p.smem));
        k_eig_cta<true><<<grid, EIG_CTA_T, p.smem, st>>>(*e, ws, slab_doubles);
    } else {
        static SmemOptIn opt(48 * 1024);
        CUDA_TRY(opt.ensure(k_eig_cta<false>, p.smem));
        k_eig_cta<false><<<grid, EIG_CTA_T, p.smem, st>>>(*e, ws, slab_doubles);
    }
    g_launches++;
    disp_launch(RAFTK_FAMILY_EIGEN, p.kernel, EIG_CTA_T);
    CUDA_TRY(cudaGetLastError());
    return RAFTK_OK;
}

extern "C" int raftk_eigen_host(const raftk_eigen *e)
{
    disp_reset();
    int rc = eig_check(e);
    if (rc) return rc;
    const size_t nS = e->n_systems, n = e->n, wb = raftk_eigen_workspace_bytes(e);
    raftk_eigen d = *e;
    char *ws;
    Staging S("raftk_eigen_host");
    S.in(d.M, e->M, nS * n * n); S.in(d.C, e->C, nS * n * n);
    S.out(d.lam, nS * n * 2, e->lam); S.out(d.modes, e->modes ? nS * n * n * 2 : 0, e->modes); S.out(d.info, nS, e->info);
    S.buf(ws, wb);
    if ((rc = S.commit()) || (rc = raftk_eigen_dev(&d, ws, wb, nullptr))) return rc;
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
