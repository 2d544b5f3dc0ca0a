/*
 * raftk.h -- C ABI of the H100-native RAO-solve hot path (libraftk.so, sm_90a).
 *
 * The reference (WISDEM/RAFT) has no FFI: its boundary for this path is Python-method level.
 * Every entry point below therefore cites the reference method(s) it replaces
 * (paths relative to /root/reference/raft/).  INTEGRATION.md shows the ctypes stub a RAFT
 * maintainer would add at those call sites.
 *
 * Conventions
 *   - plain C: pointers + sizes, no C++/torch types; all entry points return 0 on success or a
 *     negative RAFTK_E* code, never throw; raftk_last_error() gives the message (thread-local).
 *   - all floating point is IEEE float64; complex128 is interleaved (re, im) pairs.
 *   - array layouts follow the reference's NumPy arrays (frequency is the fastest axis), so a
 *     live RAFT array can be passed without a transpose.
 *   - *_dev entry points take DEVICE pointers and a cudaStream_t (as void*); they allocate
 *     nothing: the caller owns a workspace sized by raftk_workspace_bytes().  They are
 *     asynchronous w.r.t. the host and re-entrant per stream.
 *   - *_host entry points take HOST pointers, stage through an internal device arena
 *     (one per device, grown on demand, shared by every *_host call), and are synchronous.
 *
 * Scope: rigid 6-DOF FOWTs, strip-theory members (+ optional BEM tables, + optional external QTF or slender-body QTF for
 * second-order difference-frequency forces), one wave train drives the drag linearisation (raft_fowt.py:1910); coupled
 * farms (6N DOF); FOWTs with generalised degrees of freedom (flexible members) through raftk_general_*; the multi-GPU
 * exchange of the responses fused into the solve (raftk_peers).  See DESIGN.md for what is out of scope.
 */
#ifndef RAFTK_H
#define RAFTK_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RAFTK_VERSION 132 /* 0.1.3.2: + raftk_last_dispatch (which kernel variant the last call launched) */

enum {
    RAFTK_OK = 0,
    RAFTK_EINVAL = -1,    /* bad argument / unsupported size            */
    RAFTK_ECUDA = -2,     /* CUDA runtime error (see raftk_last_error)  */
    RAFTK_ENOMEM = -3,    /* workspace too small / allocation failed    */
    RAFTK_ESPECTRUM = -4  /* unknown wave spectrum id (ValueError at raft_fowt.py:1774) */
};

/* wave_spectrum ids (raft_fowt.py:1761-1772) */
enum { RAFTK_SPEC_JONSWAP = 0, RAFTK_SPEC_UNIT = 1, RAFTK_SPEC_CONSTANT = 2, RAFTK_SPEC_NONE = 3 };

/* status word per (design, case): int32[4] = {passes, converged, flags, reserved} */
enum { RAFTK_FLAG_NAN = 1, RAFTK_FLAG_SINGULAR = 2, RAFTK_FLAG_PLAN = 4 /* step-class tables overflowed the hint */,
       RAFTK_FLAG_XCHG = 8 /* the fused solver's exchange between a unit's CTAs timed out: the unit's results are invalid */ };

/*
 * A batch of nD FOWT designs that share one frequency grid (w, k), water depth and density.
 * Member / node tables are concatenated over designs (CSR offsets).  Only submerged strip
 * nodes (r_z < 0; raft_member.py:1935,1979,2058) are listed.  Replaces the per-object state
 * the reference keeps in Member (raft_member.py:258-309, 368-377) and FOWT (raft_fowt.py:
 * 1045-1047 sums).  All coefficient columns are iteration invariant.
 */
typedef struct raftk_designs {
    int32_t n_designs;          /* nD                                                          */
    int32_t nw;                 /* frequency bins                                              */
    int32_t n_members_total;    /* sum of members with >= 1 submerged node                     */
    int32_t n_nodes_total;      /* sum of submerged strip nodes (NsTot)                        */
    int32_t max_nodes;          /* max submerged nodes of any one design (table stride)        */
    int32_t max_members;        /* max members of any one design                               */
    int32_t max_w_classes;      /* hints for the fused solver's on-chip tables: max number of distinct     */
    int32_t max_h_classes;      /* (q_x,q_y)*step resp. q_z*step node spacings of any design; 0 = worst case */
    int32_t max_z_classes;      /* max distinct first-node depths z0 of any design's members; 0 = worst case   */
    int32_t walk_exact;         /* 1: the fused solvers' node walk is exact for every member on this grid: no deep-water
                                   bin with k |z0| > 700 and no finite-depth bin with k (z0 - z_min) > 10 (DESIGN.md
                                   section 4; raft_b200.solver.fused_walk_exact); 0 = not, or not known: the v1 solver runs */
    double depth, rho, g, dw;   /* site (raft_fowt.py:167-173); dw = w[1]-w[0]                  */
    const double *w;            /* [nw] rad/s           raft_model.py:57                       */
    const double *k;            /* [nw] wave numbers    raft_fowt.py:170 (helpers.py:377)      */
    const int32_t *member_offset; /* [nD+1] into member arrays                                 */
    /* member table [n_members_total] */
    const double *mem_frame;    /* [.,9]  q, p1, p2 unit vectors   raft_member.py:368-372      */
    const double *mem_rA;       /* [.,3]  global position of end A (wave phase / depth)        */
    const double *mem_arm;      /* [.,3]  rA - reference point of the reduced DOFs (lever arm) */
    const int32_t *mem_node_start; /* [.+1] first node of each member in the node arrays       */
    const int32_t *mem_circ;    /* [.]    1 circular, 0 rectangular  raft_member.py:2033       */
    /* node table [n_nodes_total]; node position = rA + ls*q (raft_member.py:360-362) */
    const double *node_ls;      /* distance along the member axis                              */
    const double *node_cd_q;    /* sqrt(8/pi)*rho/2*(a_q*Cd_q + a_End*Cd_End)  member:2093,2110 */
    const double *node_cd_p1;   /* sqrt(8/pi)*rho/2*a_p1*Cd_p1                member:2094       */
    const double *node_cd_p2;   /* sqrt(8/pi)*rho/2*a_p2*Cd_p2                member:2095       */
    const double *node_in_q;    /* Imat = in_q qq' + in_p1 p1p1' + in_p2 p2p2' member:1423,1442 */
    const double *node_in_p1;
    const double *node_in_p2;
    const double *node_pa;      /* rho*g*a_i (signed end area)                 member:1343,1988 */
    /* optional MacCamy-Fuchs tables: complex [n_nodes_total,nw] transverse inertia coefficients that
       replace in_p1/in_p2 (Imat_MCF, raft_member.py:1415-1420,1446,1984-1985); both or neither NULL */
    const double *node_in_p1_w;
    const double *node_in_p2_w;
    /* system matrices, row-major 6x6 per design (raft_model.py:1045-1047) */
    const double *M0;           /* [nD,36] M_struc + A_hydro_morison (+ M_moor + A_moor)        */
    const double *B0;           /* [nD,36] B_struc + sum B_gyro (+ B_moor)                      */
    const double *C0;           /* [nD,36] C_struc + C_hydro + C_moor + C_elast                 */
    const double *A_w;          /* [nD,36,nw] A_BEM + sum A_aero, or NULL                       */
    const double *B_w;          /* [nD,36,nw] B_BEM + sum B_aero, or NULL                       */
    /* BEM excitation (raft_fowt.py:1796-1849), or n_bem_head = 0 */
    int32_t n_bem_head;
    int32_t _pad0;
    const double *bem_headings; /* [n_bem_head] deg, ascending (shared by all designs)          */
    const double *X_BEM;        /* complex [nD, n_bem_head, 6, nw]                              */
    const double *bem_xyh;      /* [nD,3] x_ref, y_ref, heading_adjust(deg)                     */
    /* external difference-frequency QTF (potSecOrder 2: the state FOWT.readQTF leaves behind,
       raft_fowt.py:2081-2128), or n_qtf_w = 0 */
    int32_t n_qtf_w;            /* QTF frequencies (w1_2nd == w2_2nd, raft_fowt.py:2105-2110)   */
    int32_t n_qtf_head;         /* unidirectional QTF headings (heads_2nd)                      */
    int32_t qtf_shared;         /* 0: one table per design; 1: ONE table used by every design (no design axis);
                                   2: one table per (design, case) -- the slender-body QTF depends on the body motions */
    int32_t _pad2;
    const double *qtf_w;        /* [n_qtf_w] rad/s, ascending                                   */
    const double *qtf_heads;    /* [n_qtf_head] rad, ascending                                  */
    const double *qtf;          /* complex [nD or 1 or nD*nC, n_qtf_w, n_qtf_w, n_qtf_head, 6]: fowt.qtf, dimensional,
                                   Hermitian-filled (raft_fowt.py:2112-2128)                     */
    /* inertial wave excitation of submerged rotors (MHK turbines, hub below the waterline; raft_fowt.py:1859-1888), or
       max_rotors = 0.  Rotor r of design d adds G ud(r3) to F_iner, ud = i w u the wave acceleration of getWaveKin at its hub
       (helpers.py:188-236), G = T_node^T ([I3; H(r3 - r6)] I[:3,:3] + [0; I[3:,:3]]) with I = rotateMatrix6(I_hydro, R_q) and
       T_node the hub node's 6 rows of fowt.T (raft_b200.packer.pack_rotor_excitation).  As in the reference, only the last
       wave train of a case gets the term: a row of the case table when it ends its group of cases.primary (every row without
       primary), so the groups must be contiguous with their primary first (*_host entries refuse other maps).  The rotor's added mass is the caller's, in M0 (the reference has it in A_hydro_morison).  *_host entries
       check rot_count in [0, max_rotors], r3[2] < 0 and a finite G; *_dev entries the counts and pointers only. */
    int32_t max_rotors;         /* table stride: the most rotors of any design                  */
    int32_t _pad3;
    const int32_t *rot_count;   /* [nD] submerged rotors of each design                         */
    const double *rot_r3;       /* [nD, max_rotors, 3] global hub positions (x_ref, y_ref included) */
    const double *rot_G;        /* [nD, max_rotors, 6, 3] row-major                              */
} raftk_designs;

/* Load cases, shared by all designs: units of work are (design, case) pairs.
 * First wave train of each RAFT case (raft_fowt.py:1742-1774). */
typedef struct raftk_cases {
    int32_t n_cases;
    int32_t _pad0;
    const double *Hs;        /* [nC] wave_height                                                */
    const double *Tp;        /* [nC] wave_period                                                */
    const double *gamma;     /* [nC] wave_gamma (0 -> IEC auto, helpers.py:733-740)             */
    const double *beta_deg;  /* [nC] wave_heading [deg]                                         */
    const int32_t *spec;     /* [nC] RAFTK_SPEC_*                                               */
    const double *zeta;      /* optional [nC,nw] explicit amplitudes (overrides spec) or NULL   */
    const int32_t *primary;  /* optional [nC]: wave trains of one RAFT case (raft_fowt.py:1742-1752).  primary[c] == c:
                                the case drives its own drag linearisation; primary[c] = p != c: secondary train --
                                its response uses the impedance and per-node drag coefficients of case p
                                (raft_model.py:1200-1236; p must be a primary).  NULL: all cases independent.
                                raftk_solve_dynamics_* (needs raftk_solve_workspace_bytes() of workspace) and
                                raftk_general_solve_dynamics_*. */
    const double *F_2nd;     /* optional real [nD,nC,6,nw]: second-order force amplitudes (fowt.Fhydro_2nd, from
                                raftk_second_order_force_*) added to the linear excitation F_BEM + F_iner of every
                                unit (raft_model.py:1048, :1212).  NULL: none, or computed by the solve (see below). */
    const double *Xi_init;   /* optional complex [nD,nC,6,nw]: start the fixed-point loop from this iterate instead of the
                                constant opts.xi_start (the loop that continues after the slender-body QTF has been
                                added, raft_model.py:1106-1131).  Fused solver only. */
    const int32_t *op;       /* optional [nC]: operating point of every case (calcTurbineConstants(case), raft_fowt.py:1514-1586);
                                NULL: none.  A secondary train must name its primary's operating point.  Unit (d, c) solves with
                                M0 + (A_w + op_A_w[op[c]]) and B0 + B_drag + (B_w + op_B_w[op[c]]) (the design's and the operating
                                point's tables summed first; a design without A_w takes the operating point's alone), so a call
                                equals one call per operating point with that point's tables summed into A_w / B_w, bit for bit.
                                Honoured by raftk_solve_dynamics_*, the farm entries, raftk_solve_dynamics_slender_* and every
                                raftk_general_* solve (there the tables are given on the support of raftk_general_fd: see below);
                                ignored by the entries that assemble no impedance (excitation, linearisation, second-order force).
                                The *_host entries refuse an index outside [0, n_op) and a secondary train whose point differs from
                                its primary's; the rigid and farm *_dev entries check n_op, op_shared and the tables but do not read
                                op back (no host synchronisation): its values must be valid.  The raftk_general_* *_dev entries
                                read op back in the same wait as fd_idx and check it as the *_host entries do. */
    int32_t n_op;            /* operating points, >= 1 when op is given                                                   */
    int32_t op_shared;       /* 0: tables per design [nD, n_op, 36, nw]; 1: one set for every design [n_op, 36, nw]
                                (generalised DOFs: [nD, n_op, n_fd, n_fd, nw] / [n_op, n_fd, n_fd, nw])                   */
    const double *op_A_w;    /* sum_r A_aero                  -- added to M0 + A_w                                         */
    const double *op_B_w;    /* sum_r B_aero + sum_r B_gyro   -- added to B0 + B_w                                         */
} raftk_cases;

/* Fixed-point loop controls (raft_model.py:966 tol, :977 nIter, :978 XiStart, :1133 relaxation).  The kernels test
 * |Xi - XiLast| / (|Xi| + tol) < tol in forms that square or take sqrt(d.d); with tol >= RAFTK_TOL_MIN those squares
 * stay in the normal range wherever they decide (|Xi| below ~1e150), so every kernel decides as the reference does.  tol = 0 (never
 * converge, run n_iter + 1 passes) is accepted too; a tol in (0, RAFTK_TOL_MIN), negative or NaN is refused. */
#define RAFTK_TOL_MIN 1e-70
typedef struct raftk_solve_opts {
    int32_t n_iter;          /* settings.nIter; the loop runs at most n_iter+1 passes           */
    int32_t cluster_size;    /* CTAs per (design,case): 0 = auto, else 1,2,4,8                  */
    double tol;              /* 0.01; 0 or >= RAFTK_TOL_MIN, else RAFTK_EINVAL                  */
    double xi_start;         /* settings.XiStart                                                */
    int32_t flags;           /* RAFTK_SOLVE_* bits, 0 = none                                    */
    int32_t _pad0;
} raftk_solve_opts;

/* raftk_solve_opts.flags.  REUSE_PLAN (raftk_*_dev only): the caller asserts that the design tables, the case count and the
 * workspace are exactly those of its previous solve call -- the per-design plan blobs (step classes, staged tables: a
 * pre-pass over the designs like the reference's calcHydroConstants, independent of the load cases' sea states) are then
 * still in the workspace and k_fused_plan is not launched again. */
enum { RAFTK_SOLVE_REUSE_PLAN = 1 };

/* Outputs.  Any pointer may be NULL (that output is skipped) except Xi/status where noted. */
typedef struct raftk_outputs {
    double *Xi;       /* complex [nD,nC,6,nw]  response amplitudes  (Model.Xi[0], fowt.Xi[0])   */
    int32_t *status;  /* [nD,nC,4]                                                              */
    double *B_drag;   /* [nD,nC,36] last linearised drag damping (fowt.B_hydro_drag)            */
    double *F_drag;   /* complex [nD,nC,6,nw] last drag excitation (fowt.F_hydro_drag)          */
    double *F_iner;   /* complex [nD,nC,6,nw] strip inertial excitation (fowt.F_hydro_iner[0])  */
    double *F_BEM;    /* complex [nD,nC,6,nw] BEM excitation (fowt.F_BEM[0])                    */
    double *zeta;     /* [nC,nw] wave amplitudes (fowt.zeta[0])                                 */
    double *F_2nd;    /* real [nD,nC,6,nw] difference-frequency force amplitudes (fowt.Fhydro_2nd)  */
    double *F_2nd_mean; /* [nD,nC,6] mean drift force (fowt.Fhydro_2nd_mean)                        */
    double *Xi_last;  /* complex [nD,nC,6,nw] the iterate the LAST pass linearised about (XiLast at raft_model.py:1063
                         when the loop stopped).  Fused solver only. */
} raftk_outputs;

int raftk_version(void);
const char *raftk_last_error(void);

/* Number of CUDA kernel launches issued by this library since load (bench.py "gpu_launches"). */
long long raftk_launch_count(void);

/*
 * Which kernel variant the last call on the calling host thread launched.  The entry points pick among several kernels by
 * shape, workspace size and RAFTK_* environment switches; the launch sites themselves fill this record, so it describes what
 * ran, not a plan recomputed afterwards.  Every entry point of the solve, second-order force, generalised-DOF, farm and
 * system-solve and eigen families clears it first; a call that fails before its launch leaves it cleared.  When one call launches
 * several families (a solve that computes its second-order force first, a farm host call) the last launch is reported.
 * Host bookkeeping only: no device work, no synchronisation.
 */
enum { RAFTK_FAMILY_NONE = 0, RAFTK_FAMILY_SOLVE = 1, RAFTK_FAMILY_QTF = 2, RAFTK_FAMILY_GENERAL = 3, RAFTK_FAMILY_FARM = 4,
       RAFTK_FAMILY_SYSTEM = 5, RAFTK_FAMILY_EIGEN = 6 };
enum {
    RAFTK_KERNEL_NONE = 0,
    RAFTK_KERNEL_V1 = 1,              /* k_depth_table + k_excitation (+ k_drag_solve), tables in the workspace          */
    RAFTK_KERNEL_FUSED128 = 2,        /* k_rao_fused<128>                                                                 */
    RAFTK_KERNEL_FUSED256 = 3,        /* k_rao_fused<256>                                                                 */
    RAFTK_KERNEL_FUSED2_CLUSTER = 4,  /* k_rao_fused2<false>: per-unit sums exchanged through distributed shared memory   */
    RAFTK_KERNEL_FUSED2_GRID = 5,     /* k_rao_fused2<true>: per-unit sums exchanged through the workspace                */
    RAFTK_KERNEL_QTF_TILES = 6,       /* k_qtf_tiles + k_qtf_finish                                                       */
    RAFTK_KERNEL_QTF_DIAG = 7,        /* k_qtf_force<false> (one QTF heading)                                             */
    RAFTK_KERNEL_QTF_DIAG_MIX = 8,    /* k_qtf_force<true> (heading interpolation)                                        */
    RAFTK_KERNEL_GEN_BLOCKED = 9,     /* k_gen_solve_blocked                                                              */
    RAFTK_KERNEL_GEN_UNBLOCKED = 10,  /* retired (the column-at-a-time k_gen_solve): never reported, kept for the numbering  */
    RAFTK_KERNEL_FARM_ROWS12 = 11,    /* k_farm_rows<12>                                                                  */
    RAFTK_KERNEL_FARM_WARP = 12,      /* k_farm_response<true>                                                            */
    RAFTK_KERNEL_FARM_BLOCK = 13,     /* k_farm_response<false>                                                           */
    RAFTK_KERNEL_SYS_UNBLOCKED = 14,  /* k_system_solve, column-at-a-time LU (n <= 24)                                    */
    RAFTK_KERNEL_SYS_BLOCKED = 15,    /* k_system_solve, blocked LU (n > 24)                                              */
    RAFTK_KERNEL_FARM_GLOBAL = 16,    /* k_farm_response_global: system in a workspace slab, LU blocked in global memory   */
    RAFTK_KERNEL_SYS_GLOBAL = 17,     /* k_system_solve_global: Z factored in place, LU blocked in global memory           */
    RAFTK_KERNEL_EIG_SMALL = 18,      /* k_eig_small: one system per thread (n <= 12)                                      */
    RAFTK_KERNEL_EIG_CTA_SMEM = 19,   /* k_eig_cta<true>: one system per CTA, H in shared memory                           */
    RAFTK_KERNEL_EIG_CTA_SLAB = 20    /* k_eig_cta<false>: one system per CTA, H in the workspace slab                     */
};
typedef struct raftk_dispatch {
    int32_t family;           /* RAFTK_FAMILY_*                                                                          */
    int32_t kernel;           /* RAFTK_KERNEL_*                                                                          */
    int32_t cluster_size;     /* CTAs per unit (solve family), else 0                                                    */
    int32_t bins_per_cta;     /* frequency bins per CTA (solve family), else 0                                           */
    int32_t threads_per_cta;
    int32_t f0_global;        /* k_rao_fused keeps the linear excitation F0 in the workspace instead of shared memory    */
    int32_t direct_d2h;       /* host entry point: the solve kernel stored Xi (and status) straight into page-locked host memory */
    int32_t trains;           /* cases.primary: the fused solver ran its two wave-train phases, or the generalised-DOF
                                 solve its secondary-train step                                                          */
    int32_t chunks;           /* v1 solver: launches over design chunks (1 = the whole batch at once)                    */
    int32_t inexact_walk;     /* the v1 solver ran because designs.walk_exact is 0                                       */
    int32_t farm_classes;     /* farm family: bit (1 << RAFTK_KERNEL_FARM_*) of every farm kernel the call launched (the
                                 kernel's bit for a uniform farm or batch; one per kernel class its farms occupy for a
                                 ragged batch)                                                                           */
} raftk_dispatch;
int raftk_last_dispatch(raftk_dispatch *out);

/* Per-kernel device timing for the roofline report.  When enabled, every *_dev / *_host call
 * brackets each kernel it launches with CUDA events on the launching stream.
 * raftk_profile_read synchronises those events and returns, for the LAST call, the summed device
 * milliseconds of ms[0] = depth-table kernel, ms[1] = excitation kernel, ms[2] = drag-linearise +
 * impedance-solve kernel, and launches[0..2] = how many launches each sum covers. */
void raftk_profile_enable(int on);
int raftk_profile_read(double ms[3], int launches[3]);

/* Bytes of device workspace the *_dev entry points need for (designs, n_cases): the wave-kinematics
 * tables of raftk_hydro_excitation_dev / raftk_hydro_linearization_dev (capped at 8 GiB; solves chunk). */
size_t raftk_workspace_bytes(const raftk_designs *d, int32_t n_cases);

/* Bytes raftk_solve_dynamics_dev alone needs: the fused solver keeps its tables in shared memory and only
 * parks the linear excitation in the workspace (16*6*nw bytes per unit); falls back to the value above when
 * a design's frequency slice does not fit on chip. */
size_t raftk_solve_workspace_bytes(const raftk_designs *d, int32_t n_cases);

/*
 * FOWT.calcHydroExcitation (raft_fowt.py:1732-1888) + Member.computeWaveKinematics /
 * calcHydroExcitation (raft_member.py:1899-1992) + helpers.getWaveKin/JONSWAP for every
 * (design, case).  Fills out->F_iner / F_BEM / zeta (those that are non-NULL) and leaves the
 * wave-kinematics tables in the workspace for raftk_hydro_linearization_dev.
 */
int raftk_hydro_excitation_dev(const raftk_designs *d, const raftk_cases *c, const raftk_outputs *out,
                               void *workspace, size_t workspace_bytes, void *stream);

/*
 * FOWT.calcHydroLinearization(Xi) + calcDragExcitation(0) (raft_fowt.py:1891-1957,
 * raft_member.py:1995-2152) for every (design, case), with Xi_in complex [nD,nC,6,nw] given.
 * Requires raftk_hydro_excitation_dev on the same workspace first (the reference has the same
 * ordering contract: mem.u must exist).  Fills out->B_drag, out->F_drag.
 */
int raftk_hydro_linearization_dev(const raftk_designs *d, const raftk_cases *c, const double *Xi_in,
                                  const raftk_outputs *out, void *workspace, size_t workspace_bytes,
                                  void *stream);

/*
 * Model.solveDynamics (raft_model.py:966-1302) for one FOWT per design and every case:
 * excitation, drag-linearisation fixed-point loop with the 6x6 complex impedance solve at
 * every frequency, convergence test and relaxation.  out->Xi and out->status are required.
 */
int raftk_solve_dynamics_dev(const raftk_designs *d, const raftk_cases *c, const raftk_solve_opts *o,
                             const raftk_outputs *out, void *workspace, size_t workspace_bytes,
                             void *stream);

/*
 * FOWT.calcHydroForce_2ndOrd(beta, S0), interpMode 'qtf' (raft_fowt.py:2158-2253) for every (design, case):
 * heading interpolation of the designs' QTF table, bilinear interpolation onto the model grid, the
 * difference-frequency sums  f(mu) = 4 dw sqrt(sum_i S(w_i) S(w_i+mu) |Q(w_i, w_i+mu)|^2)  shifted by one bin
 * (:2244-2245), and the mean drift  2 dw sum_i S(w_i) Re Q(w_i, w_i).  S is each case's wave spectrum
 * (raft_fowt.py:1758-1772; zeta^2 / (2 dw) for explicit amplitudes).  Needs designs.qtf; reads only the grid,
 * site and QTF fields of `d`.  Fills out->F_2nd (required) and out->F_2nd_mean (optional).
 *
 * Model.solveDynamics adds this force to the linear excitation when potSecOrder == 2 (raft_model.py:1035-1048,
 * :1210-1212).  raftk_solve_dynamics_dev does so when cases.F_2nd is given; when the designs carry a QTF and
 * cases.F_2nd is NULL it computes the force itself into out->F_2nd (then required as the buffer).
 * raftk_solve_dynamics_host always computes it when the designs carry a QTF (out->F_2nd optional).
 */
int raftk_second_order_force_dev(const raftk_designs *d, const raftk_cases *c, const raftk_outputs *out, void *stream);
int raftk_second_order_force_host(const raftk_designs *d, const raftk_cases *c, const raftk_outputs *out);

/*
 * Slender-body difference-frequency QTF (potSecOrder 1): FOWT.calcQTF_slenderBody (raft_fowt.py:1988-2078) with
 * Member.calcQTF_slenderBody + correction_KAY (raft_member.py:1488-1792) and the second-order wave kinematics of
 * helpers.py:239-373, for ONE design and n_cases (heading, motion RAO) pairs.  Tables: the submerged strip nodes of the
 * design (same nodes and order as raftk_designs) with the volumes / coefficients the reference evaluates inside its
 * frequency-pair loop, per-member waterline data, and the integration segments of the Kim & Yue correction
 * (raft_b200.packer.pack_qtf_members).  Xi_rao complex [n_cases,6,nw]: motion RAOs on the second-order grid
 * (raft_fowt.py:2021-2023; zeros = fixed body).  qtf complex [n_cases,nw,nw,6], Hermitian-filled (:2068-2070) --
 * the layout raftk_designs.qtf takes with qtf_shared = 2 and one heading.
 */
typedef struct raftk_slender {
    int32_t n_nodes, n_members, n_seg, nw;   /* nw: second-order frequencies (w1_2nd)                      */
    double depth, rho, g;
    const double *w, *k;            /* [nw] w1_2nd, k1_2nd (raft_fowt.py:419-426)                           */
    const double *mem_q, *mem_p1, *mem_p2;   /* [n_members,3]                                               */
    const int32_t *mem_mcf;         /* [n_members] 1: Kim & Yue correction applies (mem.MCF, crosses z = 0)  */
    const int32_t *mem_wl;          /* [n_members] 1: the member crosses the mean waterline                  */
    const double *mem_r_int;        /* [n_members,3] intersection with z = 0        raft_member.py:1528      */
    const double *mem_a_wl;         /* [n_members] cross-section area at the waterline      :1660-1674       */
    const double *mem_rwl;          /* [n_members,3] Kim & Yue: waterline point from rA, rB :1723            */
    const double *mem_R_wl;         /* [n_members] Kim & Yue: radius at z = 0               :1725            */
    const int32_t *mem_node_start;  /* [n_members+1]                                                         */
    const double *node_r;           /* [n_nodes,3] global node positions                                     */
    const double *node_v_side;      /* [n_nodes] strip volume, waterline-scaled             :1565-1571       */
    const double *node_Ca_p1, *node_Ca_p2, *node_Ca_End;  /* [n_nodes] interpolated coefficients :1560-1562  */
    const double *node_v_end;       /* [n_nodes] end volume                                 :1620-1625       */
    const double *node_a_i;         /* [n_nodes] signed end area (mem.a_i)                                   */
    const int32_t *seg_mem;         /* [n_seg] Kim & Yue integration segments               :1741-1760       */
    const double *seg_z1, *seg_z2, *seg_R, *seg_rmid;     /* [n_seg], [n_seg], [n_seg], [n_seg,3]            */
    const double *M_struc;          /* [36] fowt.M_struc (Pinkster IV term, raft_fowt.py:2044)               */
} raftk_slender;

size_t raftk_qtf_slender_workspace_bytes(const raftk_slender *s, int32_t n_cases);
int raftk_qtf_slender_dev(const raftk_slender *s, int32_t n_cases, const double *beta_rad, const double *Xi_rao, double *qtf,
                          void *workspace, size_t workspace_bytes, void *stream);
int raftk_qtf_slender_host(const raftk_slender *s, int32_t n_cases, const double *beta_rad, const double *Xi_rao, double *qtf);

/*
 * Model.solveDynamics with potSecOrder 1 (raft_model.py:1052-1142) for every (design, case), in one call on one stream:
 * loop A (the plain solve) -> motion RAOs of the units whose loop A converged, interpolated onto the second-order grid
 * (helpers.getRAO + np.interp, same bits) -> slender-body QTF per unit (the kernels of raftk_qtf_slender_*, same bits per
 * design) -> second-order force (qtf_shared = 2, one heading) -> loop B from loop A's last iterate (cases.Xi_init) with the
 * force added (cases.F_2nd) and n_iter - 1 -> merge.  Units whose loop A did not converge keep loop A's outputs and get zero
 * F_2nd, F_2nd_mean and qtf; elsewhere passes add up and the flags are OR-ed.  No host synchronisation.
 *
 * raftk_slender_batch: the raftk_slender tables of nD designs on ONE second-order grid, concatenated in design order.  cols.n_nodes /
 * n_members / n_seg are the totals; design d owns nodes node_offset[d] .. node_offset[d+1]-1 (likewise members, segments);
 * cols.mem_node_start holds each design's own [n_members_d + 1] starts (n_members_total + n_designs entries); seg_mem indexes the
 * design's own members; cols.M_struc is [nD,36].  max_*: the largest per-design counts (at least every design's).
 * raftk_slender_outputs (may be NULL): qtf complex [nD,nC,nw2,nw2,6] and Xi_rao complex [nD,nC,6,nw2], both optional;
 * qtf_chunk: units whose QTF tables are built at once in the workspace (0: all; at most 65535 per chunk).  Each unit's QTF
 * takes 96 nw2^2 bytes and its tables 16 nw2 (22 max_nodes + 10 max_members) bytes, so large batches want a chunk.
 * The designs must not carry an external QTF; cases.primary, F_2nd and Xi_init must be NULL; n_iter >= 1.  The second-order
 * force's tile kernel sums with atomics: the last bits of F_2nd, and so of loop B, vary run to run (RAFTK_QTF_DIAG=1: fixed).
 */
typedef struct raftk_slender_batch {
    int32_t n_designs, max_nodes, max_members, max_seg;
    const int32_t *node_offset, *member_offset, *seg_offset;   /* [n_designs+1] */
    raftk_slender cols;
} raftk_slender_batch;

typedef struct raftk_slender_outputs {
    double *qtf;                    /* optional complex [nD,nC,nw2,nw2,6]                                     */
    double *Xi_rao;                 /* optional complex [nD,nC,6,nw2]: the RAOs the QTFs were computed from    */
    int32_t qtf_chunk;              /* units per QTF chunk, 0 = all                                            */
    int32_t _pad0;
} raftk_slender_outputs;

size_t raftk_solve_dynamics_slender_workspace_bytes(const raftk_designs *d, const raftk_slender_batch *s, int32_t n_cases, int32_t qtf_chunk);
int raftk_solve_dynamics_slender_dev(const raftk_designs *d, const raftk_slender_batch *s, const raftk_cases *c, const raftk_solve_opts *o,
                                     const raftk_outputs *out, const raftk_slender_outputs *so, void *workspace, size_t workspace_bytes,
                                     void *stream);
int raftk_solve_dynamics_slender_host(const raftk_designs *d, const raftk_slender_batch *s, const raftk_cases *c, const raftk_solve_opts *o,
                                      const raftk_outputs *out, const raftk_slender_outputs *so);

/*
 * Model.solveDynamics for ONE FOWT with generalised degrees of freedom (flexible members, n_dof > 6; raft_fowt.py:1854-1857,
 * 1886-1888, 1913-1929; raft_model.py:1052-1142) and n_cases cases or wave trains.  Every submerged strip node carries the
 * 6 x n_dof block of fowt.T of its structural node (Tn) and its offset from that node (rr; zero on flexible members):
 * node motion = Tn Xi, node load -> Tn^T [f ; rr x f].  M, B, C: the constant system matrices of raft_model.py:1045-1047.
 * Xi complex [n_cases,n_dof,nw]; status [n_cases,4] = passes, converged, flags, 0.  The n_dof x n_dof impedance of every (case,
 * frequency, pass) is solved by a blocked LU with partial pivoting (LAPACK's pivot rule and elimination order); validated on
 * the GPU against the reference's 150-DOF VolturnUS-S-flexible run (tests/test_general_dofs.py, 1e-10).  n_dof <= 256.
 * Status flags: RAFTK_FLAG_NAN for NaN in a response, RAFTK_FLAG_SINGULAR for an exactly zero pivot at some bin (its
 * response is NaN as well); either stops the case.  A secondary train solved with its primary's singular factors carries both.
 * Wave trains (cases.primary, raft_model.py:1200-1236): a secondary train runs no pass of its own; its response is solved with
 * the LU factors of its primary's last impedance and the drag excitation of its own wave kinematics with the primary's last
 * node drag coefficients.  Primaries keep the loop's final Xi.  Status rows of secondaries: 0, 1, flags, primary + 1.
 * cases.F_2nd and cases.Xi_init are rejected (second-order loads: raftk_general_qtf below).  raftk_general_workspace_bytes() covers any primary map; the pivot rows kept for
 * the trains take n_cases * nw * n_dof * 4 bytes of it (rounded up to 256) whether or not the call has trains.
 */
typedef struct raftk_general {
    int32_t n_dof, nw, n_nodes, _pad0;
    double depth, rho, dw;
    const double *w, *k;            /* [nw]                                                          */
    const double *node_r;           /* [n_nodes,3]                                                   */
    const double *node_frame;       /* [n_nodes,9] q, p1, p2 of the node's member                    */
    const int32_t *node_circ;       /* [n_nodes]                                                     */
    const double *node_Imat;        /* [n_nodes,9]                                                   */
    const double *node_Imat_w;      /* complex [n_nodes,9,nw] MacCamy-Fuchs Imat_MCF, or NULL        */
    const double *node_a_i;         /* [n_nodes] signed end area                                     */
    const double *node_cd;          /* [n_nodes,4] a_q Cd_q, a_p1 Cd_p1, a_p2 Cd_p2, a_End Cd_End    */
    const double *Tn;               /* [n_nodes,6,n_dof]                                             */
    const double *rr;               /* [n_nodes,3]                                                   */
    const double *M, *B, *C;        /* [n_dof,n_dof]                                                 */
} raftk_general;

size_t raftk_general_workspace_bytes(const raftk_general *g, int32_t n_cases);
int raftk_general_solve_dynamics_dev(const raftk_general *g, const raftk_cases *c, const raftk_solve_opts *o, double *Xi,
                                     int32_t *status, void *workspace, size_t workspace_bytes, void *stream);
int raftk_general_solve_dynamics_host(const raftk_general *g, const raftk_cases *c, const raftk_solve_opts *o, double *Xi,
                                      int32_t *status);

/*
 * Frequency-dependent terms of the generalised-DOF solve (raft_model.py:1005-1010, 1045-1048): the added mass and damping
 * of operating rotors (sum A_aero, B_aero; raft_fowt.py:1557-1562) and of potential-flow coefficients (A_BEM, B_BEM, lumped on
 * reduced DOFs 0-5 by readHydro, raft_fowt.py:1479-1480), and the BEM wave excitation F_BEM = T^T F_BEM_fullDOF
 * (raft_fowt.py:1796-1849, 1885-1887).  raft_b200.packer.pack_general_matrices builds it.
 * The matrices are given on their support fd_idx only: every entry outside it is zero, so the restricted table gives the same
 * impedance as the dense [n_dof,n_dof,nw] sum.  On the support, M = M + A_w, B = (B + B_w) + B_drag and
 * Z = fma(-w^2, M, C) + i w B (the rigid solver's grouping); every other entry is computed exactly as without fd.
 * The BEM force of every case (secondary trains included) is added to the inertial excitation before the drag excitation:
 * (F_BEM + F_iner) + F_drag.
 * Pointers are device pointers for *_dev and host pointers for *_host.  Rejected with RAFTK_EINVAL before any launch: n_fd
 * outside [0, n_dof], fd_idx out of range, repeated or unsorted, n_bem_head < 0, a missing table for a nonzero count, headings
 * that decrease or fall outside [0, 360) (equal neighbours are legal).  The *_dev entry reads fd_idx and bem_headings back
 * to the host for these checks (a copy on the caller's stream and a wait for it).
 *
 * Per-case operating points (raftk_cases.op; calcTurbineConstants(case), raft_fowt.py:1514-1586) on a generalised-DOF FOWT:
 * every raftk_general_* solve (plain, _fd, _qtf, _stream, _batch; _host and _dev) takes them on the support of fd, in the
 * same [n_fd,n_fd,nw] layout as A_w / B_w: op_A_w, op_B_w are [nD,n_op,n_fd,n_fd,nw], or [n_op,n_fd,n_fd,nw] with
 * op_shared = 1 (single-design entries: nD = 1).  Unit (d, c) solves with M + (A_w + op_A_w[op[c]]) and
 * (B + (B_w + op_B_w[op[c]])) + B_drag on the support and exactly as without them off it, so a call equals one call per
 * operating point with that point's tables summed into fd.A_w / fd.B_w, bit for bit (except the k_qtf_tiles atomics: see
 * RAFTK_QTF_DIAG).  A batch unit reads table op_shared ? 0 : d.  Rejected with RAFTK_EINVAL before any launch: op without fd
 * or with n_fd = 0, n_op < 1, op_shared not 0 or 1, a missing table, an index outside [0, n_op), a secondary train whose
 * point differs from its primary's.  The *_dev entries read op (and primary) back in the same wait as fd_idx.  Workspace
 * sizes do not depend on them.
 */
typedef struct raftk_general_fd {
    int32_t n_fd, n_bem_head;
    const int32_t *fd_idx;          /* [n_fd] reduced DOFs carrying frequency-dependent terms, strictly increasing        */
    const double *A_w, *B_w;        /* [n_fd,n_fd,nw] (the reference's [n,n,nw] layout restricted to fd_idx); NULL if n_fd = 0 */
    const double *bem_headings;     /* [n_bem_head] deg, non-decreasing in [0,360)                                         */
    const double *X_BEM;            /* complex [n_bem_head,6,nw], heading-relative (packer.pack_bem_excitation's table)      */
    const double *T0;               /* [6,n_dof]: rows 0..5 of fowt.T (maps the full-DOF BEM force to reduced DOFs)          */
    double x_ref, y_ref, heading_adjust;
} raftk_general_fd;

/* fd = NULL: the constant-matrix solve of raftk_general_solve_dynamics_*, bit for bit (those entry points call these).
 * F_BEM: optional output, complex [n_cases,n_dof,nw] in reduced DOFs (zero without BEM tables), or NULL. */
size_t raftk_general_fd_workspace_bytes(const raftk_general *g, const raftk_general_fd *fd, int32_t n_cases);
int raftk_general_solve_dynamics_fd_dev(const raftk_general *g, const raftk_general_fd *fd, const raftk_cases *c, const raftk_solve_opts *o,
                                        double *Xi, int32_t *status, double *F_BEM, void *workspace, size_t workspace_bytes, void *stream);
int raftk_general_solve_dynamics_fd_host(const raftk_general *g, const raftk_general_fd *fd, const raftk_cases *c, const raftk_solve_opts *o,
                                         double *Xi, int32_t *status, double *F_BEM);

/*
 * Second-order wave loads of the generalised-DOF solve (potSecOrder 2; raft_model.py:1035-1048, 1210-1212): the external
 * difference-frequency QTF of the FOWT, the state FOWT.readQTF leaves behind (raft_fowt.py:2081-2128) with the DOF axis cut
 * to the 6 rows a .12d file fills -- the reference lumps the force on reduced DOFs 0-5 ("Lumping at the first 6dofs",
 * raft_model.py:1034), rows 6 and up are zero.  raft_b200.packer.pack_general_qtf builds it.  Same layout as
 * raftk_designs.qtf for one FOWT.
 * Every row of the case table, secondary trains included, gets F_2nd / F_2nd_mean of its own spectrum and heading
 * (raftk_second_order_force_*: FOWT.calcHydroForce_2ndOrd, interpMode 'qtf'), computed on the call's stream before the loop
 * and added to the real part of reduced rows 0-5 of the inertial excitation after the BEM force:
 * ((F_BEM + F_iner) + F_2nd) + F_drag in every pass, and for the secondary trains.  k_qtf_tiles combines partial sums with
 * atomic adds, so the last bits of F_2nd, and therefore of Xi, vary from run to run (as on the rigid path);
 * RAFTK_QTF_DIAG=1 selects the diagonal kernel, which is reproducible.
 * Rejected with RAFTK_EINVAL before any launch: n_qtf_w < 2, n_qtf_head < 1, a missing table, n_dof < 6, nw above the force
 * kernel's shared-memory limit (nw * 20 bytes <= 227 KB), frequencies that do not strictly increase or headings that do not
 * strictly increase.  The *_dev entry reads qtf_w and qtf_heads back to the host for these checks (a copy on the caller's
 * stream and a wait for it).
 */
typedef struct raftk_general_qtf {
    int32_t n_qtf_w, n_qtf_head;
    const double *qtf_w;            /* [n_qtf_w] rad/s, strictly increasing (w1_2nd == w2_2nd)                              */
    const double *qtf_heads;        /* [n_qtf_head] rad, strictly increasing (heads_2nd)                                    */
    const double *qtf;              /* complex [n_qtf_w, n_qtf_w, n_qtf_head, 6]: fowt.qtf[..., :6], dimensional, Hermitian-filled */
} raftk_general_qtf;

/* qtf = NULL: raftk_general_solve_dynamics_fd_*, bit for bit (those entry points call these).  F_2nd: optional output, real
 * [n_cases,6,nw] (the one-bin-shifted amplitudes; last bin zero); F_2nd_mean: optional output [n_cases,6]; without a table both
 * are left untouched.  When NULL, the workspace holds them. */
size_t raftk_general_qtf_workspace_bytes(const raftk_general *g, const raftk_general_fd *fd, const raftk_general_qtf *qtf, int32_t n_cases);
int raftk_general_solve_dynamics_qtf_dev(const raftk_general *g, const raftk_general_fd *fd, const raftk_general_qtf *qtf, const raftk_cases *c,
                                         const raftk_solve_opts *o, double *Xi, int32_t *status, double *F_BEM, double *F_2nd,
                                         double *F_2nd_mean, void *workspace, size_t workspace_bytes, void *stream);
int raftk_general_solve_dynamics_qtf_host(const raftk_general *g, const raftk_general_fd *fd, const raftk_general_qtf *qtf, const raftk_cases *c,
                                          const raftk_solve_opts *o, double *Xi, int32_t *status, double *F_BEM, double *F_2nd,
                                          double *F_2nd_mean);

/*
 * The generalised-DOF solve of a case table of any size through a bounded workspace.  The table is cut into chunks of at most
 * max_chunk_cases cases (0: all cases in one chunk), each made of whole train groups -- a primary and every secondary train that
 * points at it (cases.primary) stay in one chunk, because the secondaries are solved from the primary's LU factors.  Groups are
 * packed greedily in table order.  Every chunk runs the launch sequence of raftk_general_solve_dynamics_qtf_dev on views of the
 * case columns and outputs advanced to its first case, one after the other on the caller's stream in one workspace sized for the
 * largest chunk, with no host synchronisation between chunks.  Every output equals the single-table entry's bit for bit (up to
 * the atomic sums of k_qtf_tiles, see raftk_general_qtf); status word 3 of a secondary train still holds its primary's index in
 * the whole table + 1.  Arguments are those of raftk_general_solve_dynamics_qtf_* plus max_chunk_cases; n_cases may exceed
 * 65535 when max_chunk_cases <= 65535.
 * raftk_general_stream_workspace_bytes(.., n_cases, K) = raftk_general_qtf_workspace_bytes(.., min(K, n_cases)), plus the chunk's
 * rebased primary map (K * 4 bytes rounded up to 256) when K < n_cases.
 * Rejected with RAFTK_EINVAL before any launch, in addition to the checks of the qtf entry: max_chunk_cases < 0 or a chunk of
 * more than 65535 cases; a primary map whose train groups interleave (a group not contiguous in the table;
 * raft_b200.packer.pack_case_trains never builds one); a group with more than max_chunk_cases cases; a workspace smaller than
 * the query.  The *_dev entry reads cases.primary back to the host once to plan the chunks (a copy on the caller's stream and a
 * wait for it), as it reads fd and qtf tables for their checks.
 */
size_t raftk_general_stream_workspace_bytes(const raftk_general *g, const raftk_general_fd *fd, const raftk_general_qtf *qtf, int32_t n_cases,
                                            int32_t max_chunk_cases);
int raftk_general_solve_dynamics_stream_dev(const raftk_general *g, const raftk_general_fd *fd, const raftk_general_qtf *qtf,
                                            const raftk_cases *c, const raftk_solve_opts *o, double *Xi, int32_t *status, double *F_BEM,
                                            double *F_2nd, double *F_2nd_mean, void *workspace, size_t workspace_bytes,
                                            int32_t max_chunk_cases, void *stream);
int raftk_general_solve_dynamics_stream_host(const raftk_general *g, const raftk_general_fd *fd, const raftk_general_qtf *qtf,
                                             const raftk_cases *c, const raftk_solve_opts *o, double *Xi, int32_t *status, double *F_BEM,
                                             double *F_2nd, double *F_2nd_mean, int32_t max_chunk_cases);

/*
 * Design batches of FOWTs with generalised degrees of freedom: n_designs flexible designs that share n_dof (one FE topology),
 * the frequency grid (w, k, nw, dw), depth and rho, solved over one case table in one call.  raft_b200.solver.GeneralBatch
 * builds the tables.
 *   raftk_general g:  n_nodes = the total node count; every node array (node_r .. rr, Tn) is the designs' arrays concatenated,
 *                     design d owning nodes node_offset[d] .. node_offset[d+1]-1 (a design with no submerged node is legal);
 *                     M, B, C are [n_designs,n_dof,n_dof].
 *   raftk_general_fd: n_fd and n_bem_head are the same for every design; fd_idx [nD,n_fd], A_w / B_w [nD,n_fd,n_fd,nw],
 *                     bem_headings [nD,n_bem_head], X_BEM complex [nD,n_bem_head,6,nw], T0 [nD,6,n_dof]; x_ref, y_ref,
 *                     heading_adjust per design in raftk_general_batch (NULL: fd's scalars for every design).
 *   raftk_general_qtf: one grid (qtf_w, qtf_heads); the table is per design [nD, n_qtf_w, n_qtf_w, n_qtf_head, 6], or one table
 *                     for every design (qtf_shared = 1).
 * Units are (design, case) pairs, design-major (unit d * n_cases + c): every design runs the whole case table, train groups
 * included.  Xi complex [nD,n_cases,n_dof,nw], status [nD,n_cases,4]; optional F_BEM complex [nD,n_cases,n_dof,nw], F_2nd
 * [nD,n_cases,6,nw], F_2nd_mean [nD,n_cases,6].  Xi[d] equals raftk_general_solve_dynamics_* on design d alone bit for bit (up
 * to the atomic sums of k_qtf_tiles, see raftk_general_qtf); status word 3 of a secondary train holds its primary's case index
 * + 1 within the design.  The units run in chunks of at most max_chunk_units (0: all units in one chunk), cut only at train-group
 * boundaries and possibly across designs, one after the other on the caller's stream in one workspace sized for the largest
 * chunk, with no host synchronisation between chunks (the launch sequence of raftk_general_solve_dynamics_stream_*, whose
 * kernels map every unit to its design's nodes, matrices and tables).  n_designs * n_cases may exceed 65535 when chunks do not.
 * raftk_general_batch_workspace_bytes(.., K) = raftk_general_qtf_workspace_bytes of min(K, units) units with max_nodes node
 * rows each, plus the chunk's primary map (K * 4 bytes rounded up to 256) when K < units or n_designs > 1.
 * Rejected with RAFTK_EINVAL before any launch: every check of the qtf entry, applied to every design's fd rows; n_designs <= 0;
 * node_offset missing, not starting at 0, decreasing, not ending at n_nodes, or a design with more than max_nodes nodes;
 * qtf_shared not 0 or 1; max_chunk_units < 0 or a chunk of more than 65535 units; interleaved train groups; a train group with
 * more cases than max_chunk_units; a workspace smaller than the query.  The *_dev entry reads node_offset, cases.primary, the fd
 * index and heading rows and the QTF grid back to the host with one wait per call.
 */
typedef struct raftk_general_batch {
    int32_t n_designs;
    int32_t max_nodes;              /* >= the largest node_offset[d+1] - node_offset[d] (node rows of the workspace)           */
    int32_t qtf_shared;             /* 0: qtf per design [nD, ...]; 1: one table for every design                            */
    int32_t _pad0;
    const int32_t *node_offset;     /* [n_designs + 1] CSR offsets into g's node arrays                                       */
    const double *x_ref, *y_ref, *heading_adjust;   /* [n_designs] BEM reference point and heading adjustment, or NULL       */
} raftk_general_batch;

size_t raftk_general_batch_workspace_bytes(const raftk_general *g, const raftk_general_batch *b, const raftk_general_fd *fd,
                                           const raftk_general_qtf *qtf, int32_t n_cases, int32_t max_chunk_units);
int raftk_general_batch_solve_dynamics_dev(const raftk_general *g, const raftk_general_batch *b, const raftk_general_fd *fd,
                                           const raftk_general_qtf *qtf, const raftk_cases *c, const raftk_solve_opts *o, double *Xi,
                                           int32_t *status, double *F_BEM, double *F_2nd, double *F_2nd_mean, void *workspace,
                                           size_t workspace_bytes, int32_t max_chunk_units, void *stream);
int raftk_general_batch_solve_dynamics_host(const raftk_general *g, const raftk_general_batch *b, const raftk_general_fd *fd,
                                            const raftk_general_qtf *qtf, const raftk_cases *c, const raftk_solve_opts *o, double *Xi,
                                            int32_t *status, double *F_BEM, double *F_2nd, double *F_2nd_mean, int32_t max_chunk_units);

/*
 * Output channels of FOWT.saveTurbineOutputs for a FOWT with generalised degrees of freedom (raft_fowt.py:2299-2604): PRP
 * motions, nacelle accelerations and flexible-tower base loads are real linear functionals of the reduced response,
 *   Y_ch(w) = w^wpow[ch] sum_b R[ch,b] Xi[b,w]     (raft_b200.packer.pack_general_channels; rad2deg folded into R)
 * -> std = sqrt(1/2 sum_w |Y|^2), PSD(w) = 1/2 |Y|^2 / dw, amp = Y, with the reduction of raftk_channel_stats_*.
 * w [nw] rad/s; R [n_ch,n_dof]; wpow [n_ch] 0, 1 or 2 (displacement, velocity, acceleration); Xi complex [n_units,n_dof,nw]
 * -> std [n_units,n_ch], psd [n_units,n_ch,nw] or NULL, amp complex [n_units,n_ch,nw] or NULL.  Any other wpow is refused
 * with RAFTK_EINVAL before any launch; the _dev entry reads wpow back on its stream for that check (one synchronisation).
 */
int raftk_general_channel_stats_dev(int32_t n_units, int32_t n_dof, int32_t n_ch, int32_t nw, double dw, const double *w,
                                    const double *R, const int32_t *wpow, const double *Xi, double *std, double *psd, double *amp,
                                    void *stream);
int raftk_general_channel_stats_host(int32_t n_units, int32_t n_dof, int32_t n_ch, int32_t nw, double dw, const double *w,
                                     const double *R, const int32_t *wpow, const double *Xi, double *std, double *psd, double *amp);

/*
 * Multi-GPU exchange of the responses (SURVEY.md 8e; the reference's sweep driver parametersweep.py:49-95 collects
 * every design's results in one array).  One process per GPU; rank r solves its shard of units.  Instead of a separate
 * all-gather after the solve, the solve kernel itself stores each finished unit's Xi into EVERY rank's copy of the
 * gathered array through peer-mapped pointers (NVLink stores, overlapped with the units still computing), and
 * raftk_peer_barrier_dev makes the stream wait until every peer's stores into THIS rank's copy have landed.
 *
 * Setup (once): each rank allocates its copy with raftk_peer_alloc -- plain cudaMalloc memory plus the 64-byte CUDA IPC
 * handle --, the handles are exchanged out of band (torch.distributed all_gather_object in raft_b200.sweep) and opened
 * with raftk_peer_open.  A copy holds complex [n_ranks, units_per_rank, 6, nw] responses, uint32 [n_ranks] arrival flags
 * and optionally int32 [n_ranks, units_per_rank, 4] status words; gathered[p] / flags[p] / status[p] below are rank p's
 * copy as mapped in THIS process.  A rank may run one step ahead of a peer, so consumers that read other ranks' blocks
 * should alternate between two copies (raft_b200.sweep.PeerExchange does).
 */
#define RAFTK_MAX_PEERS 16
typedef struct raftk_peers {
    int32_t n_ranks, rank;
    uint32_t epoch;          /* step counter, > 0 and increasing by one per exchange (the barrier waits for flags >= epoch) */
    int32_t _pad0;
    size_t block_elems;      /* complex elements per rank block = units_per_rank * 6 * nw                              */
    double *gathered[RAFTK_MAX_PEERS];     /* [p]: base of rank p's gathered array (p == rank: the local allocation)    */
    uint32_t *flags[RAFTK_MAX_PEERS];      /* [p]: rank p's arrival flags uint32[n_ranks]                               */
    int32_t *status[RAFTK_MAX_PEERS];      /* [p]: rank p's gathered status int32 [n_ranks, units_per_rank, 4]; all NULL: not exchanged */
} raftk_peers;

int raftk_peer_alloc(size_t bytes, void **dev_ptr, unsigned char handle[64]);
int raftk_peer_free(void *dev_ptr);
int raftk_peer_open(const unsigned char handle[64], void **dev_ptr);
int raftk_peer_close(void *dev_ptr);
/* raftk_solve_dynamics_dev with the exchange fused into the kernel's epilogue: out->Xi must be
 * peers->gathered[rank] + 2 * rank * block_elems (the rank's own block of its own copy). */
int raftk_solve_dynamics_gather_dev(const raftk_designs *d, const raftk_cases *c, const raftk_solve_opts *o,
                                    const raftk_outputs *out, const raftk_peers *peers, void *workspace,
                                    size_t workspace_bytes, void *stream);
/* Enqueue: tell every peer "my stores of this epoch are done", then wait (bounded: ~4 s, then *timeout_flag = 1 if
 * given) until every peer said so.  After it, gathered[rank] holds all ranks' blocks of this epoch. */
int raftk_peer_barrier_dev(const raftk_peers *peers, int32_t *timeout_flag, void *stream);
/* Generalised-DOF shards (raft_b200.sweep.ShardedGeneralSolve): a copy's responses are complex [n_ranks * rows_per_rank, n_dof,
 * nw] (block_elems = rows_per_rank * n_dof * nw) and its status int32 [n_ranks * rows_per_rank, 4].  Enqueue stores of n_rows
 * finished rows -- Xi complex [n_rows, n_dof, nw] and status [n_rows, 4] (or NULL) on this device -- into rows [row0, row0 +
 * n_rows) of EVERY rank's copy through the peer-mapped pointers; status word 3 of a secondary train (primary + 1) is shifted by
 * primary_base, so a shard solved as a table of its own publishes indices into the whole table.  Follow with
 * raftk_peer_barrier_dev.  Rows past n_ranks * block_elems, or status without every rank's status copy: RAFTK_EINVAL. */
int raftk_general_publish_dev(const raftk_peers *peers, const double *Xi, const int32_t *status, int32_t row0, int32_t n_rows,
                              int32_t n_dof, int32_t nw, int32_t primary_base, void *stream);

/* Same three operations with HOST pointers everywhere (tables, cases, outputs). */
int raftk_hydro_excitation_host(const raftk_designs *d, const raftk_cases *c, const raftk_outputs *out);
int raftk_hydro_linearization_host(const raftk_designs *d, const raftk_cases *c, const double *Xi_in,
                                   const raftk_outputs *out);
int raftk_solve_dynamics_host(const raftk_designs *d, const raftk_cases *c, const raftk_solve_opts *o,
                              const raftk_outputs *out);

/*
 * System (farm) response, raft_model.py:1164-1216: for every frequency solve the dense
 * n x n complex system Z_sys(w) Xi = F for nrhs right-hand sides (n = 6N).
 * Z complex [nw,n,n] row-major (destroyed), F complex [nw,n,nrhs] (overwritten with Xi).
 * info [nw]: 0, or k+1 of the first zero pivot.  Any n: a system whose [n][n+nrhs] augmented matrix fits in the device's
 * opt-in shared memory next to the kernel's static shared memory is solved there (k_system_solve); larger ones are factored
 * in place in Z (k_system_solve_global).  Both pivot on |re| + |im| (first maximum wins) with the same elimination order.
 */
int raftk_system_solve_dev(int32_t n, int32_t nw, int32_t nrhs, double *Z, double *F, int32_t *info,
                           void *stream);
int raftk_system_solve_host(int32_t n, int32_t nw, int32_t nrhs, double *Z, double *F, int32_t *info);

/*
 * Farm system response computed on the device from the per-FOWT solves (raft_model.py:1164-1236): the designs of the
 * batch are the N FOWTs of the array (each at its own x_ref / y_ref), the drag linearisation of every FOWT runs as in
 * raftk_solve_dynamics_*, then for every case and frequency
 *     Z_sys = blockdiag_i( -w^2 (M0_i + A_w,i) + i w (B0_i + B_drag_i + B_w,i) + C0_i ) + ( -w^2 M_arr + i w B_arr + C_arr )
 *     Xi_sys = Z_sys^-1 [ F_BEM_i + F_iner_i + F_drag_i (+ F_2nd_i) ]_i
 * M_arr / B_arr / C_arr: array-level mooring matrices [6N,6N] row-major (model.ms.getCoupledStiffnessA for moorMod 0/1;
 * getCoupledDynamicMatrices for moorMod 2), any may be NULL.  Xi_sys complex [nC, 6N, nw] (Model.Xi[ih] per case / train),
 * info [nC, nw]: 0, or k+1 of the first zero pivot (numpy.linalg.inv raises LinAlgError there).
 * _dev: `solved` holds the DEVICE outputs of a preceding raftk_solve_dynamics_dev of the same (d, c): B_drag, F_drag, F_iner
 * (and F_BEM when the designs carry BEM excitation) are required.  _host: one call does both steps from host buffers;
 * `out` may request any of the per-FOWT outputs as usual.
 */
typedef struct raftk_farm {
    int32_t n_fowt;          /* must equal designs.n_designs                                    */
    int32_t _pad0;
    const double *M_arr, *B_arr, *C_arr;
    double *Xi_sys;
    int32_t *info;
} raftk_farm;

int raftk_farm_response_dev(const raftk_designs *d, const raftk_cases *c, const raftk_outputs *solved, const raftk_farm *f,
                            void *stream);
/*
 * Farms of any size.  While a [6N][6N+1] complex system fits in the device's opt-in shared memory next to the static shared
 * memory of the one-CTA-per-system kernel (on an H100: N <= 20 with the sm_90a build), the shared-memory kernels solve the
 * farm and no workspace is used.  Larger farms are solved by k_farm_response_global: persistent CTAs, each assembling and
 * factoring one (case, frequency) system after another in its own [6N][6N+1] slab of the workspace.
 * raftk_farm_workspace_bytes: 0 when the shared-memory kernels take the shape; else the bytes of a full persistent grid
 * (resident CTAs x slab, at most nC * nw slabs).  Without a device it answers for an H100 (132 SMs, 227 KB opt-in).
 * raftk_farm_response_ws_dev: raftk_farm_response_dev with a device workspace; accepts every N.  Fewer bytes than the query
 * returned run fewer CTAs with bit-identical results; less than one slab is RAFTK_EINVAL before any launch.
 * raftk_farm_response_dev is the same call without a workspace, so it refuses the farms that need one.
 * raftk_solve_dynamics_farm_host reserves the workspace itself and accepts every N.
 */
size_t raftk_farm_workspace_bytes(const raftk_designs *d, const raftk_cases *c, const raftk_farm *f);
int raftk_farm_response_ws_dev(const raftk_designs *d, const raftk_cases *c, const raftk_outputs *solved, const raftk_farm *f,
                               void *workspace, size_t workspace_bytes, void *stream);
int raftk_solve_dynamics_farm_host(const raftk_designs *d, const raftk_cases *c, const raftk_solve_opts *o,
                                   const raftk_outputs *out, const raftk_farm *f);

/*
 * Batches of farms (array layout and shared-mooring studies): n_farms arrays of n_fowt FOWTs each over one case table in
 * one call.  Design f * n_fowt + i of the batch is FOWT i of farm f; the farms share the turbine count, frequency grid,
 * depth and rho, and differ in positions (hence wave phasing), platforms and array matrices.  Every system is assembled and
 * solved exactly as raftk_farm's: a farm's Xi_sys and info do not depend on the batch it is in, and the raftk_farm entries
 * are n_farms = 1 launches of the same kernels.
 * M_arr / B_arr / C_arr: [6N,6N] used by every farm when arr_shared = 1, [n_farms,6N,6N] when 0; any may be NULL.
 * Xi_sys complex [n_farms, nC, 6N, nw]; info [n_farms, nC, nw] or NULL: a zero pivot is flagged in its own farm's rows only.
 * Limits: with the system in shared memory or registers (N <= 20 on an H100) the grid is (frequency groups, case, farm), so
 * at most 65535 cases and 65535 farms per call; larger farms walk a list of n_farms * nC * nw systems and have no such limit.
 * raftk_farm_batch_workspace_bytes: as raftk_farm_workspace_bytes with n_farms * nC * nw systems (0 for N <= 20).
 * raftk_farm_batch_response_ws_dev: `solved` holds the device outputs of raftk_solve_dynamics_dev on the same (d, c).
 * RAFTK_EINVAL before any launch: n_farms or n_fowt < 1, n_farms * n_fowt != designs.n_designs, arr_shared not 0 or 1, no
 * Xi_sys, a missing per-FOWT output (B_drag, F_drag, F_iner; F_BEM with BEM excitation), a grid limit above, or less than
 * one slab of workspace when the shape needs one.
 */
typedef struct raftk_farm_batch {
    int32_t n_farms, n_fowt;        /* n_farms * n_fowt must equal designs.n_designs */
    int32_t arr_shared, _pad0;      /* 1: one M_arr/B_arr/C_arr for every farm; 0: [n_farms,6N,6N] */
    const double *M_arr, *B_arr, *C_arr;
    double *Xi_sys;
    int32_t *info;
} raftk_farm_batch;

size_t raftk_farm_batch_workspace_bytes(const raftk_designs *d, const raftk_cases *c, const raftk_farm_batch *f);
int raftk_farm_batch_response_ws_dev(const raftk_designs *d, const raftk_cases *c, const raftk_outputs *solved,
                                     const raftk_farm_batch *f, void *workspace, size_t workspace_bytes, void *stream);
int raftk_solve_dynamics_farm_batch_host(const raftk_designs *d, const raftk_cases *c, const raftk_solve_opts *o,
                                         const raftk_outputs *out, const raftk_farm_batch *f);

/*
 * Ragged farm batches (array-size studies: 4-, 6- and 9-turbine clusters, or how many turbines a lease area takes, in one
 * call): n_farms farms of N_f FOWTs each, N_f = farm_fowt0[f + 1] - farm_fowt0[f].  The designs of the batch are every farm's
 * FOWTs in order, farm after farm; all farms share the case table, frequency grid, depth and rho.  Each farm is assembled and
 * solved exactly as raftk_farm or a uniform batch of its N solves it alone: its Xi_sys and info are bit-identical.
 * Farms go to the kernel a uniform batch picks for their N (k_farm_rows<12> for N = 2, k_farm_response's warp form for
 * 6N <= 24, its CTA form while the [6N][6N+1] system fits in shared memory, k_farm_response_global above); each class that
 * occurs gets one launch over its own farms, which read their first design, N and output / matrix offsets from a descriptor
 * table the entry writes at the head of the workspace.
 * farm_fowt0 [n_farms + 1], HOST: farm_fowt0[0] = 0, strictly increasing, farm_fowt0[n_farms] = designs.n_designs.
 * M_arr / B_arr / C_arr, any may be NULL: arr_shared = 1: one [6N,6N] set for every farm (only when every N_f is equal);
 *   arr_shared = 0: farm f's [6N_f,6N_f] matrix starts at arr_offset[f] doubles, arr_offset [n_farms + 1] HOST with
 *   arr_offset[0] = 0 and arr_offset[f + 1] - arr_offset[f] = 36 N_f^2 (NULL allowed when every matrix is NULL).
 * Xi_sys complex, flat: farm f's [nC, 6N_f, nw] block starts at 6 nC nw farm_fowt0[f] complex values (n_designs nC 6 nw in
 *   all); info [n_farms, nC, nw] or NULL: a zero pivot is flagged in its own farm's rows only.
 * raftk_farm_ragged_workspace_bytes: the descriptor table plus, when a farm needs k_farm_response_global, its slabs (one
 *   [6N_max][6N_max+1] per resident CTA, N_max the largest such farm, no more than that class's systems); 0 for a bad shape.
 *   A smaller workspace that holds the table and one slab gives the same results with fewer CTAs.
 * raftk_farm_ragged_response_ws_dev: `solved` holds the device outputs of raftk_solve_dynamics_dev on the same (d, c);
 *   farm_fowt0 / arr_offset stay on the host, everything else is device memory.  _host: host pointers everywhere.
 * RAFTK_EINVAL before any launch, with a named reason: n_farms < 1, no farm_fowt0, a CSR that does not start at 0, is not
 * increasing (an empty farm) or does not end at n_designs, arr_shared not 0 or 1, arr_shared = 1 with unequal N_f, matrix
 * offsets that do not match the farm sizes, no Xi_sys, a missing per-FOWT output (B_drag, F_drag, F_iner; F_BEM with BEM
 * excitation), more than 65535 cases or 65535 farms of one on-chip class, or a workspace without the table and one slab.
 */
typedef struct raftk_farm_ragged {
    int32_t n_farms;
    int32_t arr_shared;             /* 1: one M_arr/B_arr/C_arr for every farm (equal N_f only); 0: CSR by arr_offset */
    const int32_t *farm_fowt0;      /* HOST [n_farms + 1] */
    const int64_t *arr_offset;      /* HOST [n_farms + 1] doubles, or NULL (arr_shared = 1, or no matrices) */
    const double *M_arr, *B_arr, *C_arr;
    double *Xi_sys;
    int32_t *info;
} raftk_farm_ragged;

size_t raftk_farm_ragged_workspace_bytes(const raftk_designs *d, const raftk_cases *c, const raftk_farm_ragged *f);
int raftk_farm_ragged_response_ws_dev(const raftk_designs *d, const raftk_cases *c, const raftk_outputs *solved,
                                      const raftk_farm_ragged *f, void *workspace, size_t workspace_bytes, void *stream);
int raftk_solve_dynamics_farm_ragged_host(const raftk_designs *d, const raftk_cases *c, const raftk_solve_opts *o,
                                          const raftk_outputs *out, const raftk_farm_ragged *f);

/*
 * Ragged farm batches sharded over GPUs (raft_b200.sweep.ShardedFarmSolve(farm_sizes=...)): rank r solves a contiguous run of
 * whole farms, farms [farm_row0, farm_row0 + f->n_farms) of the n_farms_total, whose FOWTs are designs [fowt_row0,
 * fowt_row0 + d->n_designs) of the whole batch, and stores their results at their global offsets of EVERY rank's copy (no
 * padding).  Rank p's copy holds
 *     gathered[p]: complex Xi_sys, flat as raftk_farm_ragged's (n_ranks * peers.block_elems >= 6 nC nw n_designs_total)
 *     status[p]:   int32 info [n_farms_total, nC, nw], followed by the per-FOWT status [n_designs_total, nC, 4]
 * f describes this rank's farms (farm_fowt0 from 0, arr_offset from 0); f->Xi_sys and f->info must be their rows of this
 * rank's own copy.  The farms are solved as raftk_farm_ragged_response_ws_dev solves them (same bits), then k_farm_publish
 * copies the rank's three contiguous runs (Xi_sys, info, status) to the other copies; follow with raftk_peer_barrier_dev.
 * RAFTK_EINVAL before any launch, besides every refusal of raftk_farm_ragged_response_ws_dev: a bad raftk_peers, no info or
 * per-FOWT status, a rank's status pointer missing, farm rows outside [0, n_farms_total), copies too small for this rank's
 * FOWTs, and Xi_sys / info that are not this rank's rows of its own copy.
 */
int raftk_farm_ragged_response_gather_dev(const raftk_designs *d, const raftk_cases *c, const raftk_outputs *solved,
                                          const raftk_farm_ragged *f, const raftk_peers *peers, int32_t farm_row0, int32_t fowt_row0,
                                          int32_t n_farms_total, void *workspace, size_t workspace_bytes, void *stream);

/*
 * Farm batches sharded over GPUs (raft_b200.sweep.ShardedFarmSolve): rank r solves a contiguous run of whole farms and stores
 * their results into EVERY rank's gathered copy (raftk_peers above); a farm is never split across ranks.  F_max is the largest
 * shard: smaller shards leave their last farm slots unwritten.  Rank p's copy holds
 *     gathered[p]: complex Xi_sys [n_ranks * F_max, nC, 6N, nw]    (peers.block_elems = F_max * nC * 6N * nw)
 *     status[p]:   int32 info [n_ranks * F_max, nC, nw], followed by the per-FOWT status [n_ranks * F_max * N, nC, 4]
 *     flags[p]:    the arrival flags of raftk_peer_barrier_dev.
 * raftk_farm_batch_response_gather_dev is raftk_farm_batch_response_ws_dev for this rank's f->n_farms farms, which are farms
 * [farm_row0, farm_row0 + n_farms) of the gathered copies (farm_row0 = rank * F_max); f->Xi_sys and f->info must be those rows of
 * this rank's own copy, and `solved` must carry the per-FOWT status of raftk_solve_dynamics_dev.  The farms are solved as
 * raftk_farm_batch_response_ws_dev solves them, then a second kernel, k_farm_publish, copies the rank's Xi_sys, info and
 * per-FOWT status rows to the other ranks' copies (and the status rows to its own), so a call makes two launches whatever the
 * farm size; the results are identical to raftk_farm_batch_response_ws_dev's, bit for bit.  Follow with
 * raftk_peer_barrier_dev; a rank without farms (more ranks than farms) calls only the barrier.
 * RAFTK_EINVAL before any launch, besides every refusal of raftk_farm_batch_response_ws_dev: NULL peers, n_ranks outside
 * [1, RAFTK_MAX_PEERS] or rank outside [0, n_ranks), a rank's gathered / flags / status pointer missing, no info or per-FOWT
 * status, block_elems not a positive multiple of nC * 6N * nw, n_farms > F_max, farm_row0 other than rank * F_max, and
 * Xi_sys / info that are not this rank's rows of its own copy.
 */
int raftk_farm_batch_response_gather_dev(const raftk_designs *d, const raftk_cases *c, const raftk_outputs *solved,
                                         const raftk_farm_batch *f, const raftk_peers *peers, int32_t farm_row0, void *workspace,
                                         size_t workspace_bytes, void *stream);

/*
 * Output channels of farm batches: mooring line tensions (the array level of Model.analyzeCases, raft_model.py:371-433, and
 * a FOWT's own lines, raft_fowt.py:2355-2399, moorMod 0) and any other real linear functional of the coupled response,
 *   Y[f,r,ch,w] = w^wpow[ch] sum_b R_f[ch,b] Xi_sys[f,r,b,w]
 * -> std = sqrt(1/2 sum_w |Y|^2), PSD(w) = 1/2 |Y|^2 / dw, amp = Y, for n_farms farms x n_rows rows (cases or wave trains)
 * x n_ch channels.  Tensions: R = dT/dx, the line-end tension Jacobian (MoorPy getCoupledStiffness(tensions=True)[1]).
 * dw is a parameter because the reference's Tmoor_PSD divides by w[0], not by the bin width w[1] - w[0]; pass w[0] to match it.
 * Every std, PSD and amplitude is bit-identical to raftk_general_channel_stats_* on the same R and Xi (same per-bin
 * summation order, same reduction), and a farm's values do not depend on the batch it is in or on the tile width.
 * Xi_sys complex [n_farms, n_rows, n_dof, nw] (raftk_farm_batch's output, n_dof = 6N); w [nw] (may be NULL when every wpow
 * is 0).  std [n_farms, n_rows, n_ch]; psd [n_farms, n_rows, n_ch, nw] or NULL; amp complex [n_farms, n_rows, n_ch, nw] or NULL.
 * Kernels: one CTA per (farm, row, bin tile) stages the tile of Xi_sys in shared memory and computes every channel from it
 * (bins per tile from n_dof and the opt-in shared-memory limit; Xi_sys is read from L2 when not even one bin fits), then one
 * CTA per (farm, row, channel) reduces over frequency.  |Y|^2 passes through psd, or through the workspace when psd is NULL:
 * raftk_farm_channel_stats_workspace_bytes is 0 with psd, else n_farms * n_rows * n_ch * nw doubles.
 * _dev: device R, Xi_sys, w and outputs, caller-owned workspace, enqueued on `stream` without synchronising.  _host: host
 * pointers everywhere.  wpow is HOST memory in both, read during the call.
 * RAFTK_EINVAL before any launch: a count below 1, more than RAFTK_FARM_CH_MAX channels, R_shared not 0 or 1, a wpow
 * outside {0, 1, 2}, NULL R, Xi_sys or std, no w while a wpow is not 0, dw <= 0, or (_dev) a workspace that is too small.
 */
#define RAFTK_FARM_CH_MAX 4096
#define RAFTK_FARM_TILE_L2 (-1)
typedef struct raftk_farm_channels {
    int32_t n_ch;
    int32_t R_shared;        /* 1: R [n_ch, n_dof] for every farm; 0: R [n_farms, n_ch, n_dof]                     */
    const double *R;
    const int32_t *wpow;     /* HOST [n_ch] 0, 1 or 2 (displacement, velocity, acceleration), or NULL: all 0      */
    double dw;               /* PSD divisor (> 0)                                                                  */
    double *std, *psd, *amp;
    int32_t tile_w;          /* 0: automatic; > 0: at most tile_w bins per CTA; RAFTK_FARM_TILE_L2: read Xi_sys from L2 */
    int32_t _pad0;
} raftk_farm_channels;

size_t raftk_farm_channel_stats_workspace_bytes(int32_t n_farms, int32_t n_rows, int32_t nw, const raftk_farm_channels *ch);
int raftk_farm_channel_stats_dev(int32_t n_farms, int32_t n_rows, int32_t n_dof, int32_t nw, const double *w, const double *Xi_sys,
                                 const raftk_farm_channels *ch, void *workspace, size_t workspace_bytes, void *stream);
int raftk_farm_channel_stats_host(int32_t n_farms, int32_t n_rows, int32_t n_dof, int32_t nw, const double *w, const double *Xi_sys,
                                  const raftk_farm_channels *ch);

/*
 * Channels of a ragged farm batch (raftk_farm_ragged's flat Xi_sys): farm f has n_dof_f = 6 N_f, N_f = farm_fowt0[f + 1] -
 * farm_fowt0[f], and channels [ch0[f], ch0[f + 1]) of the n_ch = ch0[n_farms] in all.  farm_fowt0 and ch0 are HOST arrays
 * starting at 0 and strictly increasing.  ch->R packs every R_f [n_ch_f, n_dof_f] farm after farm (R_shared must be 0); wpow
 * [n_ch] as the uniform entry's.  Outputs farm after farm: std [n_rows, n_ch_f] at n_rows ch0[f], psd / amp [n_rows, n_ch_f, nw]
 * at n_rows ch0[f] nw.  Each farm's values are bit-identical to raftk_farm_channel_stats_* on that farm alone.  The workspace
 * holds the farm descriptors (the query's 256-aligned head) and, without psd, |Y|^2.  Refusals: those of the uniform entry
 * plus a bad CSR, n_ch != ch0[n_farms] and R_shared != 0.
 */
size_t raftk_farm_ragged_channel_stats_workspace_bytes(int32_t n_farms, int32_t n_rows, int32_t nw, const int32_t *farm_fowt0,
                                                       const int32_t *ch0, const raftk_farm_channels *ch);
int raftk_farm_ragged_channel_stats_dev(int32_t n_farms, int32_t n_rows, int32_t nw, const int32_t *farm_fowt0, const int32_t *ch0,
                                        const double *w, const double *Xi_sys, const raftk_farm_channels *ch, void *workspace,
                                        size_t workspace_bytes, void *stream);
int raftk_farm_ragged_channel_stats_host(int32_t n_farms, int32_t n_rows, int32_t nw, const int32_t *farm_fowt0, const int32_t *ch0,
                                         const double *w, const double *Xi_sys, const raftk_farm_channels *ch);

/*
 * Rotor speed, generator torque and blade pitch statistics (FOWT.saveTurbineOutputs raft_fowt.py:2610-2679) for
 * n_units units (designs or farms) x n_cases cases x n_rot rotors.  Per (unit u, case c, rotor k) and row h of the case:
 *   y_h(w) = sum_b R[k,b] Xi[u, h, col0[k] + b, w]           (the hub row XiHub[h, ir], a real functional of the response)
 *   phi_h = C y_h for every row of the case, plus one wind row phi = -C V_w / (j w)   (:2643-2646)
 *   omega = j w phi, torque = (j w kp_tau + ki_tau) phi, bPitch = (j w kp_beta + ki_beta) phi   (:2649-2651)
 * std[u,c,k,:] = sqrt(1/2 sum_rows sum_w |.|^2) and psd[u,c,k,:,w] = 1/2 sum_rows |.|^2 / dw of (omega, torque, bPitch),
 * omega in rpm (/ 0.1047, the reference's radps2rpm; PSD times its square), torque in N m, bPitch in degrees (x
 * 57.29577951308232; PSD times its square).  A (case, rotor) with C = 0 and V_w = 0 gives exact zeros (the reference's
 * outputs when aeroServoMod <= 1 or the inflow speed is 0).  Means and bounds (omega_avg = Omega_case, avg +- 2 std, ...)
 * are the caller's.
 * Xi complex [n_units, n_rows, n_dof, nw]; the rows of case c are case_row0[c] .. case_row0[c+1]-1 (its wave trains).
 * w [nw], every bin > 0: the wind row divides by w, so a bin at w <= 0 has no finite value (the reference's grids start at
 * min_freq > 0); _host refuses such a w, _dev cannot read it and leaves NaN in that (unit, case, rotor)'s outputs.
 * One CTA per (unit, case, rotor); a result does not depend on which units, cases or rotors share the call.
 * _dev: device w, Xi, R, C, V_w, gains and outputs, enqueued on `stream` without synchronising.  _host: host pointers
 * everywhere.  col0 and case_row0 are HOST memory in both, read during the call.
 * RAFTK_EINVAL before any launch: a count below 1, n_r > n_dof, a col0 < 0 or col0 + n_r > n_dof, a case_row0 that does not
 * start at 0 or end at n_rows or has an empty or decreasing case, R_shared or tf_shared not 0 or 1, a NULL w, Xi, R, C, V_w,
 * gains, std, col0 or case_row0, dw <= 0, or (_host) a w <= 0.
 */
typedef struct raftk_rotor_outputs {
    int32_t n_cases, n_rot;
    int32_t n_r;               /* hub-row length: 6 for rigid FOWTs and farm FOWTs, n_dof for generalised DOFs        */
    int32_t R_shared;          /* 1: R [n_rot, n_r] for every unit; 0: R [n_units, n_rot, n_r]                      */
    int32_t tf_shared;         /* 1: C, V_w, gains [n_cases, n_rot, ...] for every unit; 0: [n_units, n_cases, n_rot, ...] */
    int32_t _pad0;
    const int32_t *col0;       /* HOST [n_rot]: first response column of each rotor's hub row                       */
    const int32_t *case_row0;  /* HOST [n_cases + 1]                                                                 */
    const double *R;
    const double *C, *V_w;     /* complex [..., nw]: control transfer function, turbulent-wind amplitudes          */
    const double *gains;       /* [..., 4]: kp_tau, ki_tau, kp_beta, ki_beta                                        */
    double dw;                 /* PSD divisor (> 0)                                                                 */
    double *std;               /* [n_units, n_cases, n_rot, 3]                                                       */
    double *psd;               /* [n_units, n_cases, n_rot, 3, nw] or NULL                                           */
} raftk_rotor_outputs;

int raftk_rotor_stats_dev(int32_t n_units, int32_t n_rows, int32_t n_dof, int32_t nw, const double *w, const double *Xi,
                          const raftk_rotor_outputs *ro, void *stream);
int raftk_rotor_stats_host(int32_t n_units, int32_t n_rows, int32_t n_dof, int32_t nw, const double *w, const double *Xi,
                           const raftk_rotor_outputs *ro);

/*
 * Fatigue damage-equivalent loads (DELs) by spectral methods, for n_units units (designs, farms or designs of a flexible
 * batch) x n_cases cases x n_ch channels.  Per (unit u, case c, channel ch), over the rows h of the case (its wave trains):
 *   real form:    Y_h(w) = w^wpow[ch] sum_b R[ch,b] Xi[u,h,b,w]          (as raftk_general_channel_stats / raftk_farm_channel_stats)
 *   complex form: Y_h(w) = sum_b coef[ch,b,w] Xi[u,h,b,w]                 (as raftk_channel_stats, e.g. a rigid tower's Mbase)
 *   moments lambda_k = sum_h sum_j w_j^k 1/2 |Y_h(w_j)|^2, k = 0, 1, 2, 4  (rad/s, one-sided; lambda_0 = std^2)
 * Dirlik (RAFTK_FATIGUE_DIRLIK): xm = (l1/l0) sqrt(l2/l4), g = l2 / sqrt(l0 l4), E[P] = sqrt(l4/l2) / 2 pi,
 *   D1 = 2 (xm - g^2) / (1 + g^2), R = (g - xm - D1^2) / (1 - g - D1 + D1^2), D2 = (1 - g - D1 + D1^2) / (1 - R),
 *   D3 = 1 - D1 - D2, Q = 1.25 (g - D3 - D2 R) / D1,
 *   E[S^m] = (2 sqrt(l0))^m [D1 Q^m Gamma(1+m) + 2^(m/2) Gamma(1+m/2) (D2 |R|^m + D3)],  d = E[P] E[S^m]  (S: stress range).
 * Narrow band (RAFTK_FATIGUE_NARROWBAND, and Dirlik's fallback): d = sqrt(l2/l0) / 2 pi (2 sqrt(2 l0))^m Gamma(1+m/2).
 * DEL[u,c,ch] = (d / f_eq)^(1/m[ch]); DEL_life[u,ch] = (sum_c p_c d_c / (f_eq sum_c p_c))^(1/m[ch]) with p = weights (NULL:
 * every case weighs 1).  No mean-stress correction; one S-N slope per channel.
 * info[u,c,ch]: RAFTK_FATIGUE_ZERO when l0 or l2 is 0 (DEL exactly 0: e.g. a rotor channel at wind 0, a zero Jacobian row);
 * RAFTK_FATIGUE_NARROWBAND when the narrow-band form gave the value -- requested, or a Dirlik request with
 * 1 - g < RAFTK_FATIGUE_NB_SWITCH, a D1, Q or R that is not finite and positive (the narrow-band limit g -> 1, D1 -> 0,
 * R = 0/0; a single-bin spectrum) or D2 |R|^m + D3 <= 0.  Across the switch the DEL moves by less than 1e-6 relative.
 * d is evaluated in the log domain (lgamma, m log(2 sqrt(l0))) and exponentiated after the 1/m root, so a DEL is finite
 * whenever it is representable, also for large loads and exponents; DEL_life sums p_c d_c scaled by its largest term.
 * Xi complex [n_units, n_rows, n_dof, nw]; w [nw] rad/s.  Exactly one of R (R_shared 1: [n_ch, n_dof]; 0: [n_units, n_ch,
 * n_dof]) and coef (complex; coef_mode RAFTK_FATIGUE_COEF_SHARED [n_ch, n_dof, nw], _UNIT [n_units, n_ch, n_dof, nw], _ROW
 * [n_units, n_rows, n_ch, n_dof, nw]) is given.  Outputs: moments [n_units, n_cases, n_ch, 4] (l0, l1, l2, l4) or NULL,
 * DEL and info [n_units, n_cases, n_ch], DEL_life [n_units, n_ch] or NULL.
 * Kernels: one CTA per (unit, row, bin tile) stages the tile of Xi in shared memory (read from L2 when not even 32 bins fit)
 * and reduces each channel's moments per 32-bin chunk with a fixed warp tree into the workspace; one thread per (unit, case,
 * channel) sums the chunks in order and applies the closed form; one thread per (unit, channel) sums the cases.  No
 * atomics: a result does not depend on the batch, the other cases or channels, or the tile width.  FP64 throughout.
 * raftk_fatigue_workspace_bytes: n_units * n_rows * ceil(nw / 32) * n_ch * 4 doubles, plus n_units * n_cases * n_ch doubles
 * with DEL_life.
 * _dev: device Xi, w, R / coef and outputs, caller-owned workspace (32-byte aligned), enqueued on `stream`; it allocates
 * nothing and never synchronises.  _host: host pointers everywhere, staged through the device arena.  case_row0, wpow, m and weights are HOST
 * memory in both, read during the call.
 * RAFTK_EINVAL before any launch: a count below 1, more than RAFTK_FATIGUE_CH_MAX channels, not exactly one of R and coef,
 * R_shared not 0 or 1, an unknown coef_mode or method, a wpow outside {0, 1, 2}, a NULL w, Xi, m, case_row0, DEL or info, a
 * case_row0 that does not start at 0 or end at n_rows or has an empty or decreasing case, an m that is not finite and > 0,
 * an f_eq that is not finite and > 0, a negative or non-finite weight or all-zero weights, or (_dev) a workspace that is too small
 * or not 32-byte aligned.
 */
#define RAFTK_FATIGUE_CH_MAX 4096
#define RAFTK_FATIGUE_NB_SWITCH 1e-6
enum { RAFTK_FATIGUE_DIRLIK = 0, RAFTK_FATIGUE_NARROWBAND_METHOD = 1 };
enum { RAFTK_FATIGUE_ZERO = 1, RAFTK_FATIGUE_NARROWBAND = 2 };
enum { RAFTK_FATIGUE_COEF_SHARED = 0, RAFTK_FATIGUE_COEF_UNIT = 1, RAFTK_FATIGUE_COEF_ROW = 2 };
typedef struct raftk_fatigue {
    int32_t n_cases, n_ch;
    int32_t method;            /* RAFTK_FATIGUE_DIRLIK or RAFTK_FATIGUE_NARROWBAND_METHOD                                */
    int32_t tile_w;            /* 0: automatic; > 0: at most tile_w bins per CTA (whole 32-bin chunks); RAFTK_FARM_TILE_L2 */
    const int32_t *case_row0;  /* HOST [n_cases + 1]                                                                    */
    const double *R;           /* real form, or NULL                                                                    */
    const int32_t *wpow;       /* HOST [n_ch] 0, 1 or 2, or NULL: all 0 (real form only)                                */
    const double *coef;        /* complex form, or NULL                                                                 */
    int32_t R_shared, coef_mode;
    const double *m;           /* HOST [n_ch] Woehler exponents                                                          */
    const double *weights;     /* HOST [n_cases] or NULL                                                                 */
    double f_eq;               /* equivalent frequency (Hz), e.g. 1 for the 1 Hz DEL                                     */
    double *moments, *DEL;
    int32_t *info;
    double *DEL_life;
} raftk_fatigue;

size_t raftk_fatigue_workspace_bytes(int32_t n_units, int32_t n_rows, int32_t nw, const raftk_fatigue *fa);
int raftk_fatigue_dev(int32_t n_units, int32_t n_rows, int32_t n_dof, int32_t nw, const double *w, const double *Xi,
                      const raftk_fatigue *fa, void *workspace, size_t workspace_bytes, void *stream);
int raftk_fatigue_host(int32_t n_units, int32_t n_rows, int32_t n_dof, int32_t nw, const double *w, const double *Xi,
                       const raftk_fatigue *fa);

/*
 * Tower-base axial stress around the circumference (the reference's helpers.getSigmaXPSD, helpers.py:1164), for n_units units
 * x n_cases cases x n_rings rings (tower bases) x n_angles angles.  Per (unit u, case c, ring), over the rows h of the case, the
 * fore-aft moment a_h and the side-side moment b_h in the channel forms of raftk_fatigue (ring k's channels read the n_r columns
 * col0[k] .. col0[k] + n_r - 1 of Xi, e.g. 6 i for FOWT i of a farm's Xi_sys):
 *   real form:    a_h(w) = w^wpow[k,0] sum_j R[k,0,j] Xi[u,h,col0[k]+j,w], b_h the same with row 1
 *   complex form: a_h(w) = sum_j coef[k,0,j,w] Xi[u,h,col0[k]+j,w], b_h the same with row 1
 * n_ch = 1 gives the fore-aft moment only (b = 0: a rigid tower's Mbase, which has no side-side moment).  Thin-wall section:
 *   Izz = pi/8 t d^3, c = (d/2) / Izz / 1e6, sigma_h(theta, w) = c (a_h cos theta - b_h sin theta)  (MPa for N m and m)
 *   S_xy,k = sum_h sum_j w_j^k 1/2 Re(x_h conj(y_h)) for xy = aa, bb, ab and k = 0, 1, 2, 4
 *   lambda_k(theta) = c^2 (cos^2 S_aa,k - 2 sin cos S_ab,k + sin^2 S_bb,k)
 *   std = sqrt(lambda_0), avg = c (cos theta mean_a - sin theta mean_b), max / min = avg +- 3 std
 *   DEL (m > 0): raftk_fatigue's closed form on lambda_k(theta) (Dirlik, narrow band as the fallback or on request, f_eq),
 *     info as raftk_fatigue's; DEL_life (weights or not) as raftk_fatigue's DEL_life, per angle.
 *   hot [.., 6] = {angle of the largest std on the grid, that std, angle of the largest DEL, that DEL (0, 0 without m), the
 *     largest std over the whole circle c sqrt(mu) with mu the larger eigenvalue of [[S_aa,0, S_ab,0], [S_ab,0, S_bb,0]], its
 *     angle in [0, pi)}; ties go to the first angle.  hot_life [.., 2] = {angle of the largest DEL_life, that DEL_life}.
 *   psd (optional, output-bound): per bin sum_h 1/2 |sigma_h(theta, w)|^2 / dw.
 * Xi complex [n_units, n_rows, n_dof, nw]; w [nw] rad/s.  Exactly one of R (R_shared 1: [n_rings, n_ch, n_r]; 0: [n_units,
 * n_rings, n_ch, n_r]) and coef (complex; coef_mode RAFTK_FATIGUE_COEF_SHARED [n_rings, n_ch, n_r, nw], _UNIT [n_units, ...],
 * _ROW [n_units, n_rows, ...]).  mean [n_units, n_cases, n_rings, n_ch] (device) or NULL (0).  Outputs [n_units, n_cases,
 * n_rings, n_angles]: std, avg, max, min (required), DEL and info (required with m > 0); hot [n_units, n_cases, n_rings, 6] or
 * NULL; DEL_life [n_units, n_rings, n_angles] and hot_life [n_units, n_rings, 2] or NULL; psd [n_units, n_cases, n_rings,
 * n_angles, nw] or NULL.  Kernels: one CTA per (unit, row, bin tile) forms the twelve sums per 32-bin chunk into the
 * workspace; one thread per (unit, case, ring, angle) sums them in (row, chunk) order and finishes; one thread per (unit, case,
 * ring) finds the hot spot.  No atomics: a result does not depend on the batch, the other cases, rings or angles, or the tile
 * width.  FP64 throughout.
 * raftk_stress_ring_workspace_bytes: n_units * n_rows * ceil(nw / 32) * n_rings * 12 doubles, plus n_units * n_cases *
 * n_rings * n_angles doubles with DEL_life.
 * _dev: device Xi, w, R / coef, mean and outputs, caller-owned workspace (32-byte aligned), enqueued on `stream`; it
 * allocates nothing and never synchronises.  _host: host pointers everywhere, staged through the device arena.  case_row0,
 * col0, wpow, angles and weights are HOST memory in both, read during the call.
 * RAFTK_EINVAL before any launch: a count below 1, n_ch not 1 or 2, more than RAFTK_STRESS_RING_MAX rings or
 * RAFTK_STRESS_ANGLE_MAX angles, n_r above n_dof, a col0 outside [0, n_dof - n_r], not exactly one of R and coef, R_shared not 0
 * or 1, an unknown coef_mode or method, a wpow outside {0, 1, 2}, a NULL w, Xi, angles, case_row0, std, avg, max or min, an
 * angle that is not finite, a d or t that is not finite and > 0, an m that is not 0 or finite and > 0, m > 0 without DEL and
 * info, DEL_life without m, hot_life without DEL_life, psd without a finite dw > 0, an f_eq that is not finite and > 0, a
 * case_row0 as raftk_fatigue refuses it, weights as raftk_fatigue refuses them, or (_dev) a workspace that is too small or
 * not 32-byte aligned.
 */
#define RAFTK_STRESS_RING_MAX 64
#define RAFTK_STRESS_ANGLE_MAX 256
typedef struct raftk_stress_ring {
    int32_t n_cases, n_rings, n_ch, n_r, n_angles;
    int32_t method;            /* RAFTK_FATIGUE_DIRLIK or RAFTK_FATIGUE_NARROWBAND_METHOD                                */
    int32_t tile_w;            /* 0: automatic; > 0: at most tile_w bins per CTA (whole 32-bin chunks); RAFTK_FARM_TILE_L2 */
    int32_t R_shared, coef_mode, _pad0;
    const int32_t *case_row0;  /* HOST [n_cases + 1]                                                                    */
    const int32_t *col0;       /* HOST [n_rings] or NULL: all 0                                                          */
    const int32_t *wpow;       /* HOST [n_rings, n_ch] 0, 1 or 2, or NULL: all 0 (real form only)                        */
    const double *R, *coef;
    const double *angles;      /* HOST [n_angles] rad                                                                    */
    double d, t;               /* tower-base diameter and wall thickness (m)                                            */
    double m;                  /* Woehler exponent, or 0: no DEL                                                         */
    double f_eq;               /* equivalent frequency (Hz) of the DEL                                                   */
    double dw;                 /* PSD divisor (with psd)                                                                 */
    const double *weights;     /* HOST [n_cases] or NULL                                                                 */
    const double *mean;
    double *std, *avg, *max, *min, *DEL;
    int32_t *info;
    double *hot, *DEL_life, *hot_life, *psd;
} raftk_stress_ring;

size_t raftk_stress_ring_workspace_bytes(int32_t n_units, int32_t n_rows, int32_t nw, const raftk_stress_ring *sr);
int raftk_stress_ring_dev(int32_t n_units, int32_t n_rows, int32_t n_dof, int32_t nw, const double *w, const double *Xi,
                          const raftk_stress_ring *sr, void *workspace, size_t workspace_bytes, void *stream);
int raftk_stress_ring_host(int32_t n_units, int32_t n_rows, int32_t n_dof, int32_t nw, const double *w, const double *Xi,
                           const raftk_stress_ring *sr);

/*
 * Natural frequencies and mode shapes (Model.solveEigen raft_model.py:436-547, FOWT.solveEigen raft_fowt.py:1646-1729): the
 * eigenvalues and right eigenvectors of M^-1 C for n_systems systems of n DOFs, what np.linalg.eig(np.linalg.solve(M, C))
 * returns, in the reference's output order.  Per system: LU of M with partial pivoting, A = M^-1 C, power-of-two balancing,
 * Householder Hessenberg reduction, Francis double-shift QR (at most 30 n iterations), eigenvectors by back-substitution on
 * the real Schur form, un-balanced and scaled to unit 2-norm; a complex vector is rotated so that its largest component is
 * real.  FP64 throughout.
 * sort RAFTK_EIG_SORT_DOF: rows n-1..0 of |V| each claim the column of their largest entry (first index on a tie; a claimed
 * column is zeroed and the search repeated), the claims reversed (raft_model.py:490-516).  A row that claims nothing leaves
 * NaN in the last slot(s) of lam and modes, where the reference returns fewer modes.
 * sort RAFTK_EIG_SORT_ASCENDING: by real part, then imaginary part (np.argsort of complex values); ties keep LAPACK's order.
 * Kernels: n <= 12 one system per thread (k_eig_small, no workspace); n > 12 one system per CTA (k_eig_cta), persistent CTAs
 * with Q and the back-substitution in a per-CTA workspace slab, H in shared memory while it fits the opt-in limit (n up to
 * 167 on an H100) and in the slab beyond.  A system's outputs do not depend on the batch or the workspace size.
 * info flags per system: RAFTK_EIG_SMALL_DIAG a diagonal of M or C below 1 (the reference's viability check, on the inputs);
 * RAFTK_EIG_NONPOSITIVE an eigenvalue with real part <= 0; RAFTK_EIG_COMPLEX a complex eigenvalue (informational);
 * RAFTK_EIG_SINGULAR an exactly zero pivot of M; RAFTK_EIG_NOCONV the QR iteration did not converge.  The last two leave
 * NaN in the system's lam and modes.  fns = sqrt(lam) / 2 pi is left to the caller.
 * raftk_eigen_workspace_bytes: 0 for n <= 12, else whole slabs: one per resident CTA, at most one per system (without a
 * device it answers for an H100).  Fewer bytes run fewer CTAs with the same results.
 * RAFTK_EINVAL before any launch: n < 1, n_systems < 1, an unknown sort, a NULL M, C, lam or info, n too large for the
 * per-system vectors in shared memory, or less than one slab of workspace when one is needed.
 */
enum { RAFTK_EIG_SORT_DOF = 0, RAFTK_EIG_SORT_ASCENDING = 1 };
enum { RAFTK_EIG_SMALL_DIAG = 1, RAFTK_EIG_NONPOSITIVE = 2, RAFTK_EIG_COMPLEX = 4, RAFTK_EIG_SINGULAR = 8, RAFTK_EIG_NOCONV = 16 };
typedef struct raftk_eigen {
    int32_t n_systems, n, sort, _pad0;
    const double *M, *C;   /* [n_systems, n, n] row-major                                    */
    double *lam;           /* complex [n_systems, n]: eigenvalues of M^-1 C in output order    */
    double *modes;         /* complex [n_systems, n, n] (column j = mode j) or NULL            */
    int32_t *info;         /* [n_systems] RAFTK_EIG_* flags                                    */
} raftk_eigen;
size_t raftk_eigen_workspace_bytes(const raftk_eigen *e);
int raftk_eigen_dev(const raftk_eigen *e, void *workspace, size_t workspace_bytes, void *stream);
int raftk_eigen_host(const raftk_eigen *e);

/*
 * Response statistics of FOWT.saveTurbineOutputs (raft_fowt.py:2299-2353) as reductions over Xi:
 * for every unit (design, case) and DOF   std = sqrt(1/2 sum_w |Xi|^2)   (helpers.getRMS, helpers.py:678-684)
 * and, if psd != NULL,                    PSD(w) = 1/2 |Xi(w)|^2 / dw    (helpers.getPSD, helpers.py:687-700).
 * Rotational DOFs (3..5) are converted to degrees first when rot_deg != 0, like the reference's roll/pitch/yaw.
 * Xi complex [n_units,6,nw] -> std [n_units,6], psd [n_units,6,nw].
 */
int raftk_response_stats_dev(int32_t n_units, int32_t nw, double dw, int32_t rot_deg, const double *Xi,
                             double *std, double *psd, void *stream);
int raftk_response_stats_host(int32_t n_units, int32_t nw, double dw, int32_t rot_deg, const double *Xi,
                              double *std, double *psd);

/*
 * Output channels of FOWT.saveTurbineOutputs beyond the platform DOFs -- nacelle accelerations
 * (raft_fowt.py:2401-2444) and the tower-base fore-aft bending moment of a rigid tower (:2504-2538).  Each is a
 * linear functional of the response, Y_ch(w) = sum_dof coef[ch,dof,w] Xi[dof,w]  (e.g. AxRNA: w^2 times the hub
 * node's row of fowt.T; Mbase: m hArm w^2 (Xi_0 + zCG Xi_4) + (ICG w^2 + m g hArm + aero reaction) Xi_4), so the
 * caller packs the turbine constants into coef once per design (raft_b200.packer.pack_turbine_channels) and gets
 *   std = sqrt(1/2 sum_w |Y|^2) (helpers.getRMS),  PSD(w) = 1/2 |Y|^2 / dw (helpers.getPSD),  amp = Y (optional).
 * coef complex [n_designs,n_ch,6,nw]; Xi complex [n_designs,n_cases,6,nw] -> std [n_designs,n_cases,n_ch],
 * psd [n_designs,n_cases,n_ch,nw] or NULL, amp complex [n_designs,n_cases,n_ch,nw] or NULL.
 */
int raftk_channel_stats_dev(int32_t n_designs, int32_t n_cases, int32_t n_ch, int32_t nw, double dw, const double *coef,
                            const double *Xi, double *std, double *psd, double *amp, void *stream);
int raftk_channel_stats_host(int32_t n_designs, int32_t n_cases, int32_t n_ch, int32_t nw, double dw, const double *coef,
                             const double *Xi, double *std, double *psd, double *amp);

/* Pinned host memory for the *_host paths and the e2e benchmark (cudaHostAlloc / cudaFreeHost). */
void *raftk_host_alloc(size_t bytes);
void raftk_host_free(void *p);

/* FP64 FMA micro-benchmark: returns achieved GFLOP/s on the current device (roofline denominator). */
double raftk_fp64_peak_gflops(int iters);

/*
 * Native node-table builder for a FAMILY of designs on one topology (a design sweep, the reference's parametersweep.py:29-95):
 * what Member.__init__ / setPosition / calcHydroConstants / calcImat (raft_member.py:190-271, 312-377, 1261-1448) and
 * FOWT.calcHydroConstants (raft_fowt.py:1589-1625) leave behind per design, written straight into the CSR tables of
 * raftk_designs.  Pure host code (no CUDA).  One raftk_family_member per member COPY (a member entry with several headings
 * appears once per heading); per-design geometry arrays have n_designs rows.  Rigid circular / rectangular members without
 * MacCamy-Fuchs tables.  raftk_family_sizes returns the totals the caller needs to allocate raftk_family_tables;
 * raftk_build_family_host fills them (error -1: an end point on the waterplane or stations not ascending, as the reference raises).
 */
typedef struct raftk_family_member {
    int32_t n_stations;        /* n                                                              */
    int32_t circular;          /* 1 circular (d [nD][n][1]), 0 rectangular (d [nD][n][2])      */
    int32_t pot_mod;           /* strips carry drag only (inertia from BEM)                      */
    int32_t _pad0;
    double gamma_deg, heading_deg, dls_max;
    const double *stations;    /* [n] as in the design file                                     */
    const double *rA, *rB;     /* [nD][3] end points before the heading rotation                */
    const double *d;           /* [nD][n][1 or 2]                                               */
    const double *Cd_q, *Cd_p1, *Cd_p2, *Cd_End, *Ca_p1, *Ca_p2, *Ca_End;   /* [n] per station  */
} raftk_family_member;

typedef struct raftk_family {
    int32_t n_designs, n_members;
    double rho, g;
    double Rp[9];              /* platform rotation (helpers.rotationMatrix of r6[3:6]), row-major */
    double r0[3];              /* platform reference point r6[0:3]                               */
    const raftk_family_member *members;
} raftk_family;

typedef struct raftk_family_tables {
    int32_t *member_offset;    /* [nD+1]                                                         */
    int32_t *mem_node_start;   /* [n_members_total+1]                                            */
    int32_t *mem_circ;         /* [n_members_total]                                              */
    double *mem_frame, *mem_rA, *mem_arm;      /* [n_members_total][9], [..][3], [..][3]        */
    double *node_ls, *node_cd_q, *node_cd_p1, *node_cd_p2, *node_in_q, *node_in_p1, *node_in_p2, *node_pa;   /* [n_nodes_total] */
    double *A_morison;         /* [nD][36]  A_hydro_morison about r0                             */
    int32_t max_nodes, max_members, max_w_classes, max_h_classes, max_z_classes, _pad0;        /* out */
} raftk_family_tables;

int raftk_family_sizes(const raftk_family *f, int32_t *n_members_total, int32_t *n_nodes_total);
int raftk_build_family_host(const raftk_family *f, raftk_family_tables *t);

#ifdef __cplusplus
}
#endif
#endif /* RAFTK_H */
