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
    int32_t _pad1;
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
} raftk_cases;

/* Fixed-point loop controls (raft_model.py:966 tol, :977 nIter, :978 XiStart, :1133 relaxation) */
typedef struct raftk_solve_opts {
    int32_t n_iter;          /* settings.nIter; the loop runs at most n_iter+1 passes           */
    int32_t cluster_size;    /* CTAs per (design,case): 0 = auto, else 1,2,4,8                  */
    double tol;              /* 0.01                                                            */
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
 * system-solve families clears it first; a call that fails before its launch leaves it cleared.  When one call launches
 * several families (a solve that computes its second-order force first, a farm host call) the last launch is reported.
 * Host bookkeeping only: no device work, no synchronisation.
 */
enum { RAFTK_FAMILY_NONE = 0, RAFTK_FAMILY_SOLVE = 1, RAFTK_FAMILY_QTF = 2, RAFTK_FAMILY_GENERAL = 3, RAFTK_FAMILY_FARM = 4,
       RAFTK_FAMILY_SYSTEM = 5 };
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
    RAFTK_KERNEL_GEN_UNBLOCKED = 10,  /* k_gen_solve                                                                      */
    RAFTK_KERNEL_FARM_ROWS12 = 11,    /* k_farm_rows<12>                                                                  */
    RAFTK_KERNEL_FARM_WARP = 12,      /* k_farm_response<true>                                                            */
    RAFTK_KERNEL_FARM_BLOCK = 13,     /* k_farm_response<false>                                                           */
    RAFTK_KERNEL_SYS_UNBLOCKED = 14,  /* k_system_solve, column-at-a-time LU (n <= 24)                                    */
    RAFTK_KERNEL_SYS_BLOCKED = 15,    /* k_system_solve, blocked LU (n > 24)                                              */
    RAFTK_KERNEL_FARM_GLOBAL = 16,    /* k_farm_response_global: system in a workspace slab, LU blocked in global memory   */
    RAFTK_KERNEL_SYS_GLOBAL = 17      /* k_system_solve_global: Z factored in place, LU blocked in global memory           */
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
    int32_t _pad0;
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
