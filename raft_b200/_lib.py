"""ctypes binding of libraftk.so (include/raftk.h).  No CPU fallback: if the CUDA library is not
built, importing this module raises -- the product path must fail loudly, never degrade.

The shared object is mapped on the first call into it (``lib.<symbol>``), not at import: the pure-NumPy
host helpers of the package (grid, packer, member builder) can then be imported by a process that must
not load CUDA code -- ``bench.py --impl reference`` -- while every product call still goes through
``lib`` and a missing file is an ImportError at import time."""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("RAFTK_LIB", os.path.join(HERE, "csrc", "libraftk.so"))   # RAFTK_LIB: A/B builds of the same ABI

c_double_p = C.POINTER(C.c_double)
c_int32_p = C.POINTER(C.c_int32)


class RaftkDesigns(C.Structure):
    _fields_ = [
        ("n_designs", C.c_int32), ("nw", C.c_int32), ("n_members_total", C.c_int32), ("n_nodes_total", C.c_int32),
        ("max_nodes", C.c_int32), ("max_members", C.c_int32), ("max_w_classes", C.c_int32), ("max_h_classes", C.c_int32), ("max_z_classes", C.c_int32), ("walk_exact", C.c_int32),
        ("depth", C.c_double), ("rho", C.c_double), ("g", C.c_double), ("dw", C.c_double),
        ("w", C.c_void_p), ("k", C.c_void_p), ("member_offset", C.c_void_p),
        ("mem_frame", C.c_void_p), ("mem_rA", C.c_void_p), ("mem_arm", C.c_void_p),
        ("mem_node_start", C.c_void_p), ("mem_circ", C.c_void_p),
        ("node_ls", C.c_void_p), ("node_cd_q", C.c_void_p), ("node_cd_p1", C.c_void_p), ("node_cd_p2", C.c_void_p),
        ("node_in_q", C.c_void_p), ("node_in_p1", C.c_void_p), ("node_in_p2", C.c_void_p), ("node_pa", C.c_void_p),
        ("node_in_p1_w", C.c_void_p), ("node_in_p2_w", C.c_void_p),
        ("M0", C.c_void_p), ("B0", C.c_void_p), ("C0", C.c_void_p), ("A_w", C.c_void_p), ("B_w", C.c_void_p),
        ("n_bem_head", C.c_int32), ("_pad0", C.c_int32),
        ("bem_headings", C.c_void_p), ("X_BEM", C.c_void_p), ("bem_xyh", C.c_void_p),
        ("n_qtf_w", C.c_int32), ("n_qtf_head", C.c_int32), ("qtf_shared", C.c_int32), ("_pad2", C.c_int32),
        ("qtf_w", C.c_void_p), ("qtf_heads", C.c_void_p), ("qtf", C.c_void_p),
        ("max_rotors", C.c_int32), ("_pad3", C.c_int32), ("rot_count", C.c_void_p), ("rot_r3", C.c_void_p), ("rot_G", C.c_void_p),
    ]


class RaftkCases(C.Structure):
    _fields_ = [
        ("n_cases", C.c_int32), ("_pad0", C.c_int32),
        ("Hs", C.c_void_p), ("Tp", C.c_void_p), ("gamma", C.c_void_p), ("beta_deg", C.c_void_p),
        ("spec", C.c_void_p), ("zeta", C.c_void_p), ("primary", C.c_void_p), ("F_2nd", C.c_void_p), ("Xi_init", C.c_void_p),
        ("op", C.c_void_p), ("n_op", C.c_int32), ("op_shared", C.c_int32), ("op_A_w", C.c_void_p), ("op_B_w", C.c_void_p),
    ]


class RaftkSolveOpts(C.Structure):
    _fields_ = [("n_iter", C.c_int32), ("cluster_size", C.c_int32), ("tol", C.c_double), ("xi_start", C.c_double),
                ("flags", C.c_int32), ("_pad0", C.c_int32)]


class RaftkOutputs(C.Structure):
    _fields_ = [("Xi", C.c_void_p), ("status", C.c_void_p), ("B_drag", C.c_void_p), ("F_drag", C.c_void_p),
                ("F_iner", C.c_void_p), ("F_BEM", C.c_void_p), ("zeta", C.c_void_p),
                ("F_2nd", C.c_void_p), ("F_2nd_mean", C.c_void_p), ("Xi_last", C.c_void_p)]


MAX_PEERS = 16


class RaftkPeers(C.Structure):
    """include/raftk.h raftk_peers: peer-mapped gathered arrays of the fused multi-GPU exchange."""
    _fields_ = [("n_ranks", C.c_int32), ("rank", C.c_int32), ("epoch", C.c_uint32), ("_pad0", C.c_int32),
                ("block_elems", C.c_size_t), ("gathered", C.c_void_p * MAX_PEERS), ("flags", C.c_void_p * MAX_PEERS),
                ("status", C.c_void_p * MAX_PEERS)]


class RaftkFarm(C.Structure):
    """include/raftk.h raftk_farm: array-level matrices and outputs of the coupled 6N-DOF system response."""
    _fields_ = [("n_fowt", C.c_int32), ("_pad0", C.c_int32), ("M_arr", C.c_void_p), ("B_arr", C.c_void_p), ("C_arr", C.c_void_p),
                ("Xi_sys", C.c_void_p), ("info", C.c_void_p)]


class RaftkFarmBatch(C.Structure):
    """include/raftk.h raftk_farm_batch: n_farms arrays of n_fowt FOWTs each, solved over one case table in one call."""
    _fields_ = [("n_farms", C.c_int32), ("n_fowt", C.c_int32), ("arr_shared", C.c_int32), ("_pad0", C.c_int32),
                ("M_arr", C.c_void_p), ("B_arr", C.c_void_p), ("C_arr", C.c_void_p), ("Xi_sys", C.c_void_p), ("info", C.c_void_p)]


class RaftkFarmRagged(C.Structure):
    """include/raftk.h raftk_farm_ragged: n_farms farms of their own N_f FOWTs each (farm_fowt0, arr_offset: host CSR arrays)."""
    _fields_ = [("n_farms", C.c_int32), ("arr_shared", C.c_int32), ("farm_fowt0", C.c_void_p), ("arr_offset", C.c_void_p),
                ("M_arr", C.c_void_p), ("B_arr", C.c_void_p), ("C_arr", C.c_void_p), ("Xi_sys", C.c_void_p), ("info", C.c_void_p)]


SLENDER_ARRAYS = ("w", "k", "mem_q", "mem_p1", "mem_p2", "mem_mcf", "mem_wl", "mem_r_int", "mem_a_wl", "mem_rwl", "mem_R_wl", "mem_node_start",
                  "node_r", "node_v_side", "node_Ca_p1", "node_Ca_p2", "node_Ca_End", "node_v_end", "node_a_i",
                  "seg_mem", "seg_z1", "seg_z2", "seg_R", "seg_rmid", "M_struc")


GENERAL_ARRAYS = ("w", "k", "node_r", "node_frame", "node_circ", "node_Imat", "node_Imat_w", "node_a_i", "node_cd", "Tn", "rr", "M", "B", "C")


class RaftkGeneral(C.Structure):
    """Generalised degrees of freedom (flexible members), include/raftk.h raftk_general."""
    _fields_ = ([("n_dof", C.c_int32), ("nw", C.c_int32), ("n_nodes", C.c_int32), ("_pad0", C.c_int32),
                 ("depth", C.c_double), ("rho", C.c_double), ("dw", C.c_double)] + [(n, C.c_void_p) for n in GENERAL_ARRAYS])


class RaftkGeneralFd(C.Structure):
    """Frequency-dependent terms of the generalised-DOF solve, include/raftk.h raftk_general_fd."""
    _fields_ = [("n_fd", C.c_int32), ("n_bem_head", C.c_int32), ("fd_idx", C.c_void_p), ("A_w", C.c_void_p), ("B_w", C.c_void_p),
                ("bem_headings", C.c_void_p), ("X_BEM", C.c_void_p), ("T0", C.c_void_p),
                ("x_ref", C.c_double), ("y_ref", C.c_double), ("heading_adjust", C.c_double)]


class RaftkGeneralQtf(C.Structure):
    """Second-order wave loads of the generalised-DOF solve, include/raftk.h raftk_general_qtf."""
    _fields_ = [("n_qtf_w", C.c_int32), ("n_qtf_head", C.c_int32), ("qtf_w", C.c_void_p), ("qtf_heads", C.c_void_p), ("qtf", C.c_void_p)]


class RaftkGeneralBatch(C.Structure):
    """A design batch of the generalised-DOF solve, include/raftk.h raftk_general_batch."""
    _fields_ = [("n_designs", C.c_int32), ("max_nodes", C.c_int32), ("qtf_shared", C.c_int32), ("_pad0", C.c_int32),
                ("node_offset", C.c_void_p), ("x_ref", C.c_void_p), ("y_ref", C.c_void_p), ("heading_adjust", C.c_void_p)]


class RaftkFarmChannels(C.Structure):
    """include/raftk.h raftk_farm_channels: channels Y = w^wpow R_f Xi_sys of farm batches (mooring tensions) and their outputs."""
    _fields_ = [("n_ch", C.c_int32), ("R_shared", C.c_int32), ("R", C.c_void_p), ("wpow", C.c_void_p), ("dw", C.c_double),
                ("std", C.c_void_p), ("psd", C.c_void_p), ("amp", C.c_void_p), ("tile_w", C.c_int32), ("_pad0", C.c_int32)]


class RaftkRotorOutputs(C.Structure):
    """include/raftk.h raftk_rotor_outputs: hub rows, control transfer functions and gains of rotors, and their statistics."""
    _fields_ = [("n_cases", C.c_int32), ("n_rot", C.c_int32), ("n_r", C.c_int32), ("R_shared", C.c_int32), ("tf_shared", C.c_int32),
                ("_pad0", C.c_int32), ("col0", C.c_void_p), ("case_row0", C.c_void_p), ("R", C.c_void_p), ("C", C.c_void_p),
                ("V_w", C.c_void_p), ("gains", C.c_void_p), ("dw", C.c_double), ("std", C.c_void_p), ("psd", C.c_void_p)]


class RaftkFatigue(C.Structure):
    """include/raftk.h raftk_fatigue: channels, S-N exponents and case weights of spectral fatigue DELs, and their outputs."""
    _fields_ = [("n_cases", C.c_int32), ("n_ch", C.c_int32), ("method", C.c_int32), ("tile_w", C.c_int32), ("case_row0", C.c_void_p),
                ("R", C.c_void_p), ("wpow", C.c_void_p), ("coef", C.c_void_p), ("R_shared", C.c_int32), ("coef_mode", C.c_int32),
                ("m", C.c_void_p), ("weights", C.c_void_p), ("f_eq", C.c_double), ("moments", C.c_void_p), ("DEL", C.c_void_p),
                ("info", C.c_void_p), ("DEL_life", C.c_void_p)]


class RaftkStressRing(C.Structure):
    """include/raftk.h raftk_stress_ring: tower-base moments, section, angles and S-N options of the circumferential axial
    stress, and its outputs."""
    _fields_ = [("n_cases", C.c_int32), ("n_rings", C.c_int32), ("n_ch", C.c_int32), ("n_r", C.c_int32), ("n_angles", C.c_int32),
                ("method", C.c_int32), ("tile_w", C.c_int32), ("R_shared", C.c_int32), ("coef_mode", C.c_int32), ("_pad0", C.c_int32),
                ("case_row0", C.c_void_p), ("col0", C.c_void_p), ("wpow", C.c_void_p), ("R", C.c_void_p), ("coef", C.c_void_p),
                ("angles", C.c_void_p), ("d", C.c_double), ("t", C.c_double), ("m", C.c_double), ("f_eq", C.c_double), ("dw", C.c_double),
                ("weights", C.c_void_p), ("mean", C.c_void_p), ("std", C.c_void_p), ("avg", C.c_void_p), ("max", C.c_void_p),
                ("min", C.c_void_p), ("DEL", C.c_void_p), ("info", C.c_void_p), ("hot", C.c_void_p), ("DEL_life", C.c_void_p),
                ("hot_life", C.c_void_p), ("psd", C.c_void_p)]


class RaftkEigen(C.Structure):
    """include/raftk.h raftk_eigen: eigenvalues and right eigenvectors of M^-1 C for a batch of systems."""
    _fields_ = [("n_systems", C.c_int32), ("n", C.c_int32), ("sort", C.c_int32), ("_pad0", C.c_int32),
                ("M", C.c_void_p), ("C", C.c_void_p), ("lam", C.c_void_p), ("modes", C.c_void_p), ("info", C.c_void_p)]


class RaftkSlender(C.Structure):
    _fields_ = ([("n_nodes", C.c_int32), ("n_members", C.c_int32), ("n_seg", C.c_int32), ("nw", C.c_int32),
                 ("depth", C.c_double), ("rho", C.c_double), ("g", C.c_double)] + [(n, C.c_void_p) for n in SLENDER_ARRAYS])


class RaftkSlenderBatch(C.Structure):
    """include/raftk.h raftk_slender_batch: the slender-body tables of several designs, concatenated (CSR offsets)."""
    _fields_ = [("n_designs", C.c_int32), ("max_nodes", C.c_int32), ("max_members", C.c_int32), ("max_seg", C.c_int32),
                ("node_offset", C.c_void_p), ("member_offset", C.c_void_p), ("seg_offset", C.c_void_p), ("cols", RaftkSlender)]


class RaftkSlenderOutputs(C.Structure):
    _fields_ = [("qtf", C.c_void_p), ("Xi_rao", C.c_void_p), ("qtf_chunk", C.c_int32), ("_pad0", C.c_int32)]


class RaftkDispatch(C.Structure):
    """include/raftk.h raftk_dispatch: the kernel variant the last call on this thread launched."""
    _fields_ = [(n, C.c_int32) for n in ("family", "kernel", "cluster_size", "bins_per_cta", "threads_per_cta", "f0_global", "direct_d2h",
                                         "trains", "chunks", "inexact_walk", "farm_classes")]


# every symbol include/raftk.h declares (tests/test_abi.py checks the header against this list)

class RaftkFamilyMember(C.Structure):
    """include/raftk.h raftk_family_member: one member copy of a design family (template constants + per-design geometry)."""
    _fields_ = [("n_stations", C.c_int32), ("circular", C.c_int32), ("pot_mod", C.c_int32), ("_pad0", C.c_int32),
                ("gamma_deg", C.c_double), ("heading_deg", C.c_double), ("dls_max", C.c_double),
                ("stations", C.c_void_p), ("rA", C.c_void_p), ("rB", C.c_void_p), ("d", C.c_void_p),
                ("Cd_q", C.c_void_p), ("Cd_p1", C.c_void_p), ("Cd_p2", C.c_void_p), ("Cd_End", C.c_void_p),
                ("Ca_p1", C.c_void_p), ("Ca_p2", C.c_void_p), ("Ca_End", C.c_void_p)]


class RaftkFamily(C.Structure):
    _fields_ = [("n_designs", C.c_int32), ("n_members", C.c_int32), ("rho", C.c_double), ("g", C.c_double),
                ("Rp", C.c_double * 9), ("r0", C.c_double * 3), ("members", C.POINTER(RaftkFamilyMember))]


class RaftkFamilyTables(C.Structure):
    _fields_ = [("member_offset", C.c_void_p), ("mem_node_start", C.c_void_p), ("mem_circ", C.c_void_p),
                ("mem_frame", C.c_void_p), ("mem_rA", C.c_void_p), ("mem_arm", C.c_void_p),
                ("node_ls", C.c_void_p), ("node_cd_q", C.c_void_p), ("node_cd_p1", C.c_void_p), ("node_cd_p2", C.c_void_p),
                ("node_in_q", C.c_void_p), ("node_in_p1", C.c_void_p), ("node_in_p2", C.c_void_p), ("node_pa", C.c_void_p),
                ("A_morison", C.c_void_p),
                ("max_nodes", C.c_int32), ("max_members", C.c_int32), ("max_w_classes", C.c_int32), ("max_h_classes", C.c_int32),
                ("max_z_classes", C.c_int32), ("_pad0", C.c_int32)]


SYMBOLS = [
    "raftk_version", "raftk_last_error", "raftk_launch_count", "raftk_last_dispatch", "raftk_profile_enable", "raftk_profile_read",
    "raftk_workspace_bytes", "raftk_solve_workspace_bytes",
    "raftk_hydro_excitation_dev", "raftk_hydro_linearization_dev", "raftk_solve_dynamics_dev",
    "raftk_hydro_excitation_host", "raftk_hydro_linearization_host", "raftk_solve_dynamics_host",
    "raftk_second_order_force_dev", "raftk_second_order_force_host",
    "raftk_qtf_slender_workspace_bytes", "raftk_qtf_slender_dev", "raftk_qtf_slender_host",
    "raftk_solve_dynamics_slender_workspace_bytes", "raftk_solve_dynamics_slender_dev", "raftk_solve_dynamics_slender_host",
    "raftk_general_workspace_bytes", "raftk_general_solve_dynamics_dev", "raftk_general_solve_dynamics_host",
    "raftk_general_fd_workspace_bytes", "raftk_general_solve_dynamics_fd_dev", "raftk_general_solve_dynamics_fd_host",
    "raftk_general_qtf_workspace_bytes", "raftk_general_solve_dynamics_qtf_dev", "raftk_general_solve_dynamics_qtf_host",
    "raftk_general_stream_workspace_bytes", "raftk_general_solve_dynamics_stream_dev", "raftk_general_solve_dynamics_stream_host",
    "raftk_general_batch_workspace_bytes", "raftk_general_batch_solve_dynamics_dev", "raftk_general_batch_solve_dynamics_host",
    "raftk_system_solve_dev", "raftk_system_solve_host", "raftk_response_stats_dev", "raftk_response_stats_host",
    "raftk_channel_stats_dev", "raftk_channel_stats_host", "raftk_general_channel_stats_dev", "raftk_general_channel_stats_host",
    "raftk_host_alloc", "raftk_host_free",
    "raftk_fp64_peak_gflops",
    "raftk_peer_alloc", "raftk_peer_free", "raftk_peer_open", "raftk_peer_close",
    "raftk_solve_dynamics_gather_dev", "raftk_peer_barrier_dev", "raftk_general_publish_dev",
    "raftk_farm_response_dev", "raftk_solve_dynamics_farm_host", "raftk_farm_workspace_bytes", "raftk_farm_response_ws_dev",
    "raftk_farm_batch_workspace_bytes", "raftk_farm_batch_response_ws_dev", "raftk_solve_dynamics_farm_batch_host",
    "raftk_farm_batch_response_gather_dev",
    "raftk_farm_ragged_workspace_bytes", "raftk_farm_ragged_response_ws_dev", "raftk_solve_dynamics_farm_ragged_host",
    "raftk_farm_ragged_response_gather_dev", "raftk_farm_ragged_channel_stats_workspace_bytes", "raftk_farm_ragged_channel_stats_dev",
    "raftk_farm_ragged_channel_stats_host",
    "raftk_family_sizes", "raftk_build_family_host",
    "raftk_eigen_workspace_bytes", "raftk_eigen_dev", "raftk_eigen_host",
    "raftk_farm_channel_stats_workspace_bytes", "raftk_farm_channel_stats_dev", "raftk_farm_channel_stats_host",
    "raftk_rotor_stats_dev", "raftk_rotor_stats_host",
    "raftk_fatigue_workspace_bytes", "raftk_fatigue_dev", "raftk_fatigue_host",
    "raftk_stress_ring_workspace_bytes", "raftk_stress_ring_dev", "raftk_stress_ring_host",
]


class RaftkError(RuntimeError):
    pass


def _require():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "raft_b200: CUDA library %s is missing. Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). There is no CPU fallback." % LIB_PATH)


def _load():
    _require()
    lib = C.CDLL(LIB_PATH)
    P = C.POINTER
    lib.raftk_version.restype = C.c_int
    lib.raftk_last_error.restype = C.c_char_p
    lib.raftk_launch_count.restype = C.c_longlong
    lib.raftk_last_dispatch.argtypes = [P(RaftkDispatch)]
    lib.raftk_last_dispatch.restype = C.c_int
    lib.raftk_profile_enable.argtypes = [C.c_int]
    lib.raftk_profile_read.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_int)]
    lib.raftk_profile_read.restype = C.c_int
    lib.raftk_workspace_bytes.restype = C.c_size_t
    lib.raftk_workspace_bytes.argtypes = [P(RaftkDesigns), C.c_int32]
    lib.raftk_solve_workspace_bytes.restype = C.c_size_t
    lib.raftk_solve_workspace_bytes.argtypes = [P(RaftkDesigns), C.c_int32]
    lib.raftk_hydro_excitation_dev.argtypes = [P(RaftkDesigns), P(RaftkCases), P(RaftkOutputs), C.c_void_p, C.c_size_t, C.c_void_p]
    lib.raftk_hydro_linearization_dev.argtypes = [P(RaftkDesigns), P(RaftkCases), C.c_void_p, P(RaftkOutputs), C.c_void_p, C.c_size_t, C.c_void_p]
    lib.raftk_solve_dynamics_dev.argtypes = [P(RaftkDesigns), P(RaftkCases), P(RaftkSolveOpts), P(RaftkOutputs), C.c_void_p, C.c_size_t, C.c_void_p]
    lib.raftk_hydro_excitation_host.argtypes = [P(RaftkDesigns), P(RaftkCases), P(RaftkOutputs)]
    lib.raftk_hydro_linearization_host.argtypes = [P(RaftkDesigns), P(RaftkCases), C.c_void_p, P(RaftkOutputs)]
    lib.raftk_solve_dynamics_host.argtypes = [P(RaftkDesigns), P(RaftkCases), P(RaftkSolveOpts), P(RaftkOutputs)]
    lib.raftk_second_order_force_dev.argtypes = [P(RaftkDesigns), P(RaftkCases), P(RaftkOutputs), C.c_void_p]
    lib.raftk_second_order_force_host.argtypes = [P(RaftkDesigns), P(RaftkCases), P(RaftkOutputs)]
    lib.raftk_qtf_slender_workspace_bytes.restype = C.c_size_t
    lib.raftk_qtf_slender_workspace_bytes.argtypes = [P(RaftkSlender), C.c_int32]
    lib.raftk_qtf_slender_dev.argtypes = [P(RaftkSlender), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    lib.raftk_qtf_slender_host.argtypes = [P(RaftkSlender), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.raftk_qtf_slender_dev.restype = C.c_int
    lib.raftk_qtf_slender_host.restype = C.c_int
    lib.raftk_solve_dynamics_slender_workspace_bytes.restype = C.c_size_t
    lib.raftk_solve_dynamics_slender_workspace_bytes.argtypes = [P(RaftkDesigns), P(RaftkSlenderBatch), C.c_int32, C.c_int32]
    lib.raftk_solve_dynamics_slender_dev.argtypes = [P(RaftkDesigns), P(RaftkSlenderBatch), P(RaftkCases), P(RaftkSolveOpts), P(RaftkOutputs),
                                                     P(RaftkSlenderOutputs), C.c_void_p, C.c_size_t, C.c_void_p]
    lib.raftk_solve_dynamics_slender_host.argtypes = [P(RaftkDesigns), P(RaftkSlenderBatch), P(RaftkCases), P(RaftkSolveOpts), P(RaftkOutputs),
                                                      P(RaftkSlenderOutputs)]
    lib.raftk_solve_dynamics_slender_dev.restype = C.c_int
    lib.raftk_solve_dynamics_slender_host.restype = C.c_int
    lib.raftk_general_workspace_bytes.restype = C.c_size_t
    lib.raftk_general_workspace_bytes.argtypes = [P(RaftkGeneral), C.c_int32]
    lib.raftk_general_solve_dynamics_dev.argtypes = [P(RaftkGeneral), P(RaftkCases), P(RaftkSolveOpts), C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    lib.raftk_general_solve_dynamics_host.argtypes = [P(RaftkGeneral), P(RaftkCases), P(RaftkSolveOpts), C.c_void_p, C.c_void_p]
    lib.raftk_general_solve_dynamics_dev.restype = C.c_int
    lib.raftk_general_solve_dynamics_host.restype = C.c_int
    lib.raftk_general_fd_workspace_bytes.restype = C.c_size_t
    lib.raftk_general_fd_workspace_bytes.argtypes = [P(RaftkGeneral), P(RaftkGeneralFd), C.c_int32]
    lib.raftk_general_solve_dynamics_fd_dev.argtypes = [P(RaftkGeneral), P(RaftkGeneralFd), P(RaftkCases), P(RaftkSolveOpts), C.c_void_p, C.c_void_p,
                                                        C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    lib.raftk_general_solve_dynamics_fd_host.argtypes = [P(RaftkGeneral), P(RaftkGeneralFd), P(RaftkCases), P(RaftkSolveOpts), C.c_void_p, C.c_void_p,
                                                         C.c_void_p]
    lib.raftk_general_solve_dynamics_fd_dev.restype = C.c_int
    lib.raftk_general_solve_dynamics_fd_host.restype = C.c_int
    lib.raftk_general_qtf_workspace_bytes.restype = C.c_size_t
    lib.raftk_general_qtf_workspace_bytes.argtypes = [P(RaftkGeneral), P(RaftkGeneralFd), P(RaftkGeneralQtf), C.c_int32]
    lib.raftk_general_solve_dynamics_qtf_dev.argtypes = [P(RaftkGeneral), P(RaftkGeneralFd), P(RaftkGeneralQtf), P(RaftkCases), P(RaftkSolveOpts),
                                                         C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                                         C.c_void_p]
    lib.raftk_general_solve_dynamics_qtf_host.argtypes = [P(RaftkGeneral), P(RaftkGeneralFd), P(RaftkGeneralQtf), P(RaftkCases), P(RaftkSolveOpts),
                                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.raftk_general_solve_dynamics_qtf_dev.restype = C.c_int
    lib.raftk_general_solve_dynamics_qtf_host.restype = C.c_int
    lib.raftk_general_stream_workspace_bytes.restype = C.c_size_t
    lib.raftk_general_stream_workspace_bytes.argtypes = [P(RaftkGeneral), P(RaftkGeneralFd), P(RaftkGeneralQtf), C.c_int32, C.c_int32]
    lib.raftk_general_solve_dynamics_stream_dev.argtypes = [P(RaftkGeneral), P(RaftkGeneralFd), P(RaftkGeneralQtf), P(RaftkCases),
                                                            P(RaftkSolveOpts), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                            C.c_void_p, C.c_size_t, C.c_int32, C.c_void_p]
    lib.raftk_general_solve_dynamics_stream_host.argtypes = [P(RaftkGeneral), P(RaftkGeneralFd), P(RaftkGeneralQtf), P(RaftkCases),
                                                             P(RaftkSolveOpts), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                             C.c_int32]
    lib.raftk_general_solve_dynamics_stream_dev.restype = C.c_int
    lib.raftk_general_solve_dynamics_stream_host.restype = C.c_int
    lib.raftk_general_batch_workspace_bytes.restype = C.c_size_t
    lib.raftk_general_batch_workspace_bytes.argtypes = [P(RaftkGeneral), P(RaftkGeneralBatch), P(RaftkGeneralFd), P(RaftkGeneralQtf), C.c_int32,
                                                        C.c_int32]
    lib.raftk_general_batch_solve_dynamics_dev.argtypes = [P(RaftkGeneral), P(RaftkGeneralBatch), P(RaftkGeneralFd), P(RaftkGeneralQtf),
                                                           P(RaftkCases), P(RaftkSolveOpts), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                           C.c_void_p, C.c_void_p, C.c_size_t, C.c_int32, C.c_void_p]
    lib.raftk_general_batch_solve_dynamics_host.argtypes = [P(RaftkGeneral), P(RaftkGeneralBatch), P(RaftkGeneralFd), P(RaftkGeneralQtf),
                                                            P(RaftkCases), P(RaftkSolveOpts), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                            C.c_void_p, C.c_int32]
    lib.raftk_general_batch_solve_dynamics_dev.restype = C.c_int
    lib.raftk_general_batch_solve_dynamics_host.restype = C.c_int
    lib.raftk_system_solve_dev.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.raftk_system_solve_host.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.raftk_response_stats_dev.argtypes = [C.c_int32, C.c_int32, C.c_double, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.raftk_response_stats_host.argtypes = [C.c_int32, C.c_int32, C.c_double, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.raftk_channel_stats_dev.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_double] + [C.c_void_p] * 6
    lib.raftk_channel_stats_host.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_double] + [C.c_void_p] * 5
    lib.raftk_general_channel_stats_dev.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_double] + [C.c_void_p] * 8
    lib.raftk_general_channel_stats_host.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_double] + [C.c_void_p] * 7
    lib.raftk_general_channel_stats_dev.restype = C.c_int
    lib.raftk_general_channel_stats_host.restype = C.c_int
    lib.raftk_channel_stats_dev.restype = C.c_int
    lib.raftk_channel_stats_host.restype = C.c_int
    lib.raftk_response_stats_dev.restype = C.c_int
    lib.raftk_response_stats_host.restype = C.c_int
    lib.raftk_host_alloc.restype = C.c_void_p
    lib.raftk_host_alloc.argtypes = [C.c_size_t]
    lib.raftk_host_free.argtypes = [C.c_void_p]
    lib.raftk_fp64_peak_gflops.restype = C.c_double
    lib.raftk_fp64_peak_gflops.argtypes = [C.c_int]
    lib.raftk_peer_alloc.argtypes = [C.c_size_t, P(C.c_void_p), C.c_char_p]
    lib.raftk_peer_open.argtypes = [C.c_char_p, P(C.c_void_p)]
    lib.raftk_peer_free.argtypes = [C.c_void_p]
    lib.raftk_peer_close.argtypes = [C.c_void_p]
    lib.raftk_solve_dynamics_gather_dev.argtypes = [P(RaftkDesigns), P(RaftkCases), P(RaftkSolveOpts), P(RaftkOutputs), P(RaftkPeers),
                                                    C.c_void_p, C.c_size_t, C.c_void_p]
    lib.raftk_peer_barrier_dev.argtypes = [P(RaftkPeers), C.c_void_p, C.c_void_p]
    lib.raftk_general_publish_dev.argtypes = [P(RaftkPeers), C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                              C.c_void_p]
    lib.raftk_farm_response_dev.argtypes = [P(RaftkDesigns), P(RaftkCases), P(RaftkOutputs), P(RaftkFarm), C.c_void_p]
    lib.raftk_solve_dynamics_farm_host.argtypes = [P(RaftkDesigns), P(RaftkCases), P(RaftkSolveOpts), P(RaftkOutputs), P(RaftkFarm)]
    lib.raftk_farm_response_dev.restype = C.c_int
    lib.raftk_solve_dynamics_farm_host.restype = C.c_int
    lib.raftk_farm_workspace_bytes.argtypes = [P(RaftkDesigns), P(RaftkCases), P(RaftkFarm)]
    lib.raftk_farm_workspace_bytes.restype = C.c_size_t
    lib.raftk_farm_response_ws_dev.argtypes = [P(RaftkDesigns), P(RaftkCases), P(RaftkOutputs), P(RaftkFarm), C.c_void_p, C.c_size_t, C.c_void_p]
    lib.raftk_farm_response_ws_dev.restype = C.c_int
    lib.raftk_farm_batch_workspace_bytes.argtypes = [P(RaftkDesigns), P(RaftkCases), P(RaftkFarmBatch)]
    lib.raftk_farm_batch_workspace_bytes.restype = C.c_size_t
    lib.raftk_farm_batch_response_ws_dev.argtypes = [P(RaftkDesigns), P(RaftkCases), P(RaftkOutputs), P(RaftkFarmBatch), C.c_void_p, C.c_size_t,
                                                     C.c_void_p]
    lib.raftk_farm_batch_response_ws_dev.restype = C.c_int
    lib.raftk_solve_dynamics_farm_batch_host.argtypes = [P(RaftkDesigns), P(RaftkCases), P(RaftkSolveOpts), P(RaftkOutputs), P(RaftkFarmBatch)]
    lib.raftk_solve_dynamics_farm_batch_host.restype = C.c_int
    lib.raftk_farm_batch_response_gather_dev.argtypes = [P(RaftkDesigns), P(RaftkCases), P(RaftkOutputs), P(RaftkFarmBatch), P(RaftkPeers),
                                                         C.c_int32, C.c_void_p, C.c_size_t, C.c_void_p]
    lib.raftk_farm_batch_response_gather_dev.restype = C.c_int
    lib.raftk_farm_ragged_workspace_bytes.argtypes = [P(RaftkDesigns), P(RaftkCases), P(RaftkFarmRagged)]
    lib.raftk_farm_ragged_workspace_bytes.restype = C.c_size_t
    lib.raftk_farm_ragged_response_ws_dev.argtypes = [P(RaftkDesigns), P(RaftkCases), P(RaftkOutputs), P(RaftkFarmRagged), C.c_void_p,
                                                      C.c_size_t, C.c_void_p]
    lib.raftk_farm_ragged_response_ws_dev.restype = C.c_int
    lib.raftk_solve_dynamics_farm_ragged_host.argtypes = [P(RaftkDesigns), P(RaftkCases), P(RaftkSolveOpts), P(RaftkOutputs),
                                                          P(RaftkFarmRagged)]
    lib.raftk_solve_dynamics_farm_ragged_host.restype = C.c_int
    lib.raftk_farm_ragged_response_gather_dev.argtypes = [P(RaftkDesigns), P(RaftkCases), P(RaftkOutputs), P(RaftkFarmRagged), P(RaftkPeers),
                                                          C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_size_t, C.c_void_p]
    lib.raftk_farm_ragged_response_gather_dev.restype = C.c_int
    lib.raftk_farm_ragged_channel_stats_workspace_bytes.argtypes = [C.c_int32] * 3 + [C.c_void_p, C.c_void_p, P(RaftkFarmChannels)]
    lib.raftk_farm_ragged_channel_stats_workspace_bytes.restype = C.c_size_t
    lib.raftk_farm_ragged_channel_stats_dev.argtypes = [C.c_int32] * 3 + [C.c_void_p] * 4 + [P(RaftkFarmChannels), C.c_void_p, C.c_size_t,
                                                                                          C.c_void_p]
    lib.raftk_farm_ragged_channel_stats_dev.restype = C.c_int
    lib.raftk_farm_ragged_channel_stats_host.argtypes = [C.c_int32] * 3 + [C.c_void_p] * 4 + [P(RaftkFarmChannels)]
    lib.raftk_farm_ragged_channel_stats_host.restype = C.c_int
    lib.raftk_eigen_workspace_bytes.argtypes = [P(RaftkEigen)]
    lib.raftk_eigen_workspace_bytes.restype = C.c_size_t
    lib.raftk_eigen_dev.argtypes = [P(RaftkEigen), C.c_void_p, C.c_size_t, C.c_void_p]
    lib.raftk_eigen_dev.restype = C.c_int
    lib.raftk_eigen_host.argtypes = [P(RaftkEigen)]
    lib.raftk_eigen_host.restype = C.c_int
    lib.raftk_farm_channel_stats_workspace_bytes.argtypes = [C.c_int32, C.c_int32, C.c_int32, P(RaftkFarmChannels)]
    lib.raftk_farm_channel_stats_workspace_bytes.restype = C.c_size_t
    lib.raftk_farm_channel_stats_dev.argtypes = [C.c_int32] * 4 + [C.c_void_p, C.c_void_p, P(RaftkFarmChannels), C.c_void_p, C.c_size_t,
                                                                   C.c_void_p]
    lib.raftk_farm_channel_stats_dev.restype = C.c_int
    lib.raftk_farm_channel_stats_host.argtypes = [C.c_int32] * 4 + [C.c_void_p, C.c_void_p, P(RaftkFarmChannels)]
    lib.raftk_farm_channel_stats_host.restype = C.c_int
    lib.raftk_rotor_stats_dev.argtypes = [C.c_int32] * 4 + [C.c_void_p, C.c_void_p, P(RaftkRotorOutputs), C.c_void_p]
    lib.raftk_rotor_stats_dev.restype = C.c_int
    lib.raftk_rotor_stats_host.argtypes = [C.c_int32] * 4 + [C.c_void_p, C.c_void_p, P(RaftkRotorOutputs)]
    lib.raftk_rotor_stats_host.restype = C.c_int
    lib.raftk_fatigue_workspace_bytes.argtypes = [C.c_int32] * 3 + [P(RaftkFatigue)]
    lib.raftk_fatigue_workspace_bytes.restype = C.c_size_t
    lib.raftk_fatigue_dev.argtypes = [C.c_int32] * 4 + [C.c_void_p, C.c_void_p, P(RaftkFatigue), C.c_void_p, C.c_size_t, C.c_void_p]
    lib.raftk_fatigue_dev.restype = C.c_int
    lib.raftk_fatigue_host.argtypes = [C.c_int32] * 4 + [C.c_void_p, C.c_void_p, P(RaftkFatigue)]
    lib.raftk_fatigue_host.restype = C.c_int
    lib.raftk_stress_ring_workspace_bytes.argtypes = [C.c_int32] * 3 + [P(RaftkStressRing)]
    lib.raftk_stress_ring_workspace_bytes.restype = C.c_size_t
    lib.raftk_stress_ring_dev.argtypes = [C.c_int32] * 4 + [C.c_void_p, C.c_void_p, P(RaftkStressRing), C.c_void_p, C.c_size_t, C.c_void_p]
    lib.raftk_stress_ring_dev.restype = C.c_int
    lib.raftk_stress_ring_host.argtypes = [C.c_int32] * 4 + [C.c_void_p, C.c_void_p, P(RaftkStressRing)]
    lib.raftk_stress_ring_host.restype = C.c_int
    lib.raftk_family_sizes.argtypes = [P(RaftkFamily), P(C.c_int32), P(C.c_int32)]
    lib.raftk_build_family_host.argtypes = [P(RaftkFamily), P(RaftkFamilyTables)]
    lib.raftk_family_sizes.restype = C.c_int
    lib.raftk_build_family_host.restype = C.c_int
    for fn in ("raftk_peer_alloc", "raftk_peer_open", "raftk_peer_free", "raftk_peer_close", "raftk_solve_dynamics_gather_dev",
               "raftk_peer_barrier_dev", "raftk_general_publish_dev"):
        getattr(lib, fn).restype = C.c_int
    for fn in ("raftk_hydro_excitation_dev", "raftk_hydro_linearization_dev", "raftk_solve_dynamics_dev",
               "raftk_hydro_excitation_host", "raftk_hydro_linearization_host", "raftk_solve_dynamics_host",
               "raftk_system_solve_dev", "raftk_system_solve_host",
               "raftk_second_order_force_dev", "raftk_second_order_force_host"):
        getattr(lib, fn).restype = C.c_int
    return lib


class _LazyLib:
    """Proxy that dlopens libraftk.so on first attribute access (see the module docstring)."""
    _real = None

    def __getattr__(self, name):
        if _LazyLib._real is None:
            _LazyLib._real = _load()
        return getattr(_LazyLib._real, name)


_require()          # fail loudly at import when the library has not been built
lib = _LazyLib()


def loaded():
    """True once the shared object has been mapped into this process."""
    return _LazyLib._real is not None


def check(rc):
    """Translate a negative return code into an exception carrying raftk_last_error()."""
    if rc != 0:
        msg = lib.raftk_last_error().decode("utf-8", "replace")
        if rc == -4:
            raise ValueError("Wave spectrum input not recognized. (%s)" % msg)
        raise RaftkError("raftk error %d: %s" % (rc, msg))
