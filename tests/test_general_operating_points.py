"""Per-case operating points on flexible FOWTs (raftk_cases.op on every raftk_general_* solve, ``solver.CaseTable(ops=)``,
``packer.pack_general_operating_points``, ``packer.pack_general_matrices(fowt, states=...)``, ``general_analyze_cases*(ops=)``):
every load case solved with its own aero-servo added mass, damping and gyroscopic damping, as the reference's
calcTurbineConstants(case) makes them (raft_fowt.py:1514-1586), on the support of the frequency-dependent terms.

Fixtures flexops_{strip,bem}_VolturnUS-S-flexible (tests/golden/make_golden_flexops.py): the unmodified reference with a
seeded calcAero stand-in, five cases (12 m/s, 8 m/s with two trains, 12 m/s with another sea state, 18 m/s, wind 0), strip
theory only (the support comes from the operating points alone) and marin_semi BEM (the union with DOFs 0-5).
Without a GPU: the packer (sums over rotors, the gyroscopic term in every bin, deduplication, the union support, refusals),
pack_general_matrices without states bit-identical to the flexfd fixture's, the refusals of every entry before any launch,
and the CPU checker with each case's point folded into fd against both fixtures (XI_RTOL).  On the GPU: general_analyze_cases
(ops=) against both fixtures (Xi of every train, channel statistics, rotor keys), solving every case at case 0's point misses them by more than 1e-3, and a call with operating points bit for bit
equal to one call per operating point with its tables folded into fd, for both LU kernels, wave trains, a QTF
(RAFTK_QTF_DIAG=1), the streamed entry, design batches, the sessions and a one-rank ShardedGeneralSolve."""
import ctypes as C
import json
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest

from conftest import GOLDEN, relerr

gpu = pytest.mark.gpu
FIXTURES = ("strip", "bem")
# The impedance has cond ~1e6 and the reference sums the turbine, structural and hydrodynamic terms in another order than the
# packed M + (A_w + A_op): responses agree to rounding amplified by that, measured <= 1.8e-10 (the 8 m/s secondary train and
# the 18 m/s case of the strip design, CPU checker), so 3e-10.  Statistics: 1e-9 (measured <= 9e-10 from the checker's
# response), except yaw, the smallest channel by far, whose PSD carries that rounding at up to 7.2e-9 of its own peak: 2e-8.
XI_RTOL, STAT_RTOL, YAW_RTOL = 3e-10, 1e-9, 2e-8


# ---- fixtures and inputs --------------------------------------------------------------------------------------------
def load_flexops(name):
    """-> (P, M, B, C, fd, ops, z): the packed design (flex fixture's tables overlaid with the fixture's), the constant matrices
    and fd of pack_general_matrices(fowt, states=...), the operating points packed from the stored snapshots, the fixture."""
    from raft_b200 import packer
    base = np.load(os.path.join(GOLDEN, "flex_VolturnUS-S-flexible.npz"))
    z = np.load(os.path.join(GOLDEN, "flexops_%s_VolturnUS-S-flexible.npz" % name))
    keys = set(z["P_keys"].tolist())
    P = {k[2:]: base[k] for k in base.files if k.startswith("P_") and k[2:] in keys}
    P.update({k[2:]: z[k] for k in z.files if k.startswith("P_") and k != "P_keys"})
    fd = {k[3:]: z[k] for k in z.files if k.startswith("fd_")}
    ops = packer.pack_general_operating_points([snapshots(z, int(P["gen_nDOF"]))], fd["fd_idx"])
    return P, z["M"], z["B"], z["C"], fd, ops, z


def snapshots(z, n):
    """The fixture's calcTurbineConstants snapshots, scattered back to dense [n,n,nw,nrot] / [n,n,nrot] dicts."""
    out = []
    for c in range(int(z["n_cases"])):
        idx = z["op_c%d_idx" % c]
        s = {}
        for k in ("A_aero", "B_aero", "B_gyro"):
            v = z["op_c%d_%s" % (c, k)]
            d = np.zeros((n, n) + v.shape[2:])
            d[np.ix_(idx, idx)] = v
            s[k] = d
        out.append(s)
    return out


def fold(fd, A, B):
    """fd with one operating point's tables summed into A_w / B_w (the kernels' order: the design's table + the point's)."""
    return dict(fd, A_w=np.asarray(fd["A_w"]) + A, B_w=np.asarray(fd["B_w"]) + B)


def _cases_json(z):
    return json.loads(str(z["cases_json"]))


def _train_table(z):
    from raft_b200 import packer
    return packer.pack_case_trains(_cases_json(z))


def _channels(z):
    names = []
    for s in z["ch_names"]:
        nm, ir = str(s).split(":")
        names.append((nm, None if ir == "" else int(ir)))
    return dict(names=names, R=z["ch_R"], wpow=z["ch_wpow"], avg=z["ch_avg"])


# ---- without a GPU --------------------------------------------------------------------------------------------------
def _gsnap(rng, n, nw, dofs, nrot=2, gyro=True):
    A, B, G = np.zeros([n, n, nw, nrot]), np.zeros([n, n, nw, nrot]), np.zeros([n, n, nrot])
    ix = np.ix_(dofs, dofs)
    A[ix] = rng.normal(size=(len(dofs), len(dofs), nw, nrot))
    B[ix] = np.abs(rng.normal(size=(len(dofs), len(dofs), nw, nrot)))
    if gyro:
        G[ix] = rng.normal(size=(len(dofs), len(dofs), nrot))
    return dict(A_aero=A, B_aero=B, B_gyro=G)


def test_pack_general_operating_points_sums_folds_and_deduplicates():
    from raft_b200 import packer
    rng = np.random.default_rng(3)
    n, nw = 11, 7
    idx = np.array([2, 5, 9, 10], dtype=np.int32)
    s = [_gsnap(rng, n, nw, [5, 9, 10]) for _ in range(3)]
    t = [_gsnap(rng, n, nw, [2, 9]) for _ in range(3)]
    live = NS(**{k: v.copy() for k, v in s[2].items()})                     # a live FOWT works like a dict
    states = [[s[0], s[1], live, dict(s[0])], [t[0], t[1], t[2], dict(t[0])]]
    p = packer.pack_general_operating_points(states, idx)
    assert p["op"].dtype == np.int32 and p["op"].tolist() == [0, 1, 2, 0] and p["n_op"] == 3
    assert p["A_w"].shape == p["B_w"].shape == (2, 3, 4, 4, nw)
    sub = np.ix_(idx, idx)
    for d, row in enumerate(states):
        for c, x in enumerate(row):
            g = (lambda k: x[k]) if isinstance(x, dict) else (lambda k: getattr(x, k))
            assert np.array_equal(p["A_w"][d, p["op"][c]], g("A_aero").sum(axis=3)[sub])
            B = g("B_aero").sum(axis=3) + g("B_gyro").sum(axis=2)[:, :, None]         # the gyroscopic term in every bin
            assert np.array_equal(p["B_w"][d, p["op"][c]], B[sub])
    # equal on design 0 but not on design 1: two points; per-design supports [nD, n_fd]
    q = packer.pack_general_operating_points([[s[0], s[0]], [t[0], t[1]]], np.stack([idx, idx]))
    assert q["op"].tolist() == [0, 1]
    # no rotors: zero tables, one point
    z = packer.pack_general_operating_points([[dict(A_aero=np.zeros([n, n, nw, 0]), B_aero=np.zeros([n, n, nw, 0]),
                                                    B_gyro=np.zeros([n, n, 0]))] * 2], idx)
    assert z["n_op"] == 1 and not z["A_w"].any()


@pytest.mark.parametrize("bad", ["off_support", "gyro_off_support", "nw", "B_shape", "gyro", "count", "idx"])
def test_pack_general_operating_points_refusals(bad):
    from raft_b200 import packer
    rng = np.random.default_rng(4)
    n, nw = 9, 5
    idx = np.array([1, 4, 8])
    a, b = _gsnap(rng, n, nw, [1, 4]), _gsnap(rng, n, nw, [4, 8])
    if bad == "off_support":
        b["A_aero"][0, 4, 2, 1] = 1e-300
    elif bad == "gyro_off_support":
        b["B_gyro"][8, 3, 0] = 1.0
    elif bad == "nw":
        b = _gsnap(rng, n, nw + 1, [4])
    elif bad == "B_shape":
        b["B_aero"] = b["B_aero"][..., :1]
    elif bad == "gyro":
        b["B_gyro"] = b["B_gyro"][..., :1]
    elif bad == "idx":
        idx = np.array([1, 4, 9])
    states = [[a, b]] if bad != "count" else [[a, b], [a]]
    with pytest.raises(ValueError):
        packer.pack_general_operating_points(states, idx)


def _ns_fowt(rng, n, nw, bem_dofs=(), nrot=1):
    """A duck-typed generalised-DOF FOWT with a last-case turbine state on DOFs 6, 7 and BEM terms on ``bem_dofs``."""
    f = NS(nDOF=n, w=np.linspace(0.1, 1.0, nw), T=rng.normal(size=(n, n)), nrotors=nrot)
    for k in ("M_struc", "A_hydro_morison", "B_struc", "C_struc", "C_hydro", "C_moor", "C_elast"):
        setattr(f, k, rng.normal(size=(n, n)))
    s = _gsnap(rng, n, nw, [6, 7], nrot)
    f.A_aero, f.B_aero, f.B_gyro = s["A_aero"], s["B_aero"], s["B_gyro"]
    if len(bem_dofs):
        f.A_BEM, f.B_BEM = np.zeros([n, n, nw]), np.zeros([n, n, nw])
        f.A_BEM[np.ix_(bem_dofs, bem_dofs)] = rng.normal(size=(len(bem_dofs), len(bem_dofs), nw))
        f.B_BEM[np.ix_(bem_dofs, bem_dofs)] = rng.normal(size=(len(bem_dofs), len(bem_dofs), nw))
    return f


def test_pack_general_matrices_with_states_takes_the_union_support():
    from raft_b200 import packer
    rng = np.random.default_rng(5)
    n, nw = 12, 6
    f = _ns_fowt(rng, n, nw, bem_dofs=[0, 1, 2])
    old = packer.pack_general_matrices(f)
    assert old["fd"]["fd_idx"].tolist() == [0, 1, 2, 6, 7] and "ops" not in old
    assert np.array_equal(old["B"], f.B_struc + f.B_gyro.sum(axis=2))
    states = [_gsnap(rng, n, nw, [7, 10]), _gsnap(rng, n, nw, [4], gyro=False), _gsnap(rng, n, nw, [7, 10])]
    g = packer.pack_general_matrices(f, states=states)
    idx = g["fd"]["fd_idx"]
    assert idx.dtype == np.int32 and idx.tolist() == [0, 1, 2, 4, 7, 10]          # BEM support | every state's (not the FOWT's own)
    assert np.array_equal(g["B"], f.B_struc) and np.array_equal(g["M"], old["M"]) and np.array_equal(g["C"], old["C"])
    sub = np.ix_(idx, idx)
    assert np.array_equal(g["fd"]["A_w"], f.A_BEM[sub]) and np.array_equal(g["fd"]["B_w"], f.B_BEM[sub])   # BEM terms alone
    ref = packer.pack_general_operating_points([states], idx)
    assert g["ops"]["op"].tolist() == ref["op"].tolist() == [0, 1, 2]
    assert np.array_equal(g["ops"]["A_w"], ref["A_w"]) and np.array_equal(g["ops"]["B_w"], ref["B_w"])
    # a FOWT without BEM: the support is the states' alone, fd's tables zero
    h = packer.pack_general_matrices(_ns_fowt(rng, n, nw), states=states[1:2])
    assert h["fd"]["fd_idx"].tolist() == [4] and not h["fd"]["A_w"].any() and not h["fd"]["B_w"].any()


def test_pack_general_matrices_without_states_is_unchanged():
    """pack_general_matrices(fowt) of the reference's live flexfd FOWT equals the flexfd fixture's packed M, B, C and fd bit
    for bit (the fixture was made before ``states`` existed); skipped without the reference tree."""
    from oracle import ref_harness as rh
    if not rh.reference_available():
        pytest.skip("the reference tree is not available")
    import sys
    sys.path.insert(0, GOLDEN)
    import make_golden_flexfd
    from raft_b200 import packer
    z = np.load(os.path.join(GOLDEN, "flexfd_VolturnUS-S-flexible.npz"))
    _, fowt = make_golden_flexfd.build(os.path.join(rh.REF_ROOT, "tests", "test_data", "VolturnUS-S-flexible.yaml"))
    G = packer.pack_general_matrices(fowt)
    assert set(G) == {"M", "B", "C", "fd"}
    for k in ("M", "B", "C"):
        assert np.array_equal(G[k], z[k]), k
    assert sorted(G["fd"]) == sorted(k[3:] for k in z.files if k.startswith("fd_"))
    for k, v in G["fd"].items():
        assert np.array_equal(np.asarray(v), z["fd_" + k]), k


def test_case_table_checks():
    from raft_b200 import solver
    nw, nf = 5, 4
    c = dict(Hs=np.ones(3), Tp=np.full(3, 8.0), gamma=np.zeros(3), beta_deg=np.zeros(3), spec=np.zeros(3, dtype=np.int32))
    A = np.zeros([2, nf, nf, nw])
    ct = solver.CaseTable(c, ops=dict(op=[0, 1, 1], A_w=A, B_w=A))
    assert (ct.n_op, ct.op_shared) == (2, 1)
    ct.check_general_ops(nf, 3, nw)
    for args in ((nf + 1, 1, nw), (nf, 1, nw + 1), (0, 1, nw)):
        with pytest.raises(ValueError):
            ct.check_general_ops(*args)
    with pytest.raises(ValueError, match="6 x 6"):
        ct.check_ops(NS(nw=nw, n_designs=1))                                         # rigid solves take 6 x 6 tables only
    per = solver.CaseTable(c, ops=dict(op=[0, 1, 1], A_w=np.zeros([3, 2, nf, nf, nw]), B_w=np.zeros([3, 2, nf, nf, nw])))
    per.check_general_ops(nf, 3, nw)
    with pytest.raises(ValueError):
        per.check_general_ops(nf, 2, nw)                                              # three designs' tables for two
    with pytest.raises(ValueError):
        solver.CaseTable(c, ops=dict(op=[0, 1, 1], A_w=np.zeros([2, nf, nf + 1, nw]), B_w=np.zeros([2, nf, nf + 1, nw])))


# every entry, host and dev, refuses before any launch
REFUSALS = [("no_fd", "n_fd >= 1"), ("n_fd0", "n_fd >= 1"), ("n_op", "n_op must be >= 1"), ("shared", "op_shared must be 0 or 1"),
            ("A_null", "op_A_w and op_B_w"), ("B_null", "op_B_w"), ("neg", "outside [0, n_op"), ("big", "outside [0, n_op"),
            ("train", "secondary train")]
HOST_ONLY = ("neg", "big", "train")                # the *_dev entries read op back for these: on the GPU (below)


def _abi_inputs(case):
    """Host structs of a synthetic 9-DOF design (and a two-design batch of it) with a valid operating-point table, broken by
    ``case``; the arrays stay alive in the result."""
    import general_synth as gs
    from raft_b200 import solver
    from raft_b200._lib import RaftkSolveOpts
    n, nw, nC = 9, 12, 3
    P, M, B, Cm = gs.design(n, nw, seed=1)
    idx = gs.support(n)
    fd = gs.fd_tables(P, M, B, idx, seed=1)
    nf = len(idx)
    keep = dict(op=np.zeros(nC, dtype=np.int32), A=np.zeros([2 * 2 * nf * nf * nw]), buf=np.zeros(1 << 16))
    cases = dict(Hs=np.ones(nC), Tp=np.full(nC, 8.0), gamma=np.zeros(nC), beta_deg=np.zeros(nC), spec=np.zeros(nC, dtype=np.int32))
    ct = solver.CaseTable(cases)
    c = ct.struct(lambda k: ct.arrays[k].ctypes.data)
    c.op, c.n_op, c.op_shared = keep["op"].ctypes.data, 2, 0
    c.op_A_w = c.op_B_w = keep["A"].ctypes.data
    ptr = lambda name, a: keep.setdefault(name, a).ctypes.data        # noqa: E731
    g = solver._general_struct(P, M, B, Cm, ptr)
    f = solver._general_fd_struct(fd, n, nw, lambda name, a: keep.setdefault("f_" + name, a).ctypes.data)
    bt = solver.GeneralBatch([dict(P=P, M=M, B=B, Cm=Cm, fd=fd)] * 2)
    bg, bb, bf, _ = bt.structs(lambda name, a: keep.setdefault("b_" + name, a).ctypes.data)
    if case == "no_fd":
        f = bf = None
    elif case == "n_fd0":
        f.n_fd = bf.n_fd = 0
    elif case == "n_op":
        c.n_op = 0
    elif case == "shared":
        c.op_shared = 2
    elif case == "A_null":
        c.op_A_w = None
    elif case == "B_null":
        c.op_B_w = None
    elif case == "neg":
        keep["op"][1] = -1
    elif case == "big":
        keep["op"][2] = 2
    elif case == "train":
        keep["prim"] = np.array([0, 0, 2], dtype=np.int32)
        keep["op"][:] = [0, 1, 1]
        c.primary = keep["prim"].ctypes.data
    return g, f, bg, bb, bf, c, RaftkSolveOpts(4, 0, 0.01, 0.0, 0, 0), keep


@pytest.mark.parametrize("case,msg", REFUSALS)
def test_refusals_before_any_launch(case, msg):
    from raft_b200._lib import lib
    g, f, bg, bb, bf, c, o, keep = _abi_inputs(case)
    R = lambda s: C.byref(s) if s is not None else None      # noqa: E731
    X = S = keep["buf"].ctypes.data
    ws = keep["buf"].ctypes.data
    host = [lambda: lib.raftk_general_solve_dynamics_host(C.byref(g), C.byref(c), C.byref(o), X, S),
            lambda: lib.raftk_general_solve_dynamics_fd_host(C.byref(g), R(f), C.byref(c), C.byref(o), X, S, None),
            lambda: lib.raftk_general_solve_dynamics_qtf_host(C.byref(g), R(f), None, C.byref(c), C.byref(o), X, S, None, None, None),
            lambda: lib.raftk_general_solve_dynamics_stream_host(C.byref(g), R(f), None, C.byref(c), C.byref(o), X, S, None, None, None, 0),
            lambda: lib.raftk_general_batch_solve_dynamics_host(C.byref(bg), C.byref(bb), R(bf), None, C.byref(c), C.byref(o), X, S,
                                                               None, None, None, 0)]
    dev = [lambda: lib.raftk_general_solve_dynamics_dev(C.byref(g), C.byref(c), C.byref(o), X, S, ws, 1 << 19, None),
           lambda: lib.raftk_general_solve_dynamics_fd_dev(C.byref(g), R(f), C.byref(c), C.byref(o), X, S, None, ws, 1 << 19, None),
           lambda: lib.raftk_general_solve_dynamics_qtf_dev(C.byref(g), R(f), None, C.byref(c), C.byref(o), X, S, None, None, None,
                                                            ws, 1 << 19, None),
           lambda: lib.raftk_general_solve_dynamics_stream_dev(C.byref(g), R(f), None, C.byref(c), C.byref(o), X, S, None, None, None,
                                                               ws, 1 << 19, 0, None),
           lambda: lib.raftk_general_batch_solve_dynamics_dev(C.byref(bg), C.byref(bb), R(bf), None, C.byref(c), C.byref(o), X, S,
                                                              None, None, None, ws, 1 << 19, 0, None)]
    before = lib.raftk_launch_count()
    plain = (host[0], dev[0])                                 # no fd: op is refused there whatever else is wrong
    for call in [c for c in host[1:] + ([] if case in HOST_ONLY else dev[1:])]:
        assert call() == -1 and msg in lib.raftk_last_error().decode(), lib.raftk_last_error()
    for call in plain:
        assert call() == -1 and "n_fd >= 1" in lib.raftk_last_error().decode(), lib.raftk_last_error()
    assert lib.raftk_launch_count() == before


def test_python_entries_refuse_before_any_launch():
    from raft_b200 import solver
    from raft_b200._lib import lib
    P, M, B, Cm, fd, ops, z = load_flexops("bem")
    table, owner, first = _train_table(z)
    before = lib.raftk_launch_count()
    with pytest.raises(ValueError, match="not supported for generalised-DOF"):
        solver.general_solve_dynamics(P, M, B, Cm, solver.CaseTable(table, ops=dict(ops, op=ops["op"][owner])), fd=None)
    bad = dict(ops, A_w=ops["A_w"][..., :-1, :], B_w=ops["B_w"][..., :-1, :])
    with pytest.raises(ValueError):
        solver.CaseTable(table, ops=dict(bad, op=ops["op"][owner]))
    with pytest.raises(ValueError):                                                  # one point per RAFT case, not per train
        solver.general_analyze_cases(P, M, B, Cm, _cases_json(z), fd=fd, ops=dict(ops, op=ops["op"][owner]))
    with pytest.raises(NotImplementedError, match="states="):
        solver.general_analyze_cases(P, M, B, Cm, _cases_json(z), fd=fd, turbine_constants=[[{}]])
    with pytest.raises(ValueError):
        solver.general_solve_dynamics_batch([dict(P=P, M=M, B=B, Cm=Cm, fd=fd)] * 3,
                                            solver.CaseTable(table, ops=dict(ops, op=ops["op"][owner])))     # tables for one design
    assert lib.raftk_launch_count() == before


@pytest.mark.parametrize("name", FIXTURES)
def test_fixture_snapshots_pack_onto_the_support(name):
    P, M, B, Cm, fd, ops, z = load_flexops(name)
    want = [144, 146, 147, 148, 149] if name == "strip" else list(range(6)) + [144, 146, 147, 148, 149]
    assert fd["fd_idx"].tolist() == want
    assert ops["op"].tolist() == [0, 1, 0, 2, 3]                  # case 2 shares case 0's point (12 m/s)
    assert not ops["A_w"][0, 3].any() and not ops["B_w"][0, 3].any()          # wind 0: no terms
    assert len(z["op_c4_idx"]) == 0
    if name == "strip":
        assert not fd["A_w"].any() and not fd["B_w"].any()
    n = int(P["gen_nDOF"])
    assert set(z["op_c0_idx"].tolist()) == {144, 146, 147, 148, 149} and n == 150


@pytest.mark.parametrize("name", FIXTURES)
def test_checker_with_each_point_folded_vs_reference(name, oracle):
    """tests/general_fd_checker.py with each case's packed point folded into fd reproduces the reference's Xi of every case and
    train at 1e-10 and its pass counts: the packing matches what the reference adds."""
    import general_fd_checker as gfc
    P, M, B, Cm, fd, ops, z = load_flexops(name)
    for ic in range(int(z["n_cases"])):
        k = ops["op"][ic]
        tr = z["ref_run_case%d_trains" % ic]
        Xi, st, _ = gfc.solve_trains_fd(oracle, P, M, B, Cm, fold(fd, ops["A_w"][0, k], ops["B_w"][0, k]), tr, nIter=int(z["n_iter"]),
                                        XiStart=float(z["xi_start"]))
        assert st[0] == int(z["ref_run_case%d_passes" % ic]) and st[2] == 0, (ic, st)
        for h in range(len(tr)):
            assert relerr(Xi[h], z["ref_run_case%d_Xi" % ic][h]) < XI_RTOL, (ic, h, relerr(Xi[h], z["ref_run_case%d_Xi" % ic][h]))


# ---- on the GPU -----------------------------------------------------------------------------------------------------
def _env(monkeypatch, **env):
    monkeypatch.delenv("RAFTK_QTF_DIAG", raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


@gpu
@pytest.mark.parametrize("name", FIXTURES)
def test_analyze_cases_vs_reference(name):
    """general_analyze_cases(ops=, rotors=) on the fixture: Xi of every train (XI_RTOL), the motion and tower-base statistics
    and the rotor keys of every case (STAT_RTOL); the batch entry with
    two designs and per-design tables gives the same; every case at case 0's point misses the reference by more than 1e-3."""
    from test_rotor_outputs import _fixture_rotors
    from raft_b200 import solver
    from raft_b200.packer import ROTOR_KEYS
    P, M, B, Cm, fd, ops, z = load_flexops(name)
    cases = _cases_json(z)
    kw = dict(n_iter=int(z["n_iter"]), xi_start=float(z["xi_start"]))
    ch, rot = _channels(z), _fixture_rotors(z, 0)
    res = solver.general_analyze_cases(P, M, B, Cm, cases, channels=ch, fd=fd, rotors=rot, ops=ops, **kw)
    per = dict(ops, A_w=np.concatenate([ops["A_w"]] * 2), B_w=np.concatenate([ops["B_w"]] * 2))
    rb = solver.general_analyze_cases_batch([dict(P=P, M=M, B=B, Cm=Cm, fd=fd)] * 2, cases, channels=[ch, ch], rotors=[rot, rot],
                                            ops=per, **kw)
    keys = [k[len("ref_run_case0_"):] for k in z.files if k.startswith("ref_run_case0_") and k[14:] not in ("Xi", "passes", "trains")]
    for ic in range(len(cases)):
        ref = z["ref_run_case%d_Xi" % ic]
        for r in [res] + rb:
            assert len(r["Xi_trains"][ic]) == len(ref)
            for h in range(len(ref)):
                assert relerr(r["Xi_trains"][ic][h], ref[h]) < XI_RTOL, (ic, h, relerr(r["Xi_trains"][ic][h], ref[h]))
            assert r["status"][ic, 0] == int(z["ref_run_case%d_passes" % ic])
            m = r["case_metrics"][ic]
            for k in keys:
                want, got = z["ref_run_case%d_%s" % (ic, k)], np.asarray(m[k])
                assert got.shape == want.shape, (ic, k)
                tol = YAW_RTOL if k.startswith("yaw") else STAT_RTOL
                assert (relerr(got, want) < tol) if np.abs(want).max() > 0 else not np.any(got), (ic, k, relerr(got, want))
            rk = [k for k in ROTOR_KEYS + ("wind_PSD",) if "fowt0_%s_c%d" % (k, ic) in z.files]
            assert sorted(k for k in m if k in ROTOR_KEYS + ("wind_PSD",)) == sorted(rk), (ic, sorted(m))
            for k in rk:
                want = z["fowt0_%s_c%d" % (k, ic)]
                assert np.shape(m[k]) == want.shape and ((relerr(m[k], want) < STAT_RTOL) if np.abs(want).max() > 0 else not np.any(m[k])), (ic, k)
        for d in range(2):
            assert np.array_equal(np.concatenate(rb[d]["Xi_trains"]), np.concatenate(res["Xi_trains"]))
    one = dict(ops, op=np.zeros_like(ops["op"]))
    miss = solver.general_analyze_cases(P, M, B, Cm, cases, fd=fd, ops=one, **kw)
    worst = max(relerr(miss["Xi_trains"][ic][0], z["ref_run_case%d_Xi" % ic][0]) for ic in range(len(cases)))
    assert worst > 1e-3, worst


def _per_point(solve, ops, table, owner):
    """For every operating point k: (rows of the train table at k, the solve of those rows with k's tables folded into fd)."""
    from test_operating_points import _sub_cases
    from raft_b200 import solver
    op = ops["op"][owner]
    out = []
    for k in range(ops["n_op"]):
        rows = np.nonzero(op == k)[0]
        if len(rows):
            out.append((rows, solve(k, solver.CaseTable(_sub_cases(table, rows)))))
    return out


def _same(got, ref, rows):
    Xi, st = got[0][..., rows, :, :], got[1][..., rows, :]
    assert np.array_equal(Xi, ref[0]), np.abs(Xi - ref[0]).max()
    assert np.array_equal(st[..., :3], ref[1][..., :3])
    for a, b in zip(got[2:], ref[2:]):
        assert np.array_equal(a[..., rows, :, :] if a.ndim == ref[0].ndim else a[..., rows, :], b)


@gpu
@pytest.mark.parametrize("kernel", ["gen-blocked"])
def test_equals_one_call_per_point(kernel, monkeypatch):
    from raft_b200 import solver
    _env(monkeypatch)
    P, M, B, Cm, fd, ops, z = load_flexops("bem")
    table, owner, first = _train_table(z)
    assert "primary" in table                                                  # wave trains
    kw = dict(n_iter=int(z["n_iter"]), xi_start=float(z["xi_start"]), F_BEM=True)
    got = solver.general_solve_dynamics(P, M, B, Cm, solver.CaseTable(table, ops=dict(ops, op=ops["op"][owner])), fd=fd, **kw)
    rec = solver.last_dispatch()
    assert rec["kernel"] == kernel and rec["trains"], rec
    for rows, ref in _per_point(lambda k, ct: solver.general_solve_dynamics(P, M, B, Cm, ct, fd=fold(fd, ops["A_w"][0, k], ops["B_w"][0, k]), **kw),
                                ops, table, owner):
        assert solver.last_dispatch()["kernel"] == kernel
        _same(got, ref, rows)
    # one shared set equals the per-design replica
    sh = solver.general_solve_dynamics(P, M, B, Cm, solver.CaseTable(table, ops=dict(op=ops["op"][owner], A_w=ops["A_w"][0], B_w=ops["B_w"][0])),
                                       fd=fd, **kw)
    for a, b in zip(got, sh):
        assert np.array_equal(a, b)


@gpu
def test_qtf_equals_one_call_per_point(monkeypatch, tmp_path):
    """With second-order loads (the flexqtf fixture's design and QTF, seeded points on its fd support) under RAFTK_QTF_DIAG=1."""
    from test_general_qtf_oracle import load_flexqtf
    from raft_b200 import solver
    _env(monkeypatch, RAFTK_QTF_DIAG="1")
    P, M, B, Cm, fd, qtf, z = load_flexqtf(tmp_path)
    zo = load_flexops("bem")[-1]                                                  # its five cases and trains
    nf, nw = len(fd["fd_idx"]), len(P["w"])
    rng = np.random.default_rng(7)
    A = rng.normal(size=(3, nf, nf, nw)) * 1e-2 * np.abs(M).max()
    Bt = np.abs(rng.normal(size=(3, nf, nf, nw))) * 1e5
    table, owner, first = _train_table(zo)
    op = np.array([0, 1, 0, 2, 1])[owner].astype(np.int32)
    ops = dict(op=np.array([0, 1, 0, 2, 1], dtype=np.int32), A_w=A, B_w=Bt, n_op=3)
    kw = dict(n_iter=int(z["n_iter"]), qtf=qtf, F_2nd=True)
    got = solver.general_solve_dynamics(P, M, B, Cm, solver.CaseTable(table, ops=dict(op=op, A_w=A, B_w=Bt)), fd=fd, **kw)
    assert solver.last_dispatch()["kernel"] == "gen-blocked"
    for rows, ref in _per_point(lambda k, ct: solver.general_solve_dynamics(P, M, B, Cm, ct, fd=fold(fd, A[k], Bt[k]), **kw),
                                ops, table, owner):
        _same(got, ref, rows)


@gpu
@pytest.mark.parametrize("chunk", [1, 2, 0])
def test_stream_equals_one_launch(chunk):
    """The streamed entry with operating points (the op column follows the chunks) equals the one-launch entry bit for bit;
    chunk 1 runs the single-train rows (a two-train group does not fit)."""
    from test_operating_points import _sub_cases
    from raft_b200 import solver
    P, M, B, Cm, fd, ops, z = load_flexops("strip")
    table, owner, first = _train_table(z)
    rows = np.arange(len(owner)) if chunk != 1 else np.nonzero(np.bincount(owner)[owner] == 1)[0]
    sub = _sub_cases(table, rows)
    ct = solver.CaseTable(sub, ops=dict(ops, op=ops["op"][owner][rows]))
    kw = dict(n_iter=int(z["n_iter"]), xi_start=float(z["xi_start"]), fd=fd)
    one = solver.general_solve_dynamics(P, M, B, Cm, ct, **kw)
    st = solver.general_solve_dynamics(P, M, B, Cm, ct, max_chunk_cases=chunk, **kw)
    assert np.array_equal(one[0], st[0]) and np.array_equal(one[1], st[1])
    if chunk:
        assert solver.last_dispatch()["chunks"] > 1


@gpu
def test_batch_per_design_tables_and_shared():
    """A two-design batch (the bem design and a stiffer copy) with per-design tables: design d's rows equal its own call with
    each point folded in; one shared set equals per-design replicas of it."""
    from raft_b200 import solver
    P, M, B, Cm, fd, ops, z = load_flexops("bem")
    table, owner, first = _train_table(z)
    C2 = Cm * 1.05
    designs = [dict(P=P, M=M, B=B, Cm=Cm, fd=fd), dict(P=P, M=M, B=B, Cm=C2, fd=fd)]
    A = np.stack([ops["A_w"][0], ops["A_w"][0][::-1] * 0.5])                     # design 1: other points
    Bt = np.stack([ops["B_w"][0], ops["B_w"][0][::-1] * 0.5])
    op = ops["op"][owner]
    kw = dict(n_iter=int(z["n_iter"]), xi_start=float(z["xi_start"]))
    got = solver.general_solve_dynamics_batch(designs, solver.CaseTable(table, ops=dict(op=op, A_w=A, B_w=Bt)), **kw)
    for d, Cd in enumerate((Cm, C2)):
        ref = [(rows, r) for rows, r in _per_point(lambda k, ct: solver.general_solve_dynamics(P, M, B, Cd, ct, fd=fold(fd, A[d, k], Bt[d, k]), **kw),
                                                   ops, table, owner)]
        for rows, r in ref:
            _same((got[0][d], got[1][d]), r, rows)
    sh = solver.general_solve_dynamics_batch(designs, solver.CaseTable(table, ops=dict(op=op, A_w=A[0], B_w=Bt[0])), **kw)
    rep = solver.general_solve_dynamics_batch(designs, solver.CaseTable(table, ops=dict(op=op, A_w=np.stack([A[0]] * 2),
                                                                                        B_w=np.stack([Bt[0]] * 2))), max_chunk_units=3, **kw)
    assert np.array_equal(sh[0], rep[0]) and np.array_equal(sh[1][..., :3], rep[1][..., :3])


@gpu
def test_sessions_and_sharded_equal_host_path():
    import torch
    from raft_b200 import solver, sweep
    P, M, B, Cm, fd, ops, z = load_flexops("bem")
    table, owner, first = _train_table(z)
    ct = solver.CaseTable(table, ops=dict(op=ops["op"][owner], A_w=ops["A_w"][0], B_w=ops["B_w"][0]))     # shared: any design count
    kw = dict(n_iter=int(z["n_iter"]), xi_start=float(z["xi_start"]))
    rX, rS = solver.general_solve_dynamics(P, M, B, Cm, ct, fd=fd, **kw)
    for chunk in (None, 2):
        s = solver.GeneralSession(P, M, B, Cm, ct, fd=fd, max_chunk_cases=chunk)
        X, S = s.solve(**kw)
        torch.cuda.synchronize()
        assert np.array_equal(X.cpu().numpy(), rX) and np.array_equal(S.cpu().numpy(), rS)
    bs = solver.GeneralBatchSession([dict(P=P, M=M, B=B, Cm=Cm, fd=fd)] * 2, ct, max_chunk_units=4)
    X, S = bs.solve(**kw)
    torch.cuda.synchronize()
    for d in range(2):
        assert np.array_equal(X[d].cpu().numpy(), rX) and np.array_equal(S[d].cpu().numpy()[..., :3], rS[..., :3])
    sh = sweep.ShardedGeneralSolve(P, M, B, Cm, ct, fd=fd, max_chunk_cases=3, exchange="nccl")
    X, S = sh.step(**kw)
    torch.cuda.synchronize()
    assert np.array_equal(X.cpu().numpy(), rX) and np.array_equal(S.cpu().numpy(), rS)
    sh.close()


@gpu
@pytest.mark.parametrize("case,msg", [("big", "outside [0, n_op"), ("neg", "outside [0, n_op"), ("train", "secondary train")])
def test_dev_entries_check_op_values(case, msg):
    """The *_dev entries read op back with fd_idx and refuse bad values before any launch: a session whose device op column
    was overwritten after the table's own checks."""
    import torch
    from raft_b200 import solver
    from raft_b200._lib import lib
    P, M, B, Cm, fd, ops, z = load_flexops("strip")
    table, owner, first = _train_table(z)
    ct = solver.CaseTable(table, ops=dict(op=ops["op"][owner], A_w=ops["A_w"][0], B_w=ops["B_w"][0]))
    bad = ops["op"][owner].astype(np.int32).copy()
    if case == "big":
        bad[0] = ops["n_op"]
    elif case == "neg":
        bad[-1] = -1
    else:
        sec = int(np.nonzero(table["primary"] != np.arange(len(owner)))[0][0])
        bad[sec] = (bad[sec] + 1) % ops["n_op"]
    sessions = [solver.GeneralSession(P, M, B, Cm, ct, fd=fd), solver.GeneralSession(P, M, B, Cm, ct, fd=fd, max_chunk_cases=2),
                solver.GeneralBatchSession([dict(P=P, M=M, B=B, Cm=Cm, fd=fd)] * 2, ct)]
    for s in sessions:
        s.ct["op"].copy_(torch.from_numpy(bad))
    torch.cuda.synchronize()
    before = lib.raftk_launch_count()
    for s in sessions:
        with pytest.raises(RuntimeError, match=msg.replace("[", r"\[")):
            s.solve(n_iter=int(z["n_iter"]))
    assert lib.raftk_launch_count() == before
