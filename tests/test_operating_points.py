"""Per-case operating points (raftk_cases.op, ``solver.CaseTable(ops=)``, ``packer.pack_operating_points``,
``Model(turbine_constants=)``): every load case solved with its own aero-servo added mass and damping, as the reference's
calcTurbineConstants(case) makes them (raft_fowt.py:1514-1586, raft_model.py:1005-1010, 1045-1046).
Without a GPU: the header and ctypes layout of the new fields, every refusal of the rigid, farm, slender and generalised-DOF
entries, and the packer (sums over rotors, B_gyro folded into B, deduplication, shapes, refusals).  On the GPU, for every solve
variant (v1, fused128, fused256, fused2 cluster / grid) and every farm variant (rows12, warp, block, global), each asserted
through last_dispatch(): a call with operating points is bit-identical to one call per operating point with that point's
tables summed into the design-level A_w / B_w, one shared set equals per-design replicas bit for bit, wave-train cases
included; the same for the potSecOrder 1 flow; and Model(turbine_constants=) equals the Model whose matrices carry each case's
terms."""
import ctypes as C
import os
import subprocess
from types import SimpleNamespace as NS

import numpy as np
import pytest

from conftest import ROOT, load_golden

gpu = pytest.mark.gpu
HEADER = os.path.join(ROOT, "include", "raftk.h")


# ---- inputs ---------------------------------------------------------------------------------------------------------
def _op_tables(rng, P, n_op, nD):
    """Seeded operating points of a realistic size for design P: [nD, n_op, 6, 6, nw] added mass (a few per cent of M0,
    symmetric) and positive damping (surge / pitch dominated, like an operating rotor's)."""
    nw = len(P["w"])
    M0 = np.abs(np.asarray(P["M0"])).max()
    A = rng.normal(size=(nD, n_op, 6, 6, nw)) * 0.01 * M0 / 36
    A = 0.5 * (A + np.swapaxes(A, 2, 3))
    B = np.abs(rng.normal(size=(nD, n_op, 6, 6, nw))) * 2e4
    B[:, :, 0, 0] += rng.uniform(1e5, 6e5, size=(nD, n_op, 1))
    B[:, :, 4, 4] += rng.uniform(1e9, 6e9, size=(nD, n_op, 1))
    return A, B


def _fold(P, A, B):
    """Design P with an operating point's tables summed into its A_w / B_w (the kernels' order: design's + point's)."""
    Q = dict(P)
    Q["A_w"] = (np.asarray(P["A_w"]) + A) if P.get("A_w") is not None else A.copy()
    Q["B_w"] = (np.asarray(P["B_w"]) + B) if P.get("B_w") is not None else B.copy()
    return Q


def _sub_cases(cases, rows):
    """Rows of a case dict as a table of their own (primaries rebased)."""
    sub = {k: np.asarray(v)[rows] for k, v in cases.items() if k != "primary"}
    if "primary" in cases:
        pos = {r: i for i, r in enumerate(rows)}
        sub["primary"] = np.array([pos[int(p)] for p in np.asarray(cases["primary"])[rows]], dtype=np.int32)
    return sub


def _cases(n, seed, trains):
    rng = np.random.default_rng(seed)
    c = dict(Hs=rng.uniform(1, 9, n), Tp=rng.uniform(6, 17, n), gamma=np.zeros(n), beta_deg=rng.uniform(-180, 180, n),
             spec=np.zeros(n, dtype=np.int32))
    if trains:
        c["primary"] = np.array([0, 0, 2, 3, 3][:n], dtype=np.int32)
    return c


OP = np.array([0, 0, 1, 2, 2], dtype=np.int32)          # trains 0/1 and 3/4 share their primary's point


# ---- without a GPU --------------------------------------------------------------------------------------------------
def test_struct_layout_matches_header(tmp_path):
    from raft_b200 import _lib
    S = _lib.RaftkCases
    fields = [n for n, _ in S._fields_ if not n.startswith("_")]
    assert fields[-5:] == ["op", "n_op", "op_shared", "op_A_w", "op_B_w"]
    src = tmp_path / "t.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "raftk.h"\nint main(void){printf("%%zu %s\\n", sizeof(raftk_cases), %s);'
                   'return 0;}\n' % (" ".join(["%zu"] * len(fields)), ", ".join("offsetof(raftk_cases, %s)" % n for n in fields)))
    exe = tmp_path / "t"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert got == [C.sizeof(S)] + [getattr(S, n).offset for n in fields]


def _structs(nD=1, nC=3, nw=8, n_op=2, shared=0):
    """Host structs that pass every other check, with an operating-point table; the arrays are kept alive in the result."""
    from raft_b200 import solver
    P = load_golden("cfg2_VolturnUS-S_nw64")[1]
    batch = solver.DesignBatch([P] * nD)
    cases = _cases(nC, 1, False)
    ct = solver.CaseTable(cases)
    keep = dict(op=np.zeros(nC, dtype=np.int32), A=np.zeros(((1 if shared else nD) * n_op, 36, batch.nw)))
    c = ct.struct(lambda k: ct.arrays[k].ctypes.data)
    c.op, c.n_op, c.op_shared = keep["op"].ctypes.data, n_op, shared
    c.op_A_w = c.op_B_w = keep["A"].ctypes.data
    d = batch.struct(lambda k: batch.arrays[k].ctypes.data)
    return batch, ct, d, c, keep


REFUSALS = [("n_op", "n_op must be >= 1"), ("shared", "op_shared must be 0 or 1"), ("A_null", "op_A_w and op_B_w"),
            ("B_null", "op_A_w and op_B_w"), ("neg", "outside [0, n_op"), ("big", "outside [0, n_op"), ("train", "secondary train")]


def _break(case, c, keep, ct):
    if case == "n_op":
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


@pytest.mark.parametrize("case,msg", REFUSALS)
def test_rigid_and_farm_refusals_before_any_launch(case, msg):
    from raft_b200._lib import RaftkFarm, RaftkFarmBatch, RaftkOutputs, RaftkSolveOpts, lib
    batch, ct, d, c, keep = _structs(nD=2)
    _break(case, c, keep, ct)
    buf = np.zeros(1 << 16)
    o = RaftkOutputs()
    o.Xi = o.status = o.B_drag = o.F_drag = o.F_iner = buf.ctypes.data
    opts = RaftkSolveOpts(10, 0, 0.01, 0.0, 0, 0)
    f = RaftkFarm()
    f.n_fowt, f.Xi_sys = 2, buf.ctypes.data
    fb = RaftkFarmBatch()
    fb.n_farms, fb.n_fowt, fb.arr_shared, fb.Xi_sys = 1, 2, 1, buf.ctypes.data
    before = lib.raftk_launch_count()
    for call in (lambda: lib.raftk_solve_dynamics_host(C.byref(d), C.byref(c), C.byref(opts), C.byref(o)),
                 lambda: lib.raftk_solve_dynamics_farm_host(C.byref(d), C.byref(c), C.byref(opts), C.byref(o), C.byref(f)),
                 lambda: lib.raftk_solve_dynamics_farm_batch_host(C.byref(d), C.byref(c), C.byref(opts), C.byref(o), C.byref(fb))):
        assert call() == -1 and msg in lib.raftk_last_error().decode(), lib.raftk_last_error()
    if case in ("n_op", "shared", "A_null", "B_null"):          # the *_dev entries check these without reading device memory
        for call in (lambda: lib.raftk_solve_dynamics_dev(C.byref(d), C.byref(c), C.byref(opts), C.byref(o), None, 0, None),
                     lambda: lib.raftk_farm_response_ws_dev(C.byref(d), C.byref(c), C.byref(o), C.byref(f), None, 0, None),
                     lambda: lib.raftk_farm_batch_response_ws_dev(C.byref(d), C.byref(c), C.byref(o), C.byref(fb), None, 0, None)):
            assert call() == -1 and msg in lib.raftk_last_error().decode(), lib.raftk_last_error()
    assert lib.raftk_launch_count() == before


@pytest.mark.parametrize("case,msg", [r for r in REFUSALS if r[0] != "train"])
def test_slender_refusals_before_any_launch(case, msg):
    from raft_b200 import solver
    from raft_b200._lib import RaftkOutputs, RaftkSlenderOutputs, RaftkSolveOpts, lib
    z = np.load(os.path.join(ROOT, "tests", "golden", "slender_VolturnUS-S.npz"))
    P = {k[2:]: z[k] for k in z.files if k.startswith("P_")}
    batch, sb, _ = solver._slender_inputs([P], solver.CaseTable(_cases(3, 1, False)))
    _, ct, _, c, keep = _structs(nD=1)
    _break(case, c, keep, ct)
    d = batch.struct(lambda k: batch.arrays[k].ctypes.data)
    s = sb.struct(lambda k: sb.arrays[k].ctypes.data)
    buf = np.zeros(1 << 16)
    o = RaftkOutputs()
    o.Xi = o.status = buf.ctypes.data
    before = lib.raftk_launch_count()
    rc = lib.raftk_solve_dynamics_slender_host(C.byref(d), C.byref(s), C.byref(c), C.byref(RaftkSolveOpts(4, 0, 0.01, 0.0, 0, 0)),
                                               C.byref(o), C.byref(RaftkSlenderOutputs(None, None, 0, 0)))
    assert rc == -1 and msg in lib.raftk_last_error().decode(), lib.raftk_last_error()
    assert lib.raftk_launch_count() == before


def test_generalised_dof_entries_refuse_operating_points():
    from raft_b200 import packer, solver
    from raft_b200._lib import lib
    z = np.load(os.path.join(ROOT, "tests", "golden", "flex_VolturnUS-S-flexible.npz"))
    P = {k[2:]: z[k] for k in z.files if k.startswith("P_")}
    n, nw = int(P["gen_nDOF"]), len(P["w"])
    M = np.eye(n) * 1e6
    ops = dict(op=np.zeros(3, dtype=np.int32), A_w=np.zeros([1, 6, 6, nw]), B_w=np.zeros([1, 6, 6, nw]))
    before = lib.raftk_launch_count()
    with pytest.raises(Exception, match="not supported for generalised-DOF"):
        solver.general_solve_dynamics(P, M, M * 0, M, solver.CaseTable(_cases(3, 1, False), ops=ops), n_iter=2)
    with pytest.raises(NotImplementedError):
        solver.general_analyze_cases(P, M, M * 0, M, [dict(wave_height=2.0, wave_period=8.0)], turbine_constants=[[{}]])
    with pytest.raises(NotImplementedError):
        solver.general_analyze_cases_batch([P], [dict(wave_height=2.0, wave_period=8.0)], turbine_constants=[[{}]])
    with pytest.raises(NotImplementedError, match="follow-up"):
        packer.pack_operating_points([[dict(A_aero=np.zeros([12, 12, nw, 1]), B_aero=np.zeros([12, 12, nw, 1]), B_gyro=np.zeros([12, 12, 1]))]])
    assert lib.raftk_launch_count() == before


def _snap(rng, nw, nrot=2, gyro=True):
    return dict(A_aero=rng.normal(size=(6, 6, nw, nrot)), B_aero=np.abs(rng.normal(size=(6, 6, nw, nrot))),
                B_gyro=rng.normal(size=(6, 6, nrot)) if gyro else np.zeros([6, 6, nrot]))


def test_pack_operating_points_sums_folds_and_deduplicates():
    from raft_b200 import packer
    rng = np.random.default_rng(3)
    nw = 7
    s = [_snap(rng, nw) for _ in range(3)]
    t = [_snap(rng, nw) for _ in range(3)]
    live = NS(nDOF=6, **{k: v.copy() for k, v in s[2].items()})            # a live FOWT works like a dict
    # design 0: cases 0 and 3 equal, case 2 a live object equal to case 1's dict on design 0 only; design 1 splits 1 / 2
    states = [[s[0], s[1], live, dict(s[0])], [t[0], t[1], t[2], dict(t[0])]]
    p = packer.pack_operating_points(states)
    assert p["op"].dtype == np.int32 and p["op"].tolist() == [0, 1, 2, 0] and p["n_op"] == 3
    assert p["A_w"].shape == p["B_w"].shape == (2, 3, 6, 6, nw)
    for d, row in enumerate(states):
        for c, x in enumerate(row):
            g = (lambda k: x[k]) if isinstance(x, dict) else (lambda k: getattr(x, k))
            assert np.array_equal(p["A_w"][d, p["op"][c]], g("A_aero").sum(axis=3))
            assert np.array_equal(p["B_w"][d, p["op"][c]], g("B_aero").sum(axis=3) + g("B_gyro").sum(axis=2)[:, :, None])
    # equal on design 0 but not on design 1: two points
    q = packer.pack_operating_points([[s[0], s[0]], [t[0], t[1]]])
    assert q["op"].tolist() == [0, 1]
    # no rotors: zero tables, one point
    z = packer.pack_operating_points([[dict(A_aero=np.zeros([6, 6, nw, 0]), B_aero=np.zeros([6, 6, nw, 0]), B_gyro=np.zeros([6, 6, 0]))] * 2])
    assert z["n_op"] == 1 and not z["A_w"].any()


@pytest.mark.parametrize("bad", ["nw", "B_shape", "gyro", "count"])
def test_pack_operating_points_refusals(bad):
    from raft_b200 import packer
    rng = np.random.default_rng(4)
    a, b = _snap(rng, 5), _snap(rng, 5)
    if bad == "nw":
        b = _snap(rng, 6)
    elif bad == "B_shape":
        b["B_aero"] = b["B_aero"][..., :1]
    elif bad == "gyro":
        b["B_gyro"] = b["B_gyro"][..., :1]
    states = [[a, b]] if bad != "count" else [[a, b], [a]]
    with pytest.raises(ValueError):
        packer.pack_operating_points(states)


def test_case_table_refusals():
    from raft_b200 import solver
    nw = 5
    A = np.zeros([2, 6, 6, nw])
    c = _cases(3, 1, False)
    with pytest.raises(ValueError):
        solver.CaseTable(c, ops=dict(op=[0, 1], A_w=A, B_w=A))                          # one per case
    with pytest.raises(ValueError):
        solver.CaseTable(c, ops=dict(op=[0, 1, 2], A_w=A, B_w=A))                       # outside [0, n_op)
    with pytest.raises(ValueError):
        solver.CaseTable(c, ops=dict(op=[0, 1, 1], A_w=A, B_w=A[..., :4]))
    with pytest.raises(ValueError):
        solver.CaseTable(dict(c, primary=np.array([0, 0, 2], dtype=np.int32)), ops=dict(op=[0, 1, 1], A_w=A, B_w=A))
    ct = solver.CaseTable(c, ops=dict(op=[0, 1, 1], A_w=A, B_w=A))
    assert (ct.n_op, ct.op_shared) == (2, 1)
    P = load_golden("cfg2_VolturnUS-S_nw64")[1]
    with pytest.raises(ValueError):
        ct.check_ops(solver.DesignBatch(P))                                            # 64 bins, tables on 5
    with pytest.raises(ValueError):
        solver.solve_dynamics(solver.DesignBatch(P), ct)
    per = solver.CaseTable(c, ops=dict(op=[0, 1, 1], A_w=np.zeros([3, 2, 6, 6, 64]), B_w=np.zeros([3, 2, 6, 6, 64])))
    with pytest.raises(ValueError):
        per.check_ops(solver.DesignBatch([P, P]))                                      # three designs' tables for two


def test_model_turbine_constants_refusals():
    from raft_b200.model import Model
    z = load_golden("cfg2_VolturnUS-S_nw64")
    m = _model(z, [[]])
    with pytest.raises(ValueError, match="iCase"):
        m.solveDynamics(dict(wave_height=2.0, wave_period=8.0, wave_heading=0.0))
    with pytest.raises(ValueError):
        Model(_design(), matrices=_mats(z[1]), turbine_constants=[[], []])               # two FOWTs' lists for one FOWT


# ---- the Model on the rigid fixture -----------------------------------------------------------------------------------
def _design():
    import json
    with open(os.path.join(ROOT, "tests", "golden", "designs.json")) as fh:
        return json.load(fh)["cfg2_VolturnUS-S_nw64"]


def _mats(P):
    return dict(M_struc=np.asarray(P["M0"]) - 0.0, C_struc=np.asarray(P["C0"]), B_struc=np.asarray(P["B0"]))


def _model(z, tc):
    from raft_b200.model import Model
    return Model(_design(), matrices=_mats(z[1]), turbine_constants=tc)


# ---- on the GPU -----------------------------------------------------------------------------------------------------
SOLVE_SHAPES = [("cfg2", 201, 2, {}, "fused128"), ("cfg2", 333, 2, {}, "fused256"), ("cfg3", 333, 2, {}, "fused256"),
                ("cfg2", 501, 2, {"RAFTK_FUSED2_XCHG": "cluster"}, "fused2-cluster"),
                ("cfg2", 501, 2, {"RAFTK_FUSED2_XCHG": "grid"}, "fused2-grid"),
                ("cfg3", 501, 2, {"RAFTK_FUSED2_XCHG": "grid"}, "fused2-grid"),
                ("cfg2", 201, 1, {"RAFTK_FORCE_V1": "1"}, "v1"), ("cfg3", 201, 1, {"RAFTK_FORCE_V1": "1"}, "v1")]


def _env(monkeypatch, env):
    for k in ("RAFTK_FORCE_V1", "RAFTK_FUSED2_XCHG", "RAFTK_FARM_SMEM", "RAFTK_QTF_DIAG"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def _same(a, b, keys, keep=None):
    """Bit-identical outputs; B_drag only on the rows ``keep`` (a secondary train's B_drag row is not written by the solve)."""
    for k in keys:
        x, y = (a[k], b[k]) if k != "B_drag" or keep is None else (a[k][:, keep], b[k][:, keep])
        if k == "status":                   # word 3 of a secondary train is its primary's index in its own table, + 1
            x, y = x[..., :3], y[..., :3]
        assert np.array_equal(x, y), k


@gpu
@pytest.mark.parametrize("shape", SOLVE_SHAPES, ids=lambda s: "%s-nw%d-%s" % (s[0], s[1], s[4]))
def test_solve_with_operating_points_equals_one_call_per_point(shape, monkeypatch):
    from test_dispatch_solve import _design as dispatch_design
    from raft_b200 import solver
    name, nw, cs, env, kernel = shape
    _env(monkeypatch, env)
    P = dispatch_design(name, nw)
    trains = kernel != "v1"                                    # wave trains need the fused solvers
    cases = _cases(5, 7, trains)
    rng = np.random.default_rng(11)
    A, B = _op_tables(rng, P, 3, 2)
    batch = solver.DesignBatch([P, P])
    want = ("Xi", "status", "B_drag", "F_drag")
    got = solver.solve_dynamics(batch, solver.CaseTable(cases, ops=dict(op=OP, A_w=A, B_w=B)), cluster_size=cs, want=want)
    rec = solver.last_dispatch()
    assert rec["kernel"] == kernel and rec["trains"] == trains, rec
    moved = False
    for k in range(3):
        rows = np.nonzero(OP == k)[0]
        ref = solver.solve_dynamics(solver.DesignBatch([_fold(P, A[d, k], B[d, k]) for d in range(2)]),
                                    solver.CaseTable(_sub_cases(cases, rows)), cluster_size=cs, want=want)
        assert solver.last_dispatch()["kernel"] == kernel
        keep = [i for i, r in enumerate(rows) if not trains or cases["primary"][r] == r]
        _same({q: got[q][:, rows] for q in want}, ref, want, keep)
        base = solver.solve_dynamics(batch, solver.CaseTable(_sub_cases(cases, rows)), cluster_size=cs, want=want)
        moved |= np.abs(base["Xi"] - ref["Xi"]).max() > 1e-3 * np.abs(ref["Xi"]).max()
    assert moved                                                # the operating points change the response
    # one shared set for every design equals per-design replicas of it
    sh = solver.solve_dynamics(batch, solver.CaseTable(cases, ops=dict(op=OP, A_w=A[0], B_w=B[0])), cluster_size=cs, want=want)
    rep = solver.solve_dynamics(batch, solver.CaseTable(cases, ops=dict(op=OP, A_w=np.stack([A[0]] * 2), B_w=np.stack([B[0]] * 2))),
                                cluster_size=cs, want=want)
    assert solver.last_dispatch()["kernel"] == kernel
    prim = [r for r in range(5) if not trains or cases["primary"][r] == r]
    _same(sh, rep, want, prim)
    # calls without operating points are unchanged by the feature: a design table of zeros gives the plain solve's bits
    if P.get("A_w") is None:
        zero = solver.solve_dynamics(batch, solver.CaseTable(cases, ops=dict(op=np.zeros(5, np.int32), A_w=np.zeros_like(A[0, :1]),
                                                                             B_w=np.zeros_like(B[0, :1]))), cluster_size=cs, want=want)
        plain = solver.solve_dynamics(batch, solver.CaseTable(cases), cluster_size=cs, want=want)
        _same(zero, plain, want, prim)


def _farm_packs(N):
    zf = np.load(os.path.join(ROOT, "tests", "golden", "farm_VolturnUS-S_farm_nw48.npz"))
    packs = [{k[3:]: zf[k] for k in zf.files if k.startswith("P%d_" % i)} for i in range(int(zf["n_fowt"]))]
    return [packs[i % len(packs)] for i in range(N)], zf


FARM_SHAPES = [(2, {}, "farm-rows12"), (3, {}, "farm-warp"), (5, {}, "farm-block"), (24, {}, "farm-global")]


@gpu
@pytest.mark.parametrize("shape", FARM_SHAPES, ids=lambda s: s[2])
def test_farm_with_operating_points_equals_one_call_per_point(shape, monkeypatch):
    from raft_b200 import solver
    N, env, kernel = shape
    _env(monkeypatch, env)
    packs, zf = _farm_packs(N)
    n = 6 * N
    rng = np.random.default_rng(12)
    K = rng.normal(size=(n, n)) * 1e4
    C_arr = K @ K.T / n + np.diag([5e4] * n)
    cases = _cases(5, 8, True)
    A, B = _op_tables(rng, packs[0], 3, N)
    batch = solver.DesignBatch(packs)
    got = solver.solve_dynamics_farm(batch, solver.CaseTable(cases, ops=dict(op=OP, A_w=A, B_w=B)), C_arr=C_arr, n_iter=int(zf["n_iter"]))
    assert solver.last_dispatch()["kernel"] == kernel, solver.last_dispatch()
    for k in range(3):
        rows = np.nonzero(OP == k)[0]
        ref = solver.solve_dynamics_farm(solver.DesignBatch([_fold(P, A[d, k], B[d, k]) for d, P in enumerate(packs)]),
                                         solver.CaseTable(_sub_cases(cases, rows)), C_arr=C_arr, n_iter=int(zf["n_iter"]))
        assert solver.last_dispatch()["kernel"] == kernel
        assert np.array_equal(got["Xi_sys"][rows], ref["Xi_sys"]) and np.array_equal(got["Xi"][:, rows], ref["Xi"])
    sh = solver.solve_dynamics_farm(batch, solver.CaseTable(cases, ops=dict(op=OP, A_w=A[0], B_w=B[0])), C_arr=C_arr)
    rep = solver.solve_dynamics_farm(batch, solver.CaseTable(cases, ops=dict(op=OP, A_w=np.stack([A[0]] * N), B_w=np.stack([B[0]] * N))),
                                     C_arr=C_arr)
    assert np.array_equal(sh["Xi_sys"], rep["Xi_sys"])
    if N == 2:                                                  # a farm batch of two farms: farm f's rows alone, bit for bit
        bb = solver.DesignBatch(packs + packs)
        two = solver.solve_dynamics_farm_batch(bb, solver.CaseTable(cases, ops=dict(op=OP, A_w=np.concatenate([A, A]), B_w=np.concatenate([B, B]))),
                                               2, C_arr=C_arr, n_iter=int(zf["n_iter"]))
        assert np.array_equal(two["Xi_sys"][0], got["Xi_sys"]) and np.array_equal(two["Xi_sys"][1], got["Xi_sys"])


@gpu
def test_device_session_equals_host_path():
    """DeviceSession.solve / farm_response with one shared set of operating points (op_shared = 1, the sweep form)."""
    from raft_b200 import solver
    packs, zf = _farm_packs(2)
    rng = np.random.default_rng(13)
    cases = _cases(5, 9, True)
    A, B = _op_tables(rng, packs[0], 3, 1)
    ct = solver.CaseTable(cases, ops=dict(op=OP, A_w=A[0], B_w=B[0]))
    batch = solver.DesignBatch(packs)
    host = solver.solve_dynamics_farm(batch, ct, C_arr=zf["C_array"], n_iter=int(zf["n_iter"]))
    s = solver.DeviceSession(batch, ct, want=("Xi", "status", "B_drag", "F_drag", "F_iner", "F_BEM"))
    out = s.solve(n_iter=int(zf["n_iter"]))
    rec = solver.last_dispatch()
    assert rec["family"] == "solve" and rec["kernel"] == "fused128" and rec["trains"], rec
    xi, _ = s.farm_response(C_arr=zf["C_array"])
    assert solver.last_dispatch()["kernel"] == "farm-rows12", solver.last_dispatch()
    assert np.array_equal(out["Xi"].cpu().numpy(), host["Xi"]) and np.array_equal(xi.cpu().numpy(), host["Xi_sys"])


@gpu
def test_slender_flow_with_operating_points_equals_one_call_per_point(monkeypatch):
    from test_dispatch_second_order import _build_pair
    from raft_b200 import solver
    _env(monkeypatch, {"RAFTK_QTF_DIAG": "1"})                 # the tile kernel's atomic sums vary in the last bits
    packs = _build_pair(201)
    cases = _cases(5, 10, False)
    op = np.array([0, 1, 0, 1, 1], dtype=np.int32)
    rng = np.random.default_rng(14)
    A, B = _op_tables(rng, packs[0], 2, 2)
    want = ("Xi", "status", "F_2nd")
    got = solver.slender_flow_host(packs, solver.CaseTable(cases, ops=dict(op=op, A_w=A, B_w=B)), n_iter=4, want=want)
    rec = solver.last_dispatch()
    kernel = rec["kernel"]
    assert rec["family"] == "solve" and kernel.startswith("fused"), rec        # both loops run on the fused solver
    for k in range(2):
        rows = np.nonzero(op == k)[0]
        ref = solver.slender_flow_host([_fold(P, A[d, k], B[d, k]) for d, P in enumerate(packs)], solver.CaseTable(_sub_cases(cases, rows)),
                                       n_iter=4, want=want)
        assert solver.last_dispatch()["kernel"] == kernel
        for q in want:
            assert np.array_equal(got[q][:, rows], ref[q]), q


@gpu
def test_model_turbine_constants_equal_per_case_matrices():
    """Model(turbine_constants=).analyzeCases on VolturnUS-S with snapshots at three operating points (two cases share one):
    every case's Xi and motion statistics equal those of a Model whose A_BEM / B_BEM carry that case's terms, and
    solveDynamics(case with iCase) the case's own row."""
    from raft_b200.model import Model
    z = load_golden("cfg2_VolturnUS-S_nw64")
    m0 = Model(_design(), matrices=_mats(z[1]))
    rng = np.random.default_rng(15)
    snaps = [_snap(rng, m0.nw, nrot=1) for _ in range(3)]
    for s in snaps:
        s["A_aero"] *= 1e5
        s["B_aero"] = np.abs(s["B_aero"]) * 1e6
        s["B_gyro"] *= 1e5
    cases = [dict(wave_height=h, wave_period=t, wave_heading=b, wind_speed=u) for h, t, b, u in
             ((6.0, 12.0, 30.0, 12.0), (4.0, 10.0, 0.0, 8.0), (3.0, 9.0, -45.0, 12.0), (5.0, 11.0, 10.0, 18.0))]
    per_case = [snaps[0], snaps[1], dict(snaps[0]), snaps[2]]
    m = Model(_design(), matrices=_mats(z[1]), turbine_constants=per_case)
    res = m.analyzeCases(cases=cases)
    for ic, case in enumerate(cases):
        s = per_case[ic]
        mats = dict(_mats(z[1]), A_BEM=s["A_aero"].sum(axis=3), B_BEM=s["B_aero"].sum(axis=3) + s["B_gyro"].sum(axis=2)[:, :, None])
        r1 = Model(_design(), matrices=mats).analyzeCases(cases=[case])
        assert np.allclose(res["Xi"][ic], r1["Xi"][0], rtol=1e-12, atol=1e-12 * np.abs(r1["Xi"][0]).max())
        for nm in ("surge_std", "pitch_std", "pitch_PSD"):
            assert np.allclose(res["case_metrics"][ic][0][nm], r1["case_metrics"][0][0][nm], rtol=1e-10, atol=0)
        one = m.solveDynamics(dict(case, iCase=ic))
        assert np.allclose(one[0], res["Xi"][ic], rtol=1e-12, atol=1e-12 * np.abs(one[0]).max())
    plain = m0.analyzeCases(cases=cases)
    assert max(np.abs(plain["Xi"][c] - res["Xi"][c]).max() / np.abs(res["Xi"][c]).max() for c in range(4)) > 1e-3


# ---- the reference's own calcTurbineConstants(case) (tests/golden/make_golden_ops.py) -----------------------------------
OPS_FIXTURES = ("VolturnUS-S", "farm", "farm24")


def _ops_fixture(name):
    return np.load(os.path.join(ROOT, "tests", "golden", "ops_%s.npz" % name))


def _ops_inputs(z, pin=None):
    """Model arguments of a fixture: matrices, per-case snapshots, per-case turbine channels, rotors and array mooring.
    ``pin``: give every case that case's snapshots instead of its own (the sensitivity guard)."""
    import json
    from test_rotor_outputs import _fixture_rotors
    nF, cases = int(z["n_fowt"]), json.loads(str(z["cases_json"]))
    nC = len(cases)
    mats = [{k[len("mat%d_" % i):]: z[k] for k in z.files if k.startswith("mat%d_" % i)} for i in range(nF)]
    src = (lambda c: c) if pin is None else (lambda c: pin)
    tc = [[{k: z["op%d_c%d_%s" % (i, src(c), k)] for k in ("A_aero", "B_aero", "B_gyro", "f_aero0")} for c in range(nC)] for i in range(nF)]
    nrot = z["hubT0"].shape[0]
    names = [(nm, ir) for ir in range(nrot) for nm in ("AxRNA", "AyRNA", "AzRNA", "Mbase")]
    ch = [[dict(names=names, coef=z["ch%d_c%d_coef" % (i, c)], avg=z["ch%d_c%d_avg" % (i, c)]) for c in range(nC)] for i in range(nF)]
    kw = dict(matrices=mats if nF > 1 else mats[0], turbine_constants=tc if nF > 1 else tc[0], channels=ch if nF > 1 else ch[0],
              rotors=[_fixture_rotors(z, i) for i in range(nF)])
    if "C_array" in z.files:
        kw.update(array_stiffness=z["C_array"], array_tension_jacobian=z["arr_J"], array_mean_tensions=z["arr_T0"])
    return json.loads(str(z["design_json"])), cases, kw


@pytest.mark.parametrize("name", OPS_FIXTURES)
def test_ops_fixture_snapshots_pack_the_reference_terms(name):
    """Each snapshot is what the reference's calcTurbineConstants left: the packer's sums over rotors with B_gyro folded into B;
    equal wind speeds share one operating point and the wind-speed-0 case has none (zero tables)."""
    import json
    from raft_b200 import packer
    z = _ops_fixture(name)
    nF, cases = int(z["n_fowt"]), json.loads(str(z["cases_json"]))
    states = [[{k: z["op%d_c%d_%s" % (i, c, k)] for k in ("A_aero", "B_aero", "B_gyro")} for c in range(len(cases))] for i in range(nF)]
    p = packer.pack_operating_points(states)
    speeds = [float(c["wind_speed"]) for c in cases]
    assert p["n_op"] == len(set(speeds))
    for c, u in enumerate(speeds):
        assert p["op"][c] == p["op"][speeds.index(u)]
        for i in range(nF):
            s = states[i][c]
            assert np.array_equal(p["B_w"][i, p["op"][c]], s["B_aero"].sum(axis=3) + s["B_gyro"].sum(axis=2)[:, :, None])
            assert (np.abs(s["B_gyro"]).max() > 0) == (u > 0) and (np.abs(s["B_aero"]).max() > 0) == (u > 0)


def test_ops_fixture_vs_cpu_oracle(oracle):
    """The VolturnUS-S fixture against the CPU oracle: each one-train case solved with its operating point's tables folded into
    A_w / B_w reproduces the reference's Xi to 1e-10 (the oracle itself unchanged)."""
    from raft_b200 import packer
    from raft_b200.model import Model
    z = _ops_fixture("VolturnUS-S")
    design, cases, kw = _ops_inputs(z)
    m = Model(design, matrices=kw["matrices"])
    P = m.fowtList[0].pack()
    checked = 0
    for c, case in enumerate(cases):
        table, owner, _ = packer.pack_case_trains([case])
        if len(owner) != 1:
            continue
        s = kw["turbine_constants"][c]
        Q = _fold(P, s["A_aero"].sum(axis=3), s["B_aero"].sum(axis=3) + s["B_gyro"].sum(axis=2)[:, :, None])
        Xi, _, _ = oracle.solve_cases(oracle.OracleDesign(Q), table, nIter=m.nIter, XiStart=m.XiStart)
        ref = z["Xi_c%d" % c][0]
        assert np.abs(Xi[0] - ref).max() / np.abs(ref).max() < 1e-10, c
        checked += 1
    assert checked == 4


def _rel(a, b):
    """max |a - b| / max |b| (complex or real)."""
    a, b = np.asarray(a), np.asarray(b)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


@gpu
@pytest.mark.parametrize("name", OPS_FIXTURES)
def test_model_analyze_cases_vs_reference(name):
    """Model(turbine_constants=).analyzeCases against the reference's analyzeCases with calcTurbineConstants(case) per case, to
    1e-10: Xi per case and train, motion std / PSD, Mbase (per-case channels), the rotor keys (rotors=) and array_mooring; the
    solve runs on the kernel the planner picks (fused for one FOWT, the farm kernels for arrays).  solveDynamics(case) with
    iCase gives the case's own Xi, and f.Z holds the last case's aero terms."""
    from test_rotor_outputs import _check_metrics
    from raft_b200 import solver
    from raft_b200.model import Model
    z = _ops_fixture(name)
    design, cases, kw = _ops_inputs(z)
    nF = int(z["n_fowt"])
    m = Model(design, **kw)
    res = m.analyzeCases(cases=cases)
    rec = solver.last_dispatch()
    assert rec["family"] == ("farm" if nF > 1 else "solve"), rec
    for c in range(len(cases)):
        ref = z["Xi_c%d" % c][:-1]
        got = res["Xi_trains"][c]
        assert got.shape == ref.shape and _rel(got, ref) < 1e-10, (c, _rel(got, ref))
        for i in range(nF):
            mc = res["case_metrics"][c][i]
            for k in (k_[len("cm%d_" % i):-len("_c%d" % c)] for k_ in z.files if k_.startswith("cm%d_" % i) and k_.endswith("_c%d" % c)):
                r = z["cm%d_%s_c%d" % (i, k, c)]
                assert np.shape(mc[k]) == r.shape and _rel(mc[k], r) < 1e-10, (c, i, k, _rel(mc[k], r))
            _check_metrics(mc, z, i, c)
        for k in (k_[4:-len("_c%d" % c)] for k_ in z.files if k_.startswith("arr_T") and k_.endswith("_c%d" % c)):
            assert _rel(res["case_metrics"][c]["array_mooring"][k], z["arr_%s_c%d" % (k, c)]) < 1e-10, (c, k)
    if nF == 1:
        for c, case in enumerate(cases):
            one = m.solveDynamics(dict(case, iCase=c))
            assert _rel(one[:-1], z["Xi_c%d" % c][:-1]) < 1e-10, c
            assert solver.last_dispatch()["family"] == "solve"
        f, last = m.fowtList[0], kw["turbine_constants"][3]
        P, w = f.pack(), m.w                                      # f.Z of a table whose last case runs at 18 m/s
        m4 = Model(design, **dict(kw, turbine_constants=kw["turbine_constants"][:4], channels=kw["channels"][:4], rotors=None))
        m4.analyzeCases(cases=cases[:4])
        f4 = m4.fowtList[0]
        M = P["M0"][:, :, None] + P.get("A_w", 0.0) + last["A_aero"].sum(axis=3)
        B = (P["B0"] + f4.B_hydro_drag)[:, :, None] + P.get("B_w", 0.0) + last["B_aero"].sum(axis=3) + last["B_gyro"].sum(axis=2)[:, :, None]
        assert np.allclose(f4.Z, -w ** 2 * M + 1j * w * B + P["C0"][:, :, None], rtol=1e-14, atol=0)


@gpu
@pytest.mark.parametrize("name", ["VolturnUS-S", "farm"])
def test_ignoring_the_operating_point_misses_the_reference(name):
    """Sensitivity guard: every case solved at the first case's operating point misses the reference by more than 1e-3 on some
    case, so the parity above cannot pass by ignoring op."""
    from raft_b200.model import Model
    z = _ops_fixture(name)
    design, cases, kw = _ops_inputs(z, pin=0)
    res = Model(design, **dict(kw, rotors=None)).analyzeCases(cases=cases)
    miss = max(_rel(res["Xi_trains"][c], z["Xi_c%d" % c][:-1]) for c in range(len(cases)))
    assert miss > 1e-3, miss
