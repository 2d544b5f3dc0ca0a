"""The second-order force in every kernel that adds it to the excitation, compared with the C oracle.

``cases.F_2nd`` is read in the prologue of k_rao_fused<128/256> (F0 on chip or in global memory), of k_rao_fused2 (cluster
and grid exchange), in k_excitation (v1), in the farm assembly (k_farm_response<true/false>, k_farm_response_global) and in
k_farm_rows.  Each test reaches its kernel through the shapes that make the planner choose it, asserts the choice through
solver.last_dispatch(), and checks that the force moves the response by far more than the tolerance, so that a dropped
or misplaced term fails.

A. potSecOrder 2 (external QTF table, the cfg3q fixture's) on every rigid-solve variant: Xi and status with
   oracle.solve_cases, F_2nd / F_2nd_mean with oracle.hydro_force_2nd; both force kernels; the 4-heading table; two designs
   with their own tables and with one shared table; wave trains; page-locked outputs.
B. The farm kernels with a second-order force, against the oracle's per-FOWT solves + explicit-inverse system response.
C. potSecOrder 1 on the device (SlenderSession) on every fused variant: loop B with F_2nd and Xi_init, reusing loop A's plan,
   per unit against oracle.solve_dynamics with the slender-body tables.
D. Where only the v1 kernel fits, potSecOrder 1 is refused before anything is launched."""
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN, QTF_GOLDEN, load_golden, relerr, response_err
from test_dispatch_solve import CLUSTER, GRID, MAX_FREQ, SEEDS, SHAPES, _check_record, _design, _sea_states, _shape_id, _train_table

pytestmark = pytest.mark.gpu
RTOL = 1e-10
MOVES = 1e-4                     # the force must move the response by more than this (relative), so that dropping it fails
DEG = 0.017453292519943295
ENV = ("RAFTK_FORCE_V1", "RAFTK_FUSED2_XCHG", "RAFTK_NO_DIRECT_D2H", "RAFTK_QTF_DIAG", "RAFTK_FARM_SMEM")


@pytest.fixture(scope="module")
def solver():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from raft_b200 import solver as s
    return s


def _env(monkeypatch, env):
    for k in ENV:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


# ---- A. potSecOrder 2 on every rigid-solve variant ----------------------------------------------------------------------

def _tables():
    """-> {name: (qtf, qtf_w, qtf_heads)}: the cfg3q fixture's single-heading table (0.25-3.0 rad/s), the same table on four
    headings with a complex scale per heading, and that one reversed and scaled (a second, different 4-heading table)."""
    G, P = load_golden(QTF_GOLDEN)
    q4 = np.stack([P["qtf"][:, :, 0, :] * s for s in G["mh_scale"]], axis=2)
    return {"1h": (P["qtf"], P["qtf_w"], P["qtf_heads"]), "4h": (q4, P["qtf_w"], G["mh_heads"]),
            "4hb": (q4[:, :, ::-1, :] * (0.5 - 0.25j), P["qtf_w"], G["mh_heads"])}


TABLES = _tables()


def _with_table(P, table):
    q, qw, qh = TABLES[table]
    return dict(P, qtf=q, qtf_w=qw, qtf_heads=qh)


def _stiffer(P):
    """Another design on the same grid: the same platform with 30 % more hydrostatic / mooring stiffness."""
    return dict(P, C0=P["C0"] * 1.3)


_ORACLE_CACHE = {}


def _oracle(oracle, P, key, cs):
    """Oracle Xi / status with the design's QTF force in the loop, and that force per case (cached per design, grid, table and
    sea-state seed)."""
    if key not in _ORACLE_CACHE:
        od = oracle.OracleDesign(P)
        Xi, st, _ = oracle.solve_cases(od, cs, nIter=10)
        F2, F2m = [], []
        for c in range(len(cs["Hs"])):
            fm, f = oracle.hydro_force_2nd(od, cs["beta_deg"][c] * DEG, oracle.jonswap(P["w"], cs["Hs"][c], cs["Tp"][c], 0.0))
            F2.append(f)
            F2m.append(fm)
        _ORACLE_CACHE[key] = dict(Xi=Xi, status=st, F_2nd=np.array(F2), F_2nd_mean=np.array(F2m))
    return _ORACLE_CACHE[key]


def _solve(solver, monkeypatch, shape, packed, cases, want=("Xi", "status", "F_2nd", "F_2nd_mean"), env=None, out=None):
    _env(monkeypatch, dict(shape[3], **(env or {})))
    r = solver.solve_dynamics(solver.DesignBatch(packed), cases, n_iter=10, cluster_size=shape[2], want=want, out=out)
    return r, solver.last_dispatch()


def _check_vs_oracle(r, d, o):
    assert np.array_equal(r["status"][d, :, :2], o["status"][:, :2]) and np.all(r["status"][d, :, 2] == 0), (r["status"][d], o["status"])
    assert response_err(r["Xi"][d], o["Xi"]) < RTOL
    assert np.abs(o["F_2nd"]).max() > 0
    assert relerr(r["F_2nd"][d], o["F_2nd"]) < RTOL and relerr(r["F_2nd_mean"][d], o["F_2nd_mean"]) < RTOL


@pytest.mark.parametrize("shape", SHAPES, ids=_shape_id)
def test_qtf_force_in_branch_vs_oracle(shape, solver, monkeypatch, oracle):
    """Force computed inside the call, on the variant the planner picks: status, Xi and the force against the oracle; the
    same design without its QTF is far off.  With the diagonal force kernel, the force handed in precomputed through
    cases.F_2nd (design without its table) gives the same bits as the in-call route."""
    name, nw = shape[:2]
    P = _design(name, nw)
    Pq = _with_table(P, "1h")
    sea = _sea_states(SEEDS[name])
    ct = solver.CaseTable(sea)
    r, rec = _solve(solver, monkeypatch, shape, Pq, ct)
    _check_record(rec, shape)
    o = _oracle(oracle, Pq, (name, nw, "1h", 0), sea)
    _check_vs_oracle(r, 0, o)
    plain, rec0 = _solve(solver, monkeypatch, shape, P, ct, want=("Xi", "status"))
    _check_record(rec0, shape)
    assert response_err(plain["Xi"][0], o["Xi"]) > MOVES
    diag, rec_d = _solve(solver, monkeypatch, shape, Pq, ct, env={"RAFTK_QTF_DIAG": "1"})
    _check_record(rec_d, shape)
    f2 = solver.second_order_force(solver.DesignBatch(Pq), ct)
    assert solver.last_dispatch()["kernel"] == "qtf-diag"
    pre, rec_p = _solve(solver, monkeypatch, shape, P, solver.CaseTable(sea, F_2nd=f2["F_2nd"]), want=("Xi", "status"))
    _check_record(rec_p, shape)
    assert np.array_equal(diag["F_2nd"], f2["F_2nd"]) and np.array_equal(diag["F_2nd_mean"], f2["F_2nd_mean"])
    assert np.array_equal(pre["Xi"], diag["Xi"]) and np.array_equal(pre["status"], diag["status"])
    _check_vs_oracle(diag, 0, o)


def _pick(name, kernel, f0g=False, env=None):
    return next(s for s in SHAPES if s[0] == name and s[4] == kernel and s[5] == f0g and (env is None or s[3] == env))


MIX_SHAPES = [_pick("cfg2", "fused2-cluster"), _pick("cfg2", "fused2-grid"), _pick("cfg2", "v1", env={}),
              next(s for s in SHAPES if s[0] == "cfg2" and s[4] == "v1" and s[3] and s[2] == 4)]


@pytest.mark.parametrize("shape", MIX_SHAPES, ids=_shape_id)
def test_four_heading_table_vs_oracle(shape, solver, monkeypatch, oracle):
    """The 4-heading table (interpolated between headings, clamped at the ends) on fused2 and v1, both force kernels."""
    name, nw = shape[:2]
    Pq = _with_table(_design(name, nw), "4h")
    sea = _sea_states(SEEDS[name] + 100)
    sea["beta_deg"][0] = -135.0                           # before the first heading (-90 deg): the clamped end
    o = _oracle(oracle, Pq, (name, nw, "4h", 100), sea)
    for env in ({}, {"RAFTK_QTF_DIAG": "1"}):
        r, rec = _solve(solver, monkeypatch, shape, Pq, solver.CaseTable(sea), env=env)
        _check_record(rec, shape)
        _check_vs_oracle(r, 0, o)


DESIGN_AXIS_SHAPES = [_pick("cfg2", "fused2-cluster"), _pick("cfg2", "v1", env={}),
                      next(s for s in SHAPES if s[0] == "cfg2" and s[4] == "v1" and s[3] and s[2] == 2)]


@pytest.mark.parametrize("shared", [0, 1])
@pytest.mark.parametrize("shape", DESIGN_AXIS_SHAPES, ids=_shape_id)
def test_design_axis_vs_oracle(shape, shared, solver, monkeypatch, oracle):
    """Two designs in one call: each with its own 4-heading table (qtf_shared 0), or both on one table (qtf_shared 1).
    Design 1 reads its own rows of the force, and its own table."""
    name, nw = shape[:2]
    P = _design(name, nw)
    tb = "4h" if shared else "4hb"
    packs = [_with_table(P, "4h"), _with_table(_stiffer(P), tb)]
    if shared:
        packs[1]["qtf"] = packs[0]["qtf"]
    batch = solver.DesignBatch(packs)
    assert batch.qtf_shared == shared
    sea = _sea_states(SEEDS[name] + 200)
    for env in ({}, {"RAFTK_QTF_DIAG": "1"}):
        _env(monkeypatch, dict(shape[3], **env))
        r = solver.solve_dynamics(batch, solver.CaseTable(sea), n_iter=10, cluster_size=shape[2], want=("Xi", "status", "F_2nd", "F_2nd_mean"))
        rec = solver.last_dispatch()
        assert rec["kernel"] == shape[4] and rec["cluster_size"] == shape[2] and rec["f0_global"] == shape[5], rec
        for d, (Pd, key) in enumerate(zip(packs, ((name, nw, "4h", 200), (name + "-stiff", nw, tb, 200)))):
            _check_vs_oracle(r, d, _oracle(oracle, Pd, key, sea))
    assert response_err(r["Xi"][1], r["Xi"][0]) > MOVES
    if not shared:
        assert relerr(r["F_2nd"][1], r["F_2nd"][0]) > MOVES


TRAIN_SHAPES = [_pick("cfg2", "fused256"), _pick("cfg2", "fused2-cluster")]


@pytest.mark.parametrize("shape", TRAIN_SHAPES, ids=_shape_id)
def test_wave_trains_vs_oracle(shape, solver, monkeypatch, oracle):
    """Single-train cases and a three-train case: every train gets its own force (raft_model.py:1210-1211), the primary's
    loop uses its own; against oracle.solve_dynamics_trains."""
    name, nw = shape[:2]
    Pq = _with_table(_design(name, nw), "1h")
    tab = _train_table()
    r, rec = _solve(solver, monkeypatch, shape, Pq, solver.CaseTable(tab))
    assert rec["trains"], rec
    _check_record(dict(rec, trains=False), shape)
    od = oracle.OracleDesign(Pq)
    pr = tab["primary"]
    for p in np.unique(pr):
        rows = np.flatnonzero(pr == p)
        Xo, so = oracle.solve_dynamics_trains(od, tab["spec"][rows], tab["Hs"][rows], tab["Tp"][rows], tab["gamma"][rows], tab["beta_deg"][rows], nIter=10)
        assert np.array_equal(r["status"][0, p, :2], so[:2]), (p, r["status"][0, p], so)
        for h, row in enumerate(rows):
            assert response_err(r["Xi"][0, row], Xo[h]) < RTOL, (p, h)
            fm, f = oracle.hydro_force_2nd(od, tab["beta_deg"][row] * DEG, oracle.jonswap(Pq["w"], tab["Hs"][row], tab["Tp"][row], 0.0))
            assert relerr(r["F_2nd"][0, row], f) < RTOL and relerr(r["F_2nd_mean"][0, row], fm) < RTOL
    plain, _ = _solve(solver, monkeypatch, shape, _design(name, nw), solver.CaseTable(tab), want=("Xi", "status"))
    assert response_err(plain["Xi"][0, 1:4], r["Xi"][0, 1:4]) > MOVES


D2H_SHAPES = [_pick("cfg2", "fused128"), _pick("cfg2", "fused256"), _pick("cfg2", "fused256", True), _pick("cfg2", "fused2-cluster"),
              _pick("cfg2", "fused2-grid")]


@pytest.mark.parametrize("shape", D2H_SHAPES, ids=_shape_id)
def test_pinned_outputs_with_force(shape, solver, monkeypatch):
    """Page-locked Xi and status (the solve kernel stores them straight into host memory) with the force computed in the
    call: bit-identical to the copy path (RAFTK_NO_DIRECT_D2H=1)."""
    name, nw = shape[:2]
    Pq = _with_table(_design(name, nw), "1h")
    ct = solver.CaseTable(_sea_states(SEEDS[name]))
    nC = ct.n_cases

    def pinned():
        return dict(Xi=solver.pinned_empty([1, nC, 6, nw], np.complex128), status=solver.pinned_empty([1, nC, 4], np.int32),
                    F_2nd=solver.pinned_empty([1, nC, 6, nw], np.float64), F_2nd_mean=solver.pinned_empty([1, nC, 6], np.float64))
    direct, rec = _solve(solver, monkeypatch, shape, Pq, ct, out=pinned(), env={"RAFTK_QTF_DIAG": "1"})
    assert rec["direct_d2h"] and rec["kernel"] == shape[4] and rec["f0_global"] == shape[5], rec
    copy, rec2 = _solve(solver, monkeypatch, shape, Pq, ct, out=pinned(), env={"RAFTK_QTF_DIAG": "1", "RAFTK_NO_DIRECT_D2H": "1"})
    assert not rec2["direct_d2h"] and rec2["kernel"] == shape[4], rec2
    for k in direct:
        assert np.array_equal(direct[k], copy[k]), k
    assert np.abs(direct["F_2nd"]).max() > 0 and np.all(direct["status"][0, :, 0] > 0)


# ---- B. the farm kernels with a second-order force ---------------------------------------------------------------------

FARM_NW, FARM_MAX_FREQ = 96, 0.2            # Hz: the grid reaches 1.26 rad/s, inside the table's 0.25-3.0 rad/s
FARM_SHAPES = [(2, {}, "farm-rows12"), (2, {"RAFTK_FARM_SMEM": "1"}, "farm-warp"), (5, {}, "farm-block"), (20, {}, "farm-block"),
               (21, {}, "farm-global")]


def _farm_cases():
    return dict(Hs=np.array([6.0, 3.0]), Tp=np.array([12.0, 8.0]), gamma=np.zeros(2), beta_deg=np.array([0.0, -70.0]), spec=np.zeros(2, dtype=np.int32))


@pytest.mark.parametrize("N,env,kernel", FARM_SHAPES, ids=lambda x: x if isinstance(x, (int, str)) else "")
def test_farm_with_qtf_vs_oracle(N, env, kernel, solver, monkeypatch):
    """Every FOWT of the farm with the cfg3q table: the system response against the oracle's per-FOWT solves (force in the
    loop) + explicit-inverse system response, pass counts identical; the same farm without QTFs is far off."""
    import bench_extra
    packs, C_arr, _ = bench_extra.farm_designs(N, nw=FARM_NW, max_freq=FARM_MAX_FREQ)
    qpacks = [_with_table(P, "1h") for P in packs]
    cs = _farm_cases()
    _env(monkeypatch, env)
    out = solver.solve_dynamics_farm(solver.DesignBatch(qpacks), solver.CaseTable(cs), C_arr=C_arr, n_iter=10)
    rec = solver.last_dispatch()
    assert rec["family"] == "farm" and rec["kernel"] == kernel, rec
    Xo, passes = bench_extra._oracle_farm(qpacks, C_arr, cs)
    assert np.array_equal(passes, out["status"][:, :, 0]) and not np.any(out["info"])
    err = max(response_err(out["Xi_sys"][:, 6 * i:6 * i + 6], Xo[:, 6 * i:6 * i + 6]) for i in range(N))
    assert err < 1e-9, err
    plain = solver.solve_dynamics_farm(solver.DesignBatch(packs), solver.CaseTable(cs), C_arr=C_arr, n_iter=10)
    assert solver.last_dispatch()["kernel"] == kernel
    assert max(response_err(plain["Xi_sys"][:, 6 * i:6 * i + 6], Xo[:, 6 * i:6 * i + 6]) for i in range(N)) > MOVES


def test_slender_farm_response_vs_oracle(solver, slender_pair, monkeypatch):
    """SlenderSession.farm_response on a potSecOrder 1 pair through the shared-memory warp kernel, against the oracle's
    potSecOrder 1 solves + system response."""
    import bench_extra
    packs = slender_pair(201)
    _env(monkeypatch, {"RAFTK_FARM_SMEM": "1"})
    cs = _farm_cases()
    k = np.diag([8e4, 8e4, 0, 0, 0, 5e7])
    C_arr = np.block([[k, -k], [-k, k]])
    s = solver.SlenderSession(packs, solver.CaseTable(cs), want=("Xi", "status", "B_drag", "F_drag", "F_iner", "F_2nd"))
    s.solve(n_iter=10)
    xi, info = s.farm_response(C_arr=C_arr)
    assert solver.last_dispatch()["kernel"] == "farm-warp"
    xi, info = xi.cpu().numpy(), info.cpu().numpy()
    Xo, passes = bench_extra._oracle_farm(packs, C_arr, cs)
    assert np.array_equal(passes, s.out["status"].cpu().numpy()[:, :, 0]) and not info.any()
    assert np.abs(s.out["F_2nd"].cpu().numpy()).max() > 0
    assert max(response_err(xi[:, 6 * i:6 * i + 6], Xo[:, 6 * i:6 * i + 6]) for i in range(2)) < 1e-9


# ---- C. potSecOrder 1 on the device on every fused variant ---------------------------------------------------------------

def _slender_mats():
    z = np.load(os.path.join(GOLDEN, "slender_VolturnUS-S.npz"))
    P = {k[2:]: z[k] for k in z.files if k.startswith("P_")}
    return dict(M_struc=P["M0"] - z["A_hydro_morison"], C_struc=P["C0"] - z["C_moor"], C_moor=z["C_moor"]), float(P["depth"])


def _build_pair(nw):
    """VolturnUS-S (designs.json, potSecOrder 1) and a random strip-theory design on nw bins up to MAX_FREQ, both on the
    fixture's second-order grid (0.04 / 0.008 / 0.2 Hz); their node and member counts differ."""
    from raft_b200 import grid
    from raft_b200.fowt import FOWT
    from test_slender_qtf import _member
    mats, depth = _slender_mats()
    D = json.load(open(os.path.join(GOLDEN, "designs.json")))["test_VolturnUS-S"]
    w = grid.make_w(MAX_FREQ / nw, MAX_FREQ)
    k = grid.wave_number(w, depth)
    second = dict(min_freq2nd=0.04, df_freq2nd=0.008, max_freq2nd=0.2)
    fa = FOWT(dict(D, platform=dict(D["platform"], potSecOrder=1, **second), site=dict(D["site"], water_depth=depth)), w, depth=depth, matrices=mats, k=k)
    rng = np.random.default_rng(14)          # few step classes: the pair still fits every fused variant's shared memory
    plat = dict(potModMaster=0, dlsMax=5.0, members=[_member(rng, i, 30.0, 6.0) for i in range(4)], potSecOrder=1, **second)
    mb = dict(M_struc=np.diag([2e7, 2e7, 2e7, 1.8e10, 1.8e10, 3e10]), C_hydro=np.diag([0, 0, 4e6, 2e9, 2e9, 0.0]),
              C_moor=np.diag([7e4, 7e4, 0, 0, 0, 1.2e8]))
    fb = FOWT(dict(site=dict(water_depth=depth, rho_water=1025.0, g=9.81), platform=plat), w, depth=depth, matrices=mb, k=k)
    packs = []
    for f in (fa, fb):
        f.calcHydroConstants()
        packs.append(f.pack())
    assert np.array_equal(packs[0]["qs_w"], packs[1]["qs_w"]) and len(packs[0]["node_r"]) != len(packs[1]["node_r"])
    return packs


@pytest.fixture(scope="module")
def slender_pair():
    cache = {}

    def get(nw):
        if nw not in cache:
            cache[nw] = _build_pair(nw)
        return cache[nw]
    return get


# (nw, cluster_size, environment, kernel, f0_global) on the two-design batch
SLENDER_SHAPES = [(201, 2, {}, "fused128", False), (333, 2, {}, "fused256", False), (333, 1, {}, "fused256", True),
                  (501, 2, CLUSTER, "fused2-cluster", False), (501, 2, GRID, "fused2-grid", False)]
SL_OUTS = ("Xi", "status", "B_drag", "F_drag", "F_iner", "F_BEM", "zeta", "F_2nd", "F_2nd_mean", "Xi_last", "qtf", "Xi_rao")
SL_CASES = 8


def _sl_id(s):
    return "nw%d-cs%d%s-%s%s" % (s[0], s[1], "".join("-" + v for v in s[2].values()), s[3], "-f0g" if s[4] else "")


def _sl_cases(seed, n=SL_CASES):
    rng = np.random.default_rng(seed)
    return dict(Hs=rng.uniform(1.5, 9.0, n), Tp=rng.uniform(6.0, 17.0, n), gamma=np.zeros(n), beta_deg=rng.uniform(-180, 180, n),
                spec=np.zeros(n, dtype=np.int32))


def _session(solver, packs, ct, qtf_chunk=0, **kw):
    import torch
    s = solver.SlenderSession(packs, ct, want=SL_OUTS, qtf_chunk=qtf_chunk)
    out = s.solve(**kw)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}, solver.last_dispatch()


def _check_slender_vs_oracle(oracle, packs, cs, out, n_iter, tol=0.01, xi_start=0.0):
    """Per unit: status and Xi against oracle.solve_dynamics with the slender-body tables; F_2nd against the oracle's force
    from the unit's own QTF; units that loop A left unconverged carry no QTF, RAO or force.  -> loop A's converged mask."""
    conv = np.zeros(out["status"].shape[:2], dtype=bool)
    for d, P in enumerate(packs):
        od = oracle.OracleDesign(P)
        base = {k: v for k, v in P.items() if not k.startswith("qs_")}
        for c in range(len(cs["Hs"])):
            Xo, so = oracle.solve_dynamics(od, 0, cs["Hs"][c], cs["Tp"][c], 0.0, cs["beta_deg"][c], nIter=n_iter, tol=tol, XiStart=xi_start)
            assert np.array_equal(out["status"][d, c, :2], so[:2]) and out["status"][d, c, 2] == 0, (d, c, out["status"][d, c], so)
            assert response_err(out["Xi"][d, c], Xo) < RTOL, (d, c)
            conv[d, c] = np.any(out["qtf"][d, c] != 0)
            if not conv[d, c]:
                assert np.all(out["F_2nd"][d, c] == 0) and np.all(out["F_2nd_mean"][d, c] == 0) and np.all(out["Xi_rao"][d, c] == 0), (d, c)
                continue
            b = cs["beta_deg"][c] * DEG
            oq = oracle.OracleDesign(dict(base, qtf=out["qtf"][d, c][:, :, None, :], qtf_w=P["qs_w"], qtf_heads=np.array([b])))
            fm, f = oracle.hydro_force_2nd(oq, b, oracle.jonswap(P["w"], cs["Hs"][c], cs["Tp"][c], 0.0))
            assert np.abs(f).max() > 0 and relerr(out["F_2nd"][d, c], f) < RTOL and relerr(out["F_2nd_mean"][d, c], fm) < RTOL, (d, c)
    return conv


@pytest.mark.parametrize("shape", SLENDER_SHAPES, ids=_sl_id)
def test_slender_flow_branch_vs_oracle(shape, solver, slender_pair, monkeypatch, oracle):
    """Loop A, QTF, force and loop B (F_2nd + Xi_init on loop A's plan) on the variant the planner picks for the plain solve
    of the same batch: per unit against the oracle; with the diagonal force kernel every output bit-identical to the host
    entry point and to the host flow."""
    nw, cs_, env, kernel, f0g = shape
    packs = slender_pair(nw)
    cs = _sl_cases(nw)
    ct = solver.CaseTable(cs)
    n_iter = 3                                                  # loop A converges for some units only
    _env(monkeypatch, env)
    plain = solver.DesignBatch([{k: v for k, v in P.items() if not k.startswith("qs_")} for P in packs])
    A = solver.solve_dynamics(plain, ct, n_iter=n_iter, cluster_size=cs_)
    rec_plain = solver.last_dispatch()
    assert rec_plain["kernel"] == kernel and rec_plain["f0_global"] == f0g and rec_plain["cluster_size"] == cs_, rec_plain
    out, rec = _session(solver, packs, ct, n_iter=n_iter, cluster_size=cs_)
    assert rec["family"] == "solve" and rec["kernel"] == kernel and rec["f0_global"] == f0g and rec["cluster_size"] == cs_, rec
    conv = _check_slender_vs_oracle(oracle, packs, cs, out, n_iter)
    assert np.array_equal(conv, A["status"][..., 1] == 1)
    assert conv.any() and (~conv).any(), conv
    assert response_err(out["Xi"][conv], A["Xi"][conv]) > MOVES            # loop B moved the converged units
    monkeypatch.setenv("RAFTK_QTF_DIAG", "1")
    dev, _ = _session(solver, packs, ct, n_iter=n_iter, cluster_size=cs_)
    host = solver.slender_flow_host(packs, ct, n_iter=n_iter, cluster_size=cs_, want=SL_OUTS)
    flow = solver.solve_dynamics_slender(packs, ct, n_iter=n_iter, cluster_size=cs_, want=tuple(k for k in SL_OUTS if k not in ("qtf", "Xi_rao")))
    for k in SL_OUTS:
        assert np.array_equal(dev[k], host[k]), k
        if k in flow:
            assert np.array_equal(dev[k], flow[k]), k


# n_iter 1 and 2 with a loose tolerance, so that loop A converges for some units and loop B (n_iter 0 and 1) decides their result
SLENDER_EDGES = [dict(n_iter=1, tol=0.3), dict(n_iter=2, tol=0.3), dict(n_iter=10, tol=0.05, xi_start=0.3), dict(n_iter=6, qtf_chunk=1)]


@pytest.mark.parametrize("edge", SLENDER_EDGES, ids=lambda e: "-".join("%s%s" % kv for kv in e.items()))
def test_slender_flow_edges_on_fused2(edge, solver, slender_pair, monkeypatch, oracle):
    """k_rao_fused2 (cluster exchange) at n_iter 1 (loop B launched with n_iter 0) and 2, with another tolerance and start
    value, and with one unit per QTF chunk (the designs split across chunks): per unit against the oracle."""
    nw, cs_, env, kernel, _ = SLENDER_SHAPES[3]
    packs = slender_pair(nw)
    cs = _sl_cases(41 + edge["n_iter"])
    _env(monkeypatch, env)
    kw = {k: v for k, v in edge.items() if k != "qtf_chunk"}
    out, rec = _session(solver, packs, solver.CaseTable(cs), qtf_chunk=edge.get("qtf_chunk", 0), cluster_size=cs_, **kw)
    assert rec["kernel"] == kernel, rec
    conv = _check_slender_vs_oracle(oracle, packs, cs, out, edge["n_iter"], tol=edge.get("tol", 0.01), xi_start=edge.get("xi_start", 0.0))
    assert conv.any(), conv


# ---- D. where only the v1 kernel fits --------------------------------------------------------------------------------------

@pytest.mark.parametrize("how", ["forced", "nw601-cs1"])
def test_slender_flow_refused_on_v1(how, solver, slender_pair, monkeypatch):
    """Loop B continues from Xi_init and loop A hands over Xi_last; the v1 kernel takes neither.  potSecOrder 1 on a plan that
    can only be v1 is refused with that message by all three entry points, and nothing is launched."""
    from raft_b200 import _lib
    nw, cs_ = (333, 2) if how == "forced" else (601, 1)
    _env(monkeypatch, {"RAFTK_FORCE_V1": "1"} if how == "forced" else {})
    packs = slender_pair(nw)
    ct = solver.CaseTable(_sl_cases(5, 4))
    plain = solver.DesignBatch([{k: v for k, v in P.items() if not k.startswith("qs_")} for P in packs])
    solver.solve_dynamics(plain, ct, n_iter=4, cluster_size=cs_)
    assert solver.last_dispatch()["kernel"] == "v1"
    s = solver.SlenderSession(packs, ct, want=SL_OUTS)
    n0 = solver.launch_count()
    msg = "Xi_init / outputs.Xi_last need the fused solver"
    with pytest.raises(_lib.RaftkError, match=msg):
        s.solve(n_iter=4, cluster_size=cs_)
    with pytest.raises(_lib.RaftkError, match=msg):
        solver.slender_flow_host(packs, ct, n_iter=4, cluster_size=cs_, want=SL_OUTS)
    with pytest.raises(_lib.RaftkError, match=msg):
        solver.solve_dynamics_slender(packs, ct, n_iter=4, cluster_size=cs_)
    assert solver.launch_count() == n0
