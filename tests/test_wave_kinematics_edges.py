"""Wave kinematics of the rigid solvers at the edges of the site and the grid: high frequencies, shallow and very deep
water, members that walk down from their first node, and members that cross the surface.

The fused kernels evaluate depth_funcs once per member, at its first submerged node z0, and walk the other nodes with
exp(+-k dz) step factors (DESIGN.md section 4).  That walk is inexact where the seed exp(k z0) of a deep-water bin
underflows (k |z0| > 708) or where a member walks down far enough in finite depth for the rounding of (C-S)/2 to grow
(raft_b200.solver.fused_walk_exact); the planner sends such designs to v1, which evaluates depth_funcs at every node.

GPU part: every variant of test_dispatch_solve.SHAPES on those designs and grids, asserted through
solver.last_dispatch(), against the oracle bin by bin (response_err: per frequency, against the largest reference
amplitude of the DOF group at that bin, for Xi and F_iner alike).  The cases put weight on the high bins: a unit and a
constant spectrum next to one JONSWAP.
CPU part: depth_funcs as the oracle evaluates it against 40-digit mpmath, a host model of the walk against the direct
evaluation, and guards that each GPU shape crosses the threshold it is there for."""
import re

import numpy as np
import pytest

from conftest import load_golden, relerr, response_err

RTOL = 1e-10
DEEP_KH = 89.4

CASES = dict(Hs=np.array([1.0, 0.3, 6.0]), Tp=np.array([10.0, 10.0, 9.0]), gamma=np.zeros(3),
             beta_deg=np.array([0.0, 35.0, -120.0]), spec=np.array([1, 2, 0], dtype=np.int32))   # unit, constant, JONSWAP


def _random_member_design(seed, depth, flip=False):
    """test_gpu_parity._random_design at water depth ``depth``, its members scaled in z to stay above the seabed.  ``flip``
    defines every member top-down (rA the upper end, stations and sections reversed: the same geometry, walked from the
    top), so that surface-piercing members start above the waterline and walk down from the first submerged node."""
    from test_gpu_parity import _random_design
    rng = np.random.default_rng(seed)
    design = _random_design(rng, int(rng.integers(3, 8)))
    design["site"]["water_depth"] = float(depth)
    zmin = min(min(m["rA"][2], m["rB"][2]) for m in design["platform"]["members"])
    s = min(1.0, 0.9 * depth / -zmin)
    for m in design["platform"]["members"]:
        m["rA"][2] *= s
        m["rB"][2] *= s
        if flip and m["rA"][2] < m["rB"][2]:
            m["rA"], m["rB"] = m["rB"], m["rA"]
            m["stations"] = [1.0 - v for v in reversed(m["stations"])]
            m["d"] = list(reversed(m["d"]))
    return design, rng


def _seabed_column(design, depth):
    """One more vertical column standing on the seabed: its first node is at z = -h exactly."""
    design["platform"]["members"].append(dict(name="foot", type="rigid", rA=[5.0, -7.0, -float(depth)], rB=[5.0, -7.0, -float(depth) + 12.0],
                                              shape="circ", stations=[0.0, 1.0], d=[6.0, 6.0], gamma=0.0, potMod=False,
                                              Cd=0.8, Ca=0.9, CdEnd=0.6, CaEnd=0.6, Cd_q=0.05, dlsMax=2.0))
    return design


def _pack(design, rng, nw, fmax):
    from raft_b200 import grid
    from raft_b200.fowt import FOWT
    m = rng.uniform(0.5, 3.0) * 1e7
    mats = dict(M_struc=np.diag([m, m, m, m * 900, m * 900, m * 1500]),
                C_struc=np.diag([0, 0, 0, -m * 5, -m * 5, 0.0]),
                C_hydro=np.diag([0, 0, rng.uniform(2, 6) * 1e6, rng.uniform(1, 4) * 1e9, rng.uniform(1, 4) * 1e9, 0.0]),
                C_moor=np.diag([7e4, 7e4, 0, 0, 0, 1.2e8]), B_struc=np.diag(rng.uniform(0, 1e5, 6)))
    f = FOWT(design, grid.make_w(fmax / nw, fmax), depth=design["site"]["water_depth"], matrices=mats)
    f.calcHydroConstants()
    return f.pack()


_DESIGNS = {}


def _design(key, nw):
    """Designs by name: "cfg1@1.22" (a fixture regridded up to 1.22 Hz), "cfg1@1.0/3000m" (the same at 3000 m water
    depth), "rand5/h20" (random members at 20 m depth, grid to 0.5 Hz), "rand5/h20/foot" (plus a column on the seabed),
    "down7/h60" (random members defined top-down, grid to 0.4 Hz)."""
    from raft_b200 import grid
    if (key, nw) not in _DESIGNS:
        if key.startswith("cfg"):
            name, rest = key.split("@")
            fmax, _, site = rest.partition("/")
            fix = dict(cfg1="cfg1_OC3spar", cfg2="cfg2_VolturnUS-S_nw64")[name]
            Q = grid.regrid(load_golden(fix)[1], nw, float(fmax))
            if site:
                Q["depth"] = float(site[:-1])
                Q["k"] = grid.wave_number(Q["w"], Q["depth"])
        else:
            parts = key.split("/")
            kind, seed = re.fullmatch(r"([a-z]+)(\d+)", parts[0]).groups()
            depth = float(parts[1][1:])
            seed = int(seed)
            design, rng = _random_member_design(seed, depth, flip=kind == "down")
            if "foot" in parts:
                design = _seabed_column(design, depth)
            Q = _pack(design, rng, nw, 0.4 if kind == "down" else 0.5)
        _DESIGNS[(key, nw)] = Q
    return _DESIGNS[(key, nw)]


def _walk_exact(P):
    from raft_b200 import solver
    return solver.DesignBatch(P).walk_exact


def _node_z(P):
    ms = np.asarray(P["mem_start"])
    out = []
    for m in range(len(ms) - 1):
        ls = np.asarray(P["node_ls"][ms[m]:ms[m + 1]], dtype=float)
        if len(ls):
            out.append(float(P["mem_rA"][m][2]) + ls * float(P["mem_q"][m][2]))
    return out


# =============================================================================== CPU part

def _depth_funcs(k, h, z):
    """depth_funcs as the oracle evaluates it (oracle.wave_kin, raft_oracle.c ro_wave_kin) -> S, C, P."""
    from oracle import oracle
    u, _, p = oracle.wave_kin(np.ones(len(k)), 0.0, np.ones(len(k)), k, h, np.array([0.0, 0.0, z]), rho=1.0, g=1.0)
    return (u[2] / 1j).real, u[0].real, p.real


def _depth_funcs_mp(k, h, z):
    import mpmath as mp
    mp.mp.dps = 40
    deep = float(k) * float(h) > DEEP_KH                  # the branch is taken on the double product, as in the oracle
    k, h, z = mp.mpf(k), mp.mpf(h), mp.mpf(z)
    if z > 0:
        return 0, 0, 0
    if deep:
        e = mp.exp(k * z)
        return e, e, e + mp.exp(-k * (z + 2 * h))
    return mp.sinh(k * (z + h)) / mp.sinh(k * h), mp.cosh(k * (z + h)) / mp.sinh(k * h), mp.cosh(k * (z + h)) / mp.cosh(k * h)


@pytest.mark.parametrize("h", [20.0, 200.0, 3000.0])
def test_depth_funcs_vs_mpmath(h, oracle):
    """kh from 1e-4 to 3x past the deep-water switch at 89.4, z from the seabed to 15 m above the surface: each of S, C, P
    to 1e-13 of its own value (the finite-depth ratios are well conditioned; above the surface the oracle returns 0)."""
    kh = np.concatenate([np.geomspace(1e-4, 80.0, 40), [89.39, 89.4, 89.41], np.geomspace(90.0, 270.0, 8)])
    k = kh / h
    assert (kh > DEEP_KH).any() and (kh <= DEEP_KH).any()
    for z in np.concatenate([[-h, -h + 1e-9 * h], -h * np.geomspace(0.9, 1e-4, 12), [0.0, 1.0, 15.0]]):
        S, Cc, Pp = _depth_funcs(k, h, z)
        for i in range(len(k)):
            ref = [float(v) for v in _depth_funcs_mp(k[i], h, z)]
            for got, want in zip((S[i], Cc[i], Pp[i]), ref):
                assert abs(got - want) <= 1e-13 * abs(want) + 1e-300, (h, kh[i], z, got, want)


def test_deep_water_switch_is_continuous_at_the_surface_scale():
    """The deep-water formulas drop e^-2k(z+h) against the finite-depth ones: below 1e-30 of the surface value at the
    switch, so the branch taken at kh = 89.4 cannot be seen in the kinematics."""
    import mpmath as mp
    mp.mp.dps = 60
    h = 100.0
    k = mp.mpf(DEEP_KH + 1e-9) / h
    for z in np.linspace(-h, 0.0, 21):
        z = mp.mpf(z)
        deep = mp.exp(k * z)
        fin = mp.cosh(k * (z + h)) / mp.sinh(k * h)
        assert abs(deep - fin) < mp.mpf(1e-30), float(z)


def _walk(k, h, zs):
    """The fused kernels' walk in double: (C, S) at every node of one member from its first node's seed."""
    S0, C0, _ = _depth_funcs(k, h, zs[0])
    ap, am = 0.5 * (C0 + S0), 0.5 * (C0 - S0)
    out = []
    for j, z in enumerate(zs):
        if j:
            ap = ap * np.exp(k * (z - zs[j - 1]))
            am = am * np.exp(-k * (z - zs[j - 1]))
        out.append((ap + am, ap - am))
    return np.array(out)


def _walk_err(P):
    """Largest error of the walked C and S over every node of the design, per bin against the largest direct value of any
    node at that bin."""
    k, h = np.asarray(P["k"], dtype=float), float(P["depth"])
    err = np.zeros(len(k))
    scale = np.zeros(len(k))
    walks = []
    for zs in _node_z(P):
        W = _walk(k, h, zs)
        D = np.array([_depth_funcs(k, h, z)[1::-1] for z in zs])
        walks.append(np.abs(W - D).max(axis=(0, 1)))
        scale = np.maximum(scale, np.abs(D).max(axis=(0, 1)))
    for e in walks:
        err = np.maximum(err, e)
    return float((err / np.where(scale > 0, scale, 1.0)).max())


WALK_CASES = [("cfg1@1.0", 201, True), ("cfg1@1.22", 201, False), ("cfg1@1.3", 201, False), ("cfg1@2.0", 201, False),
              ("cfg2@2.6", 501, True), ("cfg2@3.2", 201, False), ("cfg1@1.0/3000m", 201, True),
              ("rand5/h20", 301, True), ("rand6/h35", 301, True), ("rand7/h60", 301, True), ("rand5/h20/foot", 301, True),
              ("down7/h60", 301, False), ("down8/h200", 301, False), ("down5/h20", 301, True)]


@pytest.mark.parametrize("key,nw,exact", WALK_CASES, ids=lambda x: str(x))
def test_walk_model_and_flag(key, nw, exact, oracle):
    """fused_walk_exact on each design of the GPU part, and a host model of the kernels' walk: where the flag holds, the
    walked depth factors equal the direct ones to 1e-12 per bin.  The flag is conservative: some designs it sends to v1
    would walk to 1e-12 (a downward walk whose (C-S)/2 rounds to exactly 0), none it keeps on the fused kernels walks
    worse."""
    P = _design(key, nw)
    assert _walk_exact(P) == exact
    if exact:
        assert _walk_err(P) < 1e-12


def test_thresholds_the_shapes_cross():
    """Each GPU design crosses the edge it is there for."""
    from raft_b200 import solver
    kz = {}
    for key in ("cfg1@1.0", "cfg1@1.22", "cfg1@1.3", "cfg1@2.0", "cfg2@3.2"):
        P = _design(key, 201)
        z0 = min(zs[0] for zs in _node_z(P))
        deep = P["k"] * P["depth"] > DEEP_KH
        kz[key] = float(P["k"][deep].max() * -z0)
    assert kz["cfg1@1.0"] < solver.WALK_SEED_EXP
    assert 708.4 < kz["cfg1@1.22"] < 745.0                    # the seed is subnormal
    assert kz["cfg1@1.3"] > 745.0 and kz["cfg1@2.0"] > 745.0 and kz["cfg2@3.2"] > 745.0   # the seed is exactly 0
    deep3000 = _design("cfg1@1.0/3000m", 201)
    assert np.mean(deep3000["k"] * 3000.0 > DEEP_KH) > 0.9
    for key in ("rand5/h20", "rand6/h35", "rand7/h60"):
        P = _design(key, 301)
        assert P["k"][0] * P["depth"] < 3e-2 and not np.any(P["k"] * P["depth"] > DEEP_KH)
    foot = _design("rand5/h20/foot", 301)
    assert min(zs[0] for zs in _node_z(foot)) == -20.0
    # the random designs the GPU part expects on a fused kernel fit one: the planner's workspace is not v1's tables
    import ctypes as C
    from raft_b200 import _lib
    for key in ("rand5/h20", "rand6/h35", "rand7/h60", "rand5/h20/foot", "down5/h20"):
        b = solver.DesignBatch(_design(key, 301))
        d = b.struct(lambda name: b.arrays[name].ctypes.data)
        assert _lib.lib.raftk_solve_workspace_bytes(C.byref(d), 3) < _lib.lib.raftk_workspace_bytes(C.byref(d), 3), key
    for key in ("down7/h60", "down8/h200", "down5/h20"):
        zs = _node_z(_design(key, 301))
        assert any(len(z) > 1 and z[-1] < z[0] - 5.0 for z in zs)                    # members walk down
    # the deep-water switch between the two bins of one k_rao_fused2 thread (bins t and t + 128 of a 251-bin slice)
    for key, first_half in (("cfg2@2.6", True), ("cfg2@0.9", False)):
        P = _design(key, 501)
        s = int(np.argmax(P["k"] * P["depth"] > DEEP_KH))
        assert 0 < s < 251 and (s < 128) == first_half, s


# =============================================================================== GPU part

FORCE = {"RAFTK_FORCE_V1": "1"}
CLUSTER = {"RAFTK_FUSED2_XCHG": "cluster"}
GRID = {"RAFTK_FUSED2_XCHG": "grid"}
# (nw, cluster_size, environment, kernel, f0_global) of test_dispatch_solve.SHAPES for the fixtures
VARIANTS = [(201, 2, {}, "fused128", False), (333, 2, {}, "fused256", False), (501, 1, {}, "fused256", True),
            (501, 2, CLUSTER, "fused2-cluster", False), (501, 2, GRID, "fused2-grid", False), (601, 1, {}, "v1", False),
            (201, 1, FORCE, "v1", False)]
CFG2_VARIANTS = [(201, 2, {}, "fused128", False), (333, 1, {}, "fused256", True), (501, 2, CLUSTER, "fused2-cluster", False),
                 (501, 2, GRID, "fused2-grid", False), (201, 1, FORCE, "v1", False)]
SHAPES = ([("cfg1@%s" % f,) + v for f in ("1.0", "1.22", "1.3", "2.0") for v in VARIANTS]
          + [("cfg2@%s" % f,) + v for f in ("3.2",) for v in CFG2_VARIANTS]
          + [("cfg2@%s" % f,) + v for f in ("2.6", "0.9") for v in CFG2_VARIANTS if v[3].startswith("fused2")]
          + [("cfg1@1.0/3000m",) + v for v in VARIANTS if v[3] in ("fused128", "fused2-cluster", "v1")]
          + [(k, 301, 2, e, kern, False) for k in ("rand5/h20", "rand6/h35", "rand7/h60", "rand5/h20/foot", "down7/h60", "down8/h200", "down5/h20")
             for e, kern in (({}, "fused"), (FORCE, "v1"))])


def _shape_id(s):
    env = "".join("-" + v for v in s[3].values())
    return "%s-nw%d-cs%d%s-%s%s" % (s[0], s[1], s[2], env, s[4], "-f0g" if s[5] else "")


_ORACLE = {}


def _oracle(oracle, key, nw, P=None):
    if (key, nw) not in _ORACLE:
        od = oracle.OracleDesign(P if P is not None else _design(key, nw))
        Xi, st, _ = oracle.solve_cases(od, CASES, nIter=10)
        Bd, Fi = [], []
        for c in range(len(CASES["Hs"])):
            args = (int(CASES["spec"][c]), CASES["Hs"][c], CASES["Tp"][c], 0.0, CASES["beta_deg"][c])
            Bd.append(oracle.solve_dynamics(od, *args, nIter=10, want_Z=True)[3])
            Fi.append(oracle.calc_hydro_excitation(od, *args)[2])
        _ORACLE[(key, nw)] = dict(Xi=Xi, status=st, B_drag=np.array(Bd), F_iner=np.array(Fi))
    return _ORACLE[(key, nw)]


def _solve(monkeypatch, P, cs, env, cases=None):
    from raft_b200 import solver
    for k in ("RAFTK_FORCE_V1", "RAFTK_FUSED2_XCHG", "RAFTK_NO_DIRECT_D2H"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    r = solver.solve_dynamics(solver.DesignBatch(P), cases or solver.CaseTable(CASES), n_iter=10, cluster_size=cs,
                              want=("Xi", "status", "B_drag", "F_iner"))
    return r, solver.last_dispatch()


def _check(r, o):
    errs = dict(Xi=response_err(r["Xi"][0], o["Xi"]), F_iner=response_err(r["F_iner"][0], o["F_iner"]),
                B_drag=relerr(r["B_drag"][0], o["B_drag"]))
    assert np.array_equal(r["status"][0, :, :2], o["status"][:, :2]) and np.all(r["status"][0, :, 2] == 0), (r["status"][0], o["status"])
    assert max(errs.values()) < RTOL, errs


def _check_kernel(rec, shape, exact):
    key, nw, cs, env, kernel, f0g = shape
    assert rec["family"] == "solve", rec
    if env == FORCE:
        assert rec["kernel"] == "v1" and rec["inexact_walk"] == (not exact), rec
    elif not exact:
        assert rec["kernel"] == "v1" and rec["inexact_walk"], rec
    elif kernel == "fused":
        assert rec["kernel"] != "v1" and not rec["inexact_walk"], rec
    else:
        assert rec["kernel"] == kernel and rec["f0_global"] == f0g and not rec["inexact_walk"], rec
        assert rec["cluster_size"] == cs and rec["bins_per_cta"] == -(-nw // cs), rec


@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES, ids=_shape_id)
def test_solve_vs_oracle(shape, monkeypatch, oracle):
    """Xi, status, B_drag and F_iner of the variant the planner picks, bin by bin against the oracle; the planner picks the
    shape's kernel where the walk is exact and v1, marked inexact_walk, where it is not."""
    key, nw, cs, env = shape[:4]
    P = _design(key, nw)
    r, rec = _solve(monkeypatch, P, cs, env)
    _check(r, _oracle(oracle, key, nw))
    _check_kernel(rec, shape, _walk_exact(P))


@pytest.mark.gpu
@pytest.mark.parametrize("key,nw", [("cfg1@1.0", 201), ("cfg1@1.3", 201), ("cfg2@3.2", 201), ("rand5/h20", 301),
                                    ("cfg1@1.0/3000m", 201), ("down7/h60", 301)])
def test_excitation_and_linearization_vs_oracle(key, nw, oracle):
    """raftk_hydro_excitation / raftk_hydro_linearization (the v1 tables, one node at a time) on the same designs: F_iner
    per bin, and B_drag / F_drag at the oracle's converged response."""
    from raft_b200 import solver
    P = _design(key, nw)
    batch, ct = solver.DesignBatch(P), solver.CaseTable(CASES)
    exc = solver.hydro_excitation(batch, ct, want=("F_iner", "zeta"))
    o = _oracle(oracle, key, nw)
    assert response_err(exc["F_iner"][0], o["F_iner"]) < RTOL
    od = oracle.OracleDesign(P)
    lin = solver.hydro_linearization(batch, ct, o["Xi"][None], want=("B_drag", "F_drag"))
    for c in range(len(CASES["Hs"])):
        args = (int(CASES["spec"][c]), CASES["Hs"][c], CASES["Tp"][c], 0.0, CASES["beta_deg"][c])
        u = oracle.calc_hydro_excitation(od, *args)[3]
        _, B, F = oracle.calc_hydro_linearization(od, u, o["Xi"][c])
        assert relerr(lin["B_drag"][0, c], B) < RTOL
        assert response_err(lin["F_drag"][0, c], F) < RTOL


@pytest.mark.gpu
@pytest.mark.parametrize("key,nw,cs,env,kernel", [("cfg1@1.0", 501, 2, CLUSTER, "fused2-cluster"), ("cfg1@1.3", 501, 2, CLUSTER, "v1")])
def test_operating_point_vs_oracle(key, nw, cs, env, kernel, monkeypatch, oracle):
    """The operating-point instantiation (raftk_cases.op) on one exact and one inexact grid, against the oracle with the
    point's tables folded into the design."""
    from test_operating_points import _fold, _op_tables
    from raft_b200 import solver
    P = _design(key, nw)
    A, B = _op_tables(np.random.default_rng(5), P, 1, 1)
    ct = solver.CaseTable(CASES, ops=dict(op=np.zeros(3, dtype=np.int32), A_w=A[0], B_w=B[0]))
    r, rec = _solve(monkeypatch, P, cs, env, cases=ct)
    assert rec["kernel"] == kernel and rec["inexact_walk"] == (kernel == "v1"), rec
    _check(r, _oracle(oracle, key + "+op", nw, _fold(P, A[0, 0], B[0, 0])))


@pytest.mark.gpu
def test_inexact_walk_refuses_fused_only_inputs(monkeypatch):
    """Where the walk sends a design to v1, the inputs only the fused solvers take are refused with that reason before any
    launch, not answered by a kernel that walks wrong."""
    from test_dispatch_solve import _train_table
    from raft_b200 import _lib, solver
    P = _design("cfg1@1.3", 201)
    r, rec = _solve(monkeypatch, P, 2, {})
    assert rec["kernel"] == "v1" and rec["inexact_walk"], rec
    before = _lib.lib.raftk_launch_count()
    with pytest.raises(_lib.RaftkError, match="node walk is inexact"):
        solver.solve_dynamics(solver.DesignBatch(P), solver.CaseTable(_train_table()), n_iter=10)
    with pytest.raises(_lib.RaftkError, match="node walk is inexact"):
        solver.solve_dynamics(solver.DesignBatch(P), solver.CaseTable(CASES), n_iter=10, want=("Xi", "status", "Xi_last"))
    assert _lib.lib.raftk_launch_count() == before and solver.last_dispatch()["kernel"] == "none"
