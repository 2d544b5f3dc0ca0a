"""Every kernel variant the rigid solver's planner can pick (raftk.cu: plan_solve), reached by the shapes
that make the planner itself choose it, asserted through solver.last_dispatch(), and compared with the C oracle:
Xi and status with oracle.solve_cases, B_drag with oracle.solve_dynamics(want_Z=True), F_iner / F_BEM / zeta with
oracle.calc_hydro_excitation.  Frequency counts are ragged (nw % cluster_size != 0, bins per CTA not a multiple of 32).
The variants agree with each other to 1e-12 on the same inputs.  Also: v1 design chunking, the direct device-to-host
epilogue of the host entry point (page-locked Xi / status), and the inputs only the fused solvers support."""
import numpy as np
import pytest

from conftest import load_golden, relerr, response_err

pytestmark = pytest.mark.gpu
RTOL = 1e-10
MAX_FREQ = 0.4                     # Hz; min_freq = MAX_FREQ / nw
N_CASES = 3


def _sea_states(seed, n=N_CASES):
    rng = np.random.default_rng(seed)
    return dict(Hs=rng.uniform(1, 10, n), Tp=rng.uniform(5, 18, n), gamma=np.zeros(n), beta_deg=rng.uniform(-180, 180, n),
                spec=np.zeros(n, dtype=np.int32))


def _random_packed(seed):
    """The synthetic platform of test_gpu_parity.test_random_designs_vs_oracle[seed] (inclined, tapered, rectangular members)."""
    from test_gpu_parity import _random_design
    from raft_b200 import grid
    from raft_b200.fowt import FOWT
    rng = np.random.default_rng(seed)
    design = _random_design(rng, int(rng.integers(2, 9)))
    nw = int(rng.integers(40, 300))
    m = rng.uniform(0.5, 3.0) * 1e7
    mats = dict(M_struc=np.diag([m, m, m, m * 900, m * 900, m * 1500]) + rng.normal(size=(6, 6)) * m * 0.01,
                C_struc=np.diag([0, 0, 0, -m * 5, -m * 5, 0.0]),
                C_hydro=np.diag([0, 0, rng.uniform(2, 6) * 1e6, rng.uniform(1, 4) * 1e9, rng.uniform(1, 4) * 1e9, 0.0]),
                C_moor=np.diag([7e4, 7e4, 0, 0, 0, 1.2e8]), B_struc=np.diag(rng.uniform(0, 1e5, 6)))
    f = FOWT(design, grid.make_w(0.3 / nw, 0.3), depth=design["site"]["water_depth"], matrices=mats)
    f.calcHydroConstants()
    return f.pack()


def _regrid_bem(P, nw):
    """A BEM design on another grid: its frequency tables (A_w, B_w, X_BEM) linearly interpolated onto the new bins.  The
    result is a different but valid design, and the oracle reads the same tables."""
    from raft_b200 import grid
    Q = grid.regrid({k: v for k, v in P.items() if k not in ("A_w", "B_w", "X_BEM")}, nw, MAX_FREQ)
    w0, w1 = np.asarray(P["w"]), Q["w"]
    for key in ("A_w", "B_w", "X_BEM"):
        a = np.asarray(P[key])
        flat = a.reshape(-1, a.shape[-1])
        out = np.stack([np.interp(w1, w0, r.real) + (1j * np.interp(w1, w0, r.imag) if np.iscomplexobj(r) else 0) for r in flat])
        Q[key] = out.reshape(a.shape[:-1] + (len(w1),)).astype(a.dtype)
    return Q


_DESIGN_CACHE = {}


def _design(name, nw):
    key = (name, nw)
    if key not in _DESIGN_CACHE:
        from raft_b200 import grid
        if name == "cfg2":
            _DESIGN_CACHE[key] = grid.regrid(load_golden("cfg2_VolturnUS-S_nw64")[1], nw, MAX_FREQ)
        elif name == "cfg1":
            _DESIGN_CACHE[key] = grid.regrid(load_golden("cfg1_OC3spar")[1], nw, MAX_FREQ)
        elif name == "cfg3":
            _DESIGN_CACHE[key] = _regrid_bem(load_golden("cfg3_OC4semi-WAMIT_nw128")[1], nw)
        else:
            if (name, 0) not in _DESIGN_CACHE:
                _DESIGN_CACHE[(name, 0)] = _random_packed(int(name[len("rand"):]))
            _DESIGN_CACHE[key] = grid.regrid(_DESIGN_CACHE[(name, 0)], nw, MAX_FREQ)
    return _DESIGN_CACHE[key]


SEEDS = dict(cfg2=21, cfg1=22, cfg3=23, rand2=24)
FORCE = {"RAFTK_FORCE_V1": "1"}
CLUSTER = {"RAFTK_FUSED2_XCHG": "cluster"}
GRID = {"RAFTK_FUSED2_XCHG": "grid"}

# (design, nw, cluster_size, environment, kernel, f0_global).  Chosen from the planner's rules (fused2: 192 < bins per CTA
# <= 256; k_rao_fused<T>: T = 256 above 128 bins, shared-memory limits 112 / 226 KB with or without F0 on chip; v1 past
# 512 bins per CTA or when forced); the test asserts that the planner agrees.
SHAPES = [
    ("cfg2", 201, 2, {}, "fused128", False), ("cfg2", 333, 2, {}, "fused256", False), ("cfg2", 601, 2, {}, "fused256", False),
    ("cfg2", 333, 1, {}, "fused256", True), ("cfg2", 501, 2, CLUSTER, "fused2-cluster", False), ("cfg2", 501, 2, GRID, "fused2-grid", False),
    ("cfg2", 601, 1, {}, "v1", False), ("cfg2", 201, 1, FORCE, "v1", False),
    ("cfg1", 201, 2, {}, "fused128", False), ("cfg1", 333, 2, {}, "fused256", False), ("cfg1", 601, 2, {}, "fused256", False),
    ("cfg1", 501, 1, {}, "fused256", True), ("cfg1", 501, 2, CLUSTER, "fused2-cluster", False), ("cfg1", 501, 2, GRID, "fused2-grid", False),
    ("cfg1", 601, 1, {}, "v1", False),
    ("cfg3", 201, 2, {}, "fused128", False), ("cfg3", 333, 2, {}, "fused256", False), ("cfg3", 601, 2, {}, "fused256", False),
    ("cfg3", 451, 1, {}, "fused256", True), ("cfg3", 501, 2, CLUSTER, "fused2-cluster", False), ("cfg3", 501, 2, GRID, "fused2-grid", False),
    ("cfg3", 601, 1, {}, "v1", False),
    ("rand2", 151, 2, {}, "fused128", False), ("rand2", 171, 2, {}, "fused128", True), ("rand2", 301, 2, {}, "fused256", False),
    ("rand2", 371, 2, {}, "fused256", True), ("rand2", 601, 1, {}, "v1", False),
] + [(d, nw, cs, FORCE, "v1", False) for d, nw in (("cfg2", 333), ("cfg1", 333), ("cfg3", 333), ("rand2", 301)) for cs in (1, 2, 4, 8)]


def _shape_id(s):
    env = "".join("-" + v for v in s[3].values())
    return "%s-nw%d-cs%d%s-%s%s" % (s[0], s[1], s[2], env, s[4], "-f0g" if s[5] else "")


WANT = ("Xi", "status", "B_drag", "F_iner", "F_BEM", "zeta", "F_drag")
_ORACLE_CACHE = {}


def _oracle(oracle, name, nw):
    """Oracle results for every case of a (design, grid): Xi, status, B_drag, zeta, F_BEM, F_iner."""
    key = (name, nw)
    if key not in _ORACLE_CACHE:
        P = _design(name, nw)
        od = oracle.OracleDesign(P)
        cs = _sea_states(SEEDS[name])
        Xi, st, _ = oracle.solve_cases(od, cs, nIter=10)
        Bd, exc = [], []
        for c in range(N_CASES):
            _, _, _, B = oracle.solve_dynamics(od, 0, cs["Hs"][c], cs["Tp"][c], 0.0, cs["beta_deg"][c], nIter=10, want_Z=True)
            Bd.append(B)
            exc.append(oracle.calc_hydro_excitation(od, 0, cs["Hs"][c], cs["Tp"][c], 0.0, cs["beta_deg"][c])[:3])
        _ORACLE_CACHE[key] = dict(Xi=Xi, status=st, B_drag=np.array(Bd), zeta=np.array([e[0] for e in exc]),
                                  F_BEM=np.array([e[1] for e in exc]), F_iner=np.array([e[2] for e in exc]))
    return _ORACLE_CACHE[key]


def _run(monkeypatch, shape, want=WANT, cases=None, out=None):
    from raft_b200 import solver
    name, nw, cs, env = shape[:4]
    for k in ("RAFTK_FORCE_V1", "RAFTK_FUSED2_XCHG", "RAFTK_NO_DIRECT_D2H"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    ct = cases if cases is not None else solver.CaseTable(_sea_states(SEEDS[name]))
    r = solver.solve_dynamics(solver.DesignBatch(_design(name, nw)), ct, n_iter=10, cluster_size=cs, want=want, out=out)
    return r, solver.last_dispatch()


def _check_record(rec, shape):
    name, nw, cs, env, kernel, f0g = shape
    assert rec["family"] == "solve" and rec["kernel"] == kernel, rec
    assert rec["f0_global"] == f0g and not rec["trains"], rec
    assert rec["cluster_size"] == cs and rec["bins_per_cta"] == -(-nw // cs), rec
    assert rec["threads_per_cta"] == {"fused256": 256}.get(kernel, 128), rec
    assert rec["chunks"] == (1 if kernel == "v1" else 0), rec
    assert (cs == 1 or nw % cs != 0) and rec["bins_per_cta"] % 32 != 0     # ragged slices


@pytest.mark.parametrize("shape", SHAPES, ids=_shape_id)
def test_branch_vs_oracle(shape, monkeypatch, oracle):
    r, rec = _run(monkeypatch, shape)
    _check_record(rec, shape)
    o = _oracle(oracle, shape[0], shape[1])
    assert np.array_equal(r["status"][0, :, :2], o["status"][:, :2]) and np.all(r["status"][0, :, 2] == 0), (r["status"][0], o["status"])
    assert response_err(r["Xi"][0], o["Xi"]) < RTOL
    assert relerr(r["B_drag"][0], o["B_drag"]) < RTOL
    assert relerr(r["zeta"], o["zeta"]) < 1e-13
    assert relerr(r["F_iner"][0], o["F_iner"]) < RTOL
    if shape[0] == "cfg3":
        assert np.abs(o["F_BEM"]).max() > 0 and relerr(r["F_BEM"][0], o["F_BEM"]) < RTOL
    else:
        assert np.abs(r["F_BEM"]).max() == 0 and np.abs(o["F_BEM"]).max() == 0


def _groups():
    g = {}
    for s in SHAPES:
        g.setdefault((s[0], s[1]), []).append(s)
    return [(k, v) for k, v in g.items() if len(v) > 1]


@pytest.mark.parametrize("key,shapes", _groups(), ids=lambda x: "%s-nw%d" % x if isinstance(x, tuple) else "")
def test_branches_agree(key, shapes, monkeypatch):
    """Every variant on the same inputs: the same pass counts and drag matrices, responses and loads to 1e-12."""
    runs = [(_shape_id(s), _run(monkeypatch, s)[0]) for s in shapes]
    base_id, base = runs[0]
    for sid, r in runs[1:]:
        assert np.array_equal(r["status"], base["status"]), (base_id, sid)
        assert response_err(r["Xi"][0], base["Xi"][0]) < 1e-12, (base_id, sid)
        assert relerr(r["B_drag"], base["B_drag"]) < 1e-12, (base_id, sid)
        for k in ("F_iner", "F_drag", "F_BEM"):
            if np.abs(base[k]).max() > 0:
                assert relerr(r[k], base[k]) < 1e-12, (base_id, sid, k)


def test_v1_design_chunking(monkeypatch, oracle):
    """A 3-design batch on the v1 solver with a workspace that holds one design's tables: three chunk launches, results
    bit-identical to the one-launch call and equal to the oracle."""
    import torch
    from raft_b200 import grid, solver
    monkeypatch.setenv("RAFTK_FORCE_V1", "1")
    Qa, Qb = _design("cfg2", 201), grid.regrid(load_golden("cfg1_OC3spar")[1], 201, MAX_FREQ)
    Qb["depth"], Qb["k"] = Qa["depth"], Qa["k"]
    Qc = dict(Qa, C0=Qa["C0"] * 1.3)
    batch, cs = solver.DesignBatch([Qa, Qb, Qc]), _sea_states(31)
    full = solver.DeviceSession(batch, solver.CaseTable(cs), tables=True)
    a = {k: v.clone() for k, v in full.solve(n_iter=10, cluster_size=2).items()}
    torch.cuda.synchronize()
    rec_full = solver.last_dispatch()
    assert rec_full["kernel"] == "v1" and rec_full["chunks"] == 1, rec_full
    small = solver.DeviceSession(batch, solver.CaseTable(cs), tables=True, workspace_bytes=full.workspace_bytes // 2)
    b = small.solve(n_iter=10, cluster_size=2)
    torch.cuda.synchronize()
    rec = solver.last_dispatch()
    assert rec["kernel"] == "v1" and rec["chunks"] == 3 and rec["cluster_size"] == 2, rec
    for k in a:
        assert np.array_equal(a[k].cpu().numpy(), b[k].cpu().numpy()), k
    for d, Q in enumerate((Qa, Qb, Qc)):
        Xi_o, st_o, _ = oracle.solve_cases(oracle.OracleDesign(Q), cs, nIter=10)
        assert np.array_equal(b["status"][d, :, :2].cpu().numpy(), st_o[:, :2])
        assert response_err(b["Xi"][d].cpu().numpy(), Xi_o) < RTOL


def _train_table():
    from raft_b200 import packer
    cases = [dict(wave_spectrum="JONSWAP", wave_height=3.0, wave_period=9.0, wave_heading=20.0),
             dict(wave_spectrum=["JONSWAP"] * 3, wave_height=[4.0, 1.5, 2.5], wave_period=[11.0, 7.0, 14.0], wave_heading=[0.0, 60.0, -45.0],
                  wave_gamma=[0.0] * 3),
             dict(wave_spectrum="JONSWAP", wave_height=6.0, wave_period=13.0, wave_heading=-100.0)]
    return packer.pack_case_trains(cases)[0]


D2H_SHAPES = [next(s for s in SHAPES if s[0] == "cfg2" and s[4] == k and not s[5]) for k in ("fused128", "fused256", "fused2-cluster", "fused2-grid")]


@pytest.mark.parametrize("shape", D2H_SHAPES, ids=_shape_id)
@pytest.mark.parametrize("table", ["plain", "trains", "xi_init"])
def test_direct_d2h_epilogue(shape, table, monkeypatch):
    """Page-locked Xi and status: the solve kernel stores them straight into host memory.  Bit-identical to the device
    outputs of the same solve and to the copy path (RAFTK_NO_DIRECT_D2H=1)."""
    import torch
    from raft_b200 import solver
    name, nw, cs = shape[:3]
    sea = _sea_states(SEEDS[name])
    if table == "plain":
        ct = solver.CaseTable(sea)
    elif table == "trains":
        ct = solver.CaseTable(_train_table())
    else:
        first, _ = _run(monkeypatch, shape, want=("Xi", "status"))
        ct = solver.CaseTable(sea, Xi_init=first["Xi"] * (0.9 + 0.05j))
    nC = ct.n_cases

    def pinned():
        return dict(Xi=solver.pinned_empty([1, nC, 6, nw], np.complex128), status=solver.pinned_empty([1, nC, 4], np.int32))
    direct, rec = _run(monkeypatch, shape, cases=ct, out=pinned())
    assert rec["direct_d2h"] and rec["kernel"] == shape[4] and rec["trains"] == (table == "trains"), rec
    assert np.all(direct["status"][0, :, 2] == 0) and np.all(direct["status"][0, :, 0] >= 0)
    copy, rec2 = _run(monkeypatch, shape[:3] + (dict(shape[3], RAFTK_NO_DIRECT_D2H="1"),) + shape[4:], cases=ct, out=pinned())
    assert not rec2["direct_d2h"] and rec2["kernel"] == shape[4], rec2
    assert np.array_equal(direct["Xi"], copy["Xi"]) and np.array_equal(direct["status"], copy["status"])
    monkeypatch.delenv("RAFTK_NO_DIRECT_D2H")
    sess = solver.DeviceSession(solver.DesignBatch(_design(name, nw)), ct)
    dev = sess.solve(n_iter=10, cluster_size=cs)
    torch.cuda.synchronize()
    assert solver.last_dispatch()["kernel"] == shape[4]
    assert np.array_equal(dev["Xi"].cpu().numpy(), direct["Xi"]) and np.array_equal(dev["status"].cpu().numpy(), direct["status"])


def test_v1_rejects_fused_only_inputs(monkeypatch):
    """Where v1 is the only plan, wave trains, Xi_init and Xi_last are refused with their messages, not answered wrongly."""
    from raft_b200 import _lib, solver
    shape = ("cfg2", 601, 1, {}, "v1", False)
    r, rec = _run(monkeypatch, shape, want=("Xi", "status"))
    assert rec["kernel"] == "v1"
    with pytest.raises(_lib.RaftkError, match="wave-train cases"):
        _run(monkeypatch, shape, cases=solver.CaseTable(_train_table()))
    assert solver.last_dispatch()["kernel"] == "none"
    with pytest.raises(_lib.RaftkError, match="Xi_init"):
        _run(monkeypatch, shape, cases=solver.CaseTable(_sea_states(SEEDS["cfg2"]), Xi_init=r["Xi"]))
    with pytest.raises(_lib.RaftkError, match="Xi_last"):
        _run(monkeypatch, shape, want=("Xi", "status", "Xi_last"))
