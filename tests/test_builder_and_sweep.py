"""Host logic (CPU): the node-table builder against tables packed from the live reference, the Model/FOWT
mirror's construction, and the multi-GPU sharding logic on world_size-2 gloo."""
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN, load_golden, relerr

DESIGNS = json.load(open(os.path.join(GOLDEN, "designs.json")))
TABLE_KEYS = ["mem_q", "mem_p1", "mem_p2", "mem_rA", "node_r", "node_ls", "node_cd_q", "node_cd_p1", "node_cd_p2",
              "node_in_q", "node_in_p1", "node_in_p2", "node_pa", "node_a_i", "node_Imat", "k", "w"]


@pytest.mark.parametrize("name", sorted(n for n in DESIGNS if not n.startswith(("farm_", "slender_synth_"))))   # slender_synth_: per-depth tables, own test
def test_builder_matches_reference_tables(name):
    """raft_b200.member/fowt rebuild, from the design dict alone, the tables packed from the reference's objects
    (strip discretisation, frames, node positions, drag/inertia coefficients, MacCamy-Fuchs, A_hydro_morison)."""
    from raft_b200.fowt import FOWT
    G, P = load_golden(name)
    f = FOWT(DESIGNS[name], P["w"], depth=float(P["depth"]))
    A = f.calcHydroConstants()
    Q = f.pack()
    for k in TABLE_KEYS:
        assert np.asarray(Q[k]).shape == np.asarray(P[k]).shape, k
        if np.asarray(P[k]).size and np.abs(P[k]).max() > 0:
            assert relerr(Q[k], P[k]) < 1e-14, k
    assert np.array_equal(Q["mem_circ"], P["mem_circ"]) and np.array_equal(Q["mem_start"], P["mem_start"])
    if np.abs(G["A_hydro_morison"]).max() > 0:
        assert relerr(A, G["A_hydro_morison"]) < 1e-14
        if "ref_pickle_A_hydro_morison" in G:                     # the reference's own hydroConstants pickle
            assert relerr(A, G["ref_pickle_A_hydro_morison"]) < 1e-12
    if "node_in_p1_w" in P:
        assert relerr(Q["node_in_p1_w"], P["node_in_p1_w"]) < 1e-13


def test_member_input_errors():
    from raft_b200.member import Member
    base = dict(name="m", type="rigid", rA=[0, 0, -10], rB=[0, 0, 5], shape="circ", stations=[0, 1], d=2.0)
    Member(base).setPosition()
    with pytest.raises(ValueError):
        Member(dict(base, rA=[0, 0, 0]))
    with pytest.raises(ValueError):
        Member(dict(base, stations=[1, 0]))
    with pytest.raises(ValueError):
        Member(dict(base, shape="hex"))
    with pytest.raises(NotImplementedError):
        Member(dict(base, type="beam"))
    m = Member(dict(base, shape="rect", d=[2.0, 3.0], Cd=[0.5, 0.7])).setPosition()
    assert m.ds.shape == (m.ns, 2) and np.all(m.Cd_p1 == 0.5) and np.all(m.Cd_p2 == 0.7)


def test_model_construction_and_sweep_variants():
    from raft_b200 import sweep
    from raft_b200.model import Model
    G, P = load_golden("cfg2_VolturnUS-S_nw64")
    mats = dict(M_struc=P["M0"] - G["A_hydro_morison"], C_struc=P["C0"] - G["C_moor"], C_moor=G["C_moor"])
    design = dict(DESIGNS["cfg2_VolturnUS-S_nw64"], site=dict(DESIGNS["cfg2_VolturnUS-S_nw64"]["site"], water_depth=float(P["depth"])))
    m = Model(design, matrices=mats)
    assert m.nw == 64 and m.nDOF == 6 and len(m.fowtList[0].memberList) == 10
    Q = m.fowtList[0].pack()
    assert relerr(Q["M0"], P["M0"]) < 1e-14 and relerr(Q["C0"], P["C0"]) < 1e-14
    fac = sweep.sample_factors(5, seed=40)
    assert fac.shape == (5, 5) and fac.min() >= 0.75 and fac.max() <= 1.25
    V = sweep.build_variants(DESIGNS["cfg2_VolturnUS-S_nw64"], mats, fac[:3], nw=32, max_freq=0.4, depth=float(P["depth"]))
    assert len(V) == 3 and all(len(v["w"]) == 32 for v in V)
    assert not np.allclose(V[0]["node_cd_p1"][:5], V[1]["node_cd_p1"][:5])
    one = sweep.build_variants(DESIGNS["cfg2_VolturnUS-S_nw64"], mats, np.ones((1, 5)), nw=64, max_freq=0.512, depth=float(P["depth"]))[0]
    for k in ("node_ls", "node_cd_q", "node_in_p1", "mem_rA"):
        assert relerr(one[k], P[k]) < 1e-12, k


def test_shard_bounds():
    from raft_b200.sweep import shard_bounds
    for n, world in ((10000, 8), (7, 2), (3, 4), (0, 2)):
        cuts = [shard_bounds(n, r, world) for r in range(world)]
        assert cuts[0][0] == 0 and cuts[-1][1] == n
        assert all(cuts[r][1] == cuts[r + 1][0] for r in range(world - 1))
        sizes = [b - a for a, b in cuts]
        assert max(sizes) - min(sizes) <= 1


def _gloo_worker(rank, world, port, n_items, q):
    import torch
    import torch.distributed as dist
    from raft_b200.sweep import all_gather_blocks, shard_bounds
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    lo, hi = shard_bounds(n_items, rank, world)
    idx = torch.arange(lo, hi, dtype=torch.float64)
    local = (idx[:, None, None] * 10 + torch.arange(3, dtype=torch.float64)[None, :, None] + 1j * torch.arange(2)[None, None, :]).to(torch.complex128)
    full = all_gather_blocks(local, n_items)
    st = all_gather_blocks(torch.arange(lo, hi, dtype=torch.int32)[:, None].repeat(1, 4), n_items)
    q.put((rank, full.numpy(), st.numpy()))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("n_items", [6, 7])
def test_all_gather_blocks_gloo_world2(n_items):
    """The N>1 data path (contiguous design shards + one all-gather, ragged by one) on 2 gloo ranks."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29600 + n_items
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, n_items, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    want = (np.arange(n_items)[:, None, None] * 10 + np.arange(3)[None, :, None] + 1j * np.arange(2)[None, None, :])
    for rank, full, st in got:
        assert full.shape == (n_items, 3, 2) and np.array_equal(full, want)
        assert np.array_equal(st[:, 0], np.arange(n_items))


def test_turbine_channel_coefficients_vs_reference_saveTurbineOutputs():
    """packer.pack_turbine_channels (packed from the live reference FOWT when the fixture was made) reproduces the
    reference's nacelle-acceleration and tower-base-moment metrics as plain linear functionals of its own Xi."""
    z = np.load(os.path.join(GOLDEN, "turb_VolturnUS-S.npz"))
    coef, names, dw = z["ch_coef"], [n.split(":")[0] for n in z["ch_names"]], float(z["P_dw"])
    assert names == ["AxRNA", "AyRNA", "AzRNA", "Mbase"]
    for ic in range(3):
        Xi = z["ref_run_case%d_Xi" % ic]                                   # [nWaves+1, 6, nw]
        Y = np.einsum("kaw,taw->tkw", coef, Xi)
        sd = np.sqrt(0.5 * np.sum(np.abs(Y) ** 2, axis=(0, 2)))            # helpers.getRMS over trains and frequencies
        psd = np.sum(0.5 * np.abs(Y) ** 2 / dw, axis=0)                    # helpers.getPSD
        for k, nm in enumerate(names):
            assert abs(sd[k] - z["ref_run_case%d_%s_std" % (ic, nm)][0]) <= 1e-13 * sd[k]
            ref = z["ref_run_case%d_%s_PSD" % (ic, nm)][:, 0]
            assert np.abs(psd[k] - ref).max() <= 1e-13 * ref.max()
            assert abs(z["ch_avg"][k] - z["ref_run_case%d_%s_avg" % (ic, nm)][0]) <= 1e-13 * max(1.0, abs(z["ch_avg"][k]))


def test_slender_qtf_tables_from_own_builder_match_reference_tables():
    """potSecOrder 1: raft_b200.FOWT builds the second-order grid (w1_2nd, k1_2nd) and, through
    packer.pack_qtf_members, the strip / waterline / Kim & Yue tables exactly as packed from the live reference."""
    _check_slender_tables_from_own_builder("slender_VolturnUS-S", "test_VolturnUS-S", "")


@pytest.mark.parametrize("depth", [40, 1000])
def test_slender_qtf_tables_from_own_builder_synthetic_geometry(depth):
    """The same on the synthetic design (inclined tapered MacCamy-Fuchs brace with station-varying Ca, rectangular member
    with end A above water) at both of its depths."""
    _check_slender_tables_from_own_builder("slender_synth_VolturnUS-S", "slender_synth_VolturnUS-S", "d%d_" % depth)


def _check_slender_tables_from_own_builder(name, design_key, pre):
    """``pre``: depth prefix of the fixture's keys ('' for a fixture with one packed design)."""
    from raft_b200.model import Model
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    P = {k[len(pre) + 2:]: z[k] for k in z.files if k.startswith(pre + "P_")}
    D = DESIGNS[design_key]
    design = dict(D, platform=dict(D["platform"], potSecOrder=1), site=dict(D["site"], water_depth=float(P["depth"])))
    if pre:
        mats = dict(M_struc=z[pre + "M_struc"])
    else:
        mats = dict(M_struc=P["M0"] - z["A_hydro_morison"], C_struc=P["C0"] - z["C_moor"], C_moor=z["C_moor"])
    f = Model(design, matrices=mats).fowtList[0]
    assert f.potSecOrder == 1 and len(f.w1_2nd) == 23
    Q = f.pack()
    keys = sorted(k for k in P if k.startswith("qs_"))
    assert len(keys) == 28
    for k in keys:
        a, b = np.asarray(Q[k]), np.asarray(P[k])
        assert a.shape == b.shape, k
        assert np.abs(a - b).max() <= 1e-15 * max(np.abs(b).max(), 1e-300), k
    # the two MacCamy-Fuchs columns that cross the waterline carry the Kim & Yue correction
    assert int(Q["qs_mem_mcf"].sum()) >= 1 and len(Q["qs_seg_mem"]) > 0
    bad = dict(design, platform={k: v for k, v in design["platform"].items() if k != "min_freq2nd"})
    with pytest.raises(Exception, match="min_freq2nd"):
        Model(bad, matrices=mats)


def test_slender_struct_rejects_unsorted_node_members():
    """The slender-body kernels map a node to its member through mem_node_start (counts of qs_node_mem): nodes out of member
    order would be paired with the wrong member's frame and waterline data, so solver._slender_struct refuses them."""
    from raft_b200 import solver
    z = np.load(os.path.join(GOLDEN, "slender_VolturnUS-S.npz"))
    P = {k[2:]: z[k] for k in z.files if k.startswith("P_")}
    s = solver._slender_struct(P, lambda name, a: a.ctypes.data)
    nm = len(P["qs_mem_mcf"])
    assert (s.n_nodes, s.n_members, s.nw) == (len(P["qs_node_mem"]), nm, len(P["qs_w"]))
    swapped = P["qs_node_mem"].copy()
    i = int(np.flatnonzero(np.diff(swapped))[0])                   # last node of member 0 <-> first node of member 1
    swapped[i], swapped[i + 1] = swapped[i + 1], swapped[i]
    with pytest.raises(ValueError, match="non-decreasing"):
        solver._slender_struct(dict(P, qs_node_mem=swapped), lambda name, a: a.ctypes.data)
    for bad in (np.where(P["qs_node_mem"] == 0, -1, P["qs_node_mem"]), np.where(P["qs_node_mem"] == nm - 1, nm, P["qs_node_mem"])):
        with pytest.raises(ValueError, match="non-decreasing"):
            solver._slender_struct(dict(P, qs_node_mem=bad), lambda name, a: a.ctypes.data)
    # no strip nodes at all (only waterline / Kim & Yue terms) is a valid table
    empty = dict(P, qs_node_mem=np.zeros(0, dtype=np.int32))
    assert solver._slender_struct(empty, lambda name, a: a.ctypes.data).n_nodes == 0


def test_get_rao_and_second_order_case_plumbing():
    from raft_b200 import solver
    Xi = np.arange(12, dtype=float).reshape(2, 6) + 1j
    zeta = np.array([0.0, 2.0, 1e-7, 4.0, 0.5, 1e-6])
    r = solver.get_rao(Xi, zeta)                                  # helpers.getRAO: zero where |zeta| <= 1e-6
    assert np.all(r[:, [0, 2, 5]] == 0) and np.allclose(r[:, [1, 3, 4]], Xi[:, [1, 3, 4]] / zeta[[1, 3, 4]])
    ct = solver.CaseTable(dict(Hs=[1.0], Tp=[8.0], gamma=[0.0], beta_deg=[0.0], spec=[0]), F_2nd=np.zeros([1, 1, 6, 4]),
                          Xi_init=np.zeros([1, 1, 6, 4], dtype=complex))
    s = ct.struct(lambda name: ct.arrays[name].ctypes.data)
    assert s.F_2nd == ct.arrays["F_2nd"].ctypes.data and s.Xi_init == ct.arrays["Xi_init"].ctypes.data and not s.primary


def _batch_tables_equal(ref, bat, tol=1e-13):
    assert sorted(ref.arrays) == sorted(bat.arrays)
    for k in ref.arrays:
        a, b = ref.arrays[k], bat.arrays[k]
        assert a.shape == b.shape and a.dtype == b.dtype, k
        if a.dtype.kind == "i":
            assert np.array_equal(a, b), k
        elif a.size and np.abs(a).max() > 0:
            assert relerr(b, a) < tol, k
    for at in ("n_designs", "nw", "n_members_total", "n_nodes_total", "max_nodes", "max_members", "max_w_classes", "max_h_classes",
               "max_z_classes", "depth", "rho", "g", "dw"):
        assert getattr(ref, at) == getattr(bat, at), at


def test_batched_builder_matches_per_design_builder():
    """raft_b200.batch_builder (all designs in one vectorised pass) against Member + pack_members per design: every CSR
    column of the DesignBatch within rounding, identical node / member counts and step-class hints (SURVEY 8f row 1)."""
    import time
    from raft_b200 import solver, sweep
    G, P = load_golden("cfg2_VolturnUS-S_nw64")
    mats = dict(M_struc=P["M0"] - G["A_hydro_morison"], C_struc=P["C0"] - G["C_moor"], C_moor=G["C_moor"])
    base = DESIGNS["cfg2_VolturnUS-S_nw64"]
    fac = sweep.sample_factors(48, seed=40)
    per = sweep.build_variants(base, mats, fac, nw=64, max_freq=0.32, depth=float(P["depth"]))
    bat = sweep.build_variants_batched(base, mats, fac, nw=64, max_freq=0.32, depth=float(P["depth"]))
    _batch_tables_equal(solver.DesignBatch(per), bat)
    # each design alone gives the same hints as its per-design tables (they size the fused solver's on-chip tables)
    for i in (0, 7, 31):
        one = sweep.build_variants_batched(base, mats, fac[i:i + 1], nw=64, max_freq=0.32, depth=float(P["depth"]))
        _batch_tables_equal(solver.DesignBatch(per[i:i + 1]), one)
    t0 = time.perf_counter()
    big = sweep.build_variants_batched(base, mats, sweep.sample_factors(1250, seed=40), nw=512, max_freq=0.40, depth=float(P["depth"]))
    dt = time.perf_counter() - t0
    assert big.n_designs == 1250 and dt < 2.0, dt                  # ~0.25 s here: 0.2 ms per design (was 10 ms)


def test_batched_builder_general_members():
    """Headings, a rectangular tapered member, a flat step (zero-length station interval), inclined members, potMod."""
    from raft_b200 import batch_builder, grid, solver
    from raft_b200.fowt import FOWT
    members = [
        dict(name="col", type="rigid", rA=[10.0, 0, -18], rB=[10.0, 0, 12], shape="circ", stations=[0, 10, 10, 30], d=[9.0, 9.0, 6.0, 6.0],
             heading=[0.0, 120.0, 240.0], Cd=0.8, Ca=[1.0, 1.0, 0.9, 0.8], CdEnd=0.6, CaEnd=0.6),
        dict(name="pon", type="rigid", rA=[2.0, 0, -15], rB=[9.0, 1.0, -13], shape="rect", stations=[0, 1], d=[[4.0, 3.0], [3.0, 2.0]],
             heading=[60.0, 180.0], gamma=10.0, Cd=[0.9, 1.1], Ca=[0.8, 0.9], potMod=True),
        dict(name="brace", type="rigid", rA=[1.0, 0.5, -12], rB=[8.0, 2.0, 6.0], shape="circ", stations=[0, 2], d=0.9, Cd=1.0, Ca=1.0),
    ]
    base = dict(site=dict(rho_water=1025.0, g=9.81), platform=dict(potModMaster=0, dlsMax=3.0, members=members))
    rng = np.random.default_rng(3)
    nD = 9
    geom = dict(col=dict(d=np.array([[9.0, 9.0, 6.0, 6.0]]) * rng.uniform(0.8, 1.2, (nD, 1)),
                         rA=np.column_stack([np.full(nD, 10.0), np.zeros(nD), -18 * rng.uniform(0.7, 1.3, nD)])),
                pon=dict(d=np.array([[[4.0, 3.0], [3.0, 2.0]]]) * rng.uniform(0.8, 1.2, (nD, 1, 1))),
                brace=dict(rB=np.column_stack([8.0 * rng.uniform(0.9, 1.1, nD), np.full(nD, 2.0), np.full(nD, 6.0)])))
    w = grid.make_w(0.01, 0.2)
    k = grid.wave_number(w, 150.0)
    mats = dict(M_struc=np.eye(6) * 1e7, C_struc=np.eye(6) * 1e6)
    bat = batch_builder.build_family(batch_builder.DesignFamily(base, geom, nD), w, k, 150.0, mats)
    per = []
    for d in range(nD):
        des = json.loads(json.dumps(base))
        for m in des["platform"]["members"]:
            for key, v in geom[m["name"]].items():
                m[key] = np.asarray(v[d]).tolist()
        f = FOWT(des, w, depth=150.0, matrices=mats, k=k)
        f.calcHydroConstants()
        per.append(f.pack())
    _batch_tables_equal(solver.DesignBatch(per), bat)


def test_wave_number_is_the_references_scalar_iteration():
    """grid.wave_number (vectorised rounds + scalar finish for the last stragglers) against the reference's loop written out
    (helpers.py:377-392): identical bits, also where the long-wave bins need thousands of iterations."""
    from raft_b200 import grid

    def scalar(omega, h, e=0.001, g=9.81):
        k1 = omega * omega / g
        k2 = omega * omega / (np.tanh(k1 * h) * g)
        while np.abs(k2 - k1) / k1 > e:
            k1 = k2
            k2 = omega * omega / (np.tanh(k1 * h) * g)
        return k2

    for nw, max_freq, depth in ((64, 0.32, 200.0), (256, 0.256, 320.0), (80, 0.40, 50.0)):
        w = grid.make_w(max_freq / nw, max_freq)
        k = grid.wave_number(w, depth)
        assert np.array_equal(k, np.array([scalar(x, depth) for x in w]))


def test_host_struct_cache_follows_table_edits():
    """solver._host_struct: the cached C struct of the host-buffer calls is rebuilt when a table is replaced (its address
    changes) and kept when arrays are edited in place."""
    from raft_b200 import solver
    _, P = load_golden("cfg2_VolturnUS-S_nw64")
    b = solver.DesignBatch([P])
    s1 = solver._host_struct(b)
    assert solver._host_struct(b) is s1
    b.arrays["node_ls"][0] += 0.0                                  # in place: same address, same struct
    assert solver._host_struct(b) is s1 and s1.node_ls == b.arrays["node_ls"].ctypes.data
    b.arrays["node_ls"] = b.arrays["node_ls"].copy()               # replaced: new address, new struct
    s2 = solver._host_struct(b)
    assert s2 is not s1 and s2.node_ls == b.arrays["node_ls"].ctypes.data
    c = solver.CaseTable(dict(Hs=[1.0], Tp=[8.0], gamma=[0.0], beta_deg=[0.0], spec=np.zeros(1, dtype=np.int32)))
    t1 = solver._host_struct(c)
    c.arrays.update(Hs=np.array([2.0]))
    assert solver._host_struct(c) is not t1


def test_unknown_outputs_are_refused_before_any_device_use():
    """An output name an entry does not offer is the same ValueError on the host solves, the potSecOrder 1 flows and
    DeviceSession (which has no Xi_last), raised before a launch or any use of a device."""
    from raft_b200 import solver
    _, P = load_golden("cfg2_VolturnUS-S_nw64")
    _, Ps = load_golden("slender_VolturnUS-S")
    cs = dict(Hs=[6.0], Tp=[12.0], gamma=[0.0], beta_deg=[0.0], spec=np.zeros(1, dtype=np.int32))
    b, c = solver.DesignBatch([P]), solver.CaseTable(cs)
    before = solver.launch_count()
    for call in (lambda: solver.solve_dynamics(b, c, want=("Xi", "F_nope")),
                 lambda: solver.slender_flow_host([Ps], c, want=("F_nope",)),
                 lambda: solver.SlenderSession([Ps], c, want=("F_nope",)),
                 lambda: solver.DeviceSession(b, c, want=("F_nope",)),
                 lambda: solver.DeviceSession(b, c, want=("Xi_last",))):
        with pytest.raises(ValueError, match="unknown outputs"):
            call()
    assert solver.launch_count() == before


def _general_family():
    from raft_b200 import batch_builder, grid
    members = [
        dict(name="col", type="rigid", rA=[10.0, 0, -18], rB=[10.0, 0, 12], shape="circ", stations=[0, 10, 10, 30], d=[9.0, 9.0, 6.0, 6.0],
             heading=[0.0, 120.0, 240.0], Cd=0.8, Ca=[1.0, 1.0, 0.9, 0.8], CdEnd=0.6, CaEnd=0.6),
        dict(name="pon", type="rigid", rA=[2.0, 0, -15], rB=[9.0, 1.0, -13], shape="rect", stations=[0, 1], d=[[4.0, 3.0], [3.0, 2.0]],
             heading=[60.0, 180.0], gamma=10.0, Cd=[0.9, 1.1], Ca=[0.8, 0.9], potMod=True),
        dict(name="brace", type="rigid", rA=[1.0, 0.5, -12], rB=[8.0, 2.0, 6.0], shape="circ", stations=[0, 2], d=0.9, Cd=1.0, Ca=1.0),
        dict(name="vert", type="rigid", rA=[0.0, 0, -20], rB=[0.0, 0, 5.0], shape="rect", stations=[0, 5, 25], d=[[5.0, 4.0], [5.0, 4.0], [3.0, 2.5]],
             heading=[0.0, 45.0], gamma=5.0, Cd=[[0.7, 0.9], [0.7, 0.9], [0.8, 1.0]], Ca=[[1.0, 0.9], [0.9, 0.8], [0.8, 0.7]], CdEnd=0.5, CaEnd=0.7),
    ]
    base = dict(site=dict(rho_water=1025.0, g=9.81), platform=dict(potModMaster=0, dlsMax=3.0, members=members))
    rng = np.random.default_rng(3)
    nD = 9
    geom = dict(col=dict(d=np.array([[9.0, 9.0, 6.0, 6.0]]) * rng.uniform(0.8, 1.2, (nD, 1)),
                         rA=np.column_stack([np.full(nD, 10.0), np.zeros(nD), -18 * rng.uniform(0.7, 1.3, nD)])),
                pon=dict(d=np.array([[[4.0, 3.0], [3.0, 2.0]]]) * rng.uniform(0.8, 1.2, (nD, 1, 1))),
                brace=dict(rB=np.column_stack([8.0 * rng.uniform(0.9, 1.1, nD), np.full(nD, 2.0), np.full(nD, 6.0)])))
    w = grid.make_w(0.01, 0.2)
    return batch_builder.DesignFamily(base, geom, nD), w, grid.wave_number(w, 150.0)


def test_native_builder_matches_numpy_builder():
    """raftk_build_family_host (csrc/raftk_builder.h, plain C++ loops) against batch_builder.build_family: identical counts, offsets
    and step-class hints, tables to rounding -- on the sweep family, on a family with headings / tapered rectangular members / a
    flat step / inclined and vertical members / potMod, and with a rotated, shifted platform."""
    from raft_b200 import batch_builder, sweep
    G, P = load_golden("cfg2_VolturnUS-S_nw64")
    mats = dict(M_struc=P["M0"] - G["A_hydro_morison"], C_struc=P["C0"] - G["C_moor"], C_moor=G["C_moor"])
    fac = sweep.sample_factors(64, seed=41)
    num = sweep.build_variants_batched(DESIGNS["cfg2_VolturnUS-S_nw64"], mats, fac, nw=64, max_freq=0.32, depth=float(P["depth"]), native=False)
    nat = sweep.build_variants_batched(DESIGNS["cfg2_VolturnUS-S_nw64"], mats, fac, nw=64, max_freq=0.32, depth=float(P["depth"]), native=True)
    _batch_tables_equal(num, nat)
    assert relerr(nat.A_hydro_morison, num.A_hydro_morison) < 1e-13
    fam, w, k = _general_family()
    mats2 = dict(M_struc=np.eye(6) * 1e7, C_struc=np.eye(6) * 1e6)
    for r6 in (None, np.array([3.0, -2.0, 0.5, 0.02, -0.03, 0.4])):
        a = batch_builder.build_family(fam, w, k, 150.0, mats2, r6=r6)
        b = batch_builder.build_family_native(fam, w, k, 150.0, mats2, r6=r6)
        _batch_tables_equal(a, b)
        assert relerr(b.A_hydro_morison, a.A_hydro_morison) < 1e-13


def test_native_builder_errors_like_the_reference():
    from raft_b200 import _lib, batch_builder, grid
    members = [dict(name="col", type="rigid", rA=[0.0, 0, -10], rB=[0.0, 0, 0.0], shape="circ", stations=[0, 10], d=5.0)]
    base = dict(site=dict(rho_water=1025.0, g=9.81), platform=dict(potModMaster=0, dlsMax=3.0, members=members))
    w = grid.make_w(0.05, 0.2)
    with pytest.raises(_lib.RaftkError, match="cannot start or end on the waterplane"):
        batch_builder.build_family_native(batch_builder.DesignFamily(base, {}, 2), w, grid.wave_number(w, 100.0), 100.0, {})
    members[0].update(rB=[0.0, 0, 5.0], stations=[0, 10, 5])
    with pytest.raises(ValueError, match="not in ascending order"):
        batch_builder.build_family_native(batch_builder.DesignFamily(base, {}, 2), w, grid.wave_number(w, 100.0), 100.0, {})
