"""Submerged rotors (MHK turbines): the hub's inertial wave excitation on the rigid path (raft_fowt.py:1859-1888).

The reference's steps are restated here literally -- getWaveKin at the hub (the oracle's ro_wave_kin), rotateMatrix6 with its
transposed lower-left block, translateForce3to6DOF about the PRP, the hub node's rows of fowt.T -- and checked against
``packer.pack_rotor_excitation``'s collapsed G on the CPU.  On the GPU, every rigid entry point is checked against a
restatement of Model.solveDynamics's fixed-point loop (raft_model.py:1040-1135) over the oracle's strip-theory excitation and
drag linearisation, with the restated rotor term added to F_hydro_iner.  The rotor is synthetic: a hub 16 m below the
waterline of VolturnUS-S, rotated, off the platform's axis."""
import types

import numpy as np
import pytest

from conftest import load_golden, relerr, response_err

RTOL = 1e-10


def _rot(a, b, c):
    ca, sa, cb, sb, cc, sc = np.cos(a), np.sin(a), np.cos(b), np.sin(b), np.cos(c), np.sin(c)
    Rx = np.array([[1, 0, 0], [0, ca, -sa], [0, sa, ca]])
    Ry = np.array([[cb, 0, sb], [0, 1, 0], [-sb, 0, cb]])
    Rz = np.array([[cc, -sc, 0], [sc, cc, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def _H(r):
    """helpers.getH: H(r) v = v x r ... the reference's alternator; here only its use through np.cross matters."""
    return np.array([[0, r[2], -r[1]], [-r[2], 0, r[0]], [r[1], -r[0], 0]])


def _rigid_T(nodes_r, r6):
    """fowt.T of a rigid FOWT whose nodes are tied to the PRP: node displacement = x + theta x (r - r_PRP)."""
    T = np.zeros([6 * len(nodes_r), 6])
    for i, r in enumerate(nodes_r):
        d = np.asarray(r, dtype=float) - r6[:3]
        T[6 * i:6 * i + 6] = np.eye(6)
        T[6 * i:6 * i + 3, 3:] = _H(d)            # theta x d = H(d) theta with the reference's getH sign
    return T


def synthetic_fowt(seed=0, r6=(0.0, 0.0, 0.0, 0, 0, 0), hub=(-6.0, 3.5, -16.0), n_rotors=1):
    """A duck-typed live FOWT with submerged rotors: rotorList (r3, I_hydro, R_q, nodeList[0].id), T, r6."""
    rng = np.random.default_rng(seed)
    r6 = np.asarray(r6, dtype=float)
    rotors, nodes = [], [r6[:3]]
    for j in range(n_rotors):
        A = rng.normal(size=(6, 6))
        I6 = A @ A.T * 4e4 + np.diag([3e5, 8e4, 8e4, 2e6, 1e6, 1e6])
        r3 = np.asarray(hub, dtype=float) + r6[:3] + np.array([0.0, 7.0 * j, -2.0 * j])
        node_r = r3 + rng.normal(size=3)                        # the hub node need not sit at r3
        nodes.append(node_r)
        rotors.append(types.SimpleNamespace(r3=r3, I_hydro=I6, R_q=_rot(*rng.uniform(-0.4, 0.4, 3)),
                                            nodeList=[types.SimpleNamespace(id=len(nodes) - 1)]))
    return types.SimpleNamespace(rotorList=rotors, T=_rigid_T(nodes, r6), r6=r6, nDOF=6)


def reference_rotor_force(fowt, ud):
    """raft_fowt.py:1861-1888 for one frequency: ud [nrot,3] complex -> reduced force [6] (T^T F_full)."""
    F_full = np.zeros(fowt.T.shape[0], dtype=complex)
    for ir, rot in enumerate(fowt.rotorList):
        if rot.r3[2] >= 0:
            continue
        R, M = rot.R_q, rot.I_hydro
        I = np.zeros([6, 6])                                        # rotateMatrix6 (helpers.py:604-640)
        I[:3, :3] = R @ M[:3, :3] @ R.T
        I[:3, 3:] = R @ M[:3, 3:] @ R.T
        I[3:, :3] = I[:3, 3:].T
        I[3:, 3:] = R @ M[3:, 3:] @ R.T
        f3 = I[:3, :3] @ ud[ir]
        f6 = np.zeros(6, dtype=complex)
        f6[:3] = f3
        f6[3:] = np.cross(rot.r3 - fowt.r6[:3], f3)                 # translateForce3to6DOF
        f6[3:] += I[3:, :3] @ ud[ir]
        i0 = rot.nodeList[0].id * 6
        F_full[i0:i0 + 6] += f6
    return fowt.T.T @ F_full


def restated_rotor_excitation(oracle, P, zeta, beta_deg):
    """Rotor term of F_hydro_iner [6,nw] for one wave train, from the packed table's hubs and the reference's getWaveKin."""
    F = np.zeros([6, len(P["w"])], dtype=complex)
    for r3, G in zip(P.get("rot_r3", ()), P.get("rot_G", ())):
        _, ud, _ = oracle.wave_kin(zeta, np.deg2rad(beta_deg), P["w"], P["k"], float(P["depth"]), r3)
        F += np.asarray(G) @ ud
    return F


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_pack_rotor_excitation_reproduces_the_reference_steps():
    from raft_b200 import packer
    rng = np.random.default_rng(3)
    for seed, r6 in ((0, np.zeros(6)), (1, np.array([350.0, -120.0, 0, 0, 0, 0])), (2, np.array([5.0, 2.0, -0.5, 0.01, -0.02, 0.3]))):
        fw = synthetic_fowt(seed, r6=r6, n_rotors=2)
        fw.rotorList.append(types.SimpleNamespace(r3=np.array([0.0, 0.0, 90.0]), I_hydro=None, R_q=np.eye(3),
                                                  nodeList=[types.SimpleNamespace(id=0)]))   # above water: no term, no I_hydro needed
        P = packer.pack_rotor_excitation(fw)
        assert P["rot_r3"].shape == (2, 3) and P["rot_G"].shape == (2, 6, 3)
        for _ in range(4):
            ud = rng.normal(size=(3, 3)) + 1j * rng.normal(size=(3, 3))
            ref = reference_rotor_force(fw, ud)
            got = sum(P["rot_G"][j] @ ud[j] for j in range(2))
            assert relerr(got, ref) < 1e-14


def test_pack_rotor_excitation_needs_hydro_constants():
    from raft_b200 import packer
    fw = synthetic_fowt()
    fw.rotorList[0].I_hydro = None
    with pytest.raises(ValueError, match="calcHydroConstants"):
        packer.pack_rotor_excitation(fw)
    fw.rotorList = []
    assert packer.pack_rotor_excitation(fw) == {}


def test_generalised_packers_refuse_a_submerged_rotor():
    from raft_b200 import packer
    fw = synthetic_fowt()
    with pytest.raises(NotImplementedError, match="submerged rotors"):
        packer.pack_general_dofs(fw)
    with pytest.raises(NotImplementedError, match="submerged rotors"):
        packer.pack_general_matrices(fw)


def _design_with_rotor(seed=0, x_ref=0.0, y_ref=0.0):
    """cfg2's VolturnUS-S packed design with one synthetic submerged rotor (its table from pack_rotor_excitation)."""
    from raft_b200 import packer
    _, P = load_golden("cfg2_VolturnUS-S_nw64")
    P = dict(P)
    fw = synthetic_fowt(seed, r6=np.array([x_ref, y_ref, 0, 0, 0, 0]))
    P.update(packer.pack_rotor_excitation(fw))
    return P


def test_design_batch_carries_the_rotor_table():
    from raft_b200 import solver
    _, P0 = load_golden("cfg2_VolturnUS-S_nw64")
    P1, P2 = _design_with_rotor(0), _design_with_rotor(1)
    P2 = dict(P2, rot_r3=np.vstack([P2["rot_r3"], P1["rot_r3"]]), rot_G=np.vstack([P2["rot_G"], P1["rot_G"]]))
    b = solver.DesignBatch([P1, P0, P2])
    assert b.max_rotors == 2
    assert b.arrays["rot_count"].tolist() == [1, 0, 2]
    np.testing.assert_array_equal(b.arrays["rot_G"][0, 0], P1["rot_G"][0])
    np.testing.assert_array_equal(b.arrays["rot_G"][1], 0.0)
    np.testing.assert_array_equal(b.arrays["rot_r3"][2], P2["rot_r3"])
    s = b.struct(lambda n: 1)
    assert s.max_rotors == 2 and s.rot_count and s.rot_G
    t = b.take(1, 3)
    assert t.max_rotors == 2 and t.arrays["rot_count"].tolist() == [0, 2]
    np.testing.assert_array_equal(t.arrays["rot_G"][1], b.arrays["rot_G"][2])
    plain = solver.DesignBatch(P0)
    assert plain.max_rotors == 0 and "rot_count" not in plain.arrays and plain.struct(lambda n: 1).max_rotors == 0


def _mhk_matrices(seed=0):
    from raft_b200 import packer
    fw = synthetic_fowt(seed)
    rot = packer.pack_rotor_excitation(fw)
    return dict(M_struc=np.diag([2e7, 2e7, 2e7, 1.5e10, 1.5e10, 2e10]), C_hydro=np.diag([0, 0, 4e6, 2e9, 2e9, 0.0]),
                C_moor=np.diag([7e4, 7e4, 1e4, 0, 0, 1e8]), rotor_excitation=dict(r3=rot["rot_r3"], G=rot["rot_G"]),
                A_hydro_rotor=np.diag([1.1e5, 4e4, 4e4, 3e5, 2e6, 2e6]))


def _volturn_design():
    import json
    import os
    from conftest import GOLDEN
    with open(os.path.join(GOLDEN, "designs.json")) as f:
        return json.load(f)["cfg2_VolturnUS-S_nw64"]


def test_fowt_takes_injected_rotors():
    from raft_b200 import grid
    from raft_b200.fowt import FOWT
    mats = _mhk_matrices()
    design = _volturn_design()
    w = grid.make_w(0.02, 0.4)
    f = FOWT(design, w, depth=200.0, matrices=mats)
    A = f.calcHydroConstants()
    g = FOWT(design, w, depth=200.0, matrices={k: v for k, v in mats.items() if k not in ("rotor_excitation", "A_hydro_rotor")})
    A0 = g.calcHydroConstants()
    np.testing.assert_array_equal(A, A0 + mats["A_hydro_rotor"])
    P, P0 = f.pack(), g.pack()
    np.testing.assert_array_equal(P["rot_G"], mats["rotor_excitation"]["G"])
    assert relerr(np.asarray(P["M0"]) - np.asarray(P0["M0"]), mats["A_hydro_rotor"]) < 1e-9
    assert "rot_G" not in P0


def test_family_builders_copy_the_base_rotors():
    from raft_b200 import sweep
    mats = _mhk_matrices()
    design = _volturn_design()
    factors = np.array([[1, 1, 1, 1, 1], [1.05, 0.95, 1.1, 1.0, 0.9], [0.9, 1.1, 0.95, 1.05, 1.1]])
    packed = sweep.build_variants(design, mats, factors, 48, 0.4, 200.0)
    b = sweep.build_variants_batched(design, mats, factors, 48, 0.4, 200.0, native=False)
    assert b.max_rotors == 1 and b.arrays["rot_count"].tolist() == [1, 1, 1]
    for i, P in enumerate(packed):
        np.testing.assert_array_equal(b.arrays["rot_G"][i], P["rot_G"])
        np.testing.assert_array_equal(b.arrays["rot_r3"][i], P["rot_r3"])
        assert relerr(b.arrays["M0"][i], np.asarray(P["M0"]).reshape(36)) < 1e-13


# ------------------------------------------------------------------------------------------------------------------ GPU
def _cases(seed, n=3):
    rng = np.random.default_rng(seed)
    return dict(Hs=rng.uniform(2, 9, n), Tp=rng.uniform(6, 16, n), gamma=np.zeros(n), beta_deg=rng.uniform(-180, 180, n),
                spec=np.zeros(n, dtype=np.int32))


def reference_solve(oracle, P, Hs, Tp, beta_deg, n_iter=10, tol=0.01, xi_start=0.0):
    """Model.solveDynamics for one FOWT and one wave train (raft_model.py:996-1135): the oracle's strip-theory excitation and
    drag linearisation, the restated rotor term, the reference's impedance, convergence test and relaxation.
    -> Xi [6,nw], passes, F_iner [6,nw]."""
    od = oracle.OracleDesign(P)
    zeta, F_BEM, F_iner, u = oracle.calc_hydro_excitation(od, 0, Hs, Tp, 0.0, beta_deg)
    F_iner = F_iner + restated_rotor_excitation(oracle, P, zeta, beta_deg)
    w = np.asarray(P["w"])
    M0, B0, C0 = (np.asarray(P[k]).reshape(6, 6) for k in ("M0", "B0", "C0"))
    XiLast = np.zeros([6, len(w)], dtype=complex) + xi_start
    passes = 0
    for _ in range(n_iter + 1):
        _, Bd, Fd = oracle.calc_hydro_linearization(od, u, XiLast)
        F = F_BEM + F_iner + Fd
        Z = -w[:, None, None] ** 2 * M0 + 1j * w[:, None, None] * (B0 + Bd) + C0
        Xi = np.linalg.solve(Z, F.T[:, :, None])[:, :, 0].T
        passes += 1
        if (np.abs(Xi - XiLast) / (np.abs(Xi) + tol) < tol).all():
            break
        XiLast = 0.2 * XiLast + 0.8 * Xi
    return Xi, passes, F_iner


_SHAPES = [(201, 2, {}, "fused128"), (333, 2, {}, "fused256"), (501, 2, {"RAFTK_FUSED2_XCHG": "cluster"}, "fused2-cluster"),
           (501, 2, {"RAFTK_FUSED2_XCHG": "grid"}, "fused2-grid"), (201, 1, {"RAFTK_FORCE_V1": "1"}, "v1")]


def _regridded(P, nw):
    from raft_b200 import grid
    Q = grid.regrid({k: v for k, v in P.items() if not k.startswith("rot_")}, nw, 0.4)
    Q.update({k: v for k, v in P.items() if k.startswith("rot_")})
    return Q


@pytest.mark.gpu
@pytest.mark.parametrize("shape", _SHAPES, ids=[s[3] for s in _SHAPES])
def test_every_rigid_kernel_against_the_reference_loop(oracle, monkeypatch, shape):
    from raft_b200 import solver
    nw, cs, env, kernel = shape
    for k in ("RAFTK_FORCE_V1", "RAFTK_FUSED2_XCHG"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    P = _regridded(_design_with_rotor(0), nw)
    cs_ = _cases(11)
    out = solver.solve_dynamics(solver.DesignBatch(P), solver.CaseTable(cs_), n_iter=10, cluster_size=cs,
                                want=("Xi", "status", "F_iner"))
    rec = solver.last_dispatch()
    assert rec["family"] == "solve" and rec["kernel"] == kernel, rec
    plain = solver.solve_dynamics(solver.DesignBatch({k: v for k, v in P.items() if not k.startswith("rot_")}), solver.CaseTable(cs_),
                                  n_iter=10, cluster_size=cs)
    for c in range(3):
        Xi, passes, Fi = reference_solve(oracle, P, cs_["Hs"][c], cs_["Tp"][c], cs_["beta_deg"][c])
        assert response_err(out["Xi"][0, c], Xi) < RTOL, (c, response_err(out["Xi"][0, c], Xi))
        assert out["status"][0, c, 0] == passes
        assert relerr(out["F_iner"][0, c], Fi) < 1e-12
        assert response_err(plain["Xi"][0, c], Xi) > 1e-6        # the rotor term matters at this size


@pytest.mark.gpu
def test_excitation_puts_the_term_on_the_last_train_only(oracle):
    from raft_b200 import solver
    from raft_b200.fowt import FOWT
    P = _design_with_rotor(2)
    cs_ = _cases(12, 3)
    ex = solver.hydro_excitation(solver.DesignBatch(P), solver.CaseTable(cs_))
    od = oracle.OracleDesign(P)
    for c in range(3):
        zeta, _, Fi, _ = oracle.calc_hydro_excitation(od, 0, cs_["Hs"][c], cs_["Tp"][c], 0.0, cs_["beta_deg"][c])
        assert relerr(ex["F_iner"][0, c], Fi + restated_rotor_excitation(oracle, P, zeta, cs_["beta_deg"][c])) < 1e-12
    # one case of two wave trains: train 0 (the primary) has no rotor term, train 1 has it (raft_fowt.py:1866-1883)
    two = dict(cs_, Hs=cs_["Hs"][:2], Tp=cs_["Tp"][:2], gamma=cs_["gamma"][:2], beta_deg=cs_["beta_deg"][:2], spec=cs_["spec"][:2],
               primary=np.zeros(2, dtype=np.int32))
    ex2 = solver.hydro_excitation(solver.DesignBatch(P), solver.CaseTable(two))
    z0, _, F0, _ = oracle.calc_hydro_excitation(od, 0, two["Hs"][0], two["Tp"][0], 0.0, two["beta_deg"][0])
    z1, _, F1, _ = oracle.calc_hydro_excitation(od, 0, two["Hs"][1], two["Tp"][1], 0.0, two["beta_deg"][1])
    assert relerr(ex2["F_iner"][0, 0], F0) < 1e-12
    assert relerr(ex2["F_iner"][0, 1], F1 + restated_rotor_excitation(oracle, P, z1, two["beta_deg"][1])) < 1e-12
    # FOWT.calcHydroExcitation groups a case's trains the same way
    design = _volturn_design()
    from raft_b200 import grid
    f = FOWT(design, grid.make_w(0.02, 0.4), depth=200.0, matrices=_mhk_matrices())
    f.calcHydroConstants()
    case = dict(wave_spectrum=["JONSWAP", "JONSWAP"], wave_period=[9.0, 12.0], wave_height=[4.0, 2.0], wave_heading=[0.0, 40.0])
    F = f.calcHydroExcitation(case)
    Pf = f.pack()
    odf = oracle.OracleDesign(Pf)
    for ih in range(2):
        zt, _, Ft, _ = oracle.calc_hydro_excitation(odf, 0, case["wave_height"][ih], case["wave_period"][ih], 0.0, case["wave_heading"][ih])
        ref = Ft + (restated_rotor_excitation(oracle, Pf, zt, case["wave_heading"][ih]) if ih == 1 else 0)
        assert relerr(F[ih], ref) < 1e-12


@pytest.mark.gpu
def test_mixed_batch_leaves_rotor_free_designs_bit_identical():
    from raft_b200 import solver
    _, P0 = load_golden("cfg2_VolturnUS-S_nw64")
    P1 = _design_with_rotor(4)
    ct = solver.CaseTable(_cases(13))
    mixed = solver.solve_dynamics(solver.DesignBatch([P1, P0, P1]), ct, n_iter=10)
    solo = solver.solve_dynamics(solver.DesignBatch(P0), ct, n_iter=10)
    one = solver.solve_dynamics(solver.DesignBatch(P1), ct, n_iter=10)
    np.testing.assert_array_equal(mixed["Xi"][1], solo["Xi"][0])
    np.testing.assert_array_equal(mixed["status"][1], solo["status"][0])
    np.testing.assert_array_equal(mixed["Xi"][0], one["Xi"][0])
    np.testing.assert_array_equal(mixed["Xi"][2], one["Xi"][0])


@pytest.mark.gpu
def test_farms_take_the_rotor_term_through_every_entry(oracle):
    """Two FOWTs, the second offset and turned by its hub position: the per-FOWT loads inside every farm entry are the
    single solves' (checked against the reference loop), and the uniform, ragged and single-farm entries agree."""
    from raft_b200 import solver
    zf = load_golden("farm_VolturnUS-S_farm_nw48")[0]
    packs = [{k[3:]: v for k, v in zf.items() if k.startswith("P%d_" % i)} for i in range(int(zf["n_fowt"]))]
    from raft_b200 import packer
    for i, P in enumerate(packs):
        fw = synthetic_fowt(5 + i, r6=np.array([float(P.get("x_ref", 0.0)), float(P.get("y_ref", 0.0)), 0, 0, 0, 0]))
        if i == 1:
            fw.rotorList[0].R_q = _rot(0.0, 0.0, 0.7) @ fw.rotorList[0].R_q
        P.update(packer.pack_rotor_excitation(fw))
    cf = zf["cases"][:2]
    cases = dict(Hs=cf[:, 0], Tp=cf[:, 1], gamma=np.zeros(2), beta_deg=cf[:, 2], spec=np.zeros(2, dtype=np.int32))
    b, ct = solver.DesignBatch(packs), solver.CaseTable(cases)
    kw = dict(C_arr=zf["C_array"], n_iter=int(zf["n_iter"]), xi_start=float(zf["xi_start"]))
    one = solver.solve_dynamics_farm(b, ct, **kw)
    single = solver.solve_dynamics(b, ct, n_iter=int(zf["n_iter"]), xi_start=float(zf["xi_start"]))
    np.testing.assert_array_equal(one["Xi"], single["Xi"])
    for i, P in enumerate(packs):
        for c in range(2):
            Xi, passes, _ = reference_solve(oracle, P, cases["Hs"][c], cases["Tp"][c], cases["beta_deg"][c], n_iter=int(zf["n_iter"]),
                                            xi_start=float(zf["xi_start"]))
            assert response_err(single["Xi"][i, c], Xi) < RTOL and single["status"][i, c, 0] == passes
    b2 = solver.DesignBatch(packs + packs)
    bat = solver.solve_dynamics_farm_batch(b2, ct, 2, **kw)
    rag = solver.solve_dynamics_farm_ragged(b2, ct, [2, 2], **kw)
    for f in range(2):
        assert relerr(bat["Xi_sys"][f], one["Xi_sys"]) < 1e-13
        assert relerr(rag["Xi_sys"][f], one["Xi_sys"]) < 1e-13
    plain = solver.solve_dynamics_farm(solver.DesignBatch([{k: v for k, v in P.items() if not k.startswith("rot_")} for P in packs]), ct, **kw)
    assert relerr(plain["Xi_sys"], one["Xi_sys"]) > 1e-6


@pytest.mark.gpu
def test_device_session_sweep_of_mhk_variants():
    from raft_b200 import solver, sweep
    mats = _mhk_matrices()
    design = _volturn_design()
    factors = np.array([[1, 1, 1, 1, 1], [1.05, 0.95, 1.1, 1.0, 0.9], [0.9, 1.1, 0.95, 1.05, 1.1]])
    b = sweep.build_variants_batched(design, mats, factors, 64, 0.4, 200.0)
    ct = solver.CaseTable(_cases(14))
    dev = solver.DeviceSession(b, ct).solve(n_iter=10)
    host = solver.solve_dynamics(solver.DesignBatch(sweep.build_variants(design, mats, factors, 64, 0.4, 200.0)), ct, n_iter=10)
    Xi = dev["Xi"].cpu().numpy() if hasattr(dev["Xi"], "cpu") else np.asarray(dev["Xi"])
    st = dev["status"].cpu().numpy() if hasattr(dev["status"], "cpu") else np.asarray(dev["status"])
    assert response_err(Xi, host["Xi"]) < RTOL
    np.testing.assert_array_equal(st[..., 0], host["status"][..., 0])


def _farm_design():
    import json
    import os
    from conftest import GOLDEN
    with open(os.path.join(GOLDEN, "designs.json")) as f:
        return json.load(f)["farm_VolturnUS-S_farm_nw48"]


def test_model_array_places_an_injected_rotor_at_every_fowt():
    """One rotor_excitation shared by an array's FOWTs: each FOWT's hubs sit at its own (x_ref, y_ref)."""
    import copy
    from raft_b200.model import Model
    mats = _mhk_matrices()
    turned = _farm_design()
    m = Model(copy.deepcopy(turned), matrices=mats)
    if any(f.heading_adjust != 0 for f in m.fowtList):
        with pytest.raises(NotImplementedError, match="heading_adjust"):
            [f.pack() for f in m.fowtList]
    design = copy.deepcopy(turned)
    keys = design["array"]["keys"]
    if "heading_adjust" in keys:
        j = keys.index("heading_adjust")
        for row in design["array"]["data"]:
            row[j] = 0
    m = Model(design, matrices=mats)
    assert m.nFOWT >= 2
    for f in m.fowtList:
        for fw in (f,):
            fw.calcHydroConstants()
        P = f.pack()
        np.testing.assert_array_equal(P["rot_r3"], mats["rotor_excitation"]["r3"] + np.array([f.x_ref, f.y_ref, 0.0]))
        np.testing.assert_array_equal(P["rot_G"], mats["rotor_excitation"]["G"])
    assert len({tuple(f.pack()["rot_r3"][0]) for f in m.fowtList}) == m.nFOWT


@pytest.mark.gpu
def test_model_solve_dynamics_single_fowt(oracle):
    from raft_b200 import solver
    from raft_b200.model import Model
    design = dict(_volturn_design())
    design["settings"] = dict(design.get("settings", {}), min_freq=0.01, max_freq=0.4)
    m = Model(design, matrices=_mhk_matrices())
    for f in m.fowtList:
        f.calcHydroConstants()
    case = dict(wave_spectrum="JONSWAP", wave_period=11.0, wave_height=5.0, wave_heading=30.0, wave_gamma=0.0)
    Xi = m.solveDynamics(case)
    rec = solver.last_dispatch()
    assert rec["family"] == "solve", rec
    P = m.fowtList[0].pack()
    ref = solver.solve_dynamics(solver.DesignBatch(P), solver.CaseTable(dict(Hs=[5.0], Tp=[11.0], gamma=[0.0], beta_deg=[30.0], spec=[0])),
                                n_iter=m.nIter, xi_start=m.XiStart)
    np.testing.assert_array_equal(Xi[0], ref["Xi"][0, 0])
    Xr, passes, _ = reference_solve(oracle, P, 5.0, 11.0, 30.0, n_iter=m.nIter, xi_start=m.XiStart)
    assert response_err(Xi[0], Xr) < RTOL and ref["status"][0, 0, 0] == passes


@pytest.mark.gpu
def test_slender_session_equals_the_host_flow():
    from raft_b200 import packer, solver
    _, P = load_golden("slender_VolturnUS-S")
    P = dict(P, **packer.pack_rotor_excitation(synthetic_fowt(6)))
    ct = solver.CaseTable(_cases(15, 2))
    host = solver.solve_dynamics_slender(P, ct, n_iter=10)
    dev = solver.SlenderSession(P, ct).solve(n_iter=10)
    Xi = dev["Xi"].cpu().numpy() if hasattr(dev["Xi"], "cpu") else np.asarray(dev["Xi"])
    st = dev["status"].cpu().numpy() if hasattr(dev["status"], "cpu") else np.asarray(dev["status"])
    assert response_err(Xi, host["Xi"]) < RTOL
    np.testing.assert_array_equal(st[..., 0], host["status"][..., 0])
    plain = solver.solve_dynamics_slender({k: v for k, v in P.items() if not k.startswith("rot_")}, ct, n_iter=10)
    assert response_err(plain["Xi"], host["Xi"]) > 1e-6


@pytest.mark.gpu
@pytest.mark.parametrize("field,value,msg", [("rot_count", 3, "outside \\[0, max_rotors"), ("rot_r3", 1.0, "not submerged"),
                                             ("rot_G", np.nan, "non-finite")])
def test_host_entries_refuse_a_bad_rotor_table(field, value, msg):
    from raft_b200 import solver
    from raft_b200._lib import RaftkError
    b = solver.DesignBatch(_design_with_rotor(0))
    a = b.arrays[field].copy()
    if field == "rot_count":
        a[0] = value
    elif field == "rot_r3":
        a[0, 0, 2] = value
    else:
        a[0, 0, 1, 2] = value
    b.arrays[field] = a
    with pytest.raises(RaftkError, match=msg):
        solver.solve_dynamics(b, solver.CaseTable(_cases(16, 1)), n_iter=2)


@pytest.mark.gpu
def test_host_entries_refuse_interleaved_train_groups_with_rotors():
    from raft_b200 import solver
    from raft_b200._lib import RaftkError
    cs = _cases(17, 3)
    cs["primary"] = np.array([0, 1, 0], dtype=np.int32)          # train 2 belongs to group 0 but follows group 1
    with pytest.raises(RaftkError, match="contiguous"):
        solver.hydro_excitation(solver.DesignBatch(_design_with_rotor(0)), solver.CaseTable(cs))
