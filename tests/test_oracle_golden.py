"""Pin the C oracle (oracle/raft_oracle.c) against the reference: its own golden pickles and outputs of
the unmodified reference run under the stub harness (tests/golden/*.npz, made by make_golden.py)."""
import numpy as np
import pytest

from conftest import QTF_GOLDEN, golden_names, load_golden, relerr, response_err

NAMES = golden_names()
PICKLED = [n for n in NAMES if n.startswith("test_")]


def test_fixtures_present():
    assert len(NAMES) >= 6 and len(PICKLED) == 3


@pytest.mark.parametrize("name", PICKLED)
def test_excitation_vs_reference_pickle(name, oracle):
    """F_hydro_iner for the 72 (heading, period, height) cases of the reference's test_hydroExcitation."""
    G, P = load_golden(name)
    od = oracle.OracleDesign(P)
    worst = 0.0
    ref = G["ref_pickle_exc_F_hydro_iner"]
    scale = np.abs(ref).max()
    for i in range(len(ref)):
        sc = lambda x: float(np.ravel(x)[0])
        _, _, F_iner, _ = oracle.calc_hydro_excitation(od, 0, sc(G["ref_pickle_exc_height"][i]), sc(G["ref_pickle_exc_period"][i]),
                                                       0.0, sc(G["ref_pickle_exc_heading"][i]))
        if scale > 0:
            worst = max(worst, np.abs(F_iner - ref[i]).max() / scale)
        else:
            assert np.abs(F_iner).max() == 0.0
    assert worst < 1e-13


@pytest.mark.parametrize("name", PICKLED)
def test_linearization_vs_reference_pickle(name, oracle):
    """B_hydro_drag / F_hydro_drag of the reference's test_hydroLinearization (unit spectrum, synthetic Xi)."""
    G, P = load_golden(name)
    od = oracle.OracleDesign(P)
    _, _, _, u = oracle.calc_hydro_excitation(od, 1, 2.0, 10.0, 0.0, 0.0)
    _, B, F = oracle.calc_hydro_linearization(od, u, G["ref_run_lin_Xi"])
    assert relerr(B, G["ref_pickle_lin_B_hydro_drag"]) < 1e-13
    assert relerr(F, G["ref_pickle_lin_F_hydro_drag"]) < 1e-13


@pytest.mark.parametrize("name", NAMES)
def test_excitation_and_linearization_vs_reference_run(name, oracle):
    G, P = load_golden(name)
    od = oracle.OracleDesign(P)
    zeta, F_BEM, F_iner, u = oracle.calc_hydro_excitation(od, 1, 2.0, 10.0, 0.0, 0.0)
    assert relerr(zeta, G["ref_run_lin_zeta"]) < 1e-15
    for mine, key in ((F_iner, "ref_run_lin_F_hydro_iner"), (F_BEM, "ref_run_lin_F_BEM")):
        if np.abs(G[key]).max() > 0:
            assert relerr(mine, G[key]) < 1e-13
        else:
            assert np.abs(mine).max() == 0
    _, B, F = oracle.calc_hydro_linearization(od, u, G["ref_run_lin_Xi"])
    assert relerr(B, G["ref_run_lin_B_hydro_drag"]) < 1e-13
    assert relerr(F, G["ref_run_lin_F_hydro_drag"]) < 1e-13


@pytest.mark.parametrize("name", NAMES)
def test_solve_dynamics_vs_reference_run(name, oracle):
    """Full Model.solveDynamics: response amplitudes and the number of drag-linearisation passes."""
    G, P = load_golden(name)
    od = oracle.OracleDesign(P)
    for i, (Hs, Tp, beta) in enumerate(G["ref_run_solve_cases"]):
        Xi, st = oracle.solve_dynamics(od, 0, Hs, Tp, 0.0, beta, nIter=int(G["n_iter"]), XiStart=float(G["xi_start"]))
        assert st[0] == G["ref_run_solve_passes"][i]
        assert st[2] == 0
        assert response_err(Xi, G["ref_run_solve_Xi"][i]) < 1e-12


def test_helper_known_answers(oracle):
    """Literal known answers of the reference's tests/test_helpers.py (rtol 1e-5 there, same here)."""
    # test_waveKin :41-69
    w = np.array([0.1, 0.25, 0.5, 0.75])
    zeta0 = np.array([0.2, 0.2, 0.2, 0.2])
    beta, h, r = 30, 200, [30, 45, -20]
    k = np.array([oracle.wave_number(x, h) for x in w])
    np.testing.assert_allclose(k, [0.00233623, 0.0071452, 0.02548611, 0.05733945], rtol=1e-5)
    u, ud, pDyn = oracle.wave_kin(zeta0, beta, w, k, h, r)
    np.testing.assert_allclose(u, np.array(
        [[0.0069097100 + 0.0006448900j, 0.0073269700 + 0.0021436100j, 0.0048875900 + 0.0078728400j, -0.0048089800 + 0.0055581900j],
         [-0.0442590100 - 0.0041307200j, -0.0469316700 - 0.0137305200j, -0.0313066500 - 0.0504281200j, 0.0308031300 - 0.0356020400j],
         [-0.0016613100 + 0.0178002300j, -0.0119250300 + 0.0407604200j, -0.0510284000 + 0.0316793100j, -0.0360333000 - 0.0311762500j]]), rtol=1e-5)
    np.testing.assert_allclose(ud, np.array(
        [[-0.0000644885 + 0.0006909710j, -0.0005359019 + 0.0018317440j, -0.0039364177 + 0.0024438000j, -0.0041686415 - 0.0036067400j],
         [0.0004130725 - 0.0044259010j, 0.0034326291 - 0.0117329200j, 0.0252140594 - 0.0156533200j, 0.0267015296 + 0.0231023400j],
         [-0.0017800228 - 0.0001661310j, -0.0101901044 - 0.0029812600j, -0.0158396548 - 0.0255142000j, 0.0233821912 - 0.0270249700j]]), rtol=1e-5)
    np.testing.assert_allclose(pDyn, [1963.730340920 + 183.276331860j, 1703.156386190 + 498.282218140j,
                                      637.171137130 + 1026.342526750j, -417.980049950 + 483.098446900j], rtol=1e-5)
    # test_getKinematics :26-38
    Xi = np.array([[1, 2 + 1j], [0.1 + 0.2j, 0.3 + 0.4j], [0.5 + 0.6j, 0.7 + 0.8j], [0.9 + 1.0j, 1.1 + 1.2j],
                   [1.3 + 1.4j, 1.5 + 1.6j], [1.7 + 1.8j, 1.9 + 2.0j]])
    dr, v, a = oracle.get_kinematics([2, 2, 2], Xi, [0.5, 0.75])
    desired = np.array([
        [[0.2 - 0.8j, 1.2 + 0.2j], [1.7 + 1.8j, 1.9 + 2.0j], [-0.3 - 0.2j, -0.1 + 0j]],
        [[0.4 + 0.1j, -0.15 + 0.9j], [-0.9 + 0.85j, -1.5 + 1.425j], [0.1 - 0.15j, 0 - 0.075j]],
        [[-0.05 + 0.2j, -0.675 - 0.1125j], [-0.425 - 0.45j, -1.06875 - 1.125j], [0.075 + 0.05j, 0.05625 + 0j]]])
    np.testing.assert_allclose(np.array([dr, v, a]), desired, rtol=1e-5, atol=1e-15)
    # test_translateForce3to6DOF :88-94, test_translateMatrix3to6DOF :123-136
    np.testing.assert_allclose(oracle.translate_force([0.5 + 3j, 2.0 + 1.5j, 3.0 + 0.7j], [1, 2, 3]),
                               [0.5 + 3.0j, 2.0 + 1.5j, 3.0 + 0.7j, 0.0 - 3.1j, -1.5 + 8.3j, 1.0 - 4.5j], rtol=1e-5, atol=1e-15)
    Min = np.array([[0.73, 2.41, 3.88], [1.25, 9.12, 5.79], [5.37, 7.94, 8.63]])
    np.testing.assert_allclose(oracle.translate_matrix(Min, [10, 20, 30]), np.array(
        [[7.300e-01, 2.410e+00, 3.880e+00, 5.300e+00, -1.690e+01, 9.500e+00],
         [1.250e+00, 9.120e+00, 5.790e+00, -1.578e+02, -2.040e+01, 6.620e+01],
         [5.370e+00, 7.940e+00, 8.630e+00, -6.560e+01, 7.480e+01, -2.800e+01],
         [5.300e+00, -1.578e+02, -6.560e+01, 3.422e+03, 2.108e+03, -2.546e+03],
         [-1.690e+01, -2.040e+01, 7.480e+01, 8.150e+02, -1.255e+03, 5.650e+02],
         [9.500e+00, 6.620e+01, -2.800e+01, -1.684e+03, 1.340e+02, 4.720e+02]]), rtol=1e-5)


def test_wave_number_and_jonswap(oracle):
    from raft_b200 import grid
    w = grid.make_w(0.005, 0.4)
    k = grid.wave_number(w, 200.0)
    np.testing.assert_allclose(k, np.array([oracle.wave_number(x, 200.0) for x in w]), rtol=1e-14)
    S = oracle.jonswap(w, 6.0, 12.0, 0.0)
    # Hs = 4 sqrt(m0) within the truncation of the grid
    m0 = np.sum(S) * (w[1] - w[0])
    assert abs(4 * np.sqrt(m0) - 6.0) < 0.15


def test_grid_recipes():
    from raft_b200 import grid
    for nw, mf in ((1024, 0.512), (2048, 0.256), (512, 0.40), (1024, 0.1024)):
        assert len(grid.make_w(mf / nw, mf)) == nw


@pytest.mark.parametrize("name", ["cfg1_OC3spar", "cfg2_VolturnUS-S_nw64"])
def test_wave_trains_vs_reference_run(name, oracle):
    """Cases with several wave trains: Model.Xi[ih] of the unmodified reference (raft_model.py:1200-1236)."""
    G, P = load_golden(name)
    tr = G["ref_run_trains"]
    Xi, st = oracle.solve_dynamics_trains(oracle.OracleDesign(P), np.zeros(len(tr), dtype=np.int32), tr[:, 0], tr[:, 1],
                                          np.zeros(len(tr)), tr[:, 2], nIter=int(G["n_iter"]), XiStart=float(G["xi_start"]))
    for ih in range(len(tr)):
        assert response_err(Xi[ih], G["ref_run_trains_Xi"][ih]) < 1e-12


def test_second_order_force_vs_reference_run(oracle):
    """calcHydroForce_2ndOrd (potSecOrder 2, external .12d QTF) and solveDynamics with it, vs the reference run."""
    G, P = load_golden(QTF_GOLDEN)
    od = oracle.OracleDesign(P)
    cases = G["ref_run_solve_cases"]
    for i, (Hs, Tp, beta) in enumerate(cases):
        fm, f = oracle.hydro_force_2nd(od, beta * 0.017453292519943295, G["ref_run_S"][i])
        assert relerr(f, G["ref_run_F2nd"][i]) < 1e-13
        assert relerr(fm, G["ref_run_F2nd_mean"][i]) < 1e-13
        assert np.all(f[:, -1] == 0.0)                                   # raft_fowt.py:2245
        Xi, st = oracle.solve_dynamics(od, 0, Hs, Tp, 0.0, beta, nIter=int(G["n_iter"]), XiStart=float(G["xi_start"]))
        assert st[0] == G["ref_run_solve_passes"][i]
        assert response_err(Xi, G["ref_run_solve_Xi"][i]) < 1e-12
    # the force matters: without the table the response differs visibly
    P0 = {k: v for k, v in P.items() if not k.startswith("qtf")}
    Xi0, _ = oracle.solve_dynamics(oracle.OracleDesign(P0), 0, *cases[0][:2], 0.0, cases[0][2], nIter=int(G["n_iter"]),
                                   XiStart=float(G["xi_start"]))
    assert response_err(Xi0, G["ref_run_solve_Xi"][0]) > 1e-4
    # wave trains: every train gets its own second-order force (raft_model.py:1210-1212)
    tr = G["ref_run_trains"]
    Xi, _ = oracle.solve_dynamics_trains(od, [0] * len(tr), tr[:, 0], tr[:, 1], [0.0] * len(tr), tr[:, 2],
                                         nIter=int(G["n_iter"]), XiStart=float(G["xi_start"]))
    assert response_err(Xi, G["ref_run_trains_Xi"]) < 1e-12


def test_second_order_heading_interpolation_vs_reference_run(oracle):
    """4-heading synthetic table: interp1d along the heading axis incl. the clamped ends (raft_fowt.py:2178-2187)."""
    G, P = load_golden(QTF_GOLDEN)
    P = dict(P)
    P["qtf"] = np.stack([P["qtf"][:, :, 0, :] * s for s in G["mh_scale"]], axis=2)
    P["qtf_heads"] = G["mh_heads"]
    od = oracle.OracleDesign(P)
    for i, b in enumerate(G["mh_betas_deg"]):
        fm, f = oracle.hydro_force_2nd(od, b * 0.017453292519943295, G["ref_run_S"][0])
        assert relerr(f, G["ref_run_mh_F2nd"][i]) < 1e-13
        assert relerr(fm, G["ref_run_mh_F2nd_mean"][i]) < 1e-13


def test_slender_body_qtf_vs_reference_pickle_and_run(oracle):
    """potSecOrder 1: the oracle's calcQTF_slenderBody vs the reference's OWN golden pickle (fixed body; the reference's
    test allows rtol 1e-5) and vs QTFs the reference computed inside solveDynamics with the body moving; then the full
    solve with the QTF inside the loop (response, pass count)."""
    import os
    from conftest import GOLDEN
    z = np.load(os.path.join(GOLDEN, "slender_VolturnUS-S.npz"))
    P = {k[2:]: z[k] for k in z.files if k.startswith("P_")}
    od = oracle.OracleDesign(P)
    n2 = len(P["qs_w"])
    q = oracle.qtf_slender(od, z["ref_pickle_case"][2] * 0.017453292519943295, np.zeros([6, n2], dtype=complex))
    ref = z["ref_pickle_qtf"][:, :, 0, :]
    for a in range(6):
        assert relerr(q[..., a], ref[..., a]) < 1e-13, a
    cases = z["ref_run_solve_cases"]
    for i, (Hs, Tp, beta) in enumerate(cases):
        Xi0 = z["ref_run_solve_Xi0"][i]
        Xi2 = np.array([np.interp(P["qs_w"], P["w"], Xi0[a], left=0, right=0) for a in range(6)])
        q = oracle.qtf_slender(od, beta * 0.017453292519943295, Xi2)
        for a in range(6):
            assert relerr(q[..., a], z["ref_run_solve_qtf"][i][..., a]) < 1e-13, (i, a)
        Xi, st = oracle.solve_dynamics(od, 0, Hs, Tp, 0.0, beta, nIter=int(z["n_iter"]), XiStart=float(z["xi_start"]))
        assert st[0] == z["ref_run_solve_passes"][i]
        assert response_err(Xi, z["ref_run_solve_Xi"][i]) < 1e-11


def test_point_inertia_design_vs_reference_pickle_and_run(oracle):
    """Fourth rigid design of the reference's test set (VolturnUS-S-pointInertia): its golden excitation /
    linearisation pickles and reference-run responses."""
    G, P = load_golden("pin_VolturnUS-S-pointInertia")
    od = oracle.OracleDesign(P)
    ref = G["ref_pickle_exc_F_hydro_iner"]
    sc = lambda x: float(np.ravel(x)[0])
    worst = 0.0
    for i in range(len(ref)):
        _, _, F, _ = oracle.calc_hydro_excitation(od, 0, sc(G["ref_pickle_exc_height"][i]), sc(G["ref_pickle_exc_period"][i]), 0.0,
                                                  sc(G["ref_pickle_exc_heading"][i]))
        worst = max(worst, np.abs(F - ref[i]).max() / np.abs(ref).max())
    assert worst < 1e-13
    _, _, _, u = oracle.calc_hydro_excitation(od, 1, 2.0, 10.0, 0.0, 0.0)
    _, B, F = oracle.calc_hydro_linearization(od, u, G["ref_run_lin_Xi"])
    assert relerr(B, G["ref_pickle_lin_B_hydro_drag"]) < 1e-13 and relerr(F, G["ref_pickle_lin_F_hydro_drag"]) < 1e-13
    for i, (Hs, Tp, beta) in enumerate(G["ref_run_solve_cases"]):
        Xi, st = oracle.solve_dynamics(od, 0, Hs, Tp, 0.0, beta, nIter=int(G["n_iter"]), XiStart=float(G["xi_start"]))
        assert st[0] == G["ref_run_solve_passes"][i] and response_err(Xi, G["ref_run_solve_Xi"][i]) < 1e-12


def test_slender_body_qtf_second_reference_pickle(oracle):
    """The reference's other slender-body golden (VolturnUS-S-pointInertia_true_calcQTF_slenderBody.pkl) + one solve."""
    import os
    from conftest import GOLDEN
    z = np.load(os.path.join(GOLDEN, "pinq_VolturnUS-S-pointInertia.npz"))
    P = {k[2:]: z[k] for k in z.files if k.startswith("P_")}
    od = oracle.OracleDesign(P)
    q = oracle.qtf_slender(od, z["ref_pickle_case"][2] * 0.017453292519943295, np.zeros([6, len(P["qs_w"])], dtype=complex))
    for a in range(6):
        assert relerr(q[..., a], z["ref_pickle_qtf"][:, :, 0, a]) < 1e-13, a
    Hs, Tp, beta = z["ref_run_solve_cases"][0]
    Xi, st = oracle.solve_dynamics(od, 0, Hs, Tp, 0.0, beta, nIter=int(z["n_iter"]), XiStart=float(z["xi_start"]))
    assert st[0] == z["ref_run_solve_passes"][0] and response_err(Xi, z["ref_run_solve_Xi"][0]) < 1e-11


@pytest.mark.parametrize("depth", [40, 1000])
def test_slender_body_qtf_synthetic_geometry_vs_reference_run(depth, oracle):
    """The oracle's calcQTF_slenderBody against the unmodified reference on VolturnUS-S plus an inclined, tapered
    MacCamy-Fuchs brace and a rectangular member with end A above water, at 40 m (every k h < 10) and 1000 m (k h up to
    ~190): fixed body and seeded random motions, two headings, per DOF over every frequency pair."""
    import os
    from conftest import GOLDEN
    z = np.load(os.path.join(GOLDEN, "slender_synth_VolturnUS-S.npz"))
    pre = "d%d_" % depth
    P = {k[len(pre) + 2:]: z[k] for k in z.files if k.startswith(pre + "P_")}
    od = oracle.OracleDesign(P)
    n2 = len(P["qs_w"])
    kh = P["qs_k"] * depth
    assert (kh.max() < 10) if depth == 40 else (kh.min() < 10 and kh.max() > 89.4)
    for c, beta in enumerate(z[pre + "beta"]):
        Xi2 = np.array([np.interp(P["qs_w"], P["w"], z[pre + "Xi0"][c][a], left=0, right=0) for a in range(6)])
        for Xi, ref in ((np.zeros([6, n2], dtype=complex), z[pre + "qtf_fixed"][c]), (Xi2, z[pre + "qtf"][c])):
            q = oracle.qtf_slender(od, beta, Xi)
            for a in range(6):
                assert relerr(q[..., a], ref[..., a]) < 1e-13, (c, a)


def test_generalised_dofs_vs_reference_flexible_pickles(oracle):
    """Groundwork for the next row (flexible members, nDOF = 150): the oracle's generalised calcHydroExcitation /
    calcHydroLinearization with fowt.T against the reference's VolturnUS-S-flexible golden pickles."""
    import os
    from conftest import GOLDEN
    z = np.load(os.path.join(GOLDEN, "flex_VolturnUS-S-flexible.npz"))
    P = {k[2:]: z[k] for k in z.files if k.startswith("P_")}
    gd = oracle.GeneralDesign(P)
    assert gd.n == 150
    ref = z["ref_pickle_exc_F_hydro_iner"]
    worst = 0.0
    for i in range(len(ref)):
        sc = lambda x: float(np.ravel(x)[0])
        _, F, _ = oracle.general_excitation(gd, 0, sc(z["ref_pickle_exc_height"][i]), sc(z["ref_pickle_exc_period"][i]), 0.0,
                                            sc(z["ref_pickle_exc_heading"][i]))
        worst = max(worst, np.abs(F - ref[i]).max() / np.abs(ref).max())
    assert worst < 1e-13
    _, _, u = oracle.general_excitation(gd, 1, 2.0, 10.0, 0.0, 0.0)                 # the reference's own recipe (test_fowt.py:150-175)
    nw = len(P["w"])
    Xi = 0.1 * np.exp(1j * np.linspace(0, 2 * np.pi, nw * gd.n).reshape(gd.n, nw))
    B, F = oracle.general_linearization(gd, u, Xi)
    assert relerr(B, z["ref_pickle_lin_B_hydro_drag"]) < 1e-13 and relerr(F, z["ref_pickle_lin_F_hydro_drag"]) < 1e-13


def test_generalised_solve_vs_reference_run(oracle):
    """150-DOF Model.solveDynamics (flexible members) of the unmodified reference vs the oracle's generalised loop with a
    dense 150 x 150 complex LU per frequency.  The impedance of the flexible system is far worse conditioned than the
    rigid 6 x 6 one, so two independent LU implementations agree to ~1e-11 only (tolerance 1e-9 here)."""
    import os
    from conftest import GOLDEN
    z = np.load(os.path.join(GOLDEN, "flex_VolturnUS-S-flexible.npz"))
    P = {k[2:]: z[k] for k in z.files if k.startswith("P_")}
    gd = oracle.GeneralDesign(P)
    for i, (Hs, Tp, beta) in enumerate(z["ref_run_solve_cases"]):
        Xi, st = oracle.general_solve_dynamics(gd, z["gen_M"], z["gen_B"], z["gen_C"], 0, Hs, Tp, 0.0, beta, nIter=int(z["n_iter"]),
                                               XiStart=float(z["xi_start"]))
        assert st[0] == z["ref_run_solve_passes"][i]
        assert relerr(Xi, z["ref_run_solve_Xi"][i]) < 1e-9
