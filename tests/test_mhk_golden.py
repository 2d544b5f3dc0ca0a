"""Submerged rotor against the reference's own run (tests/golden/make_golden_mhk.py: VolturnUS-S with its hub 18 m below the
waterline and a seeded I_hydro on the reference's rotor; r3, R_q, the hub node and fowt.T are the reference's).

CPU: the packer's G applied to the reference's hub kinematics reproduces the rotor's share of the reference's F_hydro_iner
(one train; two trains: the last train only), and the restated solve loop of test_mhk_rotor (the oracle's excitation and
drag linearisation plus G ud) reproduces the reference's Xi and pass counts.  GPU: the solver and the stand-alone excitation
against the same run."""
import types

import numpy as np
import pytest

from conftest import load_golden, relerr, response_err
from test_mhk_rotor import reference_solve, restated_rotor_excitation

NAME = "mhk_VolturnUS-S"


def _golden():
    return load_golden(NAME)


def _live_rotor(G):
    """The fixture's raw rotor inputs as a duck-typed live FOWT (rotorList, T, r6)."""
    T = np.zeros([6 * (int(G["hub_id"]) + 1), 6])
    T[6 * int(G["hub_id"]):] = G["T_hub"]
    rot = types.SimpleNamespace(r3=G["r3"], I_hydro=G["I_hydro"], R_q=G["R_q"], nodeList=[types.SimpleNamespace(id=int(G["hub_id"]))])
    return types.SimpleNamespace(rotorList=[rot], T=T, r6=G["r6"])


def test_packer_reproduces_the_reference_rotor_excitation():
    from raft_b200 import packer
    G, P = _golden()
    R = packer.pack_rotor_excitation(_live_rotor(G))
    np.testing.assert_array_equal(R["rot_G"], P["rot_G"])          # the live reference FOWT packs the same table
    np.testing.assert_array_equal(R["rot_r3"], P["rot_r3"])
    for name in ("one", "two"):
        ud, Fr, F0 = G["exc_%s_ud" % name], G["exc_%s_F_hydro_iner_rot" % name], G["exc_%s_F_hydro_iner_plain" % name]
        last = len(ud) - 1
        for ih in range(len(ud)):
            ref = Fr[ih] - F0[ih]
            if ih != last:
                assert not np.any(ref), "the reference puts the rotor term on the last train only"
                continue
            got = R["rot_G"][0] @ ud[last]
            assert relerr(got, ref) < 1e-14


def test_restated_loop_reproduces_the_reference_run(oracle):
    G, P = _golden()
    for c, (Hs, Tp, beta) in enumerate(G["ref_run_solve_cases"]):
        Xi, passes, _ = reference_solve(oracle, P, Hs, Tp, beta, n_iter=int(G["n_iter"]), xi_start=float(G["xi_start"]))
        assert response_err(Xi, G["ref_run_solve_Xi"][c]) < 1e-10
        assert passes == G["ref_run_solve_passes"][c]
    od = oracle.OracleDesign(P)
    Hs, Tp, beta = G["exc_one_trains"][0]
    zeta, _, Fi, _ = oracle.calc_hydro_excitation(od, 0, Hs, Tp, 0.0, beta)
    assert relerr(Fi + restated_rotor_excitation(oracle, P, zeta, beta), G["exc_one_F_hydro_iner_rot"][0]) < 1e-13


@pytest.mark.gpu
@pytest.mark.parametrize("env,kernel", [({}, None), ({"RAFTK_FORCE_V1": "1"}, "v1")], ids=["planner", "v1"])
def test_solver_against_the_reference_run(monkeypatch, env, kernel):
    from raft_b200 import solver
    monkeypatch.delenv("RAFTK_FORCE_V1", raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    G, P = _golden()
    sc = G["ref_run_solve_cases"]
    n = len(sc)
    ct = solver.CaseTable(dict(Hs=sc[:, 0], Tp=sc[:, 1], gamma=np.zeros(n), beta_deg=sc[:, 2], spec=np.zeros(n, dtype=np.int32)))
    out = solver.solve_dynamics(solver.DesignBatch(P), ct, n_iter=int(G["n_iter"]), xi_start=float(G["xi_start"]))
    rec = solver.last_dispatch()
    assert rec["family"] == "solve" and (kernel is None or rec["kernel"] == kernel), rec
    assert response_err(out["Xi"][0], G["ref_run_solve_Xi"]) < 1e-10
    np.testing.assert_array_equal(out["status"][0, :, 0], G["ref_run_solve_passes"])


@pytest.mark.gpu
def test_excitation_against_the_reference_run():
    from raft_b200 import solver
    G, P = _golden()
    for name in ("one", "two"):
        tr = G["exc_%s_trains" % name]
        n = len(tr)
        cases = dict(Hs=tr[:, 0], Tp=tr[:, 1], gamma=np.zeros(n), beta_deg=tr[:, 2], spec=np.zeros(n, dtype=np.int32))
        if n > 1:
            cases["primary"] = np.zeros(n, dtype=np.int32)
        ex = solver.hydro_excitation(solver.DesignBatch(P), solver.CaseTable(cases))
        assert relerr(ex["F_iner"][0], G["exc_%s_F_hydro_iner_rot" % name]) < 1e-12
