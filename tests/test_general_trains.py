"""Wave trains and output statistics on the generalised-DOF GPU path (raftk_general_solve_dynamics_* with cases.primary,
raftk_general_channel_stats_*) against the unmodified reference's Model.solveDynamics / FOWT.saveTurbineOutputs of the
150-DOF VolturnUS-S-flexible (fixture flexout_VolturnUS-S-flexible).  Every train at 1e-10 against the reference run (cond ~1e6
impedance: the primaries agree to ~1e-11, the secondary train, solved from the primary's LU factors where the reference multiplies
by an explicit inverse (raft_model.py:1191), to 8e-11).  Statistics are compared within groups of channels that share units
(translations, rotations, accelerations, forces, moments), relative to the group's largest reference value, as
tests/conftest.response_err does for responses: 1e-10, PSDs 2e-10 (squared amplitudes).  Relative to its own size a small
channel carries the response's absolute error at a larger relative size (the yaw of the two-train case is ~1e-3 of the other
rotations)."""
import os

import numpy as np
import pytest

import general_trains_checker as gtc
from conftest import GOLDEN, relerr

pytestmark = [pytest.mark.gpu]

NAME = "flexout_VolturnUS-S-flexible"
RTOL = 1e-10


@pytest.fixture(scope="module")
def G():
    z = np.load(os.path.join(GOLDEN, NAME + ".npz"))
    return {k: z[k] for k in z.files}


def _P(G):
    return {k[2:]: v for k, v in G.items() if k.startswith("P_")}


def _case_dicts(G):
    out = []
    for ic in range(3):
        tr = G["ref_run_case%d_trains" % ic]
        out.append(dict(wave_spectrum=["JONSWAP"] * len(tr), wave_height=list(tr[:, 0]), wave_period=list(tr[:, 1]),
                        wave_heading=list(tr[:, 2]), wave_gamma=[0.0] * len(tr)))
    return out


def _channels(G):
    names = []
    for s in G["ch_names"]:
        nm, ir = str(s).split(":")
        names.append((nm, None if ir == "" else int(ir)))
    return dict(names=names, R=G["ch_R"], wpow=G["ch_wpow"], avg=G["ch_avg"])


def test_general_trains_vs_reference_run(G):
    from raft_b200 import packer, solver
    table, owner, first = packer.pack_case_trains(_case_dicts(G))
    assert list(first) == [0, 1, 2] and list(table["primary"]) == [0, 1, 2, 2]
    Xi, st = solver.general_solve_dynamics(_P(G), G["gen_M"], G["gen_B"], G["gen_C"], solver.CaseTable(table), n_iter=int(G["n_iter"]),
                                           xi_start=float(G["xi_start"]))
    for ic in range(3):
        ref = G["ref_run_case%d_Xi" % ic]
        idx = np.nonzero(owner == ic)[0]
        assert st[first[ic], 0] == int(G["ref_run_case%d_passes" % ic])
        for ih, t in enumerate(idx):
            assert relerr(Xi[t], ref[ih]) < RTOL, (ic, ih, relerr(Xi[t], ref[ih]))
    assert st[:3, 3].tolist() == [0, 0, 0] and st[3].tolist() == [0, 1, 0, 3]        # secondary: 0 passes, 1, flags, primary + 1


def test_mixed_table_leaves_independent_cases_bit_identical(G, oracle):
    from raft_b200 import packer, solver
    P, n_iter, xs = _P(G), int(G["n_iter"]), float(G["xi_start"])
    cases = _case_dicts(G)
    mixed = [cases[0], cases[2], cases[1]]
    table, owner, first = packer.pack_case_trains(mixed)
    Xi, st = solver.general_solve_dynamics(P, G["gen_M"], G["gen_B"], G["gen_C"], solver.CaseTable(table), n_iter=n_iter, xi_start=xs)
    solo, sts = solver.general_solve_dynamics(P, G["gen_M"], G["gen_B"], G["gen_C"], solver.CaseTable(packer.pack_cases([cases[0], cases[1]])),
                                              n_iter=n_iter, xi_start=xs)
    assert np.array_equal(Xi[0], solo[0]) and np.array_equal(Xi[3], solo[1])
    assert np.array_equal(st[[0, 3]], sts)
    # the trains of the middle case against the reference run; the checker's pass count.  (The checker's own responses are not
    # the yardstick here: its explicit inverse of this cond ~1e6 impedance moves by ~1e-10 with the host's LAPACK build.)
    tr = G["ref_run_case2_trains"]
    _, so, _ = gtc.solve_trains(oracle, P, G["gen_M"], G["gen_B"], G["gen_C"], tr, nIter=n_iter, XiStart=xs)
    assert st[1, 0] == so[0] == int(G["ref_run_case2_passes"]) and st[2].tolist() == [0, 1, 0, 2]
    for ih in range(len(tr)):
        ref = G["ref_run_case2_Xi"][ih]
        assert relerr(Xi[1 + ih], ref) < RTOL, (ih, relerr(Xi[1 + ih], ref))


def test_general_session_matches_host_entry_point(G):
    import torch
    from raft_b200 import packer, solver
    P, n_iter, xs = _P(G), int(G["n_iter"]), float(G["xi_start"])
    table, _, _ = packer.pack_case_trains(_case_dicts(G))
    ct = solver.CaseTable(table)
    Xh, sh = solver.general_solve_dynamics(P, G["gen_M"], G["gen_B"], G["gen_C"], ct, n_iter=n_iter, xi_start=xs)
    s = solver.GeneralSession(P, G["gen_M"], G["gen_B"], G["gen_C"], ct)
    Xd, sd_ = s.solve(n_iter=n_iter, xi_start=xs)
    ch = _channels(G)
    std_d, psd_d, amp_d = s.stats(ch["R"], ch["wpow"], psd=True, amp=True)
    torch.cuda.synchronize()
    assert np.array_equal(Xd.cpu().numpy(), Xh) and np.array_equal(sd_.cpu().numpy(), sh)
    std_h, psd_h, amp_h = solver.general_channel_stats(ch["R"], ch["wpow"], P["w"], Xh, float(P["dw"]), psd=True, amp=True)
    assert np.array_equal(std_d.cpu().numpy(), std_h) and np.array_equal(psd_d.cpu().numpy(), psd_h)
    assert np.array_equal(amp_d.cpu().numpy(), amp_h)
    Y = np.einsum("kb,tbw->tkw", ch["R"], Xh) * P["w"][None, None, :] ** ch["wpow"][None, :, None]
    assert relerr(amp_h, Y) < 1e-12
    assert relerr(std_h, np.sqrt(0.5 * np.sum(np.abs(Y) ** 2, axis=-1))) < 1e-12
    assert relerr(psd_h, 0.5 * np.abs(Y) ** 2 / float(P["dw"])) < 1e-12


def test_general_analyze_cases_vs_save_turbine_outputs(G):
    from raft_b200 import solver
    out = solver.general_analyze_cases(_P(G), G["gen_M"], G["gen_B"], G["gen_C"], _case_dicts(G), channels=_channels(G),
                                       n_iter=int(G["n_iter"]), xi_start=float(G["xi_start"]))
    assert [len(x) for x in out["Xi_trains"]] == [1, 1, 2]
    assert out["status"][:, 0].tolist() == [int(G["ref_run_case%d_passes" % ic]) for ic in range(3)]
    groups = [("surge", "sway", "heave"), ("roll", "pitch", "yaw"), ("AxRNA", "AyRNA", "AzRNA"), ("FbaseX", "FbaseY", "FbaseZ"),
              ("MbaseX", "MbaseY", "MbaseZ", "Mbase")]
    for ic in range(3):
        m = out["case_metrics"][ic]
        for grp in groups:
            for s in ("_avg", "_std", "_max", "_min", "_PSD") + (("_RA",) if grp[0] in ("surge", "roll") else ()):
                scale = max(np.abs(G["ref_run_case%d_%s%s" % (ic, c, s)]).max() for c in grp)
                for c in grp:
                    ref, got = G["ref_run_case%d_%s%s" % (ic, c, s)], np.asarray(m[c + s])
                    assert got.shape == ref.shape, (ic, c + s)
                    if scale == 0:
                        assert np.abs(got).max() == 0, (ic, c + s)
                    else:
                        err = np.abs(got - ref).max() / scale
                        assert err < (2 * RTOL if s == "_PSD" else RTOL), (ic, c + s, err)
