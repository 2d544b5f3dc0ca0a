"""Wave trains and output statistics of a FOWT with generalised degrees of freedom (150-DOF VolturnUS-S-flexible), without a
GPU: the multi-train checker (tests/general_trains_checker.py) and the packed output channels against the unmodified
reference's Model.solveDynamics and FOWT.saveTurbineOutputs (fixture flexout_VolturnUS-S-flexible, made by
tests/golden/make_golden_flexout.py).
Responses at 1e-10 (the impedance has cond ~1e6; two independent LUs agree to ~2e-11), statistics at 1e-12 -- except the
tower-base forces FbaseX/Y/Z at 1e-11: the reference forms -Kf (T Xi), tower stiffness times node displacements whose
rigid-body parts cancel, and the packed channel folds -Kf T into one row, which rounds differently (measured <= 8e-12 on
the PSDs, <= 4e-13 on the standard deviations)."""
import os

import numpy as np
import pytest

import general_trains_checker as gtc
from conftest import GOLDEN, relerr

NAME = "flexout_VolturnUS-S-flexible"
CHANNELS = ["surge", "sway", "heave", "roll", "pitch", "yaw", "AxRNA", "AyRNA", "AzRNA",
            "FbaseX", "FbaseY", "FbaseZ", "MbaseX", "MbaseY", "MbaseZ", "Mbase"]


@pytest.fixture(scope="module")
def G():
    z = np.load(os.path.join(GOLDEN, NAME + ".npz"))
    return {k: z[k] for k in z.files}


def _channels(G):
    names = []
    for s in G["ch_names"]:
        nm, ir = str(s).split(":")
        names.append((nm, None if ir == "" else int(ir)))
    return dict(names=names, R=G["ch_R"], wpow=G["ch_wpow"], avg=G["ch_avg"])


def _cases(G):
    return [G["ref_run_case%d_trains" % ic] for ic in range(3)]


def test_fixture_covers_single_and_multi_train_cases(G):
    tr = _cases(G)
    assert [len(t) for t in tr] == [1, 1, 2]
    for ic, t in enumerate(tr):
        X = G["ref_run_case%d_Xi" % ic]
        assert X.shape == (len(t) + 1, 150, len(G["P_w"])) and np.all(X[-1] == 0)


def test_checker_general_trains_vs_reference_run(G, oracle):
    P = {k[2:]: v for k, v in G.items() if k.startswith("P_")}
    n_iter, xs = int(G["n_iter"]), float(G["xi_start"])
    for ic, tr in enumerate(_cases(G)):
        X, st, (Fd_np, Fd_c) = gtc.solve_trains(oracle, P, G["gen_M"], G["gen_B"], G["gen_C"], tr, nIter=n_iter, XiStart=xs)
        ref = G["ref_run_case%d_Xi" % ic]
        assert st[0] == int(G["ref_run_case%d_passes" % ic]) and st[2] == 0, (ic, st)
        assert relerr(Fd_np, Fd_c) < 1e-13                    # the NumPy Bmat / drag excitation against the pinned C routine
        for ih in range(len(tr)):
            assert relerr(X[ih], ref[ih]) < 1e-10, (ic, ih, relerr(X[ih], ref[ih]))
    # train 0 of the multi-train case is the single-train solve of that sea state; the C checker's own solve agrees
    tr = _cases(G)[2]
    X0, s0, _ = gtc.solve_trains(oracle, P, G["gen_M"], G["gen_B"], G["gen_C"], tr[:1], nIter=n_iter, XiStart=xs)
    X2, s2, _ = gtc.solve_trains(oracle, P, G["gen_M"], G["gen_B"], G["gen_C"], tr, nIter=n_iter, XiStart=xs)
    assert np.array_equal(X0[0], X2[0]) and np.array_equal(s0, s2)
    Xc, sc = oracle.general_solve_dynamics(oracle.GeneralDesign(P), G["gen_M"], G["gen_B"], G["gen_C"], 0, tr[0, 0], tr[0, 1], 0.0, tr[0, 2],
                                           nIter=n_iter, XiStart=xs)
    assert np.array_equal(sc, s0) and relerr(X0[0], Xc) < 1e-10


def test_general_channels_numpy_vs_save_turbine_outputs(G):
    """The packed channels (R, wpow, avg) applied to the reference's own Model.Xi with NumPy, combined over the trains by
    solver.general_case_metrics, reproduce every saveTurbineOutputs entry of the fixture."""
    from raft_b200 import solver
    ch = _channels(G)
    w, dw = G["P_w"], float(G["P_dw"])
    assert [nm for nm, _ in ch["names"]] == CHANNELS[:-1]
    for ic in range(3):
        Xi = G["ref_run_case%d_Xi" % ic][:-1]                                    # the trains (the last row is zero)
        Y = np.einsum("kb,tbw->tkw", ch["R"], Xi) * w[None, None, :] ** ch["wpow"][None, :, None]
        sd = np.sqrt(0.5 * np.sum(np.abs(Y) ** 2, axis=-1))
        psd = 0.5 * np.abs(Y) ** 2 / dw
        m = solver.general_case_metrics(ch, sd, psd, Y, np.arange(len(Xi)))
        for nm in CHANNELS:
            for suffix in ("_avg", "_std", "_max", "_min", "_PSD"):
                ref, got = G["ref_run_case%d_%s%s" % (ic, nm, suffix)], np.asarray(m[nm + suffix])
                assert got.shape == ref.shape, (ic, nm, suffix, got.shape, ref.shape)
                if np.abs(ref).max() == 0:
                    assert np.abs(got).max() == 0, (ic, nm, suffix)
                else:
                    tol = 1e-11 if nm.startswith("Fbase") else 1e-12
                    assert relerr(got, ref) < tol, (ic, nm, suffix, relerr(got, ref))
        for nm in CHANNELS[:6]:
            assert relerr(m[nm + "_RA"], G["ref_run_case%d_%s_RA" % (ic, nm)]) < 1e-12, (ic, nm)


def test_combine_trains_is_the_reference_sum_of_squares():
    from raft_b200 import solver
    rng = np.random.default_rng(3)
    X = rng.normal(size=(3, 5, 16)) + 1j * rng.normal(size=(3, 5, 16))
    sd = np.sqrt(0.5 * np.sum(np.abs(X) ** 2, axis=-1))
    psd = 0.5 * np.abs(X) ** 2 / 0.1
    s, p = solver.combine_trains(sd, psd, np.array([0, 2]))
    assert relerr(s, np.sqrt(0.5 * np.sum(np.abs(X[[0, 2]]) ** 2, axis=(0, 2)))) < 1e-14     # helpers.getRMS over two trains
    assert relerr(p, np.sum(0.5 * np.abs(X[[0, 2]]) ** 2 / 0.1, axis=0)) < 1e-14             # helpers.getPSD


def test_pack_general_channels_rejects_rigid_towers():
    from raft_b200 import packer

    class Node:
        def __init__(self, i, r):
            self.id, self.r0, self.r = i, np.array(r, dtype=float), np.array(r, dtype=float)

    class Obj:
        pass
    f = Obj()
    f.T, f.g, f.r6, f.nplatmems = np.eye(12), 9.81, np.zeros(6), 0
    f.rigidBodyNode = Node(0, [0, 0, 0, 0, 0, 0])
    rot, tow = Obj(), Obj()
    rot.nodeList, tow.type = [Node(1, [0, 0, 100, 0, 0, 0])], "rigid"
    f.rotorList, f.memberList = [rot], [tow]
    with pytest.raises(NotImplementedError):
        packer.pack_general_channels(f)
