"""Mooring line tension statistics (raftk_farm_channel_stats_*, solver.farm_channel_stats, DeviceSession.farm_channel_stats,
packer.pack_mooring_tensions, Model.analyzeCases' Tmoor_* and array_mooring entries).  Without a GPU: the struct layout and
prototypes against include/raftk.h, the workspace query, every refusal, pack_mooring_tensions on a MoorPy stand-in, the
tension rows of pack_general_channels and the reference's w[0] PSD divisor.  On the GPU: the reference's own analyzeCases
tensions (fixtures tmoor_*, tests/golden/make_golden_tmoor.py), bit-identity with k_general_channel_stats on the same R and
Xi for every tile shape, batch independence, amplitudes against numpy, the session path and the Model API."""
import ctypes as C
import json
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT

HEADER = os.path.join(ROOT, "include", "raftk.h")
NEW = ("raftk_farm_channel_stats_workspace_bytes", "raftk_farm_channel_stats_dev", "raftk_farm_channel_stats_host")
RTOL = 1e-10
gpu = pytest.mark.gpu


def _fixture(name):
    return np.load(os.path.join(GOLDEN, "tmoor_%s.npz" % name))


# ---- without a GPU --------------------------------------------------------------------------------------------------
def _prototype(name):
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    m = re.search(r"\b(\w+\s*\*?)\s*\b%s\s*\(([^)]*)\)\s*;" % name, src)
    assert m, name
    return m.group(1).strip(), [a.strip() for a in m.group(2).split(",")]


@pytest.mark.parametrize("name", NEW)
def test_bindings_match_header_prototypes(name):
    from raft_b200 import _lib
    ret, params = _prototype(name)
    fn = getattr(_lib.lib, name)
    assert name in _lib.SYMBOLS and len(fn.argtypes) == len(params), (name, params)
    for decl, ct in zip(params, fn.argtypes):
        if "raftk_farm_channels" in decl:
            want = C.POINTER(_lib.RaftkFarmChannels)
        else:
            want = C.c_void_p if "*" in decl else (C.c_size_t if decl.startswith("size_t") else C.c_int32)
        assert ct is want, (name, decl, ct)
    assert fn.restype is (C.c_size_t if ret == "size_t" else C.c_int)


def test_struct_layout_matches_header(tmp_path):
    from raft_b200 import _lib
    S = _lib.RaftkFarmChannels
    fields = [n for n, _ in S._fields_]
    src = tmp_path / "t.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "raftk.h"\nint main(void){printf("%%zu %s\\n", sizeof(raftk_farm_channels), %s);'
                   'printf("%%d %%d\\n", RAFTK_FARM_CH_MAX, RAFTK_FARM_TILE_L2); return 0;}\n'
                   % (" ".join(["%zu"] * len(fields)), ", ".join("offsetof(raftk_farm_channels, %s)" % n for n in fields)))
    exe = tmp_path / "t"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert got[:-2] == [C.sizeof(S)] + [getattr(S, n).offset for n in fields]
    assert got[-2:] == [4096, -1]


def _channels(nch=4, R_shared=1, wpow=None, psd=True):
    from raft_b200 import _lib
    ch = _lib.RaftkFarmChannels()
    ch.n_ch, ch.R_shared, ch.R, ch.dw, ch.std = nch, R_shared, 0x1000, 0.1, 0x1000
    ch.psd = 0x1000 if psd else None
    keep = np.ascontiguousarray(np.zeros(nch) if wpow is None else wpow, dtype=np.int32)
    ch.wpow = keep.ctypes.data
    return ch, keep


def test_workspace_query_without_gpu():
    from raft_b200._lib import lib
    ch, _ = _channels(nch=7, psd=False)
    assert lib.raftk_farm_channel_stats_workspace_bytes(3, 5, 11, C.byref(ch)) == 3 * 5 * 7 * 11 * 8
    ch.psd = 0x1000                                                  # |Y|^2 passes through psd: no workspace
    assert lib.raftk_farm_channel_stats_workspace_bytes(3, 5, 11, C.byref(ch)) == 0
    ch.psd = None
    for F, R, nw in ((0, 5, 11), (3, 0, 11), (3, 5, 0)):
        assert lib.raftk_farm_channel_stats_workspace_bytes(F, R, nw, C.byref(ch)) == 0
    assert lib.raftk_farm_channel_stats_workspace_bytes(3, 5, 11, None) == 0


@pytest.mark.parametrize("case,msg", [
    ("n_farms", ">= 1"), ("n_rows", ">= 1"), ("n_dof", ">= 1"), ("nw", ">= 1"), ("n_ch", ">= 1"), ("n_ch_max", "at most"),
    ("wpow3", "wpow must be"), ("wpow_neg", "wpow must be"), ("R", "R, Xi_sys and std"), ("Xi", "R, Xi_sys and std"),
    ("std", "R, Xi_sys and std"), ("R_shared", "R_shared"), ("dw", "dw must be"), ("w", "w is required"), ("null", "null argument"),
])
def test_refusals_before_any_launch(case, msg):
    from raft_b200._lib import lib
    dims = dict(n_farms=2, n_rows=3, n_dof=12, nw=16)
    wpow = [0, 1, 2, 0] if case == "w" else None
    ch, keep = _channels(wpow=wpow)
    xi, w = 0x1000, (None if case == "w" else 0x1000)
    if case in dims:
        dims[case] = 0
    elif case == "n_ch":
        ch.n_ch = 0
    elif case == "n_ch_max":
        ch.n_ch = 4097
        keep = np.zeros(4097, dtype=np.int32)
        ch.wpow = keep.ctypes.data
    elif case in ("wpow3", "wpow_neg"):
        keep[2] = 3 if case == "wpow3" else -1
    elif case == "R":
        ch.R = None
    elif case == "Xi":
        xi = None
    elif case == "std":
        ch.std = None
    elif case == "R_shared":
        ch.R_shared = 2
    elif case == "dw":
        ch.dw = 0.0
    ref = None if case == "null" else C.byref(ch)
    before = lib.raftk_launch_count()
    args = (dims["n_farms"], dims["n_rows"], dims["n_dof"], dims["nw"], w, xi, ref)
    assert lib.raftk_farm_channel_stats_host(*args) == -1 and msg in lib.raftk_last_error().decode()
    assert lib.raftk_farm_channel_stats_dev(*args, 0x1000, 1 << 30, None) == -1 and msg in lib.raftk_last_error().decode()
    assert lib.raftk_launch_count() == before


def test_dev_refuses_a_small_workspace():
    from raft_b200._lib import lib
    ch, keep = _channels(nch=4, psd=False)
    need = 2 * 3 * 4 * 16 * 8
    before = lib.raftk_launch_count()
    for ws, wb in ((None, need), (0x1000, need - 8), (0x1000, 0)):
        assert lib.raftk_farm_channel_stats_dev(2, 3, 12, 16, 0x1000, 0x1000, C.byref(ch), ws, wb, None) == -1
        assert "workspace" in lib.raftk_last_error().decode()
    assert lib.raftk_launch_count() == before


def test_python_refusals():
    from raft_b200 import solver
    Xi = np.zeros([2, 3, 12, 8], dtype=complex)
    with pytest.raises(ValueError):
        solver.farm_channel_stats(np.zeros([4, 6]), Xi, 0.1)                        # wrong DOF count
    with pytest.raises(ValueError):
        solver.farm_channel_stats(np.zeros([3, 4, 12]), Xi, 0.1)                    # three farms' R for two farms
    with pytest.raises(ValueError):
        solver.farm_channel_stats(np.zeros([4, 12]), Xi, 0.1, wpow=[0, 1, 3, 0], w=np.ones(8))
    with pytest.raises(ValueError):
        solver.farm_channel_stats(np.zeros([4, 12]), Xi, 0.0)


class _FakeMoorPy:
    """The three things pack_mooring_tensions asks of a MoorPy system."""

    def __init__(self, J, T0, n_lines):
        self.J, self.T0, self.lineList = J, T0, [object()] * n_lines
        self.calls = []

    def getCoupledStiffness(self, lines_only=False, tensions=False):
        self.calls.append((lines_only, tensions))
        return np.eye(self.J.shape[1]), self.J

    def getTensions(self):
        return self.T0


def test_pack_mooring_tensions():
    from raft_b200 import packer
    rng = np.random.default_rng(1)
    J, T0 = rng.normal(size=(10, 12)), rng.uniform(1, 2, 10)
    ms = _FakeMoorPy(J, T0, 5)
    t = packer.pack_mooring_tensions(ms)
    assert ms.calls == [(True, True)]
    assert np.array_equal(t["J"], J) and np.array_equal(t["T0"], T0) and t["n_lines"] == 5
    d = packer.pack_mooring_tensions(dict(J=J, T0=T0))
    assert np.array_equal(d["J"], J) and np.array_equal(d["T0"], T0) and d["n_lines"] == 5
    with pytest.raises(ValueError):
        packer.pack_mooring_tensions(_FakeMoorPy(J, T0, 4))                       # 10 ends for 4 lines
    with pytest.raises(ValueError):
        packer.pack_mooring_tensions(dict(J=J, T0=T0[:9]))
    with pytest.raises(ValueError):
        packer.pack_mooring_tensions(dict(J=J[:9], T0=T0[:9]))                     # an odd number of line ends


@pytest.mark.parametrize("moorMod", [1, 2])
def test_pack_mooring_tensions_refuses_dynamic_moorings(moorMod):
    from raft_b200 import packer
    with pytest.raises(NotImplementedError, match="moorMod"):
        packer.pack_mooring_tensions(dict(J=np.zeros([2, 6]), T0=np.zeros(2)), moorMod=moorMod)


def test_reference_psd_divides_by_first_frequency():
    """Tmoor_PSD of the reference is 1/2 |T|^2 / w[0] summed over the wave trains (raft_fowt.py:2370, 2399), not / dw (the
    two coincide on grids that start at their step, as the reference's own do; Model.analyzeCases passes w[0])."""
    z = _fixture("VolturnUS-S")
    w = z["w"]
    for ic in range(2):
        T = np.einsum("ab,hbw->haw", z["J0"], z["Xi_c%d" % ic])
        a2 = (np.abs(T) ** 2).sum(axis=0)
        assert np.allclose(z["fowt0_Tmoor_PSD"][ic], 0.5 * a2 / w[0], rtol=1e-12, atol=0)
        assert np.allclose(z["fowt0_Tmoor_std"][ic], np.sqrt(0.5 * a2.sum(axis=1)), rtol=1e-12, atol=0)
        assert np.array_equal(z["fowt0_Tmoor_max"][ic], z["T00"] + 3 * z["fowt0_Tmoor_std"][ic])


class _Node:
    def __init__(self, i, r0):
        self.id, self.r0 = i, np.array(r0, dtype=float)


class _FlexFowt:
    """A FOWT with generalised DOFs as pack_general_channels sees it: no rotors, rigid-body node rows in T."""

    def __init__(self, rng, n=14):
        self.T = rng.normal(size=(12, n))
        self.g, self.rigidBodyNode = 9.81, _Node(0, [0.3, -0.2, -1.5])
        self.w = np.linspace(0.05, 0.5, 10)


def test_general_channels_gain_tension_rows_in_radians():
    from raft_b200 import packer, solver
    rng = np.random.default_rng(4)
    f = _FlexFowt(rng)
    J, T0 = rng.normal(size=(6, 6)), rng.uniform(1, 2, 6)
    base = packer.pack_general_channels(f)
    ch = packer.pack_general_channels(f, tensions=dict(J=J, T0=T0))
    n0 = len(base["names"])
    assert np.array_equal(ch["R"][:n0], base["R"]) and ch["tension"]["row0"] == n0
    assert ch["names"][n0:] == [("Tmoor", k) for k in range(6)] and np.all(ch["wpow"][n0:] == 0)
    R_prp = base["R"][:6].copy()
    R_prp[3:] = np.deg2rad(R_prp[3:])                                              # the motion rows carry rad2deg, tensions do not
    assert np.allclose(ch["R"][n0:], J @ R_prp, rtol=1e-13, atol=1e-12)
    assert ch["tension"]["w0"] == f.w[0]
    # the metrics: reference shapes, avg +- 3 std, PSD divided by w[0]
    nw, dw = 10, f.w[1] - f.w[0]
    sd = rng.uniform(1, 2, [2, len(ch["names"])])
    ps = rng.uniform(1, 2, [2, len(ch["names"]), nw])
    m = solver.general_case_metrics(ch, sd, ps, ps + 0j, np.arange(2), dw=dw)
    want_sd = np.sqrt((sd[:, n0:] ** 2).sum(axis=0))
    assert m["Tmoor_std"].shape == (6,) and m["Tmoor_PSD"].shape == (6, nw)
    assert np.allclose(m["Tmoor_std"], want_sd, rtol=1e-15) and np.array_equal(m["Tmoor_avg"], T0)
    assert np.allclose(m["Tmoor_max"], T0 + 3 * want_sd, rtol=1e-15) and np.allclose(m["Tmoor_min"], T0 - 3 * want_sd, rtol=1e-15)
    assert np.allclose(m["Tmoor_PSD"], ps[:, n0:].sum(axis=0) * dw / f.w[0], rtol=1e-14)
    with pytest.raises(ValueError):
        solver.general_case_metrics(ch, sd, ps, ps + 0j, np.arange(2))


# ---- on the GPU -----------------------------------------------------------------------------------------------------
def _rel(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)).max() / np.abs(np.asarray(b)).max()


@gpu
def test_rigid_fowt_tensions_vs_reference():
    """VolturnUS-S, a case with two wave trains and one with one: J applied to the reference's own Xi through the path
    Model.analyzeCases uses (channel_stats, J constant over w) and through farm_channel_stats."""
    from raft_b200 import solver
    z = _fixture("VolturnUS-S")
    w0, nw = float(z["w"][0]), len(z["w"])
    for ic in range(2):
        Xi = z["Xi_c%d" % ic]
        sd, ps, _ = solver.channel_stats(np.repeat(z["J0"][:, :, None], nw, axis=2) + 0j, Xi, w0)
        sd2, ps2, _ = solver.farm_channel_stats(z["J0"], Xi, w0)
        idx = np.arange(len(Xi))
        for s_, p_ in ((sd, ps), (sd2, ps2)):
            m = solver.tension_metrics(z["T00"], *solver.combine_trains(s_, p_, idx))
            for k in ("Tmoor_std", "Tmoor_PSD", "Tmoor_max", "Tmoor_min"):
                assert m[k].shape == z["fowt0_" + k][ic].shape and _rel(m[k], z["fowt0_" + k][ic]) < RTOL, (ic, k)
            assert np.array_equal(m["Tmoor_avg"], z["fowt0_Tmoor_avg"][ic])


@gpu
@pytest.mark.parametrize("name", ["farm", "farm24"])
def test_array_tensions_vs_reference(name):
    """The array level of analyzeCases (raft_model.py:371-433): J_arr on the reference's coupled Xi, shared-memory tiles
    for the two-FOWT farm and for farm24's 144 DOFs."""
    from raft_b200 import solver
    z = _fixture(name)
    w0 = float(z["w"][0])
    nC = z["arr_Tmoor_std"].shape[0]
    for ic in range(nC):
        Xi = z["Xi_c%d" % ic]
        sd, ps, _ = solver.farm_channel_stats(z["J_arr"], Xi, w0)
        m = solver.tension_metrics(z["T0_arr"], *solver.combine_trains(sd, ps, np.arange(len(Xi))))
        for k in ("Tmoor_std", "Tmoor_PSD", "Tmoor_max", "Tmoor_min", "Tmoor_avg"):
            assert m[k].shape == z["arr_" + k][ic].shape and _rel(m[k], z["arr_" + k][ic]) < RTOL, (ic, k)


@gpu
def test_flexible_fowt_tensions_vs_reference():
    """VolturnUS-S-flexible (150 DOFs): J applied to the reference's Xi_PRP, the motions its saveTurbineOutputs multiplies."""
    from raft_b200 import solver
    z = _fixture("VolturnUS-S-flexible")
    w0 = float(z["w"][0])
    for ic in range(z["fowt0_Tmoor_std"].shape[0]):
        X = z["Xi_PRP"][ic]
        sd, ps, _ = solver.farm_channel_stats(z["J0"], X, w0)
        m = solver.tension_metrics(z["T00"], *solver.combine_trains(sd, ps, np.arange(len(X))))
        for k in ("Tmoor_std", "Tmoor_PSD"):
            assert _rel(m[k], z["fowt0_" + k][ic]) < RTOL, (ic, k)


def _random_problem(rng, F, nR, N, nw, nch, per_farm):
    n = 6 * N
    Xi = rng.normal(size=(F, nR, n, nw)) + 1j * rng.normal(size=(F, nR, n, nw))
    R = rng.normal(size=((F,) if per_farm else ()) + (nch, n))
    wpow = rng.integers(0, 3, nch).astype(np.int32)
    w = np.linspace(0.03, 1.2, nw)
    return Xi, R, wpow, w


def _assert_same_as_general(Xi, R, wpow, w, dw, tile_w=0):
    from raft_b200 import solver
    F = Xi.shape[0]
    sd, ps, A = solver.farm_channel_stats(R, Xi, dw, w=w, wpow=wpow, psd=True, amp=True, tile_w=tile_w)
    for f in range(F):
        Rf = R[f] if R.ndim == 3 else R
        s1, p1, a1 = solver.general_channel_stats(Rf, wpow, w, Xi[f], dw, psd=True, amp=True)
        assert np.array_equal(sd[f], s1) and np.array_equal(ps[f], p1) and np.array_equal(A[f], a1), (f, tile_w)
    return sd, ps, A


@gpu
@pytest.mark.parametrize("N,nw", [(2, 64), (24, 40), (64, 24)])
def test_bit_identical_to_general_channel_stats(N, nw):
    """12N channels (wpow 0, 1, 2 mixed) over 2 farms x 2 rows, per-farm R: every std, PSD and amplitude equals
    k_general_channel_stats' on the same R and Xi, bit for bit."""
    rng = np.random.default_rng(N)
    Xi, R, wpow, w = _random_problem(rng, 2, 2, N, nw, 12 * N, per_farm=True)
    _assert_same_as_general(Xi, R, wpow, w, 0.037)


@gpu
@pytest.mark.parametrize("per_farm", [False, True])
def test_farm_in_a_batch_equals_farm_alone(per_farm):
    from raft_b200 import solver
    rng = np.random.default_rng(7 + per_farm)
    Xi, R, wpow, w = _random_problem(rng, 5, 3, 3, 50, 20, per_farm)
    sd, ps, A = solver.farm_channel_stats(R, Xi, 0.05, w=w, wpow=wpow, amp=True)
    for f in range(5):
        s1, p1, a1 = solver.farm_channel_stats(R[f] if per_farm else R, Xi[f], 0.05, w=w, wpow=wpow, amp=True)
        assert np.array_equal(sd[f], s1) and np.array_equal(ps[f], p1) and np.array_equal(A[f], a1), f
    # psd=None routes |Y|^2 through the workspace: the same std
    s0, p0, _ = solver.farm_channel_stats(R, Xi, 0.05, w=w, wpow=wpow, psd=False)
    assert p0 is None and np.array_equal(s0, sd)


@gpu
@pytest.mark.parametrize("nw,nch,tile_w", [
    (1, 9, 0), (37, 9, 8), (37, 9, 5), (64, 1, 0), (33, 300, 0), (33, 300, 7), (45, 20, -1), (1, 300, -1), (129, 3, 1)])
def test_tile_edges(nw, nch, tile_w):
    """One bin; bins not a multiple of the tile; one channel; more channels than the CTA's 256 threads; Xi_sys from L2."""
    rng = np.random.default_rng(nw * 1000 + nch)
    Xi, R, wpow, w = _random_problem(rng, 2, 2, 2, nw, nch, per_farm=True)
    _assert_same_as_general(Xi, R, wpow, w, 0.02, tile_w=tile_w)


@gpu
def test_amplitudes_are_R_times_Xi():
    from raft_b200 import solver
    rng = np.random.default_rng(11)
    Xi, R, wpow, w = _random_problem(rng, 2, 3, 4, 30, 17, per_farm=True)
    _, _, A = solver.farm_channel_stats(R, Xi, 0.1, w=w, wpow=wpow, amp=True)
    want = np.einsum("fcb,frbw->frcw", R, Xi) * (w[None, None, None, :] ** wpow[None, None, :, None])
    assert _rel(A, want) < 1e-13


@gpu
def test_session_path_equals_host_path():
    """DeviceSession.farm_channel_stats on the resident Xi_sys of farm_response(n_fowt=2), per-farm J, against the host path
    on the same Xi_sys copied back: bit for bit."""
    import torch
    from raft_b200 import solver
    zf = np.load(os.path.join(GOLDEN, "farm_VolturnUS-S_farm_nw48.npz"))
    packs = [{k[3:]: zf[k] for k in zf.files if k.startswith("P%d_" % i)} for i in range(int(zf["n_fowt"]))]
    rows = zf["cases"]
    cs = dict(Hs=rows[:, 0], Tp=rows[:, 1], gamma=np.zeros(len(rows)), beta_deg=rows[:, 2], spec=np.zeros(len(rows), dtype=np.int32))
    F = 3
    batch = solver.DesignBatch(packs * F)
    S = solver.DeviceSession(batch, solver.CaseTable(cs), want=("Xi", "status", "B_drag", "F_drag", "F_iner", "F_BEM"))
    S.solve(n_iter=int(zf["n_iter"]), xi_start=float(zf["xi_start"]))
    xi, info = S.farm_response(C_arr=zf["C_array"], n_fowt=2)
    rng = np.random.default_rng(3)
    J = rng.normal(size=(F, 10, 12)) * 1e4
    w0 = float(packs[0]["w"][0])
    sd, ps, A = S.farm_channel_stats(J, w0, psd=True, amp=True, n_fowt=2)
    torch.cuda.synchronize()
    Xh = xi.cpu().numpy()
    s1, p1, a1 = solver.farm_channel_stats(J, Xh, w0, amp=True)
    assert np.array_equal(sd.cpu().numpy(), s1) and np.array_equal(ps.cpu().numpy(), p1) and np.array_equal(A.cpu().numpy(), a1)
    # the single-farm form of the session
    S1 = solver.DeviceSession(solver.DesignBatch(packs), solver.CaseTable(cs), want=("Xi", "status", "B_drag", "F_drag", "F_iner", "F_BEM"))
    S1.solve(n_iter=int(zf["n_iter"]), xi_start=float(zf["xi_start"]))
    x1, _ = S1.farm_response(C_arr=zf["C_array"])
    sd1, ps1, _ = S1.farm_channel_stats(J[0], w0)
    torch.cuda.synchronize()
    s2, p2, _ = solver.farm_channel_stats(J[0], x1.cpu().numpy(), w0)
    assert sd1.shape == (len(rows), 10) and np.array_equal(sd1.cpu().numpy(), s2) and np.array_equal(ps1.cpu().numpy(), p2)


@gpu
def test_model_analyze_cases_tension_keys_vs_reference():
    """Model.analyzeCases on the two-FOWT farm with the fixture's array and per-FOWT tension Jacobians: the reference's keys
    and shapes ((2L,), [2L, nw]) in case_metrics[iCase]['array_mooring'] and per FOWT, its values, and wave_PSD."""
    from raft_b200.model import Model
    z = _fixture("farm")
    zf = np.load(os.path.join(GOLDEN, "farm_VolturnUS-S_farm_nw48.npz"))
    assert np.array_equal(z["C_array"], zf["C_array"])
    packs = [{k[3:]: zf[k] for k in zf.files if k.startswith("P%d_" % i)} for i in range(2)]
    D = json.load(open(os.path.join(GOLDEN, "designs.json")))["farm_VolturnUS-S_farm_nw48"]
    design = dict(settings=D["settings"], site=D["site"], platform=D["platform"], array=D["array"])
    mats = [dict(M_struc=P["M0"] - zf["A_hydro_morison%d" % i], C_struc=P["C0"] - zf["C_moor%d" % i], C_moor=zf["C_moor%d" % i])
            for i, P in enumerate(packs)]
    rng = np.random.default_rng(9)
    Jf, T0f = rng.normal(size=(6, 6)) * 1e4, rng.uniform(1e6, 2e6, 6)
    model = Model(design, matrices=mats, array_stiffness=z["C_array"], tension_jacobian=[Jf, None], mean_tensions=[T0f, None],
                  array_tension_jacobian=z["J_arr"], array_mean_tensions=z["T0_arr"])
    cases = [dict(wave_spectrum="JONSWAP", wave_height=H, wave_period=T, wave_heading=b) for H, T, b in ((6.0, 12.0, 0.0), (3.5, 9.0, 40.0))]
    res = model.analyzeCases(cases=cases)
    w0 = float(model.w[0])
    for ic in range(2):
        am = res["case_metrics"][ic]["array_mooring"]
        assert sorted(am) == ["Tmoor_PSD", "Tmoor_avg", "Tmoor_max", "Tmoor_min", "Tmoor_std"]
        for k in am:
            assert am[k].shape == z["arr_" + k][ic].shape and _rel(am[k], z["arr_" + k][ic]) < RTOL, (ic, k)
        m0, m1 = res["case_metrics"][ic][0], res["case_metrics"][ic][1]
        assert "Tmoor_std" not in m1 and m0["Tmoor_std"].shape == (6,) and m0["Tmoor_PSD"].shape == (6, model.nw)
        T = np.einsum("ab,hbw->haw", Jf, res["Xi_trains"][ic][:, 0:6])
        assert _rel(m0["Tmoor_std"], np.sqrt(0.5 * (np.abs(T) ** 2).sum(axis=(0, 2)))) < RTOL
        assert _rel(m0["Tmoor_PSD"], (0.5 * np.abs(T) ** 2 / w0).sum(axis=0)) < RTOL
        for i in range(2):
            wp = res["case_metrics"][ic][i]["wave_PSD"]
            assert wp.shape == z["fowt%d_wave_PSD" % i][ic].shape and _rel(wp, z["fowt%d_wave_PSD" % i][ic]) < RTOL, (ic, i)
