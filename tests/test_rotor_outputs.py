"""Rotor speed, generator torque and blade pitch statistics (raftk_rotor_stats_*, solver.rotor_stats, the sessions'
rotor_stats, packer.pack_rotor_outputs, solver.rotor_metrics, Model(rotors=) and general_analyze_cases(rotors=)).
Without a GPU: the struct layout and prototypes against include/raftk.h, every refusal, pack_rotor_outputs on stand-in
rotors (hub rows with the stacked-column quirk, the gate, raw torque gains, means) and a numpy restatement against the
reference's own saveTurbineOutputs (fixture rotor_VolturnUS-S, tests/golden/make_golden_rotor.py).  On the GPU: the kernel
and the whole solve against that fixture, batch independence, host = device = sessions, farm columns = rigid slices, a
sweep-sized batch against numpy, and the Model / general_analyze_cases entries."""
import ctypes as C
import json
import os
import re
import subprocess
from types import SimpleNamespace as NS

import numpy as np
import pytest

from conftest import GOLDEN, ROOT

HEADER = os.path.join(ROOT, "include", "raftk.h")
NEW = ("raftk_rotor_stats_dev", "raftk_rotor_stats_host")
RTOL = 1e-10
RPM, DEG = 1 / 0.1047, 57.29577951308232
gpu = pytest.mark.gpu


def _fixture(name):
    return np.load(os.path.join(GOLDEN, "rotor_%s.npz" % name))


def _rel(a, b):
    a, b = np.asarray(a, dtype=float), np.asarray(b, dtype=float)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


def np_rotor_stats(R, C_, V_w, gains, w, Xi, dw, case_row0, col0):
    """Numpy restatement of raft_fowt.py:2643-2675 on Xi [nU, nRows, n, nw], per-unit or shared tables."""
    nU, _, _, nw = Xi.shape
    nrot, n_r = R.shape[-2:]
    nC = len(case_row0) - 1
    R = np.broadcast_to(R, (nU, nrot, n_r))
    C_, V_w, gains = (np.broadcast_to(a, (nU,) + a.shape[-3:]) for a in (C_, V_w, gains))
    sd, P = np.zeros([nU, nC, nrot, 3]), np.zeros([nU, nC, nrot, 3, nw])
    for u in range(nU):
        for c in range(nC):
            for k in range(nrot):
                hub = np.einsum("b,hbw->hw", R[u, k], Xi[u, case_row0[c]:case_row0[c + 1], col0[k]:col0[k] + n_r])
                phi = np.vstack([C_[u, c, k] * hub, C_[u, c, k] * (0 - V_w[u, c, k] / (1j * w))])
                kp_t, ki_t, kp_b, ki_b = gains[u, c, k]
                for j, (ch, s) in enumerate(((1j * w * phi, RPM), ((1j * w * kp_t + ki_t) * phi, 1.0), ((1j * w * kp_b + ki_b) * phi, DEG))):
                    sd[u, c, k, j] = np.sqrt(0.5 * np.sum(np.abs(ch) ** 2)) * s
                    P[u, c, k, j] = s ** 2 * np.sum(0.5 * np.abs(ch) ** 2 / dw, axis=0)
    return sd, P


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
        want = C.POINTER(_lib.RaftkRotorOutputs) if "raftk_rotor_outputs" in decl else (C.c_void_p if "*" in decl else C.c_int32)
        assert ct is want, (name, decl, ct)
    assert fn.restype is C.c_int and ret == "int"


def test_struct_layout_matches_header(tmp_path):
    from raft_b200 import _lib
    S = _lib.RaftkRotorOutputs
    fields = [n for n, _ in S._fields_]
    src = tmp_path / "t.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "raftk.h"\nint main(void){printf("%%zu %s\\n", sizeof(raftk_rotor_outputs), %s);'
                   'return 0;}\n' % (" ".join(["%zu"] * len(fields)), ", ".join("offsetof(raftk_rotor_outputs, %s)" % n for n in fields)))
    exe = tmp_path / "t"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert got == [C.sizeof(S)] + [getattr(S, n).offset for n in fields]


def _outputs(n_cases=2, n_rot=3, n_r=6):
    from raft_b200 import _lib
    ro = _lib.RaftkRotorOutputs()
    ro.n_cases, ro.n_rot, ro.n_r, ro.R_shared, ro.tf_shared = n_cases, n_rot, n_r, 1, 1
    col0 = np.array([0, 6, 12][:n_rot] + [0] * max(0, n_rot - 3), dtype=np.int32)
    row0 = np.array([0, 2, 3], dtype=np.int32)
    ro.col0, ro.case_row0 = col0.ctypes.data, row0.ctypes.data
    ro.R = ro.C = ro.V_w = ro.gains = ro.std = ro.psd = 0x1000
    ro.dw = 0.1
    return ro, col0, row0


@pytest.mark.parametrize("case,msg", [
    ("n_units", ">= 1"), ("n_rows", ">= 1"), ("n_dof", ">= 1"), ("nw", ">= 1"), ("n_cases", ">= 1"), ("n_rot", ">= 1"),
    ("n_r", ">= 1"), ("n_r_big", "n_r must be"), ("col0_neg", "col0"), ("col0_end", "col0"), ("row0_start", "start at 0"),
    ("row0_end", "end at n_rows"), ("row0_empty", "at least one row"), ("row0_decreasing", "at least one row"),
    ("R_shared", "R_shared"), ("tf_shared", "tf_shared"), ("w", "are required"), ("Xi", "are required"), ("R", "are required"),
    ("C", "are required"), ("V_w", "are required"), ("gains", "are required"), ("std", "are required"), ("dw", "dw must be"),
    ("null", "null argument"),
])
def test_refusals_before_any_launch(case, msg):
    from raft_b200._lib import lib
    dims = dict(n_units=2, n_rows=3, n_dof=18, nw=16)
    ro, col0, row0 = _outputs()
    w = xi = 0x1000
    if case in dims:
        dims[case] = 0
    elif case in ("n_cases", "n_rot", "n_r"):
        setattr(ro, case, 0)
    elif case == "n_r_big":
        ro.n_r = 19
    elif case == "col0_neg":
        col0[1] = -1
    elif case == "col0_end":
        col0[2] = 13
    elif case == "row0_start":
        row0[0] = 1
    elif case == "row0_end":
        row0[2] = 4
    elif case == "row0_empty":
        row0[1] = 0
    elif case == "row0_decreasing":
        row0[:] = [0, 3, 3]
    elif case in ("R_shared", "tf_shared"):
        setattr(ro, case, 2)
    elif case == "w":
        w = None
    elif case == "Xi":
        xi = None
    elif case in ("R", "C", "V_w", "gains", "std"):
        setattr(ro, case, None)
    elif case == "dw":
        ro.dw = 0.0
    ref = None if case == "null" else C.byref(ro)
    before = lib.raftk_launch_count()
    args = (dims["n_units"], dims["n_rows"], dims["n_dof"], dims["nw"], w, xi, ref)
    assert lib.raftk_rotor_stats_host(*args) == -1 and msg in lib.raftk_last_error().decode(), lib.raftk_last_error()
    assert lib.raftk_rotor_stats_dev(*args, None) == -1 and msg in lib.raftk_last_error().decode()
    assert lib.raftk_launch_count() == before


def test_host_refuses_a_nonpositive_frequency():
    """The wind row divides by w: a bin at w <= 0 has no finite value, so the host entry refuses it before any launch."""
    from raft_b200 import solver
    from raft_b200._lib import lib
    w = np.linspace(0.0, 1.0, 8)
    Xi, C_, g = np.zeros([1, 2, 6, 8], dtype=complex), np.zeros([1, 1, 8], dtype=complex), np.zeros([1, 1, 4])
    before = lib.raftk_launch_count()
    with pytest.raises(Exception, match="w must be > 0"):
        solver.rotor_stats(np.zeros([1, 6]), C_, C_, g, w, Xi, 0.1, case_row0=[0, 2])
    assert lib.raftk_launch_count() == before


def test_python_refusals():
    from raft_b200 import solver
    Xi = np.zeros([2, 3, 12, 8], dtype=complex)
    C_, g = np.zeros([3, 2, 8], dtype=complex), np.zeros([3, 2, 4])
    with pytest.raises(ValueError):
        solver.rotor_stats(np.zeros([3, 2, 6]), C_, C_, g, np.ones(8), Xi, 0.1)                 # three units' R for two units
    with pytest.raises(ValueError):
        solver.rotor_stats(np.zeros([2, 6]), C_[..., :7], C_[..., :7], g, np.ones(8), Xi, 0.1)  # C on another grid
    with pytest.raises(ValueError):
        solver.rotor_stats(np.zeros([2, 6]), C_, C_, g[..., :3], np.ones(8), Xi, 0.1)
    with pytest.raises(ValueError):
        solver.rotor_stats(np.zeros([2, 6]), C_, C_, g, np.ones(8), Xi, 0.1, case_row0=[0, 3])  # three cases, one bound


def _stand_in_fowt(nrot, nDOF=6, seed=0):
    rng = np.random.default_rng(seed)
    nodes = [NS(id=3 + 2 * i) for i in range(nrot)]
    rotors = [NS(nodeList=[nodes[i]], r3=np.array([0.0, 0.0, 150.0]), aeroServoMod=2) for i in range(nrot)]
    return NS(rotorList=rotors, T=rng.normal(size=(6 * (3 + 2 * nrot), nDOF)), w=np.linspace(0.05, 1.0, 8)), rng


def _state(rng, nw, **kw):
    s = dict(C=rng.normal(size=nw) + 1j * rng.normal(size=nw), V_w=rng.normal(size=nw) + 0j, kp_tau=-3.0e7, ki_tau=-4.0e6,
             kp_beta=-0.01, ki_beta=-0.002, Omega_case=6.5, aero_torque=2.0e7, Ng=1.0, aero_power=1.2e7, pitch_case=3.0,
             aeroServoMod=2, r3=np.array([0.0, 0.0, 150.0]))
    s.update(kw)
    return s


def test_pack_rotor_outputs_hub_rows_keep_the_stacked_column_quirk():
    """Rotor ir's row is DOF ir % 6 of rotor ir // 6's hub (XiHub[ih, ir, :], raft_fowt.py:2402, 2423, 2644)."""
    from raft_b200 import packer
    fowt, rng = _stand_in_fowt(8, nDOF=20)
    st = [[_state(rng, 8) for _ in range(8)]]
    p = packer.pack_rotor_outputs(fowt, st, [dict(wind_speed=11.0)])
    for ir in range(8):
        hub = fowt.rotorList[ir // 6].nodeList[0].id
        assert np.array_equal(p["R"][ir], fowt.T[6 * hub + ir % 6]), ir
    assert p["R"].shape == (8, 20) and p["C"].shape == (1, 8, 8) and p["gains"].shape == (1, 8, 4)
    assert np.array_equal(p["R"][1], fowt.T[6 * 3 + 1])                        # the second rotor reads the FIRST hub's sway


def test_pack_rotor_outputs_gate_gains_and_means():
    from raft_b200 import packer
    fowt, rng = _stand_in_fowt(2)
    cases = [dict(wind_speed=11.0), dict(wind_speed=0.0), dict(wind_speed=11.0, current_speed=0.0), dict(wind_speed=9.0), {}]
    st = [[_state(rng, 8, Ng=97.0), _state(rng, 8)] for _ in cases]                # torque_avg = aero_torque / Ng
    st[2][1]["r3"] = np.array([0.0, 0.0, -20.0])                              # underwater rotor: current_speed 0 -> off
    st[3][0]["aeroServoMod"] = 1                                              # no control -> off
    st[3][1]["kp_beta"] = 0.0                                                 # calcAero's gated kp_tau would then differ
    p = packer.pack_rotor_outputs(fowt, st, cases)
    assert p["active"].tolist() == [[True, True], [False, False], [True, False], [False, True], [True, True]]
    for c in range(len(cases)):
        for k in range(2):
            if not p["active"][c, k]:
                assert not p["C"][c, k].any() and not p["V_w"][c, k].any() and not p["gains"][c, k].any()
                assert p["omega_avg"][c, k] == p["torque_avg"][c, k] == p["power_avg"][c, k] == p["bPitch_avg"][c, k] == 0.0
            else:
                s = st[c][k]
                assert np.array_equal(p["C"][c, k], s["C"]) and np.array_equal(p["V_w"][c, k], s["V_w"])
                assert p["gains"][c, k].tolist() == [s["kp_tau"], s["ki_tau"], s["kp_beta"], s["ki_beta"]]   # raw kp_tau / ki_tau
                assert p["omega_avg"][c, k] == s["Omega_case"] and p["torque_avg"][c, k] == s["aero_torque"] / s["Ng"]
                assert p["power_avg"][c, k] == s["aero_power"] and p["bPitch_avg"][c, k] == s["pitch_case"]
    assert p["wind"][1] is None and np.array_equal(p["wind"][3], st[3][1]["V_w"]) and np.array_equal(p["wind"][0], st[0][1]["V_w"])
    assert np.array_equal(p["wind"][2], st[2][0]["V_w"])
    st[0][0] = dict(st[0][0], C=None)
    with pytest.raises(NotImplementedError):
        packer.pack_rotor_outputs(fowt, st, cases)
    obj = [[NS(**_state(rng, 8)), NS(**_state(rng, 8))]]                     # rotor objects work like dicts
    assert packer.pack_rotor_outputs(fowt, obj, cases[:1])["active"].all()


FIXTURES = ("VolturnUS-S", "farm", "farm24", "VolturnUS-S-flexible")


def _fixture_rotors(z, i):
    """pack_rotor_outputs of FOWT i of a fixture: its hub rows (fowt.T at each rotor's hub node) and stand-in states."""
    from raft_b200 import packer
    hubT = z["hubT%d" % i]
    nrot = hubT.shape[0]
    fowt = NS(rotorList=[NS(nodeList=[NS(id=k)], r3=np.array([0.0, 0.0, 150.0]), aeroServoMod=2) for k in range(nrot)],
              T=hubT.reshape(6 * nrot, -1), w=z["w"])
    states = []
    for c in range(z["in%d_C" % i].shape[0]):
        row = []
        for k in range(nrot):
            kp_t, ki_t, kp_b, ki_b = z["in%d_gains" % i][c, k]
            Om, tq, Ng, pw, pc = z["in%d_means" % i][c, k]
            row.append(dict(C=z["in%d_C" % i][c, k], V_w=z["in%d_V_w" % i][c, k], kp_tau=kp_t, ki_tau=ki_t, kp_beta=kp_b, ki_beta=ki_b,
                            Omega_case=Om, aero_torque=tq, Ng=Ng, aero_power=pw, pitch_case=pc))
        states.append(row)
    return packer.pack_rotor_outputs(fowt, states, json.loads(str(z["cases_json"])))


def _check_metrics(m, z, i, c):
    """The rotor entries of one FOWT and case against the reference's: the same keys (wind_PSD only where it set it), shapes
    and, to 1e-10, values; exact zeros where the reference has them."""
    from raft_b200.packer import ROTOR_KEYS
    keys = [k for k in ROTOR_KEYS + ("wind_PSD",) if "fowt%d_%s_c%d" % (i, k, c) in z.files]
    assert sorted(k for k in m if k in ROTOR_KEYS + ("wind_PSD",)) == sorted(keys), (i, c, sorted(m), keys)
    for k in keys:
        ref = z["fowt%d_%s_c%d" % (i, k, c)]
        assert np.shape(m[k]) == ref.shape, (i, c, k)
        assert _rel(m[k], ref) < RTOL if np.abs(ref).max() > 0 else not np.any(m[k]), (i, c, k)


def _case_rows(z):
    """The trains of every case in the reference's Model.Xi (its last row is the zero row) -> (Xi [nT, n, nw], case_row0)."""
    nC = len(json.loads(str(z["cases_json"])))
    trains = [z["Xi_c%d" % c][:-1] for c in range(nC)]
    return np.concatenate(trains), np.cumsum([0] + [len(t) for t in trains])


@pytest.mark.parametrize("name", FIXTURES)
def test_numpy_restatement_and_metrics_vs_reference(name):
    """The restatement the GPU tests compare against, with pack_rotor_outputs' hub rows and rotor_metrics' keys, equals the
    reference's saveTurbineOutputs for every FOWT and case: keys, shapes, zeros and no wind_PSD with the gate off."""
    from raft_b200 import solver
    z = _fixture(name)
    w = z["w"]
    dw = w[1] - w[0]
    Xi, row0 = _case_rows(z)
    for i in range(int(z["n_fowt"])):
        p = _fixture_rotors(z, i)
        n_r = p["R"].shape[1]
        for c in range(len(row0) - 1):
            sd, P = np_rotor_stats(p["R"], p["C"][c:c + 1], p["V_w"][c:c + 1], p["gains"][c:c + 1], w, Xi[None, row0[c]:row0[c + 1]], dw,
                                   [0, row0[c + 1] - row0[c]], [6 * i if n_r == 6 else 0] * len(p["R"]))
            _check_metrics(solver.rotor_metrics(p, c, sd[0, 0], P[0, 0], dw), z, i, c)


# ---- on the GPU -----------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("name", FIXTURES)
def test_kernel_on_reference_xi_vs_reference(name):
    """One rotor_stats call per fixture on the reference's Xi, every FOWT's rotors at col0 = 6 i (0 for generalised DOFs)."""
    from raft_b200 import solver
    z = _fixture(name)
    w = z["w"]
    dw = w[1] - w[0]
    Xi, row0 = _case_rows(z)
    packs = [_fixture_rotors(z, i) for i in range(int(z["n_fowt"]))]
    cat = lambda k, ax: np.concatenate([p[k] for p in packs], axis=ax)                        # noqa: E731
    col0 = np.concatenate([np.full(len(p["R"]), 6 * i if p["R"].shape[1] == 6 else 0) for i, p in enumerate(packs)])
    sd, P = solver.rotor_stats(cat("R", 0), cat("C", 1), cat("V_w", 1), cat("gains", 1), w, Xi, dw, case_row0=row0, col0=col0)
    k0 = 0
    for i, p in enumerate(packs):
        k = slice(k0, k0 + len(p["R"]))
        k0 = k.stop
        for c in range(len(row0) - 1):
            _check_metrics(solver.rotor_metrics(p, c, sd[c, k], P[c, k], dw), z, i, c)


@gpu
@pytest.mark.parametrize("name", ["VolturnUS-S", "farm", "farm24"])
def test_model_analyze_cases_vs_reference(name):
    """Model(rotors=).analyzeCases end to end -- the project's own solve of the reference's design and cases (coupled
    through the array stiffness for farms), then its rotor entries -- against the reference's analyzeCases to 1e-10."""
    from raft_b200.model import Model
    z = _fixture(name)
    nF = int(z["n_fowt"])
    mats = [{k[len("mat%d_" % i):]: z[k] for k in z.files if k.startswith("mat%d_" % i)} for i in range(nF)]
    model = Model(json.loads(str(z["design_json"])), matrices=mats if nF > 1 else mats[0], array_stiffness=z["C_array"] if "C_array" in z.files else None,
                  rotors=[_fixture_rotors(z, i) for i in range(nF)])
    assert np.allclose(model.w, z["w"], rtol=1e-15, atol=0)
    cases = json.loads(str(z["cases_json"]))
    res = model.analyzeCases(cases=cases)
    for c in range(len(cases)):
        for i in range(nF):
            _check_metrics(res["case_metrics"][c][i], z, i, c)


@gpu
def test_general_analyze_cases_vs_reference():
    """general_analyze_cases(rotors=) and general_analyze_cases_batch(rotors=) on VolturnUS-S-flexible (150 DOFs): the
    project's generalised-DOF solve and rotor entries against the reference's solveDynamics and saveTurbineOutputs."""
    from raft_b200 import solver
    z = _fixture("VolturnUS-S-flexible")
    P = {k[2:]: z[k] for k in z.files if k.startswith("P_")}
    cases = json.loads(str(z["cases_json"]))
    rot = _fixture_rotors(z, 0)
    res = solver.general_analyze_cases(P, z["gen_M"], z["gen_B"], z["gen_C"], cases, n_iter=int(z["n_iter"]), xi_start=float(z["xi_start"]),
                                       rotors=rot)
    rb = solver.general_analyze_cases_batch([dict(P=P, M=z["gen_M"], B=z["gen_B"], Cm=z["gen_C"])] * 2, cases, n_iter=int(z["n_iter"]),
                                            xi_start=float(z["xi_start"]), rotors=[rot, rot])
    for c in range(len(cases)):
        _check_metrics(res["case_metrics"][c], z, 0, c)
        for d in range(2):
            _check_metrics(rb[d]["case_metrics"][c], z, 0, c)


def _random(rng, nU, nR, n, nw, nC, nrot, n_r, per_unit=False):
    w = np.linspace(0.02, 2.0, nw)
    Xi = rng.normal(size=(nU, nR, n, nw)) + 1j * rng.normal(size=(nU, nR, n, nw))
    lead = (nU,) if per_unit else ()
    R = rng.normal(size=lead + (nrot, n_r))
    C_ = (rng.normal(size=lead + (nC, nrot, nw)) + 1j * rng.normal(size=lead + (nC, nrot, nw))) * 0.1
    V_w = rng.normal(size=lead + (nC, nrot, nw)) + 1j * rng.normal(size=lead + (nC, nrot, nw))
    g = rng.normal(size=lead + (nC, nrot, 4)) * np.array([3e7, 4e6, 0.01, 0.002])
    cuts = np.sort(rng.choice(np.arange(1, nR), nC - 1, replace=False)) if nC > 1 else np.zeros(0, dtype=int)
    return w, Xi, R, C_, V_w, g, np.concatenate([[0], cuts, [nR]]).astype(np.int32)


@gpu
def test_batch_composition_does_not_change_a_result():
    from raft_b200 import solver
    rng = np.random.default_rng(5)
    nU, nR, n, nw, nC, nrot = 5, 9, 24, 300, 4, 3
    w, Xi, R, C_, V_w, g, row0 = _random(rng, nU, nR, n, nw, nC, nrot, 6)
    col0 = np.array([0, 6, 18], dtype=np.int32)
    dw = w[1] - w[0]
    sd, P = solver.rotor_stats(R, C_, V_w, g, w, Xi, dw, case_row0=row0, col0=col0)
    s1, p1 = solver.rotor_stats(R, C_, V_w, g, w, Xi[3:4], dw, case_row0=row0, col0=col0)        # one unit
    assert np.array_equal(s1[0], sd[3]) and np.array_equal(p1[0], P[3])
    order = [2, 0, 3, 1]                                                                           # cases reordered in blocks
    Xo = np.concatenate([Xi[:, row0[c]:row0[c + 1]] for c in order], axis=1)
    ro = np.cumsum([0] + [row0[c + 1] - row0[c] for c in order])
    s2, p2 = solver.rotor_stats(R, C_[order], V_w[order], g[order], w, Xo, dw, case_row0=ro, col0=col0)
    assert np.array_equal(s2, sd[:, order]) and np.array_equal(p2, P[:, order])
    Ra = np.concatenate([R, rng.normal(size=(2, 6))])                                              # rotors added
    ext = lambda a: np.concatenate([a, a[:, :2] * 1.5], axis=1)                                    # noqa: E731
    s3, p3 = solver.rotor_stats(Ra, ext(C_), ext(V_w), ext(g), w, Xi, dw, case_row0=row0, col0=np.append(col0, [12, 3]))
    assert np.array_equal(s3[:, :, :3], sd) and np.array_equal(p3[:, :, :3], P)
    s4, p4 = solver.rotor_stats(R, C_, V_w, g, w, Xi, dw, case_row0=row0, col0=col0, psd=False)
    assert p4 is None and np.array_equal(s4, sd)


@gpu
def test_more_cases_and_rotors_than_one_launch_holds():
    """Over 256 cases or rotors the call is split into several launches; every result is that of a small call."""
    from raft_b200 import solver
    rng = np.random.default_rng(8)
    w, Xi, R, C_, V_w, g, row0 = _random(rng, 2, 300, 6, 40, 300, 260, 6)
    dw = w[1] - w[0]
    sd, P = solver.rotor_stats(R, C_, V_w, g, w, Xi, dw, case_row0=row0)
    for c, k in ((0, 0), (299, 259), (257, 3), (17, 258)):
        s1, p1 = solver.rotor_stats(R[k:k + 1], C_[c:c + 1, k:k + 1], V_w[c:c + 1, k:k + 1], g[c:c + 1, k:k + 1], w,
                                    Xi[:, row0[c]:row0[c + 1]], dw)
        assert np.array_equal(s1[:, 0, 0], sd[:, c, k]) and np.array_equal(p1[:, 0, 0], P[:, c, k])


@gpu
def test_gate_off_gives_exact_zeros():
    from raft_b200 import solver
    rng = np.random.default_rng(2)
    w, Xi, R, C_, V_w, g, row0 = _random(rng, 2, 4, 6, 64, 2, 2, 6)
    C_[1, 0], V_w[1, 0] = 0, 0
    sd, P = solver.rotor_stats(R, C_, V_w, g, w, Xi, w[1] - w[0], case_row0=row0)
    assert not sd[:, 1, 0].any() and not P[:, 1, 0].any() and sd[:, 1, 1].all()


@gpu
@pytest.mark.parametrize("per_unit", [False, True])
def test_sweep_sized_batch_vs_numpy(per_unit):
    from raft_b200 import solver
    rng = np.random.default_rng(11 + per_unit)
    nU = 40 if per_unit else 200
    w, Xi, R, C_, V_w, g, row0 = _random(rng, nU, 8, 6, 256, 3, 1, 6, per_unit=per_unit)
    dw = w[1] - w[0]
    sd, P = solver.rotor_stats(R, C_, V_w, g, w, Xi, dw, case_row0=row0)
    sn, pn = np_rotor_stats(R, C_, V_w, g, w, Xi, dw, row0, [0])
    assert (np.abs(sd - sn) <= 1e-12 * np.abs(sn)).all()
    assert (np.abs(P - pn) <= 1e-12 * np.abs(pn) + 1e-300).all()


@gpu
def test_host_equals_dev_and_farm_columns_equal_rigid_slices():
    import torch
    from raft_b200 import solver
    rng = np.random.default_rng(13)
    F, nR, N, nw = 3, 5, 4, 200
    w, Xi, _, C_, V_w, g, row0 = _random(rng, F, nR, 6 * N, nw, 2, N, 6)
    R = rng.normal(size=(N, 6))
    col0 = 6 * np.arange(N, dtype=np.int32)
    dw = w[1] - w[0]
    sd, P = solver.rotor_stats(R, C_, V_w, g, w, Xi, dw, case_row0=row0, col0=col0)
    dev = torch.device("cuda", 0)
    sdd, Pd = solver._rotor_stats(solver._Device(dev), R, C_, V_w, g, torch.from_numpy(w).to(dev), torch.from_numpy(Xi).to(dev), dw,
                                  row0, col0, True)
    torch.cuda.synchronize()
    assert np.array_equal(sdd.cpu().numpy(), sd) and np.array_equal(Pd.cpu().numpy(), P)
    for i in range(N):
        s1, p1 = solver.rotor_stats(R[i:i + 1], C_[:, i:i + 1], V_w[:, i:i + 1], g[:, i:i + 1], w, Xi[:, :, 6 * i:6 * i + 6], dw, case_row0=row0)
        assert np.array_equal(s1[:, :, 0], sd[:, :, i]) and np.array_equal(p1[:, :, 0], P[:, :, i])


def _farm_session():
    from raft_b200 import solver
    zf = np.load(os.path.join(GOLDEN, "farm_VolturnUS-S_farm_nw48.npz"))
    packs = [{k[3:]: zf[k] for k in zf.files if k.startswith("P%d_" % i)} for i in range(int(zf["n_fowt"]))]
    cf = zf["cases"]
    cs = dict(Hs=cf[:, 0], Tp=cf[:, 1], gamma=np.zeros(len(cf)), beta_deg=cf[:, 2], spec=np.zeros(len(cf), dtype=np.int32))
    S = solver.DeviceSession(solver.DesignBatch(packs + packs), solver.CaseTable(cs),
                             want=("Xi", "status", "B_drag", "F_drag", "F_iner", "F_BEM"))
    S.solve(n_iter=int(zf["n_iter"]), xi_start=float(zf["xi_start"]))
    return S, zf, len(cf)


@gpu
def test_device_session_equals_host_path():
    import torch
    from raft_b200 import solver
    S, zf, nRows = _farm_session()
    rng = np.random.default_rng(17)
    nw = S.batch.nw
    w = S.batch.w
    dw = w[1] - w[0]
    row0 = np.array([0, 1, nRows], dtype=np.int32) if nRows > 1 else np.array([0, 1], dtype=np.int32)
    nC = len(row0) - 1
    R = rng.normal(size=(2, 6))
    C_ = rng.normal(size=(nC, 2, nw)) + 1j * rng.normal(size=(nC, 2, nw))
    V_w = rng.normal(size=(nC, 2, nw)) + 0j
    g = rng.normal(size=(nC, 2, 4))
    sd, P = S.rotor_stats(R, C_, V_w, g, dw, case_row0=row0)                                       # rigid Xi, one unit per design
    torch.cuda.synchronize()
    s1, p1 = solver.rotor_stats(R, C_, V_w, g, w, S.out["Xi"].cpu().numpy(), dw, case_row0=row0)
    assert np.array_equal(sd.cpu().numpy(), s1) and np.array_equal(P.cpu().numpy(), p1)
    xi, _ = S.farm_response(C_arr=zf["C_array"], n_fowt=2)                                         # two farms of two FOWTs
    sd, P = S.rotor_stats(R, C_, V_w, g, dw, case_row0=row0, col0=[0, 6], farm=True, n_fowt=2)
    torch.cuda.synchronize()
    s2, p2 = solver.rotor_stats(R, C_, V_w, g, w, xi.cpu().numpy(), dw, case_row0=row0, col0=[0, 6])
    assert np.array_equal(sd.cpu().numpy(), s2) and np.array_equal(P.cpu().numpy(), p2)


@gpu
def test_general_sessions_equal_host_path():
    import torch
    from conftest import load_golden
    from raft_b200 import solver
    z, P = load_golden("flex_VolturnUS-S-flexible")
    n, nw = z["gen_M"].shape[0], len(P["w"])
    cases = solver.CaseTable(dict(Hs=[6.0, 3.0, 2.0], Tp=[12.0, 9.0, 7.0], gamma=[0.0] * 3, beta_deg=[0.0, 30.0, -60.0],
                                  spec=np.zeros(3, dtype=np.int32), primary=np.array([0, 0, 2], dtype=np.int32)))
    rng = np.random.default_rng(21)
    row0 = np.array([0, 2, 3], dtype=np.int32)
    R = rng.normal(size=(2, n)) * 0.1
    C_ = rng.normal(size=(2, 2, nw)) + 1j * rng.normal(size=(2, 2, nw))
    V_w = rng.normal(size=(2, 2, nw)) + 0j
    g = rng.normal(size=(2, 2, 4))
    w, dw = np.asarray(P["w"], dtype=float), float(P["dw"])
    s = solver.GeneralSession(P, z["gen_M"], z["gen_B"], z["gen_C"], cases)
    s.solve()
    sd, ps = s.rotor_stats(R, C_, V_w, g, case_row0=row0)
    torch.cuda.synchronize()
    s1, p1 = solver.rotor_stats(R, C_, V_w, g, w, s.Xi.cpu().numpy(), dw, case_row0=row0)
    assert np.array_equal(sd.cpu().numpy(), s1) and np.array_equal(ps.cpu().numpy(), p1)
    designs = [dict(P=P, M=z["gen_M"] * (1 + 0.02 * d), B=z["gen_B"], Cm=z["gen_C"]) for d in range(3)]
    b = solver.GeneralBatchSession(designs, cases)
    b.solve()
    Rd = np.stack([R, 1.5 * R, -R])                                                                # per-design hub rows
    sd, ps = b.rotor_stats(Rd, C_, V_w, g, case_row0=row0)
    torch.cuda.synchronize()
    s2, p2 = solver.rotor_stats(Rd, C_, V_w, g, w, b.Xi.cpu().numpy(), dw, case_row0=row0)
    assert np.array_equal(sd.cpu().numpy(), s2) and np.array_equal(ps.cpu().numpy(), p2)
    # general_analyze_cases(_batch) with rotors: the same statistics in the reference's keys
    from raft_b200 import packer
    fowt = NS(rotorList=[NS(nodeList=[NS(id=0)], r3=np.array([0, 0, 150.0]), aeroServoMod=2)], T=np.vstack([R[:1], np.zeros((5, n))]), w=w)
    cl = [dict(wave_height=[6.0, 3.0], wave_period=[12.0, 9.0], wave_heading=[0.0, 30.0], wave_gamma=[0.0, 0.0],
               wave_spectrum=["JONSWAP"] * 2, wind_speed=10.0), dict(wave_height=2.0, wave_period=7.0, wave_heading=-60.0, wind_speed=0.0)]
    st = [[dict(C=C_[c, 0], V_w=V_w[c, 0], kp_tau=g[c, 0, 0], ki_tau=g[c, 0, 1], kp_beta=g[c, 0, 2], ki_beta=g[c, 0, 3], Omega_case=6.0,
                aero_torque=2e7, Ng=1.0, aero_power=1e7, pitch_case=2.0)] for c in range(2)]
    rot = packer.pack_rotor_outputs(fowt, st, cl)
    res = solver.general_analyze_cases(P, z["gen_M"], z["gen_B"], z["gen_C"], cl, rotors=rot)
    Xt = np.concatenate(res["Xi_trains"])
    s3, p3 = solver.rotor_stats(rot["R"], rot["C"], rot["V_w"], rot["gains"], w, Xt, dw, case_row0=[0, 2, 3])
    for c in range(2):
        m = res["case_metrics"][c]
        assert m["omega_std"].shape == (1,) and m["omega_PSD"].shape == (nw, 1) and ("wind_PSD" in m) == (c == 0)
        assert np.array_equal(m["torque_std"], s3[c, :, 1]) and np.array_equal(m["bPitch_PSD"][:, 0], p3[c, 0, 2])
        assert (c == 0) == bool(m["omega_std"][0]) and m["omega_max"][0] == m["omega_avg"][0] + 2 * m["omega_std"][0]
    rb = solver.general_analyze_cases_batch([dict(P=P, M=z["gen_M"], B=z["gen_B"], Cm=z["gen_C"])] * 2, cl, rotors=[rot, rot])
    for d in range(2):
        for c in range(2):
            for k, v in res["case_metrics"][c].items():
                assert np.array_equal(rb[d]["case_metrics"][c][k], v), (d, c, k)


@gpu
def test_model_analyze_cases_rotor_entries():
    """Model.analyzeCases on the coupled two-FOWT farm with rotors on FOWT 1 only: the reference's keys and shapes, and
    FOWT 1's values equal the rigid call on its 6-DOF slice of the coupled response."""
    from raft_b200 import solver
    from raft_b200.model import Model
    from raft_b200.packer import ROTOR_KEYS
    zf = np.load(os.path.join(GOLDEN, "farm_VolturnUS-S_farm_nw48.npz"))
    z = np.load(os.path.join(GOLDEN, "tmoor_farm.npz"))
    packs = [{k[3:]: zf[k] for k in zf.files if k.startswith("P%d_" % i)} for i in range(2)]
    D = json.load(open(os.path.join(GOLDEN, "designs.json")))["farm_VolturnUS-S_farm_nw48"]
    design = dict(settings=D["settings"], site=D["site"], platform=D["platform"], array=D["array"])
    mats = [dict(M_struc=P["M0"] - zf["A_hydro_morison%d" % i], C_struc=P["C0"] - zf["C_moor%d" % i], C_moor=zf["C_moor%d" % i])
            for i, P in enumerate(packs)]
    cases = [dict(wave_spectrum="JONSWAP", wave_height=[6.0, 2.0], wave_period=[12.0, 8.0], wave_heading=[0.0, 50.0], wave_gamma=[0.0, 0.0],
                  wind_speed=10.0), dict(wave_spectrum="JONSWAP", wave_height=3.5, wave_period=9.0, wave_heading=40.0, wind_speed=0.0)]
    nw = len(packs[0]["w"])
    rng = np.random.default_rng(19)
    rot = dict(R=rng.normal(size=(1, 6)), C=rng.normal(size=(2, 1, nw)) + 1j * rng.normal(size=(2, 1, nw)), V_w=rng.normal(size=(2, 1, nw)) + 0j,
               gains=rng.normal(size=(2, 1, 4)), omega_avg=np.array([[6.0], [0.0]]), torque_avg=np.array([[2e7], [0.0]]),
               power_avg=np.array([[1e7], [0.0]]), bPitch_avg=np.array([[3.0], [0.0]]), active=np.array([[True], [False]]))
    rot["C"][1], rot["V_w"][1], rot["gains"][1] = 0, 0, 0
    rot["wind"] = [rot["V_w"][0, 0], None]
    model = Model(design, matrices=mats, array_stiffness=z["C_array"], rotors=[None, rot])
    res = model.analyzeCases(cases=cases)
    dw = model.w[1] - model.w[0]
    for ic in range(2):
        m0, m1 = res["case_metrics"][ic][0], res["case_metrics"][ic][1]
        assert "omega_std" not in m0
        want = set(ROTOR_KEYS) | ({"wind_PSD"} if ic == 0 else set())
        assert want <= set(m1) and ("wind_PSD" in m1) == (ic == 0)
        for k in want:
            assert np.shape(m1[k]) == ((nw,) if k == "wind_PSD" else (nw, 1) if k.endswith("_PSD") else (1,)), k
        X = res["Xi_trains"][ic][None, :, 6:12]
        s1, p1 = solver.rotor_stats(rot["R"], rot["C"][ic:ic + 1], rot["V_w"][ic:ic + 1], rot["gains"][ic:ic + 1], model.w, X, dw,
                                    case_row0=[0, X.shape[1]])
        assert np.array_equal(m1["omega_std"], s1[0, 0, :, 0]) and np.array_equal(m1["torque_PSD"][:, 0], p1[0, 0, 0, 1])
        if ic == 1:
            assert not any(np.any(m1[k]) for k in want)
