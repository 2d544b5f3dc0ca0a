"""Tower-base axial stress around the circumference (raftk_stress_ring_*, solver.stress_ring, stress= of the analyses).

The reference's helpers.getSigmaXPSD (helpers.py:1164): thin-wall section, Izz = pi/8 t d^3, sigma_x(theta) = (TBFA cos theta
- TBSS sin theta) (d/2) / Izz / 1e6 (MPa).  Its return value, getPSD summed over axis 0 of sigmaX [rows * nw, nA], is
std(theta)^2 / dw per angle; the fixture stress_VolturnUS-S-flexible (tests/golden/make_golden_stress.py) pins it on the
reference's own tower-base loads Fi_base[:, 4] (fore-aft) and Fi_base[:, 3] (side-side) of the flexible run.

* Without a GPU: a numpy restatement of the definitions against the reference helper on the fixture; the closed form over
  angles against explicit per-angle rows; the ABI struct layout; every RAFTK_EINVAL of the header; the Python refusals.
* On an H100: std / avg / max / min against the fixture through general_analyze_cases(stress=) and GeneralBatchSession; DELs
  against solver.fatigue on the explicit rows; rigid towers (fore-aft only) through DeviceSession and Model; a farm through
  col0; bit-identical splits of units, cases, angles and tile widths; the hot spot; zero response; several wave trains per
  case; the per-bin PSD.
"""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT

GOLDEN = os.path.join(ROOT, "tests", "golden")


def _gold():
    return np.load(os.path.join(GOLDEN, "stress_VolturnUS-S-flexible.npz"))


def np_scale(d, t):
    return (d / 2) / (np.pi / 8 * t * d ** 3) / 1e6


def np_sums(a, b, w):
    """S_xy,k [3, 4] over every row and bin of amplitudes a, b [..., nw] (xy = aa, bb, ab; k = 0, 1, 2, 4)."""
    p = [0.5 * np.abs(a) ** 2, 0.5 * np.abs(b) ** 2, 0.5 * (a * np.conj(b)).real]
    return np.array([[np.sum(w ** k * q) for k in (0, 1, 2, 4)] for q in p])


def np_lambda(S, angles, c):
    """lambda_k(theta) [nA, 4] = c^2 (cos^2 S_aa,k - 2 sin cos S_ab,k + sin^2 S_bb,k)."""
    cs, sn = np.cos(angles)[:, None], np.sin(angles)[:, None]
    return c * c * (cs * cs * S[0] - 2 * sn * cs * S[2] + sn * sn * S[1])


def np_exact(S, c):
    """Largest std over the circle and its angle in [0, pi)."""
    half = 0.5 * (S[0, 0] - S[1, 0])
    A = np.hypot(half, S[2, 0])
    th = 0.5 * np.arctan2(-S[2, 0], half) if A > 0 else 0.0
    return c * np.sqrt(0.5 * (S[0, 0] + S[1, 0]) + A), th + np.pi if th < 0 else th


# ---- without a GPU ---------------------------------------------------------------------------------------------------
def test_restatement_matches_reference_helper():
    """The numpy restatement (three cross-spectral sums, closed form over the angles) equals the reference's getSigmaXPSD on
    its own tower-base loads, via std^2 / dw, to 1e-12 relative, for every case (one with two wave trains) at the helper's
    defaults and at other angles, d and t."""
    z = _gold()
    w = z["w"]
    dw = w[1] - w[0]
    for s in ("default", "other"):
        angles, c = z[s + "_angles"], np_scale(float(z[s + "_d"]), float(z[s + "_t"]))
        for ic in range(int(z["n_cases"])):
            S = np_sums(z["ref_run_case%d_FA" % ic], z["ref_run_case%d_SS" % ic], w)
            ref = z["ref_run_case%d_sigPSD_%s" % (ic, s)]
            got = np_lambda(S, angles, c)[:, 0] / dw
            assert np.allclose(got, ref, rtol=1e-12, atol=1e-12 * ref.max()), (s, ic)
    assert abs(z["ref_run_case1_FA"]).max() > 0 and abs(z["ref_run_case1_SS"]).max() > 0


def test_closed_form_equals_explicit_angle_rows():
    """lambda_k(theta) from the three cross sums equals the moments of the explicit rows sigma_theta = c (cos a - sin b) at
    every angle, and the eigenvalue form gives the largest std over the circle: no sampled angle exceeds it, and the
    sample at its angle reaches it."""
    rng = np.random.default_rng(4)
    w = np.linspace(0.05, 2.5, 90)
    a = rng.normal(size=(3, 90)) + 1j * rng.normal(size=(3, 90))
    b = 0.4 * a + rng.normal(size=(3, 90)) + 1j * rng.normal(size=(3, 90))
    c = np_scale(9.0, 0.06)
    angles = np.linspace(-1.0, 7.0, 81)
    S = np_sums(a, b, w)
    lam = np_lambda(S, angles, c)
    for j, th in enumerate(angles):
        sig = c * (np.cos(th) * a - np.sin(th) * b)
        ref = [np.sum(w ** k * 0.5 * np.abs(sig) ** 2) for k in (0, 1, 2, 4)]
        assert np.allclose(lam[j], ref, rtol=1e-12, atol=0)
    sd_max, th = np_exact(S, c)
    assert np.sqrt(lam[:, 0]).max() <= sd_max * (1 + 1e-14)
    assert np.sqrt(np_lambda(S, np.array([th, th + np.pi]), c)[:, 0]) == pytest.approx([sd_max] * 2, rel=1e-13)


def test_struct_layout_matches_header(tmp_path):
    """raftk_stress_ring's size and offsets agree with the ctypes mirror."""
    from raft_b200 import _lib
    fields = [f for f, _ in _lib.RaftkStressRing._fields_]
    prog = tmp_path / "layout.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "raftk.h"\nint main(){printf("%zu\\n", sizeof(raftk_stress_ring));'
                    + "".join('printf("%%zu\\n", offsetof(raftk_stress_ring, %s));' % f for f in fields) + "return 0;}\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got == [C.sizeof(_lib.RaftkStressRing)] + [getattr(_lib.RaftkStressRing, f).offset for f in fields]
    assert _lib.lib.raftk_version() == 132


def _base(nU=2, nR=3, n=12, nw=40):
    from raft_b200 import _lib
    rng = np.random.default_rng(0)
    shp = [nU, 2, 1, 5]
    keep = dict(Xi=np.zeros([nU, nR, n, nw], dtype=np.complex128), w=np.linspace(0.1, 2, nw), R=rng.normal(size=(1, 2, 6)),
                wpow=np.zeros(2, dtype=np.int32), row0=np.array([0, 1, nR], dtype=np.int32), col0=np.array([6], dtype=np.int32),
                angles=np.linspace(0, np.pi, 5), weights=np.ones(2), coef=np.zeros([1, 2, 6, nw], dtype=np.complex128),
                **{k: np.zeros(shp) for k in ("std", "avg", "max", "min", "DEL", "DEL_life", "psd")}, info=np.zeros(shp, dtype=np.int32))
    sr = _lib.RaftkStressRing()
    sr.n_cases, sr.n_rings, sr.n_ch, sr.n_r, sr.n_angles, sr.R_shared = 2, 1, 2, 6, 5, 1
    sr.d, sr.t, sr.m, sr.f_eq, sr.dw = 10.0, 0.083, 4.0, 1.0, 0.05
    for f in ("R", "wpow", "col0", "angles", "std", "avg", "max", "min", "DEL", "info"):
        setattr(sr, f, keep[f].ctypes.data)
    sr.case_row0 = keep["row0"].ctypes.data
    return sr, keep, (nU, nR, n, nw)


def _refusals():
    def setf(**kv):
        def f(sr, keep, dims):
            for k, v in kv.items():
                setattr(sr, k, v)
            return dims
        return f

    def arr(name, values, field, dtype=float):
        def f(sr, keep, dims):
            keep[name + "_bad"] = np.ascontiguousarray(values, dtype=dtype)
            setattr(sr, field, keep[name + "_bad"].ctypes.data)
            return dims
        return f

    def dims(i, v):
        def f(sr, keep, d):
            d = list(d)
            d[i] = v
            return tuple(d)
        return f

    def both(sr, keep, d):
        sr.coef, sr.coef_mode = keep["coef"].ctypes.data, 0
        return d
    def coef_mode(sr, keep, d):
        sr.R, sr.coef, sr.coef_mode = None, keep["coef"].ctypes.data, 3
        return d
    ge1, req, rows = ">= 1", "are required", "case_row0 must start at 0 and end at n_rows"
    col0, dt, m, de = "col0 of ring 0 outside [0, n_dof - n_r]", "d and t must be finite and > 0", "m must be 0 (no DEL) or finite and > 0", \
        "DEL and info are required with m > 0"
    return [("n_units", dims(0, 0), ge1), ("n_rows", dims(1, 0), ge1), ("n_dof", dims(2, 0), ge1), ("nw", dims(3, 0), ge1),
            ("n_cases", setf(n_cases=0), ge1), ("n_rings", setf(n_rings=0), ge1), ("n_r", setf(n_r=0), ge1), ("n_angles", setf(n_angles=0), ge1),
            ("n_ch 0", setf(n_ch=0), "n_ch must be 1"), ("n_ch 3", setf(n_ch=3), "n_ch must be 1"),
            ("rings", setf(n_rings=65), "at most 64 rings per call"), ("angles max", setf(n_angles=257), "at most 256 angles per call"),
            ("n_r above n_dof", setf(n_r=13), "n_r must not exceed n_dof"), ("col0 high", arr("col0", [7], "col0", np.int32), col0),
            ("col0 negative", arr("col0", [-1], "col0", np.int32), col0), ("no channels", setf(R=None), "give exactly one of R"),
            ("both forms", both, "give exactly one of R"), ("R_shared", setf(R_shared=2), "R_shared must be 0 or 1"),
            ("coef_mode", coef_mode, "unknown coef_mode"), ("method", setf(method=2), "unknown method"),
            ("wpow", arr("wpow", [0, 3], "wpow", np.int32), "wpow must be 0, 1 or 2"),
            ("w", lambda sr, k, d: (k.__setitem__("nullw", True), d)[1], req), ("Xi", lambda sr, k, d: (k.__setitem__("nullxi", True), d)[1], req),
            ("angles null", setf(angles=None), req), ("case_row0 null", setf(case_row0=None), req), ("std null", setf(std=None), req),
            ("avg null", setf(avg=None), req), ("max null", setf(max=None), req), ("min null", setf(min=None), req),
            ("angle nan", arr("angles", [0, np.nan, 1, 2, 3], "angles"), "every angle must be finite"), ("d", setf(d=0.0), dt),
            ("t", setf(t=-1.0), dt), ("d inf", setf(d=np.inf), dt), ("m negative", setf(m=-1.0), m), ("m nan", setf(m=np.nan), m),
            ("DEL null", setf(DEL=None), de), ("info null", setf(info=None), de),
            ("life without m", lambda sr, k, d: (setattr(sr, "DEL_life", k["DEL_life"].ctypes.data), setattr(sr, "m", 0.0), d)[2],
             "DEL_life needs m > 0"),
            ("hot_life without life", lambda sr, k, d: (setattr(sr, "hot_life", k["DEL_life"].ctypes.data), d)[1], "hot_life needs DEL_life"),
            ("psd without dw", lambda sr, k, d: (setattr(sr, "psd", k["psd"].ctypes.data), setattr(sr, "dw", 0.0), d)[2],
             "psd needs a finite dw > 0"),
            ("f_eq", setf(f_eq=0.0), "f_eq must be finite and > 0"), ("row0 start", arr("row0", [1, 1, 3], "case_row0", np.int32), rows),
            ("row0 end", arr("row0", [0, 1, 2], "case_row0", np.int32), rows),
            ("row0 empty", arr("row0", [0, 0, 3], "case_row0", np.int32), "every case needs at least one row"),
            ("weights negative", arr("weights", [1.0, -1.0], "weights"), "weights must be finite and >= 0"),
            ("weights zero", arr("weights", [0.0, 0.0], "weights"), "the weights must not all be 0"),
            ("weights nan", arr("weights", [np.nan, 1.0], "weights"), "weights must be finite and >= 0")]


@pytest.mark.parametrize("name", [r[0] for r in _refusals()])
def test_invalid_arguments_are_refused_before_any_launch(name):
    """Every refusal the header lists returns RAFTK_EINVAL from _host and _dev with its reason after the "stress ring: "
    prefix, before any launch."""
    from raft_b200 import _lib
    lib = _lib.lib
    mut, msg = {r[0]: r[1:] for r in _refusals()}[name]
    for entry in ("host", "dev"):
        sr, keep, dims = _base()
        dims = mut(sr, keep, dims)
        w = None if keep.get("nullw") else keep["w"].ctypes.data
        xi = None if keep.get("nullxi") else keep["Xi"].ctypes.data
        n0 = lib.raftk_launch_count()
        if entry == "host":
            rc = lib.raftk_stress_ring_host(*dims, w, xi, C.byref(sr))
        else:
            buf = np.zeros(1 << 16)
            rc = lib.raftk_stress_ring_dev(*dims, w, xi, C.byref(sr), (buf.ctypes.data + 31) // 32 * 32, 1 << 18, None)
        assert rc == -1, (name, entry, rc)
        assert lib.raftk_launch_count() == n0
        err = lib.raftk_last_error().decode()
        assert err.startswith("stress ring: ") and msg in err, (name, entry, err)


def test_workspace_too_small_or_misaligned_is_refused():
    from raft_b200 import _lib
    lib = _lib.lib
    sr, keep, dims = _base()
    nU, nR, n, nw = dims
    need = lib.raftk_stress_ring_workspace_bytes(nU, nR, nw, C.byref(sr))
    assert need == nU * nR * 2 * 1 * 12 * 8
    buf = np.zeros(need // 8 + 16)
    base = (buf.ctypes.data + 31) // 32 * 32
    n0 = lib.raftk_launch_count()
    assert lib.raftk_stress_ring_dev(*dims, keep["w"].ctypes.data, keep["Xi"].ctypes.data, C.byref(sr), base, need - 8, None) == -1
    assert b"too small" in lib.raftk_last_error()
    for off in (8, 16, 24):
        assert lib.raftk_stress_ring_dev(*dims, keep["w"].ctypes.data, keep["Xi"].ctypes.data, C.byref(sr), base + off, need, None) == -1
        assert b"aligned" in lib.raftk_last_error()
    assert lib.raftk_launch_count() == n0
    keep["DEL_life"] = np.zeros([nU, 1, 5])
    sr.DEL_life = keep["DEL_life"].ctypes.data
    assert lib.raftk_stress_ring_workspace_bytes(nU, nR, nw, C.byref(sr)) == need + nU * 2 * 1 * 5 * 8


def test_python_refusals():
    """stress= and stress_ring refuse bad options; an analysis whose channels have no tower-base moment is refused before
    anything is solved."""
    from raft_b200 import solver
    for bad in (dict(d=0.0), dict(t=np.nan), dict(m=-2.0), dict(method="rainflow"), dict(angles=[]), dict(angles=np.zeros(257)),
                dict(foo=1), "d=10"):
        with pytest.raises(ValueError):
            solver.stress_options(bad)
    assert solver.stress_rows([("MbaseX", 0), ("MbaseY", 0), ("MbaseX", 1), ("MbaseY", 1)]) == ([1, 3], [0, 2])
    assert solver.stress_rows([("AxRNA", 0), ("Mbase", 0)]) == ([1], None)
    with pytest.raises(ValueError):
        solver.stress_rows([("AxRNA", 0), ("surge", None)])
    g = np.load(os.path.join(GOLDEN, "flexout_VolturnUS-S-flexible.npz"))
    names = [(nm.split(":")[0], int(nm.split(":")[1]) if nm.split(":")[1] else None) for nm in g["ch_names"]]
    keep = [k for k, (nm, _) in enumerate(names) if not nm.startswith("Mbase")]
    ch = dict(names=[names[k] for k in keep], R=g["ch_R"][keep], wpow=g["ch_wpow"][keep], avg=g["ch_avg"][keep])
    P = {k[2:]: g[k] for k in g.files if k.startswith("P_")}
    with pytest.raises(ValueError, match="tower-base moment"):
        solver.general_analyze_cases(P, g["gen_M"], g["gen_B"], g["gen_C"], [dict(wave_height=2.0, wave_period=8.0, wave_heading=0.0,
                                                                                  wave_spectrum="JONSWAP", wave_gamma=0.0)],
                                     channels=ch, stress=dict(m=4.0))
    with pytest.raises(ValueError, match="ss must have"):
        solver.stress_ring(np.zeros([2, 6, 8], complex), np.linspace(0.1, 1, 8), np.ones(6), np.ones(5))


# ---- on the GPU --------------------------------------------------------------------------------------------------------
def _flex():
    from raft_b200 import packer
    g = np.load(os.path.join(GOLDEN, "flexout_VolturnUS-S-flexible.npz"))
    P = {k[2:]: g[k] for k in g.files if k.startswith("P_")}
    names = [(nm.split(":")[0], int(nm.split(":")[1]) if nm.split(":")[1] else None) for nm in g["ch_names"]]
    ch = dict(names=names, R=g["ch_R"], wpow=g["ch_wpow"], avg=g["ch_avg"])
    cases = []
    for ic in range(3):
        tr = g["ref_run_case%d_trains" % ic]
        cases.append(dict(wave_spectrum=["JONSWAP"] * len(tr), wave_height=list(tr[:, 0]), wave_period=list(tr[:, 1]),
                          wave_heading=list(tr[:, 2]), wave_gamma=[0.0] * len(tr)))
    return g, P, ch, cases, packer


def _check_golden(z, ic, s, m, atol_frac=1e-10):
    """One case's sigmaX entries [1, nA] against the reference helper (std^2 / dw) and its MbaseY / MbaseX means."""
    w = z["w"]
    dw = w[1] - w[0]
    angles, c = z[s + "_angles"], np_scale(float(z[s + "_d"]), float(z[s + "_t"]))
    ref = z["ref_run_case%d_sigPSD_%s" % (ic, s)]
    sd = np.asarray(m["sigmaX_std"])[0]
    assert np.allclose(sd ** 2 / dw, ref, rtol=1e-10, atol=1e-10 * ref.max()), (ic, s)
    avg = c * (np.cos(angles) * z["ref_run_case%d_MbaseY_avg" % ic][0] - np.sin(angles) * z["ref_run_case%d_MbaseX_avg" % ic][0])
    scale = np.abs(avg).max() + sd.max()
    assert np.allclose(m["sigmaX_avg"][0], avg, rtol=1e-10, atol=1e-10 * scale)
    assert np.allclose(m["sigmaX_max"][0], avg + 3 * sd, rtol=1e-10, atol=1e-10 * scale)
    assert np.allclose(m["sigmaX_min"][0], avg - 3 * sd, rtol=1e-10, atol=1e-10 * scale)


@pytest.mark.gpu
def test_flexible_fowt_against_reference_helper():
    """general_analyze_cases(stress=) and general_analyze_cases_batch(stress=) on the 150-DOF flexible FOWT: std, avg, max and
    min around the circumference equal the reference's getSigmaXPSD (std^2 / dw) and its MbaseY / MbaseX means at 1e-10, at
    the helper's defaults and at other angles, d and t; GeneralBatchSession.stress_ring gives the same as the host call on
    every design; without stress= the results are unchanged."""
    import torch
    from raft_b200 import solver
    z = _gold()
    g, P, ch, cases, packer = _flex()
    kw = dict(n_iter=int(g["n_iter"]), xi_start=float(g["xi_start"]))
    base = solver.general_analyze_cases(P, g["gen_M"], g["gen_B"], g["gen_C"], cases, channels=ch, **kw)
    for s in ("default", "other"):
        opt = dict(d=float(z[s + "_d"]), t=float(z[s + "_t"]), angles=z[s + "_angles"], m=4.0, psd=True)
        res = solver.general_analyze_cases(P, g["gen_M"], g["gen_B"], g["gen_C"], cases, channels=ch, stress=opt, **kw)
        for ic in range(3):
            m, b = res["case_metrics"][ic], base["case_metrics"][ic]
            assert set(m) == set(b) | {"sigmaX_avg", "sigmaX_std", "sigmaX_max", "sigmaX_min", "sigmaX_PSD", "sigmaX_DEL", "sigmaX_hot"}
            for k in b:
                assert np.array_equal(np.asarray(m[k]), np.asarray(b[k])), k
            _check_golden(z, ic, s, m)
            nA = len(opt["angles"])
            assert m["sigmaX_PSD"].shape == (1, nA, len(P["w"])) and m["sigmaX_DEL"].shape == (1, nA)
    opt = dict(m=4.0, weights=[0.5, 0.2, 0.3])
    rb = solver.general_analyze_cases_batch([dict(P=P, M=g["gen_M"], B=g["gen_B"], Cm=g["gen_C"])] * 2, cases, channels=[ch, ch],
                                            stress=opt, **kw)
    r1 = solver.general_analyze_cases(P, g["gen_M"], g["gen_B"], g["gen_C"], cases, channels=ch, stress=opt, **kw)
    for d in range(2):
        for ic in range(3):
            _check_golden(z, ic, "default", rb[d]["case_metrics"][ic])
            for k in ("sigmaX_std", "sigmaX_DEL"):
                assert np.array_equal(rb[d]["case_metrics"][ic][k], r1["case_metrics"][ic][k])
        assert rb[d]["fatigue"]["sigmaX_DEL"].shape == (1, 50) and set(rb[d]["fatigue"]["sigmaX_hot"]) == {"angle", "DEL"}
    # the session on the resident responses, one design scaled
    names = [nm for nm, _ in ch["names"]]
    fa, ss = ch["R"][names.index("MbaseY")], ch["R"][names.index("MbaseX")]
    table, owner, first = packer.pack_case_trains(cases)
    gb = solver.GeneralBatchSession([dict(P=P, M=g["gen_M"], B=g["gen_B"], Cm=g["gen_C"])] * 2, solver.CaseTable(table))
    gb.solve(**kw)
    row0 = np.r_[first, len(owner)]
    Fa, Ss = np.stack([fa[None], 2 * fa[None]]), np.stack([ss[None], 2 * ss[None]])
    dv = gb.stress_ring(Fa, Ss, m=4.0, case_row0=row0, psd=True, weights=[1.0, 1.0, 2.0])
    torch.cuda.synchronize()
    hv = solver.stress_ring(gb.Xi.cpu().numpy(), P["w"], Fa, Ss, m=4.0, case_row0=row0, psd=True, weights=[1.0, 1.0, 2.0],
                            dw=float(P["dw"]))
    for k in hv:
        assert np.array_equal(dv[k].cpu().numpy(), hv[k]), k
    w = z["w"]
    for ic in range(3):
        ref = z["ref_run_case%d_sigPSD_default" % ic]
        assert np.allclose(hv["std"][0, ic, 0] ** 2 / (w[1] - w[0]), ref, rtol=1e-10, atol=1e-10 * ref.max())
        assert np.all(hv["avg"][:, ic] == 0)
    assert np.allclose(hv["std"][1], 2 * hv["std"][0], rtol=1e-13)
    gs = solver.GeneralSession(P, g["gen_M"], g["gen_B"], g["gen_C"], solver.CaseTable(table))
    gs.solve(**kw)
    ds = gs.stress_ring(fa, ss, m=4.0, case_row0=row0)
    torch.cuda.synchronize()
    assert np.array_equal(ds["std"].cpu().numpy(), hv["std"][0])


def _random(nU=3, nR=5, n=12, nw=100, seed=1):
    rng = np.random.default_rng(seed)
    w = np.arange(1, nw + 1) * 0.03
    env = np.exp(-0.5 * ((w - 0.8) / 0.4) ** 2)
    Xi = (rng.normal(size=(nU, nR, n, nw)) + 1j * rng.normal(size=(nU, nR, n, nw))) * env * 1e6
    return rng, w, Xi


@pytest.mark.gpu
def test_del_equals_fatigue_on_explicit_rows():
    """Per-angle DELs (Dirlik and narrow band) and lifetime DELs equal solver.fatigue on the explicit rows R_theta = c (cos R_FA
    - sin R_SS) to rounding: the same closed form on the same moments, summed in another order.  std equals sqrt(l0)."""
    from raft_b200 import solver
    rng, w, Xi = _random()
    fa, ss = rng.normal(size=12), rng.normal(size=12)
    angles = np.linspace(0, 2 * np.pi, 37)
    c = np_scale(7.0, 0.05)
    row0 = np.array([0, 2, 3, 5])
    Rt = c * (np.cos(angles)[:, None] * fa - np.sin(angles)[:, None] * ss)
    for method in ("dirlik", "narrowband"):
        r = solver.stress_ring(Xi, w, fa, ss, angles, 7.0, 0.05, m=4.0, method=method, case_row0=row0, weights=[1.0, 2.0, 0.5])
        f = solver.fatigue(Xi, w, 4.0, R=Rt, case_row0=row0, method=method, weights=[1.0, 2.0, 0.5])
        assert np.allclose(r["DEL"][:, :, 0], f["DEL"], rtol=1e-11, atol=0)
        assert np.array_equal(r["info"][:, :, 0], f["info"])
        assert np.allclose(r["DEL_life"][:, 0], f["DEL_life"], rtol=1e-11, atol=0)
        assert np.allclose(r["std"][:, :, 0] ** 2, f["moments"][..., 0], rtol=1e-12, atol=0)
        h = r["hot_life"][:, 0]
        j = np.argmax(r["DEL_life"][:, 0], axis=1)
        assert np.array_equal(h[:, 0], angles[j]) and np.array_equal(h[:, 1], r["DEL_life"][np.arange(3), 0, j])


@pytest.mark.gpu
def test_rigid_tower_through_device_session_and_model():
    """A rigid tower's Mbase (complex coefficients, no side-side moment): std(theta) = |cos theta| std(Mbase) c through
    DeviceSession.stress_ring, bit-identical to the host call; Model(stress=...).analyzeCases() adds the sigmaX entries and the
    lifetime DEL and leaves every other result as it was."""
    import torch
    from raft_b200 import solver
    from raft_b200.model import Model
    from conftest import load_golden
    z = np.load(os.path.join(GOLDEN, "turb_VolturnUS-S.npz"))
    P = {k[2:]: z[k] for k in z.files if k.startswith("P_")}
    w = P["w"]
    names = [n.split(":")[0] for n in z["ch_names"]]
    k = names.index("Mbase")
    coef = z["ch_coef"][k]
    cases = dict(Hs=np.array([6.0, 8.0, 4.0]), Tp=np.array([10.0, 12.0, 8.0]), gamma=np.zeros(3), beta_deg=np.array([0.0, 30.0, 0.0]),
                 spec=np.zeros(3, dtype=np.int32))
    s = solver.DeviceSession(solver.DesignBatch([P, P]), solver.CaseTable(cases), want=("Xi", "status", "B_drag", "F_drag", "F_iner"))
    s.solve(n_iter=int(z["n_iter"]), xi_start=float(z["xi_start"]))
    angles = np.linspace(0, 2 * np.pi, 50)
    d = s.stress_ring(coef, None, angles, 10.0, 0.083, m=4.0, mean=2.0e7)
    torch.cuda.synchronize()
    Xi = s.out["Xi"].cpu().numpy()
    h = solver.stress_ring(Xi, w, coef, None, angles, 10.0, 0.083, m=4.0, mean=2.0e7, dw=float(s.batch.dw))
    for key in h:
        assert np.array_equal(d[key].cpu().numpy(), h[key]), key
    sd_M = np.sqrt(solver.fatigue(Xi, w, 4.0, coef=coef[None])["moments"][..., 0, 0])           # [2, 3]
    c = np_scale(10.0, 0.083)
    assert np.allclose(h["std"][:, :, 0], np.abs(np.cos(angles)) * sd_M[..., None] * c, rtol=1e-12, atol=1e-12 * sd_M.max() * c)
    assert np.allclose(h["avg"][:, :, 0], c * np.cos(angles) * 2.0e7, rtol=1e-13, atol=1e-6)
    assert np.allclose(h["hot"][..., 0, 4], sd_M * c, rtol=1e-13) and np.all(h["hot"][..., 0, 5] == 0.0)
    assert np.all(h["hot"][..., 0, 1] <= h["hot"][..., 0, 4] * (1 + 1e-14))
    # Model
    G0, _ = load_golden("test_VolturnUS-S")
    D = json.load(open(os.path.join(GOLDEN, "designs.json")))["test_VolturnUS-S"]
    mats = dict(M_struc=P["M0"] - G0["A_hydro_morison"], C_struc=P["C0"] - G0["C_moor"], C_moor=G0["C_moor"], B_struc=P["B0"])
    ch = dict(names=[(n.split(":")[0], int(n.split(":")[1])) for n in z["ch_names"]], coef=z["ch_coef"], avg=z["ch_avg"])
    mc = []
    for ic in range(2):
        tr = z["ref_run_case%d_trains" % ic]
        mc.append(dict(wave_spectrum=["JONSWAP"] * len(tr), wave_height=list(tr[:, 0]), wave_period=list(tr[:, 1]),
                       wave_heading=list(tr[:, 2]), wave_gamma=[0.0] * len(tr)))

    def model(**kw):
        return Model(dict(D, site=dict(D["site"], water_depth=float(P["depth"]))), matrices=mats, channels=ch, **kw)
    base = model().analyzeCases(cases=mc)
    m = model(stress=dict(m=4.0, weights=[0.4, 0.6], psd=True))
    res = m.analyzeCases(cases=mc)
    Xi_t = np.concatenate(res["Xi_trains"])
    row0 = np.cumsum([0] + [len(x) for x in res["Xi_trains"]])
    ref = solver.stress_ring(Xi_t, m.w, coef, None, m=4.0, case_row0=row0, weights=[0.4, 0.6], psd=True, mean=ch["avg"][k],
                             dw=m.w[1] - m.w[0])
    for ic in range(2):
        a, b = res["case_metrics"][ic][0], base["case_metrics"][ic][0]
        assert set(a) == set(b) | {"sigmaX_avg", "sigmaX_std", "sigmaX_max", "sigmaX_min", "sigmaX_PSD", "sigmaX_DEL", "sigmaX_hot"}
        for key in b:
            assert np.array_equal(np.asarray(a[key]), np.asarray(b[key])), key
        assert np.array_equal(a["sigmaX_std"], ref["std"][ic]) and np.array_equal(a["sigmaX_DEL"], ref["DEL"][ic])
        assert a["sigmaX_std"].shape == (1, 50) and a["sigmaX_hot"]["std_exact"].shape == (1,)
    assert np.array_equal(res["fatigue"][0]["sigmaX_DEL"], ref["DEL_life"])
    with pytest.raises(ValueError, match="tower-base moment"):
        Model(dict(D, site=dict(D["site"], water_depth=float(P["depth"]))), matrices=mats, stress=dict(m=4.0))
    no_mbase = dict(names=ch["names"][:k] + ch["names"][k + 1:], coef=np.delete(ch["coef"], k, 0), avg=np.delete(ch["avg"], k))
    with pytest.raises(ValueError, match="tower-base moment"):
        Model(dict(D, site=dict(D["site"], water_depth=float(P["depth"]))), matrices=mats, channels=no_mbase, stress=dict(m=4.0))


@pytest.mark.gpu
def test_farm_rings_through_col0():
    """A farm's Xi_sys with FOWT i's tower at col0 = 6 i: every ring equals the single-FOWT call on its columns, bit for bit,
    through the host entry and DeviceSession.stress_ring(farm=True)."""
    import torch
    from raft_b200 import solver
    z = np.load(os.path.join(GOLDEN, "turb_VolturnUS-S.npz"))
    P = {k[2:]: z[k] for k in z.files if k.startswith("P_")}
    cases = dict(Hs=np.array([6.0, 8.0]), Tp=np.array([10.0, 12.0]), gamma=np.zeros(2), beta_deg=np.array([0.0, 30.0]),
                 spec=np.zeros(2, dtype=np.int32))
    s = solver.DeviceSession(solver.DesignBatch([P, P]), solver.CaseTable(cases), want=("Xi", "status", "B_drag", "F_drag", "F_iner"))
    s.solve(n_iter=int(z["n_iter"]), xi_start=float(z["xi_start"]))
    xs, _ = s.farm_response()
    rng = np.random.default_rng(5)
    fa, ss = rng.normal(size=(2, 6)), rng.normal(size=(2, 6))
    d = s.stress_ring(fa, ss, m=3.0, col0=[0, 6], farm=True, mean=[[1e6, 2e6], [3e6, -1e6]])
    torch.cuda.synchronize()
    X = xs.cpu().numpy()
    h = solver.stress_ring(X, P["w"], fa, ss, m=3.0, col0=[0, 6], mean=[[1e6, 2e6], [3e6, -1e6]], dw=float(s.batch.dw))
    for key in h:
        assert np.array_equal(d[key].cpu().numpy(), h[key]), key
    for i in range(2):
        one = solver.stress_ring(X[:, 6 * i:6 * i + 6], P["w"], fa[i], ss[i], m=3.0, mean=[1e6, 2e6] if i == 0 else [3e6, -1e6])
        for key in ("std", "avg", "max", "min", "DEL", "info", "hot"):
            assert np.array_equal(h[key][:, i], one[key][:, 0]), (i, key)


@pytest.mark.gpu
def test_results_do_not_depend_on_batch_split_or_tile():
    """Bit-identical when units, cases or angles are split across calls, rings are split, or the tile width is forced (32
    bins, 64 bins, Xi read from L2); real and complex forms."""
    from raft_b200 import solver
    rng, w, Xi = _random(nU=4, nR=6, n=12, nw=130, seed=7)
    R = rng.normal(size=(4, 3, 2, 12))
    fa, ss = R[:, :, 0], R[:, :, 1]
    cf = rng.normal(size=(3, 12, 130)) + 1j * rng.normal(size=(3, 12, 130))
    cs = rng.normal(size=(3, 12, 130)) + 1j * rng.normal(size=(3, 12, 130))
    angles = np.linspace(0.1, 6.0, 40)
    row0 = np.array([0, 2, 3, 6])
    wts = [1.0, 0.5, 2.0]
    for A, B, kw in ((fa, ss, dict(wpow=[[0, 1], [2, 0], [1, 1]])), (cf, cs, {})):
        full = solver.stress_ring(Xi, w, A, B, angles, m=4.0, case_row0=row0, weights=wts, psd=True, **kw)
        keys = ("std", "avg", "max", "min", "DEL", "info", "hot", "psd")
        for tile in (32, 64, -1):
            t = solver.stress_ring(Xi, w, A, B, angles, m=4.0, case_row0=row0, weights=wts, psd=True, tile_w=tile, **kw)
            for key in full:
                assert np.array_equal(t[key], full[key]), (tile, key)
        per_unit = not np.iscomplexobj(A)                 # real rows per unit [4, 3, 12]; coefficients shared [3, 12, 130]
        for u in range(4):
            one = solver.stress_ring(Xi[u:u + 1], w, A[u:u + 1] if per_unit else A, B[u:u + 1] if per_unit else B, angles, m=4.0,
                                     case_row0=row0, weights=wts, psd=True, **kw)
            for key in full:
                assert np.array_equal(one[key][0], full[key][u]), (u, key)
        for c in range(3):
            one = solver.stress_ring(Xi[:, row0[c]:row0[c + 1]], w, A, B, angles, m=4.0, case_row0=[0, row0[c + 1] - row0[c]], psd=True, **kw)
            for key in keys:
                assert np.array_equal(one[key][:, 0], full[key][:, c]), (c, key)
        for sl in (slice(0, 7), slice(7, 40), slice(13, 14)):
            part = solver.stress_ring(Xi, w, A, B, angles[sl], m=4.0, case_row0=row0, weights=wts, psd=True, **kw)
            for key in ("std", "avg", "max", "min", "DEL", "info", "psd"):
                assert np.array_equal(part[key], full[key][:, :, :, sl]), key
            assert np.array_equal(part["DEL_life"], full["DEL_life"][:, :, sl])
        for ring in range(3):
            sub = dict(wpow=[kw["wpow"][ring]]) if kw else {}
            one = solver.stress_ring(Xi, w, A[:, ring:ring + 1] if per_unit else A[ring:ring + 1],
                                     B[:, ring:ring + 1] if per_unit else B[ring:ring + 1], angles, m=4.0, case_row0=row0,
                                     weights=wts, psd=True, **sub)
            for key in full:
                assert np.array_equal(one[key][:, :, 0] if key not in ("DEL_life", "hot_life") else one[key][:, 0],
                                      full[key][:, :, ring] if key not in ("DEL_life", "hot_life") else full[key][:, ring]), (ring, key)


@pytest.mark.gpu
def test_hot_spot_sampled_below_exact_and_equal_on_grid():
    """The sampled hot-spot std never exceeds the exact largest std over the circle; a grid that contains the exact angle
    reaches it; the exact value and angle equal the eigen restatement."""
    from raft_b200 import solver
    rng, w, Xi = _random(nU=2, nR=3, n=8, nw=64, seed=11)
    fa, ss = rng.normal(size=8), rng.normal(size=8)
    r = solver.stress_ring(Xi, w, fa, ss, np.linspace(0, 2 * np.pi, 17), m=4.0)
    h = r["hot"][..., 0, :]
    assert np.all(h[..., 1] <= h[..., 4] * (1 + 1e-14)) and np.all(h[..., 1] < h[..., 4])
    c = np_scale(10.0, 0.083)
    for u in range(2):
        for ic in range(3):
            a, b = fa @ Xi[u, ic], ss @ Xi[u, ic]
            sd, th = np_exact(np_sums(a, b, w), c)
            assert h[u, ic, 4] == pytest.approx(sd, rel=1e-12) and h[u, ic, 5] == pytest.approx(th, abs=1e-10)
            j = np.argmax(r["std"][u, ic, 0])
            assert h[u, ic, 0] == np.linspace(0, 2 * np.pi, 17)[j] and h[u, ic, 1] == r["std"][u, ic, 0, j]
            g = solver.stress_ring(Xi[u, ic:ic + 1], w, fa, ss, [0.3, h[u, ic, 5], 2.0], m=4.0)
            assert g["hot"][0, 0, 0] == h[u, ic, 5] and g["hot"][0, 0, 1] == pytest.approx(h[u, ic, 4], rel=1e-12)


@pytest.mark.gpu
def test_zero_response_and_several_trains():
    """A zero response gives zero stress, DEL 0 with RAFTK_FATIGUE_ZERO and a finite lifetime DEL; the rows of a case (its wave
    trains) are summed as combine_trains sums per-train statistics: std^2 and PSD add over the rows."""
    from raft_b200 import solver
    rng, w, Xi = _random(nU=1, nR=4, n=6, nw=50, seed=3)
    fa, ss = rng.normal(size=6), rng.normal(size=6)
    Z = np.zeros_like(Xi)
    r = solver.stress_ring(Z, w, fa, ss, m=4.0, weights=np.ones(4), psd=True, mean=[5e6, 0.0])
    assert np.all(r["std"] == 0) and np.all(r["DEL"] == 0) and np.all(r["info"] == solver.FATIGUE_ZERO)
    assert np.all(np.isfinite(r["DEL_life"])) and np.all(r["DEL_life"] == 0) and np.all(r["psd"] == 0)
    assert np.all(r["max"] == r["avg"]) and np.all(r["hot"][..., 4] == 0)
    one = solver.stress_ring(Xi, w, fa, ss, psd=True)
    both = solver.stress_ring(Xi, w, fa, ss, psd=True, case_row0=[0, 3, 4])
    sd, ps = solver.combine_trains(one["std"][0], one["psd"][0], [0, 1, 2])
    assert np.allclose(both["std"][0, 0], sd, rtol=1e-13) and np.allclose(both["psd"][0, 0], ps, rtol=1e-12, atol=1e-12 * ps.max())


@pytest.mark.gpu
def test_psd_equals_numpy_per_bin():
    """psd=True: per bin sum over the case's rows of 1/2 |sigma|^2 / dw, as getPSD of the explicit rows; its sum over the
    bins times dw is std^2."""
    from raft_b200 import solver
    rng, w, Xi = _random(nU=2, nR=3, n=12, nw=70, seed=9)
    fa, ss = rng.normal(size=(2, 12)), rng.normal(size=(2, 12))
    angles = np.linspace(0, np.pi, 9)
    r = solver.stress_ring(Xi, w, fa, ss, angles, 9.0, 0.07, case_row0=[0, 2, 3], col0=0, psd=True, wpow=[[0, 0], [2, 1]], dw=0.03)
    c = np_scale(9.0, 0.07)
    for u in range(2):
        for ic, rows in enumerate(([0, 1], [2])):
            for k in range(2):
                pa = 2 if k == 1 else 0
                pb = 1 if k == 1 else 0
                a, b = (fa[k] @ Xi[u, rows]) * w ** pa, (ss[k] @ Xi[u, rows]) * w ** pb
                for j, th in enumerate(angles):
                    sig = c * (np.cos(th) * a - np.sin(th) * b)
                    ref = np.sum(0.5 * np.abs(sig) ** 2 / 0.03, axis=0)
                    assert np.allclose(r["psd"][u, ic, k, j], ref, rtol=1e-12, atol=1e-13 * ref.max())
                    assert np.sum(ref) * 0.03 == pytest.approx(r["std"][u, ic, k, j] ** 2, rel=1e-12)
