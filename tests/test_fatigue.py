"""Spectral fatigue damage-equivalent loads (raftk_fatigue_*, solver.fatigue and the sessions' .fatigue).

Without a GPU: a numpy restatement of the contract (moments, Dirlik and narrow-band closed forms, DEL, info, lifetime DEL);
the closed form against mpmath quadrature of the Dirlik pdf; the narrow-band limit and the continuity of the switch; the
method against time-domain rainflow counting of random-phase realisations; the ctypes struct against the header; and every
refusal of the C ABI, with the launch count unchanged.
On an H100: the device moments against the unmodified reference's own PSDs in the committed fixtures, DEL / info / moments /
DEL_life against the restatement, batch and tile independence, and the sessions against the host entry."""
import ctypes as C
import json
import math
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT

SWITCH = 1e-6          # include/raftk.h RAFTK_FATIGUE_NB_SWITCH
ZERO, NARROWBAND = 1, 2


# ---- numpy restatement of the contract ---------------------------------------------------------------------------------
def np_amplitudes(Xi, w, R=None, wpow=None, coef=None):
    """Y [U, rows, nch, nw] of Xi [U, rows, n, nw] for real rows R ([nch, n] or [U, nch, n]) with wpow, or coef ([nch, n, nw],
    [U, nch, n, nw] or [U, rows, nch, n, nw])."""
    U, nR = Xi.shape[:2]
    if R is not None:
        R = np.broadcast_to(R, (U,) + R.shape[-2:])
        p = np.zeros(R.shape[1], dtype=int) if wpow is None else np.asarray(wpow)
        return np.einsum("ukb,urbw->urkw", R, Xi) * w[None, None, None, :] ** p[None, None, :, None]
    if coef.ndim == 3:
        return np.einsum("kbw,urbw->urkw", coef, Xi)
    if coef.ndim == 4:
        return np.einsum("ukbw,urbw->urkw", coef, Xi)
    return np.einsum("urkbw,urbw->urkw", coef, Xi)


def np_moments(Y, w, case_row0):
    """lambda_k [U, nC, nch, 4] (k = 0, 1, 2, 4) of amplitudes Y [U, rows, nch, nw], the rows of case c being case_row0[c]:[c+1]."""
    a = 0.5 * np.abs(Y) ** 2
    lam = np.stack([np.sum(a * w ** k, axis=-1) for k in (0, 1, 2, 4)], axis=-1)          # [U, rows, nch, 4]
    return np.stack([lam[:, case_row0[c]:case_row0[c + 1]].sum(axis=1) for c in range(len(case_row0) - 1)], axis=1)


def dirlik_params(l0, l1, l2, l4):
    xm = (l1 / l0) * math.sqrt(l2 / l4)
    g = l2 / math.sqrt(l0 * l4)
    D1 = 2.0 * (xm - g * g) / (1.0 + g * g)
    den = 1.0 - g - D1 + D1 * D1
    R = (g - xm - D1 * D1) / den
    D2 = den / (1.0 - R)
    D3 = 1.0 - D1 - D2
    Q = 1.25 * (g - D3 - D2 * R) / D1
    return g, D1, D2, D3, Q, R


def dirlik_ESm(l0, D1, D2, D3, Q, R, m):
    return (2.0 * math.sqrt(l0)) ** m * (D1 * Q ** m * math.gamma(1 + m) + 2 ** (m / 2) * math.gamma(1 + m / 2) * (D2 * abs(R) ** m + D3))


def np_rate(lam, m, method="dirlik", switch=SWITCH):
    """-> (damage rate d [1/s], info bits) of one moment set (l0, l1, l2, l4)."""
    l0, l1, l2, l4 = (float(x) for x in lam)
    if not (l0 > 0 and l2 > 0):
        return 0.0, ZERO
    if method == "dirlik":
        with np.errstate(all="ignore"):
            try:
                g, D1, D2, D3, Q, R = dirlik_params(l0, l1, l2, l4)
            except ZeroDivisionError:
                g = 1.0
                D1 = Q = R = float("nan")
        ok = (1 - g >= switch and all(math.isfinite(v) and v > 0 for v in (D1, Q, R)) and D2 * abs(R) ** m + D3 > 0)
        if ok:
            return math.sqrt(l4 / l2) / (2 * math.pi) * dirlik_ESm(l0, D1, D2, D3, Q, R, m), 0
    return math.sqrt(l2 / l0) / (2 * math.pi) * (2 * math.sqrt(2 * l0)) ** m * math.gamma(1 + m / 2), NARROWBAND


def np_log_rate(lam, m, method="dirlik", switch=SWITCH):
    """np_rate in the log domain, as the device evaluates it: -> (log d, info); log d = -inf for a ZERO channel."""
    l0, l1, l2, l4 = (float(x) for x in lam)
    if not (l0 > 0 and l2 > 0):
        return -math.inf, ZERO
    if method == "dirlik" and np_rate(lam, m, method, switch)[1] == 0:
        g, D1, D2, D3, Q, R = dirlik_params(l0, l1, l2, l4)
        t1 = math.log(D1) + m * math.log(Q) + math.lgamma(1 + m)
        t2 = 0.5 * m * math.log(2) + math.lgamma(1 + m / 2) + math.log(D2 * abs(R) ** m + D3)
        lb = max(t1, t2) + math.log1p(math.exp(min(t1, t2) - max(t1, t2)))
        return 0.5 * math.log(l4 / l2) - math.log(2 * math.pi) + m * (math.log(2) + 0.5 * math.log(l0)) + lb, 0
    return (0.5 * math.log(l2 / l0) - math.log(2 * math.pi) + m * (math.log(2) + 0.5 * math.log(2 * l0)) + math.lgamma(1 + m / 2),
            NARROWBAND)


def np_fatigue(lam, m, f_eq=1.0, method="dirlik", weights=None):
    """The contract on moments lam [U, nC, nch, 4]: -> dict(DEL, info, DEL_life), evaluated in the log domain so that large
    loads and exponents stay finite."""
    U, nC, nch = lam.shape[:3]
    m = np.broadcast_to(np.asarray(m, dtype=float), (nch,))
    p = np.ones(nC) if weights is None else np.asarray(weights, dtype=float)
    ld = np.zeros([U, nC, nch])
    info = np.zeros([U, nC, nch], dtype=np.int32)
    for u in range(U):
        for c in range(nC):
            for k in range(nch):
                ld[u, c, k], info[u, c, k] = np_log_rate(lam[u, c, k], m[k], method)
    with np.errstate(divide="ignore"):
        DEL = np.exp((ld - math.log(f_eq)) / m)
        lw = np.where(p[None, :, None] > 0, np.log(p)[None, :, None] + ld, -np.inf)
    mx = lw.max(axis=1)
    s = np.exp(lw - np.where(np.isfinite(mx), mx, 0)[:, None, :]).sum(axis=1)
    with np.errstate(divide="ignore"):
        life = np.where(np.isfinite(mx), np.exp((mx + np.log(s) - math.log(f_eq * p.sum())) / m), 0.0)
    return dict(DEL=DEL, info=info, DEL_life=life)


# ---- fixtures for the CPU checks ---------------------------------------------------------------------------------------
def two_bin(W, r):
    w = np.array([1.0, W])
    a = np.array([1.0, r])
    return [float(np.sum(w ** k * a)) for k in (0, 1, 2, 4)]


def dirlik_family():
    """Moment sets whose g runs from 0.2 to just below the switch, every one taking Dirlik's branch."""
    out = []
    for W, r in ((10.0, 0.01259), (10.0, 0.03), (6.0, 0.0794), (4.0, 0.1), (3.0, 0.3981), (2.0, 0.0794), (2.0, 0.0158)):   # g = 0.2 .. 0.94
        out.append(two_bin(W, r))
    w = np.linspace(0.2, 2.0, 400)
    for s in (0.3, 0.1, 3e-2, 1e-2, 3e-3):
        a = np.exp(-0.5 * ((w - 1.0) / s) ** 2) if s > 5e-3 else None
        ww = w if a is not None else np.linspace(1 - 8 * s, 1 + 8 * s, 400)
        a = a if a is not None else np.exp(-0.5 * ((ww - 1.0) / s) ** 2)
        out.append([float(np.sum(ww ** k * a)) for k in (0, 1, 2, 4)])
    out.append(two_bin(1.0 + 2e-3, 0.7))          # 1 - g = 1.5e-6, just above the switch
    return out


def test_dirlik_closed_form_against_mpmath_quadrature():
    """E[S^m] of the closed form (FP64, as the kernel evaluates it) against 40-digit quadrature of Dirlik's range pdf
    p(Z) = D1/Q e^(-Z/Q) + D2 Z/R^2 e^(-Z^2/2R^2) + D3 Z e^(-Z^2/2), Z = S / (2 sqrt(l0)), with the parameters taken to 40
    digits from the same moments: 1e-10 relative over g = 0.2 .. 1 - 1.5e-6 and m = 3, 4, 5, 8, 10."""
    mp = pytest.importorskip("mpmath")
    mp.mp.dps = 40
    gs = []
    for lam in dirlik_family():
        g, D1, D2, D3, Q, R = dirlik_params(*lam)
        assert all(v > 0 for v in (D1, Q, R)) and 1 - g >= SWITCH
        gs.append(g)
        L = [mp.mpf(x) for x in lam]
        xm = (L[1] / L[0]) * mp.sqrt(L[2] / L[3])
        G = L[2] / mp.sqrt(L[0] * L[3])
        d1 = 2 * (xm - G * G) / (1 + G * G)
        r = (G - xm - d1 * d1) / (1 - G - d1 + d1 * d1)
        d2 = (1 - G - d1 + d1 * d1) / (1 - r)
        d3 = 1 - d1 - d2
        q = mp.mpf(5) / 4 * (G - d3 - d2 * r) / d1
        pts = sorted(set([mp.mpf(0), q, 10 * q, 50 * q, r, 5 * r, mp.mpf(1), mp.mpf(5), mp.mpf(20)]))
        for m in (3, 4, 5, 8, 10):
            def f(Z):
                return Z ** m * (d1 / q * mp.exp(-Z / q) + d2 * Z / r ** 2 * mp.exp(-Z ** 2 / (2 * r ** 2)) + d3 * Z * mp.exp(-Z ** 2 / 2))
            ref = (2 * mp.sqrt(L[0])) ** m * mp.quad(f, pts + [mp.inf])
            got = dirlik_ESm(lam[0], D1, D2, D3, Q, R, m)
            assert abs(got - float(ref)) <= 1e-10 * abs(float(ref)), (g, m, got, float(ref))
    assert min(gs) < 0.2 and 1 - max(gs) < 2e-6


def test_narrowband_limit_and_switch_continuity():
    """A single-bin spectrum (g = 1, D1 = 0, R = 0/0) falls back to the narrow band exactly; across 1 - g = 1e-6 the DEL of
    Dirlik's closed form and of the narrow band differ by < 1e-6 relative (measured: 0.17 (1 - g) at m = 3, 0.23 (1 - g) at
    m = 10), on two-bin and Gaussian spectra within half a threshold of it, and the fallback engages just below it."""
    lam = [2.5, 2.5 * 0.7, 2.5 * 0.49, 2.5 * 0.7 ** 4]
    for m in (3.0, 4.0, 10.0):
        d, info = np_rate(lam, m, "dirlik")
        dn, _ = np_rate(lam, m, "narrowband")
        assert info == NARROWBAND and d == dn
        assert dn == pytest.approx(math.sqrt(0.49) / (2 * math.pi) * (2 * math.sqrt(5.0)) ** m * math.gamma(1 + m / 2), rel=1e-14)
    near = 0
    gauss = []
    for s in np.logspace(-2.8, -3.3, 8):                  # Gaussian bumps, 1 - g from about 2.5e-6 to 2.5e-7
        ww = np.linspace(1 - 8 * s, 1 + 8 * s, 400)
        a = np.exp(-0.5 * ((ww - 1.0) / s) ** 2)
        gauss.append([float(np.sum(ww ** k * a)) for k in (0, 1, 2, 4)])
    for lam in [two_bin(1.0 + s, 0.7) for s in np.logspace(-2.2, -3.2, 12)] + gauss:   # two bins: 1 - g from 1e-5 to 1e-7
        g = dirlik_params(*lam)[0]
        near += abs(1 - g - SWITCH) < 0.5 * SWITCH
        for m in (3.0, 4.0, 5.0, 8.0, 10.0):
            dd, info = np_rate(lam, m, "dirlik", switch=0.0)              # the closed form alone
            dn, _ = np_rate(lam, m, "narrowband")
            jump = abs((dd / dn) ** (1 / m) - 1)
            if abs(1 - g - SWITCH) < 0.5 * SWITCH:
                assert info == 0 and jump < 1e-6, (g, m, jump)
            assert np_rate(lam, m)[1] == (NARROWBAND if 1 - g < SWITCH else 0)
    assert near >= 4, near                                # samples on both sides of the switch, from both families


def rainflow_ranges(x):
    """ASTM E1049-85 rainflow counting (section 5.4.4) of a sequence -> (ranges, counts 1 or 0.5)."""
    d = np.diff(x)
    pv = x[np.flatnonzero(np.r_[True, np.sign(d[1:]) != np.sign(d[:-1]), True])]          # the reversals
    ranges, counts, stack = [], [], []
    for v in pv:
        stack.append(v)
        while len(stack) >= 3:
            X, Y = abs(stack[-1] - stack[-2]), abs(stack[-2] - stack[-3])
            if X < Y:
                break
            if len(stack) == 3:
                ranges.append(Y); counts.append(0.5)
                stack.pop(0)
            else:
                ranges.append(Y); counts.append(1.0)
                last = stack.pop()
                stack.pop(); stack.pop()
                stack.append(last)
    for i in range(len(stack) - 1):
        ranges.append(abs(stack[i + 1] - stack[i])); counts.append(0.5)
    return np.array(ranges), np.array(counts)


def test_rainflow_counter_on_the_standard_example():
    """ASTM E1049-85 figure 6 (-2, 1, -3, 5, -1, 3, -4, 4, -2): ranges 3, 4, 8, 9 (one half each), 4 (one full), 6, 8 (halves)."""
    r, c = rainflow_ranges(np.array([-2, 1, -3, 5, -1, 3, -4, 4, -2], dtype=float))
    got = sorted(zip(r.tolist(), c.tolist()))
    assert got == sorted([(3, 0.5), (4, 0.5), (8, 0.5), (9, 0.5), (4, 1.0), (8, 0.5), (6, 0.5)])


def _fixture_spectra():
    z = np.load(os.path.join(GOLDEN, "ops_VolturnUS-S.npz"))
    w = z["w"]
    return w, [z["cm0_Mbase_PSD_c%d" % c][:, 0] for c in range(4)]


@pytest.mark.parametrize("m", [3.0, 4.0])
def test_dirlik_against_time_domain_rainflow(m):
    """Random-phase realisations of the reference's Mbase PSDs (ops_VolturnUS-S, 40 bins at w_j = j dw, g = 0.82-0.94), each
    over one whole period 2 pi / dw sampled 64 times per shortest wave period, counted by ASTM rainflow: the damage summed
    over 24 seeded realisations gives a DEL within 6 % of Dirlik's.  Measured with this seed: Dirlik / rainflow DEL 1.001-1.018
    at m = 3 and 1.004-1.038 at m = 4, with a realisation-to-realisation spread of 6-8 % and 14-21 % in damage; the 6 % bound
    keeps a 1.6x margin over the worst case.  A range/amplitude slip (a factor 2) and a rad/s-vs-Hz slip in the rate
    ((2 pi)^(1/m) = 1.58 at m = 4, 1.85 at m = 3) miss by 50 % or more."""
    w, spectra = _fixture_spectra()
    dw = w[1] - w[0]
    T = 2 * np.pi / dw
    t = np.arange(int(64 * w[-1] / dw)) * (T / int(64 * w[-1] / dw))
    rng = np.random.default_rng(1234)
    for S in spectra:
        amp = np.sqrt(2 * S * dw)
        lam = [float(np.sum(w ** k * S * dw)) for k in (0, 1, 2, 4)]
        d_dir, info = np_rate(lam, m)
        assert info == 0
        D, Ttot = 0.0, 0.0
        for _ in range(24):
            ph = rng.uniform(0, 2 * np.pi, len(w))
            x = (amp[:, None] * np.cos(w[:, None] * t[None, :] + ph[:, None])).sum(axis=0)
            x = np.r_[x, x[0]]                                            # one closed period
            r, c = rainflow_ranges(x)
            D += float(np.sum(c * r ** m))
            Ttot += T
        ratio = (d_dir / (D / Ttot)) ** (1 / m)
        assert abs(ratio - 1) < 0.06, ratio
        assert abs(2 * ratio - 1) > 0.5 and abs((2 * np.pi) ** (1 / m) * ratio - 1) > 0.25


# ---- C ABI without a GPU -----------------------------------------------------------------------------------------------
def test_struct_layout_matches_header(tmp_path):
    from raft_b200 import _lib
    prog = tmp_path / "layout.c"
    fields = [f[0] for f in _lib.RaftkFatigue._fields_]
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "raftk.h"\nint main(){printf("%zu", sizeof(raftk_fatigue));'
                    + "".join('printf(" %%zu", offsetof(raftk_fatigue, %s));' % f for f in fields) + 'printf("\\n");return 0;}\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got == [C.sizeof(_lib.RaftkFatigue)] + [getattr(_lib.RaftkFatigue, f).offset for f in fields]
    src = open(os.path.join(ROOT, "include", "raftk.h")).read()
    assert "#define RAFTK_FATIGUE_NB_SWITCH 1e-6" in src


def _base(nU=2, nR=3, n=6, nw=40, nch=2):
    rng = np.random.default_rng(0)
    keep = dict(Xi=np.zeros([nU, nR, n, nw], dtype=np.complex128), w=np.linspace(0.1, 2, nw), R=rng.normal(size=(nch, n)),
                wpow=np.zeros(nch, dtype=np.int32), m=np.full(nch, 4.0), row0=np.array([0, 1, nR], dtype=np.int32),
                DEL=np.zeros([nU, 2, nch]), info=np.zeros([nU, 2, nch], dtype=np.int32), weights=np.ones(2),
                coef=np.zeros([nch, n, nw], dtype=np.complex128))
    from raft_b200 import _lib
    fa = _lib.RaftkFatigue()
    fa.n_cases, fa.n_ch, fa.method, fa.tile_w = 2, nch, 0, 0
    fa.case_row0, fa.R, fa.wpow, fa.R_shared = keep["row0"].ctypes.data, keep["R"].ctypes.data, keep["wpow"].ctypes.data, 1
    fa.m, fa.f_eq, fa.DEL, fa.info = keep["m"].ctypes.data, 1.0, keep["DEL"].ctypes.data, keep["info"].ctypes.data
    return fa, keep, (nU, nR, n, nw)


def _refusals():
    """(name, mutation of (fa, keep, dims) -> dims, the refusal's reason) for every refusal the header lists."""
    def setf(**kv):
        def f(fa, keep, dims):
            for k, v in kv.items():
                setattr(fa, k, v)
            return dims
        return f

    def arr(name, values, field, dtype=float):
        def f(fa, keep, dims):
            keep[name + "_bad"] = np.ascontiguousarray(values, dtype=dtype)
            setattr(fa, field, keep[name + "_bad"].ctypes.data)
            return dims
        return f

    def dims(i, v):
        def f(fa, keep, d):
            d = list(d)
            d[i] = v
            return tuple(d)
        return f
    ge1, req, rows = ">= 1", "are required", "case_row0 must start at 0 and end at n_rows"
    return [
        ("n_units", dims(0, 0), ge1), ("n_rows", dims(1, 0), ge1), ("n_dof", dims(2, 0), ge1), ("nw", dims(3, 0), ge1),
        ("n_cases", setf(n_cases=0), ge1), ("n_ch", setf(n_ch=0), ge1), ("too_many_ch", setf(n_ch=4097), "at most 4096 channels per call"),
        ("no_R_no_coef", setf(R=None), "give exactly one of R"),
        ("both_R_and_coef", lambda fa, k, d: (setattr(fa, "coef", k["coef"].ctypes.data), d)[1], "give exactly one of R"),
        ("R_shared", setf(R_shared=2), "R_shared must be 0 or 1"),
        ("coef_mode", lambda fa, k, d: (setattr(fa, "R", None), setattr(fa, "coef", k["coef"].ctypes.data), setattr(fa, "coef_mode", 3), d)[3],
         "unknown coef_mode"),
        ("method", setf(method=2), "unknown method"), ("wpow", arr("wpow", [0, 3], "wpow", np.int32), "wpow must be 0, 1 or 2"),
        ("wpow_neg", arr("wpow", [-1, 0], "wpow", np.int32), "wpow must be 0, 1 or 2"),
        ("m_null", setf(m=None), req), ("case_row0_null", setf(case_row0=None), req), ("DEL_null", setf(DEL=None), req),
        ("info_null", setf(info=None), req),
        ("row0_start", arr("row0", [1, 2, 3], "case_row0", np.int32), rows), ("row0_end", arr("row0", [0, 1, 2], "case_row0", np.int32), rows),
        ("row0_empty", arr("row0", [0, 0, 3], "case_row0", np.int32), "every case needs at least one row"),
        ("row0_decreasing", arr("row0", [0, 2, 1], "case_row0", np.int32), rows),
        ("m_zero", arr("m", [4.0, 0.0], "m"), "every m must be finite and > 0"), ("m_neg", arr("m", [-3.0, 4.0], "m"), "every m must be finite and > 0"),
        ("m_nan", arr("m", [np.nan, 4.0], "m"), "every m must be finite and > 0"), ("m_inf", arr("m", [np.inf, 4.0], "m"), "every m must be finite and > 0"),
        ("f_eq_zero", setf(f_eq=0.0), "f_eq must be finite and > 0"), ("f_eq_neg", setf(f_eq=-1.0), "f_eq must be finite and > 0"),
        ("f_eq_nan", setf(f_eq=float("nan")), "f_eq must be finite and > 0"),
        ("weights_neg", arr("weights", [1.0, -1.0], "weights"), "weights must be finite and >= 0"),
        ("weights_zero", arr("weights", [0.0, 0.0], "weights"), "the weights must not all be 0"),
        ("weights_nan", arr("weights", [np.nan, 1.0], "weights"), "weights must be finite and >= 0"),
    ]


@pytest.mark.parametrize("name", [r[0] for r in _refusals()])
def test_every_refusal_before_any_launch(name):
    """RAFTK_EINVAL (-1) from both entries with the refusal's reason after the "fatigue: " prefix, before any launch
    (raftk_launch_count unchanged), for each refusal of the header."""
    from raft_b200 import _lib
    lib = _lib.lib
    mut, msg = {r[0]: r[1:] for r in _refusals()}[name]
    for entry in ("host", "dev"):
        fa, keep, dims = _base()
        dims = mut(fa, keep, dims)
        n0 = lib.raftk_launch_count()
        if entry == "host":
            rc = lib.raftk_fatigue_host(*dims, keep["w"].ctypes.data, keep["Xi"].ctypes.data, C.byref(fa))
        else:
            rc = lib.raftk_fatigue_dev(*dims, keep["w"].ctypes.data, keep["Xi"].ctypes.data, C.byref(fa), keep["Xi"].ctypes.data, 1 << 30, None)
        assert rc == -1, (name, entry, rc)
        assert lib.raftk_launch_count() == n0
        err = lib.raftk_last_error().decode()
        assert err.startswith("fatigue: ") and msg in err, (name, entry, err)


def test_refusals_without_inputs_and_small_workspace():
    """NULL w / Xi / struct and a workspace below raftk_fatigue_workspace_bytes are refused before any launch; the size query
    matches the header's formula."""
    from raft_b200 import _lib
    lib = _lib.lib
    fa, keep, dims = _base()
    n0 = lib.raftk_launch_count()
    assert lib.raftk_fatigue_host(*dims, None, keep["Xi"].ctypes.data, C.byref(fa)) == -1
    assert lib.raftk_fatigue_host(*dims, keep["w"].ctypes.data, None, C.byref(fa)) == -1
    assert lib.raftk_fatigue_host(*dims, keep["w"].ctypes.data, keep["Xi"].ctypes.data, None) == -1
    nU, nR, n, nw = dims
    need = lib.raftk_fatigue_workspace_bytes(nU, nR, nw, C.byref(fa))
    assert need == nU * nR * ((nw + 31) // 32) * 2 * 4 * 8
    life = np.zeros([nU, 2])
    fa.DEL_life = life.ctypes.data
    assert lib.raftk_fatigue_workspace_bytes(nU, nR, nw, C.byref(fa)) == need + nU * 2 * 2 * 8
    ws = keep["Xi"].ctypes.data
    assert lib.raftk_fatigue_dev(*dims, keep["w"].ctypes.data, ws, C.byref(fa), ws, need, None) == -1
    assert lib.raftk_fatigue_dev(*dims, keep["w"].ctypes.data, ws, C.byref(fa), None, need + nU * 32, None) == -1
    assert lib.raftk_launch_count() == n0


def test_python_refusals():
    from raft_b200 import solver
    Xi = np.zeros([3, 6, 40], dtype=np.complex128)
    w = np.linspace(0.1, 2, 40)
    R = np.eye(6)[:2]
    for kw in (dict(), dict(R=R, coef=np.zeros([2, 6, 40])), dict(R=R, method="rainflow"), dict(R=R, m=0.0), dict(R=R, f_eq=0.0),
               dict(R=R, wpow=[0, 3]), dict(R=R, weights=[0.0, 0.0, 0.0]), dict(R=R, case_row0=[0, 2]), dict(R=np.eye(5)[:2]),
               dict(coef=np.zeros([2, 6, 39])), dict(coef=np.zeros([2, 6, 40]), wpow=[0, 1])):
        kw.setdefault("m", 4.0)
        with pytest.raises(ValueError):
            solver.fatigue(Xi, w, **kw)


# ---- on an H100 ----------------------------------------------------------------------------------------------------------
def _ref_moments(psd, w, div):
    """lambda_k = sum_j w_j^k PSD_j * divisor of a reference PSD [nw]."""
    return np.array([np.sum(w ** k * psd * div) for k in (0, 1, 2, 4)])


def _close(a, b, tol):
    a, b = np.asarray(a, dtype=float), np.asarray(b, dtype=float)
    return np.all(np.abs(a - b) <= tol * np.abs(b))


@pytest.mark.gpu
def test_moments_against_reference_psds_mbase():
    """Device moments of the rigid-tower Mbase (complex coefficients) against the unmodified reference's Mbase_PSD x dw:
    turb_VolturnUS-S (one coefficient set), ops_VolturnUS-S (per-case operating points: one set per row, every case in one
    call) and every FOWT of ops_farm / ops_farm24 (FOWT i's coefficients on columns 6 i .. 6 i + 5 of Xi_sys), 1e-10."""
    from raft_b200 import solver
    z = np.load(os.path.join(GOLDEN, "turb_VolturnUS-S.npz"))
    w, dw = z["P_w"], float(z["P_dw"])
    k = [n.split(":")[0] for n in z["ch_names"]].index("Mbase")
    ic = 0
    while "ref_run_case%d_Xi" % ic in z.files:
        r = solver.fatigue(z["ref_run_case%d_Xi" % ic], w, 4.0, coef=z["ch_coef"][k:k + 1], case_row0=[0, len(z["ref_run_case%d_Xi" % ic])])
        assert _close(r["moments"][0, 0], _ref_moments(z["ref_run_case%d_Mbase_PSD" % ic][:, 0], w, dw), 1e-10), ic
        ic += 1
    assert ic >= 3
    for name in ("ops_VolturnUS-S", "ops_farm", "ops_farm24"):
        z = np.load(os.path.join(GOLDEN, name + ".npz"))
        w = z["w"]
        dw = w[1] - w[0]
        nF = int(z["n_fowt"])
        nC = len([f for f in z.files if f.startswith("Xi_c")])
        Xi = np.concatenate([z["Xi_c%d" % c] for c in range(nC)])
        row0 = np.cumsum([0] + [len(z["Xi_c%d" % c]) for c in range(nC)])
        n = Xi.shape[1]
        coef = np.zeros([1, len(Xi), nF, n, len(w)], dtype=np.complex128)     # one set per row: the case's operating point
        for c in range(nC):
            for f in range(nF):
                coef[0, row0[c]:row0[c + 1], f, 6 * f:6 * f + 6] = z["ch%d_c%d_coef" % (f, c)][3]
        r = solver.fatigue(Xi, w, 4.0, coef=coef, case_row0=row0)
        for c in range(nC):
            for f in range(nF):
                ref = _ref_moments(z["cm%d_Mbase_PSD_c%d" % (f, c)][:, 0], w, dw)
                assert _close(r["moments"][c, f], ref, 1e-10), (name, c, f)


@pytest.mark.gpu
def test_moments_against_reference_psds_tensions_and_tower_loads():
    """Device moments of real rows against the reference's PSDs: Tmoor of tmoor_VolturnUS-S (J on Xi), tmoor_VolturnUS-S-
    flexible (J on the PRP motions), the arrays of tmoor_farm / tmoor_farm24 (J_arr on Xi_sys), all with the w[0] divisor of
    Tmoor_PSD; FbaseX .. MbaseZ of flexout_VolturnUS-S-flexible and flexops_{strip,bem}_VolturnUS-S-flexible (150 DOFs, the
    packed rows with their w powers, divisor dw), 1e-10."""
    from raft_b200 import solver
    for name in ("tmoor_VolturnUS-S", "tmoor_VolturnUS-S-flexible", "tmoor_farm", "tmoor_farm24"):
        z = np.load(os.path.join(GOLDEN, name + ".npz"))
        w = z["w"]
        nC = len([f for f in z.files if f.startswith("Xi_c")])
        arr = "J_arr" in z.files
        J = z["J_arr"] if arr else z["J0"]
        for c in range(nC):
            X = z["Xi_PRP"][c] if "Xi_PRP" in z.files else z["Xi_c%d" % c]
            r = solver.fatigue(X, w, 3.0, R=J, case_row0=[0, len(X)])
            ref = z["arr_Tmoor_PSD"][c] if arr else z["fowt0_Tmoor_PSD"][c]
            for k in range(J.shape[0]):
                assert _close(r["moments"][0, k], _ref_moments(ref[k], w, w[0]), 1e-10), (name, c, k)
    for name in ("flexout_VolturnUS-S-flexible", "flexops_strip_VolturnUS-S-flexible", "flexops_bem_VolturnUS-S-flexible"):
        z = np.load(os.path.join(GOLDEN, name + ".npz"))
        w, dw = z["P_w"] if "P_w" in z.files else z["w"], None
        dw = w[1] - w[0]
        names = [s.split(":")[0] for s in z["ch_names"]]
        sel = [names.index(s) for s in ("FbaseX", "FbaseY", "FbaseZ", "MbaseX", "MbaseY", "MbaseZ")]
        ic = 0
        while "ref_run_case%d_Xi" % ic in z.files:
            X = z["ref_run_case%d_Xi" % ic]
            r = solver.fatigue(X, w, 4.0, R=z["ch_R"][sel], wpow=z["ch_wpow"][sel], case_row0=[0, len(X)])
            for j, k in enumerate(sel):
                ref = z["ref_run_case%d_%s_PSD" % (ic, names[k])][:, 0]
                assert _close(r["moments"][0, j], _ref_moments(ref, w, dw), 1e-10), (name, ic, names[k])
            ic += 1
        assert ic >= 2


def _random_problem(rng, U, nR, n, nw, nch, form):
    Xi = (rng.normal(size=(U, nR, n, nw)) + 1j * rng.normal(size=(U, nR, n, nw))) * rng.uniform(0.1, 10, size=(U, 1, n, 1))
    w = np.arange(1, nw + 1) * 0.05
    if form == "R":
        return Xi, w, dict(R=rng.normal(size=(U, nch, n)), wpow=rng.integers(0, 3, size=nch).astype(np.int32))
    return Xi, w, dict(coef=rng.normal(size=(U, nR, nch, n, nw)) + 1j * rng.normal(size=(U, nR, nch, n, nw)))


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["R", "coef"])
@pytest.mark.parametrize("method", ["dirlik", "narrowband"])
def test_against_restatement(form, method):
    """DEL, info, moments and DEL_life against the numpy restatement, 1e-12 relative, with wave trains (cases of 1-3 rows),
    weights, zero channels (ZERO) and single-bin channels (the narrow-band fallback)."""
    from raft_b200 import solver
    rng = np.random.default_rng(7)
    U, n, nw, nch = 3, 6, 70, 5
    row0 = np.array([0, 1, 3, 4, 7], dtype=np.int32)
    Xi, w, ch = _random_problem(rng, U, int(row0[-1]), n, nw, nch, form)
    if form == "R":
        ch["R"][:, 4] = 0.0                                  # a zero row: exactly 0, ZERO
    else:
        ch["coef"][:, :, 4] = 0.0
        ch["coef"][:, :, 3, :, 1:] = 0.0                     # one bin only: the narrow-band limit
    m = np.array([3.0, 4.0, 5.0, 8.0, 10.0])
    weights = np.array([0.1, 0.0, 2.0, 0.5])
    r = solver.fatigue(Xi, w, m, case_row0=row0, weights=weights, method=method, **ch)
    lam = np_moments(np_amplitudes(Xi, w, **ch), w, row0)
    ref = np_fatigue(lam, m, method=method, weights=weights)
    assert _close(r["moments"], lam, 1e-12) or np.allclose(r["moments"], lam, rtol=1e-12, atol=0)
    assert np.array_equal(r["info"], ref["info"])
    assert np.all(r["DEL"][..., 4] == 0) and np.all(r["info"][..., 4] == ZERO)
    if form == "coef":
        assert np.all(r["info"][..., 3] == NARROWBAND)
    assert np.allclose(r["DEL"], ref["DEL"], rtol=1e-12, atol=0)
    assert np.allclose(r["DEL_life"], ref["DEL_life"], rtol=1e-12, atol=0)
    assert np.all(np.isfinite(r["DEL"])) and np.all(np.isfinite(r["DEL_life"]))
    f2 = solver.fatigue(Xi, w, m, case_row0=row0, method=method, f_eq=0.25, **ch)
    assert np.allclose(f2["DEL"], np_fatigue(lam, m, f_eq=0.25, method=method)["DEL"], rtol=1e-12, atol=0) and "DEL_life" not in f2


@pytest.mark.gpu
@pytest.mark.parametrize("n", [6, 48, 150, 600])
def test_batch_and_tile_independence(n):
    """Each (unit, case, channel) is bit-identical solved alone or in a batch, and for every tile width (32 .. 256 bins, and
    the L2 path); n = 600 takes the L2 path by itself (not even 32 bins fit in shared memory)."""
    from raft_b200 import solver
    rng = np.random.default_rng(n)
    U, nw, nch = 3, 100, 6
    row0 = np.array([0, 2, 3], dtype=np.int32)
    Xi, w, ch = _random_problem(rng, U, 3, n, nw, nch, "R")
    full = solver.fatigue(Xi, w, 4.0, case_row0=row0, life=True, **ch)
    for tile in (32, 64, 96, 256, -1):
        t = solver.fatigue(Xi, w, 4.0, case_row0=row0, life=True, tile_w=tile, **ch)
        for k in full:
            assert np.array_equal(t[k], full[k]), (tile, k)
    for u in range(U):
        one = solver.fatigue(Xi[u:u + 1], w, 4.0, case_row0=row0, life=True, R=ch["R"][u:u + 1], wpow=ch["wpow"])
        for k in full:
            assert np.array_equal(one[k][0], full[k][u]), (u, k)
    c1 = solver.fatigue(Xi[:, 2:3], w, 4.0, R=ch["R"], wpow=ch["wpow"])
    assert np.array_equal(c1["DEL"][:, 0], full["DEL"][:, 1])
    sub = solver.fatigue(Xi, w, 4.0, case_row0=row0, R=ch["R"][:, 2:5], wpow=ch["wpow"][2:5])
    assert np.array_equal(sub["DEL"], full["DEL"][..., 2:5]) and np.array_equal(sub["moments"], full["moments"][..., 2:5, :])


@pytest.mark.gpu
def test_sessions_match_host_entry():
    """DeviceSession.fatigue (rigid sweep, one farm and a farm batch), GeneralSession.fatigue and GeneralBatchSession.fatigue
    are bit-identical to solver.fatigue on the same Xi."""
    import torch
    from raft_b200 import solver
    z = np.load(os.path.join(GOLDEN, "turb_VolturnUS-S.npz"))
    P = {k[2:]: z[k] for k in z.files if k.startswith("P_")}
    w = P["w"]
    cases = dict(Hs=np.array([6.0, 8.0, 4.0]), Tp=np.array([10.0, 12.0, 8.0]), gamma=np.zeros(3), beta_deg=np.array([0.0, 30.0, 0.0]),
                 spec=np.zeros(3, dtype=np.int32))
    b = solver.DesignBatch([P, P])
    s = solver.DeviceSession(b, solver.CaseTable(cases), want=("Xi", "status", "B_drag", "F_drag", "F_iner"))
    s.solve(n_iter=int(z["n_iter"]), xi_start=float(z["xi_start"]))
    row0 = np.array([0, 2, 3], dtype=np.int32)
    d = s.fatigue([4.0, 3.0], coef=z["ch_coef"][2:4], case_row0=row0, weights=[1.0, 3.0])
    torch.cuda.synchronize()
    Xi = s.out["Xi"].cpu().numpy()
    h = solver.fatigue(Xi, w, [4.0, 3.0], coef=z["ch_coef"][2:4], case_row0=row0, weights=[1.0, 3.0])
    for k in h:
        assert np.array_equal(d[k].cpu().numpy(), h[k]), k
    J = np.random.default_rng(3).normal(size=(5, 12))
    xs, _ = s.farm_response(n_fowt=None)
    df = s.fatigue(3.0, R=J, farm=True)
    hf = solver.fatigue(xs.cpu().numpy(), w, 3.0, R=J)
    for k in hf:
        assert np.array_equal(df[k].cpu().numpy(), hf[k]), k
    xb, _ = s.farm_response(n_fowt=1)
    db = s.fatigue(3.0, R=J[:, :6], farm=True, n_fowt=1)
    hb = solver.fatigue(xb.cpu().numpy(), w, 3.0, R=J[:, :6])
    for k in hb:
        assert np.array_equal(db[k].cpu().numpy(), hb[k]), k
    g = np.load(os.path.join(GOLDEN, "flexout_VolturnUS-S-flexible.npz"))
    Pg = {k[2:]: g[k] for k in g.files if k.startswith("P_")}
    names = [nm.split(":")[0] for nm in g["ch_names"]]
    sel = [names.index(nm) for nm in ("FbaseX", "MbaseY")]
    from raft_b200 import packer
    tr = g["ref_run_case0_trains"]
    case = dict(wave_spectrum=["JONSWAP"] * 2, wave_height=[float(tr[0, 0]), 2.0], wave_period=[float(tr[0, 1]), 9.0],
                wave_heading=[float(tr[0, 2]), 20.0], wave_gamma=[0.0, 0.0])
    table, owner, first = packer.pack_case_trains([case, case])
    gs = solver.GeneralSession(Pg, g["gen_M"], g["gen_B"], g["gen_C"], solver.CaseTable(table))
    gs.solve(n_iter=int(g["n_iter"]), xi_start=float(g["xi_start"]))
    row0 = np.r_[first, len(table["Hs"])]
    dg = gs.fatigue(4.0, R=g["ch_R"][sel], wpow=g["ch_wpow"][sel], case_row0=row0)
    torch.cuda.synchronize()
    hg = solver.fatigue(gs.Xi.cpu().numpy(), Pg["w"], 4.0, R=g["ch_R"][sel], wpow=g["ch_wpow"][sel], case_row0=row0)
    for k in hg:
        assert np.array_equal(dg[k].cpu().numpy(), hg[k]), k
    gb = solver.GeneralBatchSession([dict(P=Pg, M=g["gen_M"], B=g["gen_B"], Cm=g["gen_C"])] * 2, solver.CaseTable(table))
    gb.solve(n_iter=int(g["n_iter"]), xi_start=float(g["xi_start"]))
    Rb = np.stack([g["ch_R"][sel], 2.0 * g["ch_R"][sel]])
    db = gb.fatigue(4.0, R=Rb, wpow=g["ch_wpow"][sel], case_row0=row0)
    torch.cuda.synchronize()
    hb = solver.fatigue(gb.Xi.cpu().numpy(), Pg["w"], 4.0, R=Rb, wpow=g["ch_wpow"][sel], case_row0=row0)
    for k in hb:
        assert np.array_equal(db[k].cpu().numpy(), hb[k]), k
    assert np.allclose(hb["DEL"][1], 2.0 * hb["DEL"][0], rtol=1e-12)


def test_misaligned_workspace_is_refused():
    """k_fatigue_finish reads the workspace's partial sums as 32-byte vectors: raftk_fatigue_dev refuses a workspace that is
    not 32-byte aligned, before any launch."""
    from raft_b200 import _lib
    lib = _lib.lib
    fa, keep, dims = _base()
    nU, nR, n, nw = dims
    need = lib.raftk_fatigue_workspace_bytes(nU, nR, nw, C.byref(fa))
    buf = np.zeros(need // 8 + 16)
    base = (buf.ctypes.data + 31) // 32 * 32
    n0 = lib.raftk_launch_count()
    for off in (8, 16, 24):
        assert lib.raftk_fatigue_dev(*dims, keep["w"].ctypes.data, keep["Xi"].ctypes.data, C.byref(fa), base + off, need, None) == -1
        assert b"aligned" in lib.raftk_last_error()
    assert lib.raftk_launch_count() == n0


def test_log_domain_restatement_matches_linear_and_stays_finite():
    """The log-domain restatement (the device's evaluation) equals the linear closed form where that is finite, and stays
    finite for a base load of 1e8 at m = 40, where (2 sqrt(l0))^m Gamma(1+m) overflows."""
    w = np.linspace(0.05, 2.0, 40)
    S = np.exp(-0.5 * ((w - 0.6) / 0.15) ** 2) + 0.2 * np.exp(-0.5 * ((w - 1.4) / 0.1) ** 2)
    for scale, ms in ((1.0, (3.0, 4.0, 10.0)), (1e16, (3.0, 4.0, 10.0))):
        lam = np.array([np.sum(w ** k * S * scale) for k in (0, 1, 2, 4)])
        for method in ("dirlik", "narrowband"):
            for m in ms:
                r = np_fatigue(lam[None, None, None], m, method=method)
                d, _ = np_rate(lam, m, method)
                assert r["DEL"][0, 0, 0] == pytest.approx(d ** (1 / m), rel=1e-13)
    lam = np.array([np.sum(w ** k * S * 1e16) for k in (0, 1, 2, 4)])
    with pytest.raises(OverflowError):
        np_rate(lam, 40.0)                                                # the linear form overflows here
    r = np_fatigue(lam[None, None, None], 40.0, weights=[1.0])
    assert np.isfinite(r["DEL"]).all() and np.isfinite(r["DEL_life"]).all()
    assert r["DEL_life"][0, 0] == pytest.approx(r["DEL"][0, 0, 0], rel=1e-13)


# ---- the analysis entry points' fatigue= option ----------------------------------------------------------------------
def _np_fatigue_call(Xi, w, m, R=None, wpow=None, coef=None, case_row0=None, f_eq=1.0, method="dirlik", weights=None, life=None,
                     moments=True, tile_w=0):
    """solver.fatigue restated in numpy (the CPU stand-in of the device call)."""
    Xi = np.asarray(Xi)
    squeeze = Xi.ndim == 3
    X = Xi[None] if squeeze else Xi
    row0 = np.arange(X.shape[1] + 1) if case_row0 is None else np.asarray(case_row0)
    lam = np_moments(np_amplitudes(X, np.asarray(w), R=R, wpow=wpow, coef=coef), np.asarray(w), row0)
    nch = lam.shape[2]
    r = np_fatigue(lam, np.broadcast_to(np.asarray(m, dtype=float), (nch,)), f_eq, method, weights)
    out = dict(DEL=r["DEL"], info=r["info"])
    if moments:
        out["moments"] = lam
    if (weights is not None) if life is None else life:
        out["DEL_life"] = r["DEL_life"]
    return {k: v[0] for k, v in out.items()} if squeeze else out


def _general_stand_in(monkeypatch, nw=24):
    """general_analyze_cases on the CPU: the device solve, channel statistics and fatigue replaced by seeded numpy stand-ins."""
    from raft_b200 import solver
    rng = np.random.default_rng(11)

    def solve(P, M, B, Cm, ct, **kw):
        nT = ct.n_cases
        X = rng.normal(size=(nT, 8, nw)) + 1j * rng.normal(size=(nT, 8, nw))
        return X, np.zeros([nT, 4], dtype=np.int32)

    def stats(R, wpow, w, Xi, dw, psd=True, amp=False):
        Y = np.einsum("kb,tbw->tkw", R, Xi) * np.asarray(w)[None, None] ** np.asarray(wpow)[None, :, None]
        return np.sqrt(0.5 * (np.abs(Y) ** 2).sum(-1)), 0.5 * np.abs(Y) ** 2 / dw, Y
    monkeypatch.setattr(solver, "general_solve_dynamics", solve)
    monkeypatch.setattr(solver, "general_channel_stats", stats)
    monkeypatch.setattr(solver, "fatigue", _np_fatigue_call)
    names = [("surge", None), ("pitch", None), ("FbaseX", 0), ("MbaseY", 0), ("Tmoor", 0), ("Tmoor", 1), ("Tmoor", 2)]
    channels = dict(names=names, R=rng.normal(size=(len(names), 8)), wpow=np.array([0, 0, 2, 2, 0, 0, 0], dtype=np.int32),
                    avg=np.zeros(len(names)), tension=dict(row0=4, T0=np.ones(3), w0=0.1))
    P = dict(w=np.arange(1, nw + 1) * 0.1, dw=0.1)
    cases = [dict(wave_spectrum="JONSWAP", wave_height=4.0, wave_period=9.0, wave_heading=0.0),
             dict(wave_spectrum=["JONSWAP"] * 2, wave_height=[4.0, 2.0], wave_period=[9.0, 12.0], wave_heading=[0.0, 30.0],
                  wave_gamma=[0.0, 0.0]),
             dict(wave_spectrum="JONSWAP", wave_height=6.0, wave_period=11.0, wave_heading=10.0)]
    return solver, P, channels, cases


def test_general_analyze_cases_fatigue_option_on_cpu(monkeypatch):
    """general_analyze_cases without fatigue= returns its usual keys (Xi_trains, status, case_metrics) and per case exactly
    the saveTurbineOutputs keys; with fatigue= it adds only the named <name>_DEL entries (Mbase_DEL the alias of MbaseY_DEL,
    Tmoor_DEL [2L], FbaseX_DEL [nrot]) with the restatement's values, and with weights results['fatigue'] the lifetime DELs;
    every other value is unchanged.  Unknown channel names and options are refused."""
    solver, P, channels, cases = _general_stand_in(monkeypatch)
    base = solver.general_analyze_cases(P, None, None, None, cases, channels=channels)
    assert sorted(base) == ["Xi_trains", "case_metrics", "status"]
    keys0 = {k for c in base["case_metrics"].values() for k in c}
    assert not any(k.endswith("_DEL") for k in keys0) and "Mbase_std" in keys0 and "Tmoor_std" in keys0
    _, P, channels, cases = _general_stand_in(monkeypatch)
    fat = dict(m={"Mbase": 4.0, "FbaseX": 5.0, "Tmoor": 3.0}, weights=[0.5, 0.3, 0.2])
    res = solver.general_analyze_cases(P, None, None, None, cases, channels=channels, fatigue=fat)
    assert sorted(res) == ["Xi_trains", "case_metrics", "fatigue", "status"]
    Xi = np.concatenate(res["Xi_trains"])
    row0 = np.cumsum([0] + [len(x) for x in res["Xi_trains"]])
    for ic, mt in res["case_metrics"].items():
        assert set(mt) == set(base["case_metrics"][ic]) | {"Mbase_DEL", "FbaseX_DEL", "Tmoor_DEL"}
        for k in base["case_metrics"][ic]:
            assert np.array_equal(np.asarray(mt[k]), np.asarray(base["case_metrics"][ic][k])), (ic, k)
        assert mt["Mbase_DEL"].shape == (1,) and mt["FbaseX_DEL"].shape == (1,) and mt["Tmoor_DEL"].shape == (3,)
    R, wp = channels["R"], channels["wpow"]
    ref = _np_fatigue_call(Xi, P["w"], [5.0, 4.0, 3.0, 3.0, 3.0], R=R[[2, 3, 4, 5, 6]], wpow=wp[[2, 3, 4, 5, 6]], case_row0=row0,
                           weights=fat["weights"])
    for ic in range(3):
        assert res["case_metrics"][ic]["FbaseX_DEL"][0] == ref["DEL"][ic, 0]
        assert res["case_metrics"][ic]["Mbase_DEL"][0] == ref["DEL"][ic, 1]
        assert np.array_equal(res["case_metrics"][ic]["Tmoor_DEL"], ref["DEL"][ic, 2:])
    assert np.array_equal(res["fatigue"]["Tmoor_DEL"], ref["DEL_life"][2:]) and res["fatigue"]["Mbase_DEL"][0] == ref["DEL_life"][1]
    for bad in (dict(m={"Nope": 3.0}), dict(m={}), dict(m={"Mbase": 0.0}), dict(m={"Mbase": 3.0}, f=1)):
        with pytest.raises(ValueError):
            solver.general_analyze_cases(P, None, None, None, cases, channels=channels, fatigue=bad)


def _model_stand_in(monkeypatch):
    """Model.analyzeCases on the CPU: the batched device solve and the device statistics replaced by numpy stand-ins."""
    from raft_b200 import solver
    from raft_b200.model import Model
    rng = np.random.default_rng(5)

    def solve_batch(self, cases, tol, icases=None):
        from raft_b200 import packer
        table, owner, first = packer.pack_case_trains(cases)
        nT = len(owner)
        X = rng.normal(size=(nT, self.nDOF, self.nw)) + 1j * rng.normal(size=(nT, self.nDOF, self.nw))
        return dict(Xi=X[first], Xi_trains=[X[owner == c] for c in range(len(cases))], status=np.zeros([len(cases), self.nFOWT, 4]),
                    Xi_all=X, owner=owner, zeta=rng.normal(size=(nT, self.nw)) + 0j)

    def response_stats(Xi, dw, psd=True, rot_deg=True):
        a = 0.5 * np.abs(Xi) ** 2
        return np.sqrt(a.sum(-1)), a / dw

    def channel_stats(coef, Xi, dw, psd=True, amp=False):
        Y = np.einsum("kaw,taw->tkw", coef, Xi) if coef.ndim == 3 else np.einsum("ckaw,cdaw->cdkw", coef, Xi)
        a = 0.5 * np.abs(Y) ** 2
        return np.sqrt(a.sum(-1)), a / dw, Y

    def farm_channel_stats(R, Xi, dw, **kw):
        a = 0.5 * np.abs(np.einsum("kb,tbw->tkw", R, Xi)) ** 2
        return np.sqrt(a.sum(-1)), a / dw, None
    monkeypatch.setattr(Model, "_solve_batch", solve_batch)
    monkeypatch.setattr(solver, "response_stats", response_stats)
    monkeypatch.setattr(solver, "channel_stats", channel_stats)
    monkeypatch.setattr(solver, "farm_channel_stats", farm_channel_stats)
    monkeypatch.setattr(solver, "fatigue", _np_fatigue_call)
    D = json.load(open(os.path.join(GOLDEN, "designs.json")))["farm_VolturnUS-S_farm_nw48"]
    design = dict(settings=D["settings"], site=D["site"], platform=D["platform"], array=D["array"])
    return Model, design, rng


def test_model_fatigue_option_on_cpu(monkeypatch):
    """Model.analyzeCases without fatigue= keeps its keys; with fatigue= (m={'Mbase': 4, 'Tmoor': 3}) every case and FOWT gets
    Mbase_DEL [nrot] (turbine channels) and Tmoor_DEL [2L] (its lines), the array gets array_mooring['Tmoor_DEL'] [2L], and
    with weights results['fatigue'] holds the lifetime DELs; all other entries are unchanged."""
    Model, design, rng = _model_stand_in(monkeypatch)
    J, T0 = rng.normal(size=(6, 6)), np.ones(6)
    Ja, T0a = rng.normal(size=(10, 12)), np.ones(10)
    cases = [dict(wave_spectrum="JONSWAP", wave_height=H, wave_period=T, wave_heading=0.0) for H, T in ((6.0, 12.0), (3.5, 9.0))]

    def run(fatigue):
        m0 = Model(json.loads(json.dumps(design)), array_stiffness=np.eye(12), tension_jacobian=[J, None], mean_tensions=[T0, None],
                   array_tension_jacobian=Ja, array_mean_tensions=T0a, channels=[ch, ch], fatigue=fatigue)
        return m0, m0.analyzeCases(cases=cases)
    nw_ = len(Model(json.loads(json.dumps(design)), array_stiffness=np.eye(12)).w)
    ch = dict(names=[("AxRNA", 0), ("Mbase", 0)], coef=rng.normal(size=(2, 6, nw_)) + 1j * rng.normal(size=(2, 6, nw_)), avg=np.zeros(2))
    state = rng.bit_generator.state
    _, base = run(None)
    rng.bit_generator.state = state
    model, res = run(dict(m={"Mbase": 4.0, "Tmoor": 3.0}, weights=[1.0, 3.0]))
    assert set(res) == set(base) | {"fatigue"} and "fatigue" not in base
    for ic in range(2):
        for i in range(2):
            a, b = res["case_metrics"][ic][i], base["case_metrics"][ic][i]
            extra = {"Mbase_DEL"} | ({"Tmoor_DEL"} if i == 0 else set())
            assert set(a) == set(b) | extra
            for k in b:
                assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), (ic, i, k)
            assert a["Mbase_DEL"].shape == (1,) and np.isfinite(a["Mbase_DEL"]).all()
        assert res["case_metrics"][ic][0]["Tmoor_DEL"].shape == (6,)
        am = res["case_metrics"][ic]["array_mooring"]
        assert set(am) == set(base["case_metrics"][ic]["array_mooring"]) | {"Tmoor_DEL"} and am["Tmoor_DEL"].shape == (10,)
    assert res["fatigue"][0]["Tmoor_DEL"].shape == (6,) and res["fatigue"]["array_mooring"]["Tmoor_DEL"].shape == (10,)
    assert res["fatigue"][1]["Mbase_DEL"].shape == (1,) and "Tmoor_DEL" not in res["fatigue"][1]
    with pytest.raises(ValueError):
        Model(json.loads(json.dumps(design)), array_stiffness=np.eye(12), fatigue=dict(m={"Mbase": 4.0}))


@pytest.mark.gpu
def test_large_loads_and_exponents_stay_finite_on_device():
    """A base load of 1e8 at m = 40 (where (2 sqrt(l0))^m Gamma(1+m) overflows in linear form): the device's log-domain DEL
    and DEL_life are finite and equal the restatement to 1e-12, for both methods."""
    from raft_b200 import solver
    rng = np.random.default_rng(21)
    nw = 60
    w = np.arange(1, nw + 1) * 0.05
    Xi = (rng.normal(size=(2, 3, 6, nw)) + 1j * rng.normal(size=(2, 3, 6, nw))) * 3e7
    R = rng.normal(size=(2, 6))
    row0 = np.array([0, 2, 3], dtype=np.int32)
    for method in ("dirlik", "narrowband"):
        r = solver.fatigue(Xi, w, [40.0, 60.0], R=R, case_row0=row0, weights=[1.0, 2.0], method=method)
        lam = np_moments(np_amplitudes(Xi, w, R=R), w, row0)
        assert lam[..., 0].min() > 1e15
        ref = np_fatigue(lam, [40.0, 60.0], method=method, weights=[1.0, 2.0])
        assert np.isfinite(r["DEL"]).all() and np.isfinite(r["DEL_life"]).all()
        assert np.allclose(r["DEL"], ref["DEL"], rtol=1e-12, atol=0) and np.allclose(r["DEL_life"], ref["DEL_life"], rtol=1e-12, atol=0)


@pytest.mark.gpu
def test_model_fatigue_fills_reference_keys():
    """Model(fatigue=dict(m={'Mbase': 4, 'Tmoor': 3}, weights=...)).analyzeCases() on VolturnUS-S with its turbine channels and a
    tension Jacobian: every case's Mbase_DEL [nrot] and Tmoor_DEL [2L] (the shapes of omdao_raft.py's stats_Mbase_DEL [n_cases]
    and stats_Tmoor_DEL [n_cases, 2 nlines] per case) equal solver.fatigue on the case's trains; results['fatigue'] the
    lifetime DELs; without fatigue= the results have the same keys and values as before."""
    from raft_b200 import solver
    from raft_b200.model import Model
    from conftest import load_golden
    z = np.load(os.path.join(GOLDEN, "turb_VolturnUS-S.npz"))
    P = {k[2:]: z[k] for k in z.files if k.startswith("P_")}
    G0, _ = load_golden("test_VolturnUS-S")
    D = json.load(open(os.path.join(GOLDEN, "designs.json")))["test_VolturnUS-S"]
    mats = dict(M_struc=P["M0"] - G0["A_hydro_morison"], C_struc=P["C0"] - G0["C_moor"], C_moor=G0["C_moor"], B_struc=P["B0"])
    ch = dict(names=[(n.split(":")[0], int(n.split(":")[1])) for n in z["ch_names"]], coef=z["ch_coef"], avg=z["ch_avg"])
    J, T0 = np.random.default_rng(2).normal(size=(6, 6)) * 1e4, np.full(6, 1e6)
    cases = []
    for ic in range(3):
        tr = z["ref_run_case%d_trains" % ic]
        cases.append(dict(wave_spectrum=["JONSWAP"] * len(tr), wave_height=list(tr[:, 0]), wave_period=list(tr[:, 1]),
                          wave_heading=list(tr[:, 2]), wave_gamma=[0.0] * len(tr)))

    def model(**kw):
        design = dict(D, site=dict(D["site"], water_depth=float(P["depth"])))
        return Model(design, matrices=mats, channels=ch, tension_jacobian=J, mean_tensions=T0, **kw)
    base = model().analyzeCases(cases=cases)
    wts = [0.2, 0.5, 0.3]
    m = model(fatigue=dict(m={"Mbase": 4.0, "Tmoor": 3.0}, weights=wts))
    res = m.analyzeCases(cases=cases)
    assert set(res) == set(base) | {"fatigue"}
    Xi = np.concatenate(res["Xi_trains"])
    row0 = np.cumsum([0] + [len(x) for x in res["Xi_trains"]])
    k = [n for n, _ in ch["names"]].index("Mbase")
    rM = solver.fatigue(Xi, m.w, 4.0, coef=z["ch_coef"][k:k + 1], case_row0=row0, weights=wts)
    rT = solver.fatigue(Xi, m.w, 3.0, R=J, case_row0=row0, weights=wts)
    for ic in range(3):
        a, b = res["case_metrics"][ic][0], base["case_metrics"][ic][0]
        assert set(a) == set(b) | {"Mbase_DEL", "Tmoor_DEL"}
        for key in b:
            assert np.array_equal(np.asarray(a[key]), np.asarray(b[key])), (ic, key)
        assert a["Mbase_DEL"].shape == (1,) and a["Tmoor_DEL"].shape == (6,)
        assert a["Mbase_DEL"][0] == rM["DEL"][ic, 0] and np.array_equal(a["Tmoor_DEL"], rT["DEL"][ic])
    assert res["fatigue"][0]["Mbase_DEL"][0] == rM["DEL_life"][0] and np.array_equal(res["fatigue"][0]["Tmoor_DEL"], rT["DEL_life"])
    stats_Mbase_DEL = np.array([res["case_metrics"][ic][0]["Mbase_DEL"][0] for ic in range(3)])
    stats_Tmoor_DEL = np.stack([res["case_metrics"][ic][0]["Tmoor_DEL"] for ic in range(3)])
    assert stats_Mbase_DEL.shape == (3,) and stats_Tmoor_DEL.shape == (3, 6) and np.all(stats_Mbase_DEL > 0)


@pytest.mark.gpu
def test_general_analyze_cases_fatigue_on_device():
    """general_analyze_cases(fatigue=) and general_analyze_cases_batch(fatigue=) on the 150-DOF flexible fixture: Mbase_DEL
    (the alias of MbaseY_DEL), FbaseX_DEL equal solver.fatigue on the returned trains; without fatigue= the results are
    unchanged; every design of the batch equals its own single-design run."""
    from raft_b200 import packer, solver
    g = np.load(os.path.join(GOLDEN, "flexout_VolturnUS-S-flexible.npz"))
    Pg = {k[2:]: g[k] for k in g.files if k.startswith("P_")}
    names = [(nm.split(":")[0], int(nm.split(":")[1]) if nm.split(":")[1] else None) for nm in g["ch_names"]]
    channels = dict(names=names, R=g["ch_R"], wpow=g["ch_wpow"], avg=g["ch_avg"])
    cases = []
    for ic in range(3):
        tr = g["ref_run_case%d_trains" % ic]
        cases.append(dict(wave_spectrum=["JONSWAP"] * len(tr), wave_height=list(tr[:, 0]), wave_period=list(tr[:, 1]),
                          wave_heading=list(tr[:, 2]), wave_gamma=[0.0] * len(tr)))
    kw = dict(n_iter=int(g["n_iter"]), xi_start=float(g["xi_start"]))
    base = solver.general_analyze_cases(Pg, g["gen_M"], g["gen_B"], g["gen_C"], cases, channels=channels, **kw)
    fat = dict(m={"Mbase": 4.0, "FbaseX": 5.0}, weights=[1.0, 1.0, 2.0])
    res = solver.general_analyze_cases(Pg, g["gen_M"], g["gen_B"], g["gen_C"], cases, channels=channels, fatigue=fat, **kw)
    Xi = np.concatenate(res["Xi_trains"])
    row0 = np.cumsum([0] + [len(x) for x in res["Xi_trains"]])
    nm = [n for n, _ in names]
    sel = [nm.index("FbaseX"), nm.index("MbaseY")]
    r = solver.fatigue(Xi, Pg["w"], [5.0, 4.0], R=g["ch_R"][sel], wpow=g["ch_wpow"][sel], case_row0=row0, weights=fat["weights"])
    for ic in range(3):
        a, b = res["case_metrics"][ic], base["case_metrics"][ic]
        assert set(a) == set(b) | {"Mbase_DEL", "FbaseX_DEL"}
        for key in b:
            assert np.array_equal(np.asarray(a[key]), np.asarray(b[key])), (ic, key)
        assert a["FbaseX_DEL"][0] == r["DEL"][ic, 0] and a["Mbase_DEL"][0] == r["DEL"][ic, 1]
    assert res["fatigue"]["Mbase_DEL"][0] == r["DEL_life"][1]
    bres = solver.general_analyze_cases_batch([dict(P=Pg, M=g["gen_M"], B=g["gen_B"], Cm=g["gen_C"])] * 2, cases,
                                              channels=[channels, channels], fatigue=fat, **kw)
    for d in range(2):
        for ic in range(3):
            for key in ("Mbase_DEL", "FbaseX_DEL"):
                assert np.allclose(bres[d]["case_metrics"][ic][key], res["case_metrics"][ic][key], rtol=1e-10, atol=0), (d, ic, key)
