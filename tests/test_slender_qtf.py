"""Slender-body QTF kernels (potSecOrder 1: k_slender_tables, k_slender_pairs, k_slender_fill) against the C oracle where the
VolturnUS-S fixture never goes: more strip nodes and members than a CTA has threads, all three depth branches of the wave
kinematics, inclined and tapered MacCamy-Fuchs members, added mass varying along a member, 1 .. 160 second-order
frequencies and 1 .. 64 (heading, RAO) pairs per call.  The Kim & Yue correction alone is also checked against a 30-digit
restatement (mpmath Hankel functions), which is the only independent check of the Bessel values of CUDA's jn / yn and
glibc's.  Further: the device entry point (bits, workspace size, argument checks) and the solve flow with two designs.

Every comparison is per DOF over all frequency pairs (|q - q_ref| max / |q_ref| max), and the lower triangle must be the
exact conjugate of the upper one."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import GOLDEN, relerr, response_err

pytestmark = pytest.mark.gpu
BOUND = 1e-12                 # per-DOF error against the oracle (fp64 both sides; the measured errors are ~1e-15)
RAFTK_EINVAL, RAFTK_ENOMEM = -1, -3


@pytest.fixture(scope="module")
def solver():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from raft_b200 import solver as s
    return s


def dof_err(q, ref):
    """max over DOFs of max |q - ref| / max |ref| over every frequency pair; a DOF that is exactly zero must stay so."""
    err = 0.0
    for a in range(6):
        d, s = np.abs(q[..., a] - ref[..., a]).max(), np.abs(ref[..., a]).max()
        assert s > 0 or d == 0, a
        err = max(err, d / s if s > 0 else 0.0)
    return err


def hermitian_exact(q):
    off = ~np.eye(q.shape[0], dtype=bool)
    return np.array_equal(q[off], np.conj(np.swapaxes(q, 0, 1))[off])


def compare_with_oracle(solver, oracle, P, betas, Xi, label):
    """All (heading, RAO) pairs in one GPU call, each against the oracle -> largest per-DOF error."""
    q = solver.qtf_slender(P, betas, Xi)
    od = oracle.OracleDesign(P)
    err = 0.0
    for c in range(len(betas)):
        assert hermitian_exact(q[c]), (label, c)
        err = max(err, dof_err(q[c], oracle.qtf_slender(od, betas[c], Xi[c])))
    print("%s: largest per-DOF error vs oracle %.2e (%d cases, nw2 %d, %d nodes, %d members)"
          % (label, err, len(betas), len(P["qs_w"]), len(P["qs_node_mem"]), len(P["qs_mem_mcf"])))
    assert err < BOUND, (label, err)
    return q


# ---- designs built by the project's own builder ------------------------------------------------------------------------

def _member(rng, i, zlo, dls):
    kind = int(rng.integers(0, 5))
    zA = -rng.uniform(0.2, 1.0) * zlo
    if kind == 0:      # vertical column through the waterline, tapered
        x, y = rng.uniform(-40, 40, 2)
        rA, rB = [x, y, zA], [x, y, rng.uniform(2, 15)]
    elif kind == 1:    # horizontal pontoon
        rA = [rng.uniform(-40, 40), rng.uniform(-40, 40), zA]
        rB = [rA[0] + rng.uniform(5, 40), rA[1] + rng.uniform(-30, 30), zA]
    elif kind == 2:    # inclined brace through the waterline
        rA = [rng.uniform(-40, 40), rng.uniform(-40, 40), zA]
        rB = [rA[0] + rng.uniform(-30, 30), rA[1] + rng.uniform(-30, 30), rng.uniform(2, 12)]
    elif kind == 3:    # submerged inclined brace
        rA = [rng.uniform(-40, 40), rng.uniform(-40, 40), zA]
        rB = [rA[0] + rng.uniform(-30, 30), rA[1] + rng.uniform(-30, 30), zA * rng.uniform(0.1, 0.9)]
    else:              # end A above water
        rA = [rng.uniform(-40, 40), rng.uniform(-40, 40), rng.uniform(2, 10)]
        rB = [rA[0] + rng.uniform(-20, 20), rA[1] + rng.uniform(-20, 20), zA]
    rect = rng.random() < 0.3
    nst = int(rng.integers(2, 5))
    st = np.sort(rng.uniform(0, 1, nst))
    st[0], st[-1] = 0.0, 1.0
    d = [[float(rng.uniform(2, 8)), float(rng.uniform(2, 8))] for _ in range(nst)] if rect else [float(rng.uniform(2, 10)) for _ in range(nst)]
    return dict(name="m%d" % i, type="rigid", rA=[float(v) for v in rA], rB=[float(v) for v in rB], shape="rect" if rect else "circ",
                stations=[float(v) for v in st], d=d, gamma=float(rng.uniform(0, 90)) if rect else 0.0,
                MCF=bool(not rect and rng.random() < 0.7), Cd=0.8,
                Ca=[[float(rng.uniform(0.4, 1.2)), float(rng.uniform(0.4, 1.2))] for _ in range(nst)],     # per station, both directions
                CaEnd=[float(rng.uniform(0.3, 1.0)) for _ in range(nst)], CdEnd=0.6, dlsMax=float(dls))


def _pile(rng, i):
    """Short vertical MacCamy-Fuchs pile through the waterline (few strip nodes, its own Kim & Yue term)."""
    x, y = rng.uniform(-60, 60, 2)
    return dict(name="p%d" % i, type="rigid", rA=[float(x), float(y), -float(rng.uniform(4, 9))], rB=[float(x), float(y), float(rng.uniform(2, 6))],
                shape="circ", stations=[0.0, 1.0], d=[float(rng.uniform(1.0, 3.0)), float(rng.uniform(1.0, 3.0))], MCF=True,
                Cd=0.8, Ca=[[0.7, 0.8], [1.0, 0.9]], CaEnd=0.6, CdEnd=0.6, dlsMax=2.0)


def slender_design(seed, depth, nw2, f_hi, n_members=0, n_piles=0, dls=(1.5, 6.0)):
    """potSecOrder-1 design from the project's builder -> packed tables (qs_* included).  The second-order grid is
    nw2 frequencies df, 2 df, .. nw2 df [Hz] with df = f_hi / nw2 (min_freq2nd = df_freq2nd = df)."""
    from raft_b200 import grid
    from raft_b200.fowt import FOWT
    rng = np.random.default_rng(seed)
    zlo = min(40.0, 0.8 * depth)
    members = [_member(rng, i, zlo, rng.uniform(*dls)) for i in range(n_members)] + [_pile(rng, i) for i in range(n_piles)]
    df = f_hi / nw2
    design = dict(site=dict(water_depth=float(depth), rho_water=1025.0, g=9.81),
                  platform=dict(potModMaster=0, dlsMax=5.0, members=members, potSecOrder=1, min_freq2nd=df, df_freq2nd=df, max_freq2nd=f_hi))
    m = rng.uniform(0.5, 3.0) * 1e7
    mats = dict(M_struc=np.diag([m, m, m, m * 900, m * 900, m * 1500]) + rng.normal(size=(6, 6)) * m * 0.01,
                C_hydro=np.diag([0, 0, 4e6, 2e9, 2e9, 0.0]), C_moor=np.diag([7e4, 7e4, 0, 0, 0, 1.2e8]))
    f = FOWT(design, grid.make_w(0.3 / 40, 0.3), depth=depth, matrices=mats)
    f.calcHydroConstants()
    P = f.pack()
    assert len(P["qs_w"]) == nw2
    return P


def headings_and_motions(seed, n, nw2):
    """Headings 0, +pi, -pi then random; case 0 a fixed body, odd cases small rotations, even cases (> 0) large ones."""
    rng = np.random.default_rng(seed)
    beta = rng.uniform(-np.pi, np.pi, n)
    beta[:min(n, 3)] = [0.0, np.pi, -np.pi][:min(n, 3)] if n > 1 else beta[:1]
    Xi = rng.normal(size=(n, 6, nw2)) + 1j * rng.normal(size=(n, 6, nw2))
    rot = np.where(np.arange(n) % 2 == 1, 0.03, 0.8)
    Xi[:, 3:] *= rot[:, None, None]
    Xi[0] = 0.0
    return beta, Xi


# id: (seed, depth [m], nw2, f_hi [Hz], n_members, n_piles, dlsMax range, n_cases)
RANDOM = {
    "over_128_nodes_1000m": (1, 1000.0, 23, 0.25, 7, 0, (0.7, 1.0), 5),     # some threads take 3 strip nodes; k h 0.7 .. 250
    "over_64_members_30m": (2, 30.0, 5, 0.2, 0, 70, (2.0, 2.0), 5),        # 70 piles: some threads take 2 members
    "nw2_1_64_cases_300m": (3, 300.0, 1, 0.12, 5, 0, (1.5, 6.0), 64),
    "nw2_2_60m": (4, 60.0, 2, 0.2, 6, 0, (1.5, 6.0), 5),
    "nw2_23_64_cases_120m": (5, 120.0, 23, 0.22, 4, 0, (2.0, 6.0), 64),
    "nw2_61_1000m": (6, 1000.0, 61, 0.25, 5, 0, (2.0, 6.0), 5),
    "nw2_160_150m": (7, 150.0, 160, 0.3, 3, 0, (3.0, 6.0), 1),
}


@pytest.mark.parametrize("label", list(RANDOM))
def test_random_designs_vs_oracle(label, solver, oracle):
    seed, depth, nw2, f_hi, nm, npile, dls, n = RANDOM[label]
    P = slender_design(seed, depth, nw2, f_hi, n_members=nm, n_piles=npile, dls=dls)
    Ns, Nm = len(P["qs_node_mem"]), len(P["qs_mem_mcf"])
    if label.startswith("over_128"):
        assert Ns > 128 and (P["qs_k"] * depth).min() < 10 < 89.4 < (P["qs_k"] * depth).max()
    if label.startswith("over_64"):
        assert Nm > 64 and int(P["qs_mem_mcf"].sum()) > 64
    assert int(P["qs_mem_wl"].sum()) > 0 or npile > 0
    beta, Xi = headings_and_motions(seed + 50, n, nw2)
    compare_with_oracle(solver, oracle, P, beta, Xi, label)


def test_random_design_mcf_and_waterline_coverage():
    """The random designs above carry what the tests rely on: inclined MacCamy-Fuchs members through the waterline (the
    Kim & Yue force gets a vertical component) and waterline members whose added mass differs between their first and
    last submerged node."""
    incl_mcf = ca_varies = 0
    for label, (seed, depth, nw2, f_hi, nm, npile, dls, n) in RANDOM.items():
        if nm == 0:
            continue
        P = slender_design(seed, depth, nw2, f_hi, n_members=nm, dls=dls)
        start = np.concatenate([[0], np.cumsum(np.bincount(P["qs_node_mem"], minlength=len(P["qs_mem_mcf"])))])
        for m in range(len(P["qs_mem_mcf"])):
            incl_mcf += int(P["qs_mem_mcf"][m] and abs(P["qs_mem_q"][m][2]) < 0.999)
            ca = P["qs_node_Ca_p1"][start[m]:start[m + 1]]
            ca_varies += int(P["qs_mem_wl"][m] and len(ca) > 1 and ca[0] != ca[-1])
    assert incl_mcf >= 3 and ca_varies >= 3, (incl_mcf, ca_varies)


# ---- hand-made tables: the member terms without strip nodes ---------------------------------------------------------------

def _frame(q):
    q = np.asarray(q, dtype=float) / np.linalg.norm(q)
    p1 = np.cross([0.0, 0.0, 1.0], q) if abs(q[2]) < 0.999 else np.array([1.0, 0.0, 0.0])
    p1 /= np.linalg.norm(p1)
    return q, p1, np.cross(q, p1)


def nodeless_tables(depth, k, members, rng):
    """qs_* tables with no strip nodes.  ``members``: dicts with q, mcf, wl, r_int, a_wl, rwl, R_wl and segs [(z1, z2, R, rmid)]."""
    g = 9.81
    k = np.asarray(k, dtype=float)
    P = dict(qs_depth=np.float64(depth), qs_rho=np.float64(1025.0), qs_g=np.float64(g), qs_k=k, qs_w=np.sqrt(g * k * np.tanh(k * depth)),
             qs_M_struc=np.diag([2e7, 2e7, 2e7, 1.5e10, 1.5e10, 2e10]) + rng.normal(size=(6, 6)) * 1e5,
             qs_node_mem=np.zeros(0, dtype=np.int32), qs_node_r=np.zeros([0, 3]))
    for nm in ("v_side", "Ca_p1", "Ca_p2", "Ca_End", "v_end", "a_i"):
        P["qs_node_" + nm] = np.zeros(0)
    fr = [_frame(m["q"]) for m in members]
    P.update(qs_mem_q=np.array([f[0] for f in fr]), qs_mem_p1=np.array([f[1] for f in fr]), qs_mem_p2=np.array([f[2] for f in fr]),
             qs_mem_mcf=np.array([m["mcf"] for m in members], dtype=np.int32), qs_mem_wl=np.array([m["wl"] for m in members], dtype=np.int32),
             qs_mem_r_int=np.array([m["r_int"] for m in members], dtype=float), qs_mem_a_wl=np.array([m["a_wl"] for m in members], dtype=float),
             qs_mem_rwl=np.array([m["rwl"] for m in members], dtype=float), qs_mem_R_wl=np.array([m["R_wl"] for m in members], dtype=float))
    segs = [(i, s) for i, m in enumerate(members) for s in m["segs"]]
    P.update(qs_seg_mem=np.array([i for i, _ in segs], dtype=np.int32), qs_seg_z1=np.array([s[0] for _, s in segs], dtype=float),
             qs_seg_z2=np.array([s[1] for _, s in segs], dtype=float), qs_seg_R=np.array([s[2] for _, s in segs], dtype=float),
             qs_seg_rmid=np.array([s[3] for _, s in segs], dtype=float).reshape(len(segs), 3))
    # the oracle's design struct needs the first-order tables too: an empty body on the same grid
    P.update(prp=np.zeros(3), w=P["qs_w"], k=k, mem_q=np.zeros([0, 3]), mem_p1=np.zeros([0, 3]), mem_p2=np.zeros([0, 3]), mem_rA=np.zeros([0, 3]),
             mem_circ=np.zeros(0, dtype=np.int32), node_r=np.zeros([0, 3]), node_mem=np.zeros(0, dtype=np.int32), node_Imat=np.zeros([0, 3, 3]),
             node_a_i=np.zeros(0), M0=np.eye(6), B0=np.zeros([6, 6]), C0=np.eye(6), depth=np.float64(depth), rho=np.float64(1025.0),
             g=np.float64(g), dw=np.float64(1.0))
    for nm in ("a_q", "a_p1", "a_p2", "a_End", "Cd_q", "Cd_p1", "Cd_p2", "Cd_End"):
        P["node_" + nm] = np.zeros(0)
    return P


def kay_reference(P, beta, dps=30):
    """correction_KAY (raft_member.py:1692-1792; Nm = 10) of every member of the tables, restated with mpmath at ``dps``
    digits from the double inputs -> qtf [nw2, nw2, 6], Hermitian-filled.  The tables have no strip nodes and the body does
    not move, so this is the whole slender-body QTF."""
    import mpmath as mp
    mp.mp.dps = dps
    w, k = [mp.mpf(float(x)) for x in P["qs_w"]], [mp.mpf(float(x)) for x in P["qs_k"]]
    n2 = len(w)
    h, rho, g = mp.mpf(float(P["qs_depth"])), mp.mpf(float(P["qs_rho"])), mp.mpf(float(P["qs_g"]))
    b = mp.mpf(float(beta))
    cb, sb = mp.cos(b), mp.sin(b)
    hank = {}

    def H(n, x):
        if (n, x) not in hank:
            hank[(n, x)] = mp.hankel1(n, x)
        return hank[(n, x)]

    def omega(k1R, k2R, n):
        HNii = (H(n - 1, k1R) - H(n + 1, k1R)) / 2
        HNjj = mp.conj(H(n - 1, k2R) - H(n + 1, k2R)) / 2
        HNm1ii = (H(n, k1R) - H(n + 2, k1R)) / 2
        HNm1jj = mp.conj(H(n, k2R) - H(n + 2, k2R)) / 2
        return 1 / (HNm1ii * HNjj) - 1 / (HNii * HNm1jj)

    def force6(f, r):
        return [f[0], f[1], f[2], f[2] * r[1] - f[1] * r[2], f[0] * r[2] - f[2] * r[0], f[1] * r[0] - f[0] * r[1]]

    q = np.zeros([n2, n2, 6], dtype=complex)
    for m in range(len(P["qs_mem_mcf"])):
        if not P["qs_mem_mcf"][m]:
            continue
        p1, p2 = [mp.mpf(float(x)) for x in P["qs_mem_p1"][m]], [mp.mpf(float(x)) for x in P["qs_mem_p2"][m]]
        d1, d2 = cb * p1[0] + sb * p1[1], cb * p2[0] + sb * p2[1]
        pf = [d1 * p1[i] + d2 * p2[i] for i in range(3)]
        nrm = mp.sqrt(sum(x * x for x in pf))
        pf = [x / nrm for x in pf]
        rwl = [mp.mpf(float(x)) for x in P["qs_mem_rwl"][m]]
        radii = [(mp.mpf(float(P["qs_mem_R_wl"][m])), None)]
        radii += [(mp.mpf(float(P["qs_seg_R"][s])), s) for s in range(len(P["qs_seg_mem"])) if P["qs_seg_mem"][s] == m]
        for i1 in range(n2):
            for i2 in range(i1, n2):
                k1, k2, w1, w2 = k[i1], k[i2], w[i1], w[i2]
                ph = mp.exp(-1j * ((k1 - k2) * cb * rwl[0] + (k1 - k2) * sb * rwl[1]))
                F = [mp.mpc(0)] * 6
                for R, s in radii:
                    k1R, k2R = k1 * R, k2 * R
                    if s is None:
                        amp = mp.re(sum(-1j * rho * g * R * 2 / mp.pi / (k1R * k2R) * omega(k1R, k2R, n) for n in range(11)))
                        r = rwl
                    else:
                        z1, z2 = mp.mpf(float(P["qs_seg_z1"][s])), mp.mpf(float(P["qs_seg_z2"][s]))
                        k1h, k2h = k1 * h, k2 * h
                        A2, A1 = mp.sinh((k1 + k2) * (z2 + h)) / (k1h + k2h), mp.sinh((k1 + k2) * (z1 + h)) / (k1h + k2h)
                        if w1 == w2:
                            B2, B1 = (z2 + h) / h, (z1 + h) / h
                        else:
                            B2, B1 = mp.sinh((k1 - k2) * (z2 + h)) / (k1h - k2h), mp.sinh((k1 - k2) * (z1 + h)) / (k1h - k2h)
                        Im, Ip = (A2 - B2 - A1 + B1) / 2, (A2 + B2 - A1 - B1) / 2
                        fac = k1h * k2h / mp.sqrt(k1h * mp.tanh(k1h)) / mp.sqrt(k2h * mp.tanh(k2h)) / mp.cosh(k1h) / mp.cosh(k2h)
                        amp = mp.re(sum(1j * rho * g * R * 2 / mp.pi / (k1R * k2R) * omega(k1R, k2R, n) * fac * (Im + Ip * n * (n + 1) / k1R / k2R)
                                        for n in range(11)))
                        r = [mp.mpf(float(x)) for x in P["qs_seg_rmid"][s]]
                    F = [a + c for a, c in zip(F, force6([amp * ph * x for x in pf], r))]
                if k1 < k2:
                    F = [mp.conj(x) for x in F]
                q[i1, i2] += np.array([complex(x) for x in F])
    iu = np.triu_indices(n2, 1)
    q[iu[1], iu[0]] = np.conj(q[iu[0], iu[1]])
    return q


def test_kim_yue_correction_alone_vs_30_digit_reference(solver, oracle):
    """No strip nodes, one inclined MacCamy-Fuchs member without a waterline term, a fixed body: the QTF is exactly the
    Kim & Yue correction (waterline Hankel term + two integration segments).  k R runs from 0.01 to 8 on a log grid,
    diagonal included; the heading has both cos and sin components so that the inclined axis tilts the force."""
    rng = np.random.default_rng(3)
    depth, R = 60.0, 4.0
    k = np.geomspace(0.01 / R, 8.0 / R, 16)
    q_ax = np.array([0.35, -0.2, 0.9])
    mem = dict(q=q_ax, mcf=1, wl=0, r_int=[0.0, 0.0, 0.0], a_wl=0.0, rwl=[3.0, -2.0, 0.0], R_wl=R,
               segs=[(-9.0, 0.0, R, [-0.5, 1.0, -4.5]), (-18.0, -9.0, 1.2 * R, [-2.0, 2.0, -13.5])])
    P = nodeless_tables(depth, k, [mem], rng)
    beta = 0.7
    ref = kay_reference(P, beta)
    Xi = np.zeros([1, 6, len(k)], dtype=complex)
    q = solver.qtf_slender(P, [beta], Xi)[0]
    qo = oracle.qtf_slender(oracle.OracleDesign(P), beta, Xi[0])
    assert hermitian_exact(q) and np.abs(ref[..., 2]).max() > 1e-3 * np.abs(ref[..., 0]).max()   # the tilt gives heave force
    e_gpu, e_orc, e_go = dof_err(q, ref), dof_err(qo, ref), dof_err(q, qo)
    print("Kim & Yue alone: GPU vs mpmath %.2e, oracle vs mpmath %.2e, GPU vs oracle %.2e" % (e_gpu, e_orc, e_go))
    assert e_gpu < 1e-11 and e_orc < 1e-11 and e_go < BOUND, (e_gpu, e_orc, e_go)


@pytest.mark.parametrize("where", ["waterline", "near_seabed"])
def test_waterline_member_without_nodes_vs_oracle(where, solver, oracle):
    """A waterline member with no strip nodes (its force then uses Ca = 0) and no Kim & Yue term.  At the waterline with
    moving bodies on a grid that spans all three depth branches; then with its intersection point placed near the seabed
    on an all-deep-water grid (k h > 89.4) and a fixed body: at z = 0 the seabed image term exp(-k (z + 2h)) of the
    deep-water pressure is below double precision, near the seabed it is within ~1e-6 of the direct term."""
    rng = np.random.default_rng(8)
    depth = 100.0
    if where == "waterline":
        k, zi, n = np.geomspace(0.02, 1.5, 20), 0.0, 5
    else:
        k, zi, n = np.linspace(0.9, 1.5, 12), -0.95 * depth, 3
    mem = dict(q=[0.3, 0.2, 0.93], mcf=0, wl=1, r_int=[4.0, -3.0, zi], a_wl=35.0, rwl=[0.0, 0.0, 0.0], R_wl=1.0, segs=[])
    P = nodeless_tables(depth, k, [mem], rng)
    beta, Xi = headings_and_motions(21, n, len(k))
    if where == "near_seabed":
        Xi[:] = 0.0
    q = compare_with_oracle(solver, oracle, P, beta, Xi, "nodeless waterline member, " + where)
    assert np.abs(q).max() > 0


# ---- the device entry point ----------------------------------------------------------------------------------------------

def _golden(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    return {k[2:]: z[k] for k in z.files if k.startswith("P_")}


def test_device_entry_point_on_a_side_stream(solver):
    """raftk_qtf_slender_dev on torch tensors and a non-default stream: the same bits as raftk_qtf_slender_host, within
    exactly raftk_qtf_slender_workspace_bytes (the bytes after it stay untouched); one byte less is RAFTK_ENOMEM, and
    65536 cases or no members are RAFTK_EINVAL -- with nothing launched."""
    import torch
    from raft_b200._lib import lib
    P = _golden("slender_VolturnUS-S")
    dev = torch.device("cuda", torch.cuda.current_device())
    keep = {}

    def to_dev(name, a):
        keep[name] = torch.from_numpy(a).to(dev)
        return keep[name].data_ptr()
    s = solver._slender_struct(P, to_dev)
    nw2, n = s.nw, 5
    beta, Xi = headings_and_motions(4, n, nw2)
    host = solver.qtf_slender(P, beta, Xi)
    beta_d = torch.from_numpy(beta).to(dev)
    Xi_d = torch.from_numpy(np.ascontiguousarray(Xi).view(np.float64)).to(dev)
    q = torch.full((n * nw2 * nw2 * 6 * 2,), float("nan"), dtype=torch.float64, device=dev)     # every element must be written
    wb = int(lib.raftk_qtf_slender_workspace_bytes(C.byref(s), n))
    guard = 1 << 16
    ws = torch.full((wb + guard,), 0xA5, dtype=torch.uint8, device=dev)
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        rc = lib.raftk_qtf_slender_dev(C.byref(s), n, beta_d.data_ptr(), Xi_d.data_ptr(), q.data_ptr(), ws.data_ptr(), wb, side.cuda_stream)
    assert rc == 0, rc
    side.synchronize()
    qd = q.cpu().numpy().view(np.complex128).reshape(n, nw2, nw2, 6)
    assert np.array_equal(qd, host)
    assert bool((ws[wb:] == 0xA5).all())
    launches = solver.launch_count()
    args = (beta_d.data_ptr(), Xi_d.data_ptr(), q.data_ptr(), ws.data_ptr())
    assert lib.raftk_qtf_slender_dev(C.byref(s), n, *args, wb - 1, side.cuda_stream) == RAFTK_ENOMEM
    assert lib.raftk_qtf_slender_dev(C.byref(s), 65536, *args, 1 << 62, side.cuda_stream) == RAFTK_EINVAL
    assert lib.raftk_qtf_slender_dev(C.byref(s), 0, *args, wb, side.cuda_stream) == RAFTK_EINVAL
    s0 = solver._slender_struct(P, to_dev)
    s0.n_members = 0
    assert lib.raftk_qtf_slender_dev(C.byref(s0), n, *args, wb, side.cuda_stream) == RAFTK_EINVAL
    assert solver.launch_count() == launches
    side.synchronize()
    assert np.array_equal(q.cpu().numpy().view(np.complex128).reshape(n, nw2, nw2, 6), host)


# ---- the solve flow with two designs ------------------------------------------------------------------------------------

def test_solve_flow_two_designs_vs_oracle(solver, oracle):
    """solve_dynamics_slender on the VolturnUS-S tables and a random design on the same grids, with n_iter small enough that
    loop (A) runs out for some units: per (design, case) status and response against the oracle's whole flow; where loop
    (A) did not converge there is no QTF and no second-order force, elsewhere the force is the QTF's."""
    z = np.load(os.path.join(GOLDEN, "slender_VolturnUS-S.npz"))
    Pa = {k[2:]: z[k] for k in z.files if k.startswith("P_")}
    from raft_b200.fowt import FOWT
    rng = np.random.default_rng(9)
    members = [_member(rng, i, 30.0, 3.0) for i in range(5)]
    plat = dict(potModMaster=0, dlsMax=5.0, members=members, potSecOrder=1, min_freq2nd=0.04, df_freq2nd=0.008, max_freq2nd=0.2)
    mats = dict(M_struc=np.diag([2e7, 2e7, 2e7, 1.8e10, 1.8e10, 3e10]), C_hydro=np.diag([0, 0, 4e6, 2e9, 2e9, 0.0]),
                C_moor=np.diag([7e4, 7e4, 0, 0, 0, 1.2e8]))
    f = FOWT(dict(site=dict(water_depth=float(Pa["depth"]), rho_water=float(Pa["rho"]), g=float(Pa["g"])), platform=plat), Pa["w"],
             depth=float(Pa["depth"]), matrices=mats)
    f.calcHydroConstants()
    Pb = f.pack()
    assert np.array_equal(Pb["qs_w"], Pa["qs_w"]) and np.array_equal(Pb["w"], Pa["w"])
    cs = dict(Hs=np.array([6.0, 2.0, 9.0, 4.0, 1.5, 7.0]), Tp=np.array([12.0, 7.5, 15.0, 9.0, 6.0, 17.0]), gamma=np.zeros(6),
              beta_deg=np.array([30.0, -75.0, 160.0, 0.0, 180.0, -110.0]), spec=np.zeros(6, dtype=np.int32))
    n_iter = 3
    out = solver.solve_dynamics_slender([Pa, Pb], solver.CaseTable(cs), n_iter=n_iter, want=("Xi", "status", "F_2nd"))
    # loop (A) alone is the plain solve: the oracle without the qs_* tables says which units it converged for
    conv = np.array([[oracle.solve_dynamics(oracle.OracleDesign({k: v for k, v in P.items() if not k.startswith("qs_")}), 0, cs["Hs"][c],
                                            cs["Tp"][c], 0.0, cs["beta_deg"][c], nIter=n_iter)[1][1] == 1 for c in range(6)] for P in (Pa, Pb)])
    assert conv.any() and (~conv).any(), conv
    for d, P in enumerate((Pa, Pb)):
        od = oracle.OracleDesign(P)
        for c in range(6):
            Xi_o, st = oracle.solve_dynamics(od, 0, cs["Hs"][c], cs["Tp"][c], 0.0, cs["beta_deg"][c], nIter=n_iter)
            assert np.array_equal(out["status"][d, c, :2], st[:2]), (d, c, out["status"][d, c], st)
            assert response_err(out["Xi"][d, c], Xi_o) < 1e-10, (d, c)
            if conv[d, c]:
                assert np.abs(out["F_2nd"][d, c]).max() > 0 and np.abs(out["qtf"][d, c]).max() > 0
                # the force is calcHydroForce_2ndOrd of this unit's QTF (the oracle's reduction of the GPU's table)
                Pq = dict(P, qtf=out["qtf"][d, c][:, :, None, :], qtf_w=P["qs_w"], qtf_heads=np.array([cs["beta_deg"][c] * 0.017453292519943295]))
                _, f2 = oracle.hydro_force_2nd(oracle.OracleDesign(Pq), cs["beta_deg"][c] * 0.017453292519943295,
                                               oracle.jonswap(P["w"], cs["Hs"][c], cs["Tp"][c], 0.0))
                assert relerr(out["F_2nd"][d, c], f2) < 1e-10, (d, c)
            else:
                assert np.all(out["F_2nd"][d, c] == 0) and np.all(out["qtf"][d, c] == 0), (d, c)
