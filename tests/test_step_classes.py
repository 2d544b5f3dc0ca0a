"""Step classes of the fused rigid solvers (DESIGN.md section 5) at node spacings a fraction of the merge tolerance apart.

k_rao_fused<T> and k_fused_plan + k_rao_fused2 walk every member with E <- E W and A+- <- A+- f+-; the factors belong to
step classes (phase keys (q_x,q_y)*step, depth keys q_z*step, first-node depths z0), and keys that agree to the tolerance
share a class.  ``spec_classes`` below is THE rule: greedy in node order, a key joins the first class whose key is within
its own tolerance, else opens one.  The kernels and all three host-side hint counters must count exactly this:

* CPU: adversarial key sets (chains 0.9 tol apart, a chain followed by a distinct key, alternating keys, the last keys
  on either side of the tolerance and of the no-step threshold, mixed signs, z0 chains on both sides of |z0| = 1), realised as packed
  designs whose node_ls / mem_rA produce them (each checks its own keys), against DesignBatch._step_classes and
  batch_builder._count_classes.
* GPU: chain designs cut from the golden packs on every kernel the planner picks, against the oracle (which evaluates
  phases and depth functions per node); hints equal to the rule's count run, one less sets RAFTK_FLAG_PLAN on every unit;
  and every entry point recovers from, or raises on, a flagged unit instead of returning results built from zeros."""
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN, load_golden, relerr, response_err


def _tols():
    from raft_b200 import solver
    return solver.STEP_RTOL, solver.STEP_ZERO, solver.Z0_RTOL


# ---- the rule ------------------------------------------------------------------------------------------------------------
def spec_classes(keys, tols):
    """Greedy classes of ``keys`` (tuples; None = no step) with per-key tolerances -> (class per key (-1: none), class keys)."""
    cls, reps = [], []
    for k, t in zip(keys, tols):
        if k is None:
            cls.append(-1)
            continue
        c = next((i for i, r in enumerate(reps) if all(abs(a - b) <= t for a, b in zip(r, k))), None)
        if c is None:
            c = len(reps)
            reps.append(k)
        cls.append(c)
    return cls, reps


def first_match_classes(keys, tols):
    """The rule the kernels used before: a key's class is the number of representatives before the FIRST earlier key within
    its tolerance (representative or not) -> (class per key, number of representatives, i.e. factor rows filled).  Only
    here to show that each adversarial set tells the two rules apart."""
    rep = []
    for j, (k, t) in enumerate(zip(keys, tols)):
        r = -1 if k is None else next((x for x in range(j) if keys[x] is not None and all(abs(a - b) <= t for a, b in zip(keys[x], k))), j)
        rep.append(r)
    return [-1 if r < 0 else sum(1 for x in range(r) if rep[x] == x) for r in rep], sum(1 for x, r in enumerate(rep) if r == x)


def design_keys(P):
    """Per-node phase and depth keys and per-member first-node depths of a packed design, formed as the kernels form
    them (q * (ls[j] - ls[j-1]); None at a member's first node and where every component is at most STEP_ZERO)."""
    _, zero, _ = _tols()
    ms = np.asarray(P["mem_start"])
    wk, hk, z0 = [], [], []
    for m in range(len(ms) - 1):
        q, ls = np.asarray(P["mem_q"][m], dtype=float), np.asarray(P["node_ls"][ms[m]:ms[m + 1]], dtype=float)
        if not len(ls):
            continue
        z0.append((float(P["mem_rA"][m][2]) + ls[0] * q[2],))
        wk.append(None)
        hk.append(None)
        for j in range(1, len(ls)):
            step = ls[j] - ls[j - 1]
            kx, ky, kz = q[0] * step, q[1] * step, q[2] * step
            wk.append((kx, ky) if abs(kx) > zero or abs(ky) > zero else None)
            hk.append((kz,) if abs(kz) > zero else None)
    return wk, hk, z0


def design_rule(P):
    """-> {"w"|"h"|"z": (class per node / member, class keys)} of a packed design by the rule."""
    rtol, _, ztol = _tols()
    wk, hk, z0 = design_keys(P)
    return dict(w=spec_classes(wk, [0 if k is None else rtol * (abs(k[0]) + abs(k[1])) for k in wk]),
                h=spec_classes(hk, [0 if k is None else rtol * abs(k[0]) for k in hk]),
                z=spec_classes(z0, [ztol * max(1.0, abs(k[0])) for k in z0]))


def rule_counts(P):
    r = design_rule(P)
    return tuple(len(r[x][1]) for x in "whz")


# ---- adversarial packed designs (CPU) --------------------------------------------------------------------------------------
def _pack(members):
    """Minimal packed design from members (q, rA, ls): the columns the class rule and DesignBatch._step_classes read."""
    starts = np.concatenate([[0], np.cumsum([len(m[2]) for m in members])]).astype(np.int32)
    return dict(mem_start=starts, mem_q=np.array([m[0] for m in members], dtype=float),
                mem_rA=np.array([m[1] for m in members], dtype=float), node_ls=np.concatenate([np.asarray(m[2], dtype=float) for m in members]))


def _ls(steps, ls0=0.0):
    return np.concatenate([[ls0], ls0 + np.cumsum(steps)])


def _adversarial():
    """name -> (packed design, expected {"w"|"h"|"z": classes}) -- expected lists only where the structure is the point."""
    rtol, zero, ztol = _tols()
    s = 4.5
    hx, vz = (1.0, 0.0, 0.0), (0.0, 0.0, 1.0)
    out = {}
    for n in range(3, 7):
        chain = [s * (1 + 0.9 * i * rtol) for i in range(n)]
        out["w-chain%d" % n] = (_pack([(hx, (0, 0, -10), _ls(chain, 1.0))]), dict(w=[-1] + [i // 2 for i in range(n)]))
        out["h-chain%d" % n] = (_pack([(vz, (0, 0, -30), _ls(chain, 1.0))]), dict(h=[-1] + [i // 2 for i in range(n)]))
    later = [s, s * (1 + 0.9 * rtol), s * (1 + 1.8 * rtol), s * (1 + 3.0 * rtol)]
    out["w-chain-then-distinct"] = (_pack([(hx, (0, 0, -10), _ls(later, 1.0))]), dict(w=[-1, 0, 0, 1, 2]))
    out["w-chain-then-member"] = (_pack([(hx, (0, 0, -10), _ls(later[:3], 1.0)), (hx, (0, 5, -10), _ls(later[3:], 2.0))]),
                                  dict(w=[-1, 0, 0, 1, -1, 2]))
    alt = [s * (1 + 0.9 * rtol * (i % 2)) for i in range(8)]
    out["alternating"] = (_pack([(vz, (0, 0, -60), _ls(alt, 1.0))]), dict(h=[-1] + [0] * 8))
    # the boundary itself: at a relative 5e-14 a thousandth of the tolerance is below one ulp of a key, so the last key that
    # joins and the first that does not are the neighbouring doubles at the boundary, on both sides (one step per member:
    # ls = [0, key] gives the key exactly)
    up = s * (1 + rtol)
    while abs(up - s) > rtol * up:
        up = np.nextafter(up, 0.0)
    while abs(np.nextafter(up, np.inf) - s) <= rtol * np.nextafter(up, np.inf):
        up = np.nextafter(up, np.inf)
    dn = s * (1 - rtol)
    while abs(dn - s) > rtol * dn:
        dn = np.nextafter(dn, np.inf)
    keys = [s, up, np.nextafter(up, np.inf), dn, np.nextafter(dn, 0.0)]
    for nm, q in (("w-tol-boundary", hx), ("h-tol-boundary", vz)):
        out[nm] = (_pack([(q, (0, 0, -10), [0.0, k]) for k in keys]), {nm[0]: [-1, 0, -1, 0, -1, 1, -1, 0, -1, 2]})
    tiny = [zero * (1 + 1e-3), zero * (1 - 1e-3), zero * (1 + 1e-3)]
    out["identity-threshold"] = (_pack([(hx, (0, 0, -10), _ls(tiny)), (vz, (0, 0, -10), _ls(tiny)),
                                        ((0.6, 0.8, 0.0), (0, 0, -10), _ls([zero * 1.5, zero * 0.8]))]),
                                 dict(w=[-1, 0, -1, 0, -1, -1, -1, -1, -1, 1, -1], h=[-1, -1, -1, -1, -1, 0, -1, 0, -1, -1, -1]))
    sq = (-0.6, 0.8, 0.0)
    out["mixed-sign"] = (_pack([(sq, (0, 0, -10), _ls([s * (1 + 0.9 * i * rtol) for i in range(3)], 1.0)),
                                ((0.6, -0.8, 0.0), (0, 0, -10), _ls([s, s], 1.0)), ((-0.6, -0.8, 0.0), (0, 0, -10), _ls([s], 1.0)),
                                (sq, (0, 0, -10), _ls([-s, -s * (1 + 0.9 * rtol), -s * (1 + 1.8 * rtol)], 30.0))]),
                         dict(w=[-1, 0, 0, 1, -1, 2, 2, -1, 3, -1, 2, 2, 4]))     # the last member's keys are the second's
    for nm, zb in (("z0-chain-small", -0.5), ("z0-chain-large", -20.0)):
        tol = ztol * max(1.0, abs(zb))
        zs = [zb - 0.9 * i * tol for i in range(4)] + [zb - 4.5 * tol]
        out[nm] = (_pack([(vz, (0, 0, z), [0.0, 1.0]) for z in zs]), dict(z=[0, 0, 1, 1, 2]))
    return out


ADV = ["w-chain3", "w-chain4", "w-chain5", "w-chain6", "h-chain3", "h-chain6", "w-chain-then-distinct", "w-chain-then-member",
       "alternating", "w-tol-boundary", "h-tol-boundary", "identity-threshold", "mixed-sign", "z0-chain-small", "z0-chain-large"]


@pytest.mark.parametrize("name", ADV)
def test_adversarial_design_has_its_structure(name):
    """The packed design realises the intended classes after ls differences are rounded, and the chains really tell the
    greedy rule from the first-match rule."""
    P, want = _adversarial()[name]
    rtol, _, ztol = _tols()
    r = design_rule(P)
    for x, cls in want.items():
        assert r[x][0] == cls, (x, r[x][0], cls)
    if "chain" in name or name == "mixed-sign":
        wk, hk, z0 = design_keys(P)
        keys = {"w": wk, "h": hk, "z": z0}[name[0] if name[0] in "hz" else "w"]
        tols = [0 if k is None else (ztol * max(1.0, abs(k[0])) if name[0] == "z" else rtol * sum(abs(v) for v in k)) for k in keys]
        cls, reps = spec_classes(keys, tols)
        assert first_match_classes(keys, tols) != (cls, len(reps))


@pytest.mark.parametrize("name", ADV)
def test_hint_counters_count_the_rule(name):
    """DesignBatch._step_classes and batch_builder._count_classes give exactly the rule's counts."""
    from raft_b200 import batch_builder, solver
    P, _ = _adversarial()[name]
    counts = rule_counts(P)
    assert solver.DesignBatch._step_classes([P]) == tuple(max(1, c) for c in counts)
    rtol, _, ztol = _tols()
    wk, hk, z0 = design_keys(P)
    for keys, tol, c in ((wk, lambda k: rtol * (abs(k[0]) + abs(k[1])), counts[0]), (hk, lambda k: rtol * abs(k[0]), counts[1]),
                         (z0, lambda k: ztol * max(1.0, abs(k[0])), counts[2])):
        nc = len(next((k for k in keys if k is not None), (0.0,)))
        K = np.array([[0.0] * nc if k is None else list(k) for k in keys])[None]
        V = np.array([k is not None for k in keys])[None]
        tl = np.array([0.0 if k is None else tol(k) for k in keys])[None]
        assert int(batch_builder._count_classes(K, V, tl)[0]) == c


def test_batched_counter_per_design():
    """Every adversarial set as one design of a single batch (ragged, padded): per-design counts equal the rule's."""
    from raft_b200 import batch_builder
    rtol, _, _ = _tols()
    sets = [design_keys(_adversarial()[n][0])[0] for n in ADV]
    Pm = max(len(k) for k in sets)
    K, V, tl = np.zeros((len(sets), Pm, 2)), np.zeros((len(sets), Pm), bool), np.zeros((len(sets), Pm))
    for d, keys in enumerate(sets):
        for j, k in enumerate(keys):
            if k is not None:
                K[d, j], V[d, j], tl[d, j] = k, True, rtol * (abs(k[0]) + abs(k[1]))
    want = [len(spec_classes(keys, [0 if k is None else rtol * (abs(k[0]) + abs(k[1])) for k in keys])[1]) for keys in sets]
    assert list(batch_builder._count_classes(K, V, tl)) == want


def test_builders_count_the_rule_on_a_sweep_family():
    """The NumPy and the native batched builder on a 64-design VolturnUS-S family: the hints are the largest per-design
    count of the rule, evaluated on the builders' own tables."""
    from raft_b200 import batch_builder, solver, sweep
    G, P = load_golden("cfg2_VolturnUS-S_nw64")
    D = json.load(open(os.path.join(GOLDEN, "designs.json")))["cfg2_VolturnUS-S_nw64"]
    mats = dict(M_struc=P["M0"] - G["A_hydro_morison"], C_struc=P["C0"] - G["C_moor"], C_moor=G["C_moor"])
    fac = sweep.sample_factors(64, seed=43)
    for native in (False, True):
        b = sweep.build_variants_batched(D, mats, fac, nw=64, max_freq=0.32, depth=float(P["depth"]), native=native)
        a = b.arrays
        best = np.zeros(3, int)
        for d in range(b.n_designs):
            m0, m1 = a["member_offset"][d], a["member_offset"][d + 1]
            Q = dict(mem_start=a["mem_node_start"][m0:m1 + 1] - a["mem_node_start"][m0], mem_q=a["mem_frame"][m0:m1, :3],
                     mem_rA=a["mem_rA"][m0:m1], node_ls=a["node_ls"][a["mem_node_start"][m0]:a["mem_node_start"][m1]])
            best = np.maximum(best, rule_counts(Q))
        assert (b.max_w_classes, b.max_h_classes, b.max_z_classes) == tuple(int(max(1, c)) for c in best), native


def test_tolerance_constants_match_the_kernels():
    """One tolerance: the Python constants are the ones the kernels and the native builder compile with."""
    import re
    from raft_b200 import solver
    src = open(os.path.join(os.path.dirname(GOLDEN), "..", "raft_b200", "csrc", "raftk_common.cuh")).read()
    for name in ("STEP_RTOL", "STEP_ZERO", "Z0_RTOL"):
        assert float(re.search(r"#define %s (\S+)" % name, src).group(1)) == getattr(solver, name)


# ---- chain designs from the golden packs (GPU) -----------------------------------------------------------------------------
def _edit_member(P, m, ls=None, dz=0.0):
    """Copy of packed design ``P`` with member ``m``'s node_ls replaced and / or its rA moved by dz along z; node_r follows."""
    P = dict(P)
    ms = P["mem_start"]
    a, b = int(ms[m]), int(ms[m + 1])
    P["node_ls"], P["node_r"], P["mem_rA"] = P["node_ls"].copy(), P["node_r"].copy(), P["mem_rA"].copy()
    if ls is not None:
        P["node_ls"][a:b] = ls
    P["mem_rA"][m, 2] += dz
    P["node_r"][a:b] = P["mem_rA"][m][None, :] + P["node_ls"][a:b, None] * P["mem_q"][m][None, :]
    return P


def _chain_ls(ls, first, factors):
    """ls with the steps first, first+1, ... scaled by ``factors`` (later nodes shifted along)."""
    steps = np.diff(ls)
    base = steps[first]
    for i, f in enumerate(factors):
        steps[first + i] = base * f
    return np.concatenate([[ls[0]], ls[0] + np.cumsum(steps)])


def _member_ls(P, m):
    return P["node_ls"][P["mem_start"][m]:P["mem_start"][m + 1]]


MAX_FREQ = 0.4


def chain_design(name, nw):
    """Adversarial designs on the golden packs (only node_ls / mem_rA edited)."""
    from raft_b200 import grid
    rtol, _, ztol = _tols()
    if name in ("wchain", "wchain+", "zchain"):
        P = grid.regrid(load_golden("cfg2_VolturnUS-S_nw64")[1], nw, MAX_FREQ)
        if name == "wchain":                   # pontoon 5 (q = -x): steps 1..3 a chain 0.9 tol apart
            return _edit_member(P, 5, _chain_ls(_member_ls(P, 5), 1, [1, 1 + 0.9 * rtol, 1 + 1.8 * rtol]))
        if name == "wchain+":                  # ... then a spacing 3.0 tol away
            return _edit_member(P, 5, _chain_ls(_member_ls(P, 5), 1, [1, 1 + 0.9 * rtol, 1 + 1.8 * rtol, 1 + 3.0 * rtol]))
        tol = ztol * 20.0                      # first-node depths of the outer columns: a chain, then a distinct depth
        for m, f in ((1, 0.9), (2, 1.8), (3, 3.0)):
            P = _edit_member(P, m, dz=-f * tol)
        return P
    P = grid.regrid(load_golden("cfg1_OC3spar")[1], nw, 0.5 if name == "alt" else MAX_FREQ)
    ls = _member_ls(P, 0)
    if name == "hchain":                       # OC3spar column: steps 1..3 a chain
        return _edit_member(P, 0, _chain_ls(ls, 1, [1, 1 + 0.9 * rtol, 1 + 1.8 * rtol]))
    steps = np.diff(ls)                        # "alt": every other step 0.9 tol longer, over the whole 120 m column
    steps[1::2] *= 1 + 0.9 * rtol
    return _edit_member(P, 0, np.concatenate([[ls[0]], ls[0] + np.cumsum(steps)]))


CHAINS = ["wchain", "wchain+", "hchain", "zchain", "alt"]
_FORCE, _CLUSTER, _GRID = {"RAFTK_FORCE_V1": "1"}, {"RAFTK_FUSED2_XCHG": "cluster"}, {"RAFTK_FUSED2_XCHG": "grid"}
# (nw, cluster_size, environment, kernel, f0_global) per base design, from test_dispatch_solve.SHAPES
VARIANTS = {"cfg2": [(201, 2, {}, "fused128", False), (333, 2, {}, "fused256", False), (333, 1, {}, "fused256", True),
                     (501, 2, _CLUSTER, "fused2-cluster", False), (501, 2, _GRID, "fused2-grid", False), (201, 1, _FORCE, "v1", False)],
            "cfg1": [(201, 2, {}, "fused128", False), (333, 2, {}, "fused256", False), (501, 1, {}, "fused256", True),
                     (501, 2, _CLUSTER, "fused2-cluster", False), (501, 2, _GRID, "fused2-grid", False), (201, 1, _FORCE, "v1", False)]}


def _base(name):
    return "cfg2" if name in ("wchain", "wchain+", "zchain") else "cfg1"


MATRIX = [(n, v) for n in CHAINS for v in VARIANTS[_base(n)]]


def _mid(p):
    n, v = p
    return "%s-nw%d-cs%d-%s%s" % (n, v[0], v[1], v[3], "-f0g" if v[4] else "")


def test_chain_designs_have_their_structure():
    """CPU check of the GPU designs: the edited member realises the chain, and the rule's counts exceed the first-match
    rule's where the kernels used to misassign."""
    for name in CHAINS:
        P = chain_design(name, 201)
        r = design_rule(P)
        if name in ("wchain", "wchain+"):
            c = r["w"][0][int(P["mem_start"][5]):int(P["mem_start"][6])]
            assert c[2] == c[3] and c[4] != c[3] and (name == "wchain" or c[5] not in (c[3], c[4])), c
        elif name == "hchain":
            c = r["h"][0][:6]
            assert c[2] == c[3] and c[4] != c[3], c
        elif name == "zchain":
            c = r["z"][0][:4]
            assert c[0] == c[1] and len({c[1], c[2], c[3]}) == 3, c
        else:                                  # merged keys up to ~0.9 tol off their class key along the whole column
            _, hk, _ = design_keys(P)
            cls, reps = r["h"]
            n = int(P["mem_start"][1])
            off = [abs(hk[j][0] - reps[cls[j]][0]) / abs(hk[j][0]) for j in range(1, n)]
            assert max(off) > 0.7 * _tols()[0] and sum(o > 0.5 * _tols()[0] for o in off) >= 8, off


_ORC = {}
SEA_SEED = 61


def _sea(n=3):
    rng = np.random.default_rng(SEA_SEED)
    return dict(Hs=rng.uniform(1, 10, n), Tp=rng.uniform(3, 18, n), gamma=np.zeros(n), beta_deg=rng.uniform(-180, 180, n),
                spec=np.zeros(n, dtype=np.int32))


def _oracle(oracle, name, nw):
    if (name, nw) not in _ORC:
        P = chain_design(name, nw)
        od, cs = oracle.OracleDesign(P), _sea()
        Xi, st, _ = oracle.solve_cases(od, cs, nIter=10)
        Bd, Fi = [], []
        for c in range(len(cs["Hs"])):
            Bd.append(oracle.solve_dynamics(od, 0, cs["Hs"][c], cs["Tp"][c], 0.0, cs["beta_deg"][c], nIter=10, want_Z=True)[3])
            Fi.append(oracle.calc_hydro_excitation(od, 0, cs["Hs"][c], cs["Tp"][c], 0.0, cs["beta_deg"][c])[2])
        _ORC[(name, nw)] = dict(Xi=Xi, status=st, B_drag=np.array(Bd), F_iner=np.array(Fi))
    return _ORC[(name, nw)]


def _env(monkeypatch, env):
    for k in ("RAFTK_FORCE_V1", "RAFTK_FUSED2_XCHG", "RAFTK_NO_DIRECT_D2H"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def _check(r, o, d=0):
    assert np.array_equal(r["status"][d, :, :2], o["status"][:, :2]) and np.all(r["status"][d, :, 2] == 0), (r["status"][d], o["status"])
    assert response_err(r["Xi"][d], o["Xi"]) < 1e-10
    if "B_drag" in r:
        assert relerr(r["B_drag"][d], o["B_drag"]) < 1e-10
    if "F_iner" in r:
        assert relerr(r["F_iner"][d], o["F_iner"]) < 1e-10


@pytest.mark.gpu
@pytest.mark.parametrize("p", MATRIX, ids=_mid)
def test_chain_vs_oracle(p, monkeypatch, oracle):
    """Every kernel variant on every chain design against the oracle: response, pass counts, converged flags, B_drag and
    F_iner to 1e-10, no flags."""
    from raft_b200 import solver
    name, (nw, cs, env, kernel, f0g) = p
    _env(monkeypatch, env)
    r = solver.solve_dynamics(solver.DesignBatch(chain_design(name, nw)), solver.CaseTable(_sea()), n_iter=10, cluster_size=cs,
                              want=("Xi", "status", "B_drag", "F_iner"))
    rec = solver.last_dispatch()
    assert rec["kernel"] == kernel and rec["f0_global"] == f0g, rec
    _check(r, _oracle(oracle, name, nw))


@pytest.mark.gpu
@pytest.mark.parametrize("name", CHAINS)
def test_chain_sweep_path_vs_oracle(name, oracle):
    """The sweep path: a DeviceSession whose hints come from the batched builder's counter (batch_builder._count_classes on
    the design's keys), and sweep.solve_sweep; both against the oracle."""
    import torch
    from raft_b200 import batch_builder, solver, sweep
    nw = 201
    P = chain_design(name, nw)
    o = _oracle(oracle, name, nw)
    rtol, _, ztol = _tols()
    wk, hk, z0 = design_keys(P)
    hints = []
    for keys, tol in ((wk, lambda k: rtol * (abs(k[0]) + abs(k[1]))), (hk, lambda k: rtol * abs(k[0])), (z0, lambda k: ztol * max(1.0, abs(k[0])))):
        nc = len(next((k for k in keys if k is not None), (0.0,)))
        K = np.array([[0.0] * nc if k is None else list(k) for k in keys])[None]
        hints.append(int(max(1, batch_builder._count_classes(K, np.array([k is not None for k in keys])[None],
                                                             np.array([0.0 if k is None else tol(k) for k in keys])[None])[0])))
    assert tuple(hints) == tuple(max(1, c) for c in rule_counts(P))
    b = solver.DesignBatch(P)
    b.max_w_classes, b.max_h_classes, b.max_z_classes = hints
    out = solver.DeviceSession(b, solver.CaseTable(_sea())).solve(n_iter=10)
    torch.cuda.synchronize()
    assert solver.last_dispatch()["kernel"] != "v1"
    _check({k: v.cpu().numpy() for k, v in out.items()}, o)
    Xi, st = sweep.solve_sweep([P], _sea(), n_iter=10)
    _check(dict(Xi=Xi.cpu().numpy(), status=st.cpu().numpy()), o)


def _session_status(P, hints, cs, cases=None):
    import torch
    from raft_b200 import solver
    b = solver.DesignBatch(P)
    b.max_w_classes, b.max_h_classes, b.max_z_classes = hints
    sess = solver.DeviceSession(b, cases if cases is not None else solver.CaseTable(_sea()))
    out = sess.solve(n_iter=10, cluster_size=cs)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}, solver.last_dispatch()


FUSED = [(n, v) for n, v in MATRIX if v[3] != "v1"]


@pytest.mark.gpu
@pytest.mark.parametrize("p", FUSED, ids=_mid)
def test_hints_are_exact_on_the_device(p, monkeypatch):
    """A hint equal to the rule's count runs without RAFTK_FLAG_PLAN; one less in w, h or z flags every unit (with exact
    zeros in Xi): the kernels count exactly what the rule counts."""
    name, (nw, cs, env, kernel, _) = p
    _env(monkeypatch, env)
    P = chain_design(name, nw)
    counts = tuple(max(1, c) for c in rule_counts(P))
    r, rec = _session_status(P, counts, cs)
    assert rec["kernel"] == kernel, rec
    assert np.all(r["status"][..., 2] == 0), r["status"]
    for i in range(3):
        if counts[i] < 2:
            continue
        h = list(counts)
        h[i] -= 1
        r, rec = _session_status(P, h, cs)
        assert np.all(r["status"][..., 2] & 4), (i, r["status"])
        assert np.all(r["status"][..., 0] == 0) and np.all(r["Xi"] == 0), i


# ---- RAFTK_FLAG_PLAN at every entry point (deliberately small hints) -------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("v", VARIANTS["cfg2"][:5], ids=lambda v: v[3] + ("-f0g" if v[4] else ""))
def test_solve_dynamics_recovers_from_small_hints(v, monkeypatch, oracle):
    """solve_dynamics re-runs flagged units with worst-case tables and agrees with the oracle."""
    from raft_b200 import solver
    nw, cs, env, kernel, _ = v
    _env(monkeypatch, env)
    b = solver.DesignBatch(chain_design("wchain+", nw))
    b.max_w_classes = b.max_h_classes = b.max_z_classes = 1
    r = solver.solve_dynamics(b, solver.CaseTable(_sea()), n_iter=10, cluster_size=cs, want=("Xi", "status", "B_drag", "F_iner"))
    rec = solver.last_dispatch()                 # the worst-case run: one class per node no longer fits a fused kernel
    assert rec["family"] == "solve" and rec["kernel"] == "v1", rec
    _check(r, _oracle(oracle, "wchain+", nw))


def _train_cases():
    from raft_b200 import packer
    cases = [dict(wave_spectrum="JONSWAP", wave_height=3.0, wave_period=9.0, wave_heading=20.0),
             dict(wave_spectrum=["JONSWAP"] * 3, wave_height=[4.0, 1.5, 2.5], wave_period=[11.0, 7.0, 14.0], wave_heading=[0.0, 60.0, -45.0],
                  wave_gamma=[0.0] * 3)]
    return packer.pack_case_trains(cases)[0]


@pytest.mark.gpu
@pytest.mark.parametrize("v", VARIANTS["cfg2"][:5], ids=lambda v: v[3] + ("-f0g" if v[4] else ""))
def test_flagged_units_hold_zeros(v, monkeypatch):
    """DeviceSession.solve with a too-small hint: Xi pre-filled with NaN comes back as exact zeros on every unit, secondary
    wave trains of a flagged primary are flagged too; the host entry's Xi_last likewise."""
    import ctypes as C
    import torch
    from raft_b200 import solver
    from raft_b200._lib import RaftkSolveOpts, check, lib
    nw, cs, env, kernel, _ = v
    _env(monkeypatch, env)
    ct = solver.CaseTable(_train_cases())
    b = solver.DesignBatch(chain_design("wchain", nw))
    b.max_w_classes = 1
    nC = ct.n_cases
    nan = dict(Xi=torch.full([1, nC, 6, nw], complex(np.nan, np.nan), dtype=torch.complex128, device="cuda"))
    out = solver.DeviceSession(b, ct, out_tensors=nan).solve(n_iter=10, cluster_size=cs)
    torch.cuda.synchronize()
    assert solver.last_dispatch()["kernel"] == kernel and solver.last_dispatch()["trains"]
    st, Xi = out["status"].cpu().numpy(), out["Xi"].cpu().numpy()
    assert np.all(st[..., 2] & solver.FLAG_PLAN) and np.all(st[..., 0] == 0), st
    assert np.all(Xi == 0)
    outs = dict(Xi=np.full([1, nC, 6, nw], np.nan + 0j), status=np.full([1, nC, 4], -1, dtype=np.int32),
                Xi_last=np.full([1, nC, 6, nw], np.nan + 0j))
    o = RaftkSolveOpts(10, cs, 0.01, 0.0, 0, 0)
    check(lib.raftk_solve_dynamics_host(C.byref(solver._host_struct(b)), C.byref(solver._host_struct(ct)), C.byref(o),
                                        C.byref(solver._out_struct(outs, lambda a: a.ctypes.data))))
    assert np.all(outs["status"][..., 2] & solver.FLAG_PLAN)
    assert np.all(outs["Xi"] == 0) and np.all(outs["Xi_last"] == 0)


@pytest.mark.gpu
def test_farm_recovers_from_small_hints():
    """solve_dynamics_farm with a too-small hint: the flagged units are solved again and Xi_sys matches the run with exact
    hints (it was assembled from zero loads before)."""
    from raft_b200 import solver
    z = np.load(os.path.join(GOLDEN, "farm_VolturnUS-S_farm_nw48.npz"))
    N = int(z["n_fowt"])
    packs = [{k[len("P%d_" % i):]: z[k] for k in z.files if k.startswith("P%d_" % i)} for i in range(N)]
    rows = z["cases"]
    cs = dict(Hs=rows[:, 0], Tp=rows[:, 1], gamma=np.zeros(len(rows)), beta_deg=rows[:, 2], spec=np.zeros(len(rows), dtype=np.int32))
    good = solver.solve_dynamics_farm(solver.DesignBatch(packs), solver.CaseTable(cs), C_arr=z["C_array"], n_iter=10)
    b = solver.DesignBatch(packs)
    b.max_w_classes = b.max_h_classes = b.max_z_classes = 1
    small = solver.solve_dynamics_farm(b, solver.CaseTable(cs), C_arr=z["C_array"], n_iter=10)
    assert np.all(small["status"][..., 2] == 0) and np.array_equal(small["status"], good["status"])
    assert np.abs(good["Xi_sys"]).max() > 0
    assert response_err(small["Xi_sys"], good["Xi_sys"]) < 1e-12


def _small_hints(monkeypatch):
    from raft_b200 import solver
    monkeypatch.setattr(solver.DesignBatch, "_step_classes", staticmethod(lambda packed: (1, 1, 1)))


@pytest.mark.gpu
def test_model_and_sweep_recover_from_small_hints(monkeypatch):
    """Model (one FOWT and a coupled array) and sweep.solve_sweep with every hint at 1: the results equal those with the
    rule's hints."""
    from raft_b200 import sweep
    from raft_b200.model import Model
    G, P = load_golden("cfg2_VolturnUS-S_nw64")
    D = json.load(open(os.path.join(GOLDEN, "designs.json")))["cfg2_VolturnUS-S_nw64"]
    mats = dict(M_struc=P["M0"] - G["A_hydro_morison"], C_struc=P["C0"] - G["C_moor"], C_moor=G["C_moor"])
    single = dict(D, site=dict(D["site"], water_depth=float(P["depth"])))
    arr = dict(settings=D["settings"], site=dict(D["site"], water_depth=float(P["depth"])), platforms=[D["platform"]],
               array=dict(keys=["ID", "turbineID", "platformID", "mooringID", "x_location", "y_location", "heading_adjust"],
                          data=[[1, 0, 1, 0, 0.0, 0.0, 0.0], [2, 0, 1, 0, 1600.0, 0.0, 0.0]]))
    rng = np.random.default_rng(1)
    A = rng.normal(size=(12, 12)) * 2e4
    C_arr = A @ A.T / 12 + np.diag([5e4] * 12)
    case = [dict(wave_spectrum="JONSWAP", wave_height=6.0, wave_period=12.0, wave_heading=20.0)]

    def run():
        r1 = Model(json.loads(json.dumps(single)), matrices=mats).analyzeCases(cases=case)
        r2 = Model(json.loads(json.dumps(arr)), matrices=mats, array_stiffness=C_arr).analyzeCases(cases=case)
        Xi, st = sweep.solve_sweep([chain_design("wchain", 201)], _sea(), n_iter=10)
        return r1["Xi"], r1["status"], r2["Xi"], r2["status"], Xi.cpu().numpy(), st.cpu().numpy()
    good = run()
    _small_hints(monkeypatch)
    small = run()
    for g, s in zip(good, small):
        if np.iscomplexobj(g):
            assert np.abs(g).max() > 0 and response_err(s, g) < 1e-12
        else:
            assert np.array_equal(s, g) and np.all(g[..., 2] == 0)
