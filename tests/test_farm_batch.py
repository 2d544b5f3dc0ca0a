"""Batches of farms in one call (raftk_farm_batch_*, solver.solve_dynamics_farm_batch, DeviceSession.farm_response(n_fowt=N)):
F arrays of N FOWTs each over one case table.  Without a GPU: the workspace query, the struct layout and prototypes against
include/raftk.h, and every refusal that is decided before a device is used.  On the GPU: farm 0 of a batch against the
reference's own runs (fixtures farm_VolturnUS-S_farm_nw48 and farm24_VolturnUS-S_farm_nw48), and every farm of a batch
against solve_dynamics_farm on that farm alone, bit for bit, on each kernel the dispatcher can pick."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, response_err

HEADER = os.path.join(ROOT, "include", "raftk.h")
NEW = ("raftk_farm_batch_workspace_bytes", "raftk_farm_batch_response_ws_dev", "raftk_solve_dynamics_farm_batch_host")
RTOL = 1e-10
gpu = pytest.mark.gpu
PER_FOWT = ("Xi", "status", "B_drag", "F_drag", "F_iner")


# ---- without a GPU --------------------------------------------------------------------------------------------------
def test_workspace_query_without_gpu():
    from raft_b200 import solver
    for N in (1, 2, 8, 20):
        for F in (1, 3, 4096):
            assert solver.farm_batch_workspace_bytes(F, N, 64, 1024) == 0, (F, N)
    for N in (21, 24, 64):
        slab = 6 * N * (6 * N + 1) * 16
        for nC, nw in ((64, 1024), (1, 3), (2, 1)):
            assert solver.farm_batch_workspace_bytes(1, N, nC, nw) == solver.farm_workspace_bytes(N, nC, nw)
        full = solver.farm_workspace_bytes(N, 64, 1024)                  # a full persistent grid
        for F in (2, 5, 1000):
            b = solver.farm_batch_workspace_bytes(F, N, 64, 1024)
            assert b == full and b % slab == 0, (F, N, b)
            assert solver.farm_batch_workspace_bytes(F, N, 1, 3) == min(3 * F * slab, full)      # never more slabs than systems
        assert solver.farm_batch_workspace_bytes(2, N, 2, 1) == 4 * slab
        assert solver.farm_batch_workspace_bytes(0, N, 2, 1) == 0


def _prototype(name):
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    m = re.search(r"\b(\w+\s*\*?)\s*\b%s\s*\(([^)]*)\)\s*;" % name, src)
    assert m, name
    return m.group(1).strip(), [a.strip() for a in m.group(2).split(",")]


@pytest.mark.parametrize("name", NEW)
def test_bindings_match_header_prototypes(name):
    from raft_b200 import _lib
    structs = (("raftk_farm_batch", _lib.RaftkFarmBatch), ("raftk_designs", _lib.RaftkDesigns), ("raftk_cases", _lib.RaftkCases),
               ("raftk_solve_opts", _lib.RaftkSolveOpts), ("raftk_outputs", _lib.RaftkOutputs))
    ret, params = _prototype(name)
    fn = getattr(_lib.lib, name)
    assert name in _lib.SYMBOLS and len(fn.argtypes) == len(params), (name, params)
    for decl, ct in zip(params, fn.argtypes):
        want = next((C.POINTER(t) for s, t in structs if s in decl), C.c_void_p if "*" in decl else C.c_size_t)
        assert ct is want, (name, decl, ct)
    assert fn.restype is (C.c_size_t if ret == "size_t" else C.c_int)


def test_struct_layout_matches_header(tmp_path):
    from raft_b200 import _lib
    fields = [n for n, _ in _lib.RaftkFarmBatch._fields_]
    src = tmp_path / "t.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "raftk.h"\nint main(void){printf("%%zu %s\\n", sizeof(raftk_farm_batch), %s);'
                   'return 0;}\n' % (" ".join(["%zu"] * len(fields)), ", ".join("offsetof(raftk_farm_batch, %s)" % n for n in fields)))
    exe = tmp_path / "t"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    B = _lib.RaftkFarmBatch
    assert got == [C.sizeof(B)] + [getattr(B, n).offset for n in fields]


def _refusal_structs(nD=6, nC=2, nw=16):
    """Structs whose pointers are never followed: every refusal below is decided from the counts and NULL tests alone."""
    from raft_b200 import _lib
    d, c = _lib.RaftkDesigns(), _lib.RaftkCases()
    d.n_designs, d.nw, d.max_nodes, d.max_members, c.n_cases = nD, nw, 8, 2, nC
    o = _lib.RaftkSolveOpts(10, 0, 0.01, 0.0, 0, 0)
    out = _lib.RaftkOutputs()
    for k in ("Xi", "status", "B_drag", "F_drag", "F_iner"):
        setattr(out, k, 0x1000)
    f = _lib.RaftkFarmBatch()
    f.n_farms, f.n_fowt, f.arr_shared, f.Xi_sys = 3, 2, 1, 0x1000
    return d, c, o, out, f


@pytest.mark.parametrize("field,value,msg", [
    ("n_farms", 0, "n_farms and n_fowt"), ("n_fowt", 0, "n_farms and n_fowt"), ("n_farms", -3, "n_farms and n_fowt"),
    ("n_farms", 2, "n_farms * n_fowt"), ("n_fowt", 3, "n_farms * n_fowt"),
    ("arr_shared", 2, "arr_shared"), ("arr_shared", -1, "arr_shared"), ("Xi_sys", None, "Xi_sys"),
])
def test_host_entry_refuses_before_any_device_use(field, value, msg):
    from raft_b200._lib import lib
    d, c, o, out, f = _refusal_structs()
    setattr(f, field, value)
    before = lib.raftk_launch_count()
    rc = lib.raftk_solve_dynamics_farm_batch_host(C.byref(d), C.byref(c), C.byref(o), C.byref(out), C.byref(f))
    assert rc == -1 and msg in lib.raftk_last_error().decode() and lib.raftk_launch_count() == before
    # the device entry decides the same from the same struct
    rc = lib.raftk_farm_batch_response_ws_dev(C.byref(d), C.byref(c), C.byref(out), C.byref(f), None, 0, None)
    assert rc == -1 and msg in lib.raftk_last_error().decode() and lib.raftk_launch_count() == before


def test_device_entry_refuses_before_any_launch():
    from raft_b200 import _lib
    lib = _lib.lib
    before = lib.raftk_launch_count()
    for missing in ("B_drag", "F_drag", "F_iner"):
        d, c, o, out, f = _refusal_structs()
        setattr(out, missing, None)
        assert lib.raftk_farm_batch_response_ws_dev(C.byref(d), C.byref(c), C.byref(out), C.byref(f), None, 0, None) == -1
        assert "B_drag, F_drag, F_iner" in lib.raftk_last_error().decode()
    d, c, o, out, f = _refusal_structs()
    d.n_bem_head = 4                                                          # designs with BEM excitation: F_BEM is part of the load
    assert lib.raftk_farm_batch_response_ws_dev(C.byref(d), C.byref(c), C.byref(out), C.byref(f), None, 0, None) == -1
    assert "F_BEM" in lib.raftk_last_error().decode()
    d, c, o, out, f = _refusal_structs(nD=48)                                 # 2 farms of 24: the system lives in a workspace slab
    f.n_farms, f.n_fowt = 2, 24
    slab = 144 * 145 * 16
    for ws, nbytes in ((None, 1 << 30), (0x1000, slab - 1), (0x1000, 0)):
        assert lib.raftk_farm_batch_response_ws_dev(C.byref(d), C.byref(c), C.byref(out), C.byref(f), ws, nbytes, None) == -1
        assert "at least one [6N][6N+1] slab" in lib.raftk_last_error().decode()
    d, c, o, out, f = _refusal_structs(nD=2 * 65536)                          # the farm index is the grid's z extent
    f.n_farms = 65536
    assert lib.raftk_farm_batch_response_ws_dev(C.byref(d), C.byref(c), C.byref(out), C.byref(f), None, 0, None) == -1
    assert "65535 farms" in lib.raftk_last_error().decode()
    assert lib.raftk_launch_count() == before


def test_python_entry_checks_shapes():
    from raft_b200 import solver
    packs, _ = _base(2)
    batch = solver.DesignBatch([packs[i % 2] for i in range(6)])
    cases = solver.CaseTable(_cases(np.array([[6.0, 12.0, 0.0]])))
    with pytest.raises(ValueError, match="n_fowt must divide"):
        solver.solve_dynamics_farm_batch(batch, cases, 4)
    with pytest.raises(ValueError, match="must all be"):
        solver.solve_dynamics_farm_batch(batch, cases, 2, C_arr=np.eye(12), M_arr=np.zeros([3, 12, 12]))
    with pytest.raises(ValueError, match="must all be"):
        solver.solve_dynamics_farm_batch(batch, cases, 2, C_arr=np.zeros([2, 12, 12]))
    with pytest.raises(ValueError, match="Xi_sys"):
        solver.solve_dynamics_farm_batch(batch, cases, 2, out=dict(Xi_sys=np.zeros([1, 12, 48], dtype=complex)))
    one = solver.DesignBatch(packs)                                           # the single-farm form: a batch of one farm
    for bad in (np.eye(6), np.zeros([2, 12, 12]), np.zeros([1, 12, 13])):
        with pytest.raises(ValueError, match=r"must all be \[12, 12\] or all be \[1, 12, 12\]"):
            solver.solve_dynamics_farm(one, cases, C_arr=bad)
    with pytest.raises(ValueError, match="must all be"):
        solver.solve_dynamics_farm(one, cases, C_arr=np.eye(12), M_arr=np.zeros([1, 12, 12]))
    for bad in (np.zeros([1, 1, 12, 48], dtype=complex), np.zeros([1, 12, 48]), np.zeros([1, 12, 96], dtype=complex)[..., ::2]):
        with pytest.raises(ValueError, match=re.escape("out['Xi_sys'] must be a C-contiguous complex128 array [1, 12, 48]")):
            solver.solve_dynamics_farm(one, cases, out=dict(Xi_sys=bad))
    with pytest.raises(ValueError, match=re.escape("out['info'] must be a C-contiguous int32 array [1, 48]")):
        solver.solve_dynamics_farm(one, cases, out=dict(info=np.zeros([1, 1, 48], dtype=np.int32)))


# ---- farm batches from the fixtures -------------------------------------------------------------------------------------
def _cases(rows, primary=None):
    n = len(rows)
    d = dict(Hs=rows[:, 0], Tp=rows[:, 1], gamma=np.zeros(n), beta_deg=rows[:, 2], spec=np.zeros(n, dtype=np.int32))
    if primary is not None:
        d["primary"] = np.asarray(primary, dtype=np.int32)
    return d


def _base(N):
    z = np.load(os.path.join(GOLDEN, ("farm24_VolturnUS-S_farm_nw48" if N == 24 else "farm_VolturnUS-S_farm_nw48") + ".npz"))
    return [{k[len("P%d_" % i):]: z[k] for k in z.files if k.startswith("P%d_" % i)} for i in range(int(z["n_fowt"]))], z


def _moved(P, dx, dy):
    """The FOWT at another position: node coordinates, member ends, reference point and BEM reference point move together."""
    Q = dict(P)
    r = np.array([dx, dy, 0.0])
    for k in ("mem_rA", "node_r", "prp"):
        Q[k] = np.asarray(P[k], dtype=float) + r
    Q["x_ref"], Q["y_ref"] = float(P["x_ref"]) + dx, float(P["y_ref"]) + dy
    return Q


def _spd(n, seed):
    A = np.random.default_rng(seed).normal(size=(n, n)) * 2e4
    return A @ A.T / n + np.diag([5e4] * n)


def _farms(N, F, nw=None, tables=False):
    """-> (packs [F][N], C_arr [F,6N,6N]).  N = 2 and N = 24: farm 0 is the fixture as it is (FOWTs, positions and C_array);
    other N take the two-FOWT fixture's FOWTs in turn on a 1600 m row.  Farms 1.. have every FOWT at another position and
    a seeded SPD array stiffness of their own.  ``nw``: the designs on another grid; ``tables``: seeded A_w / B_w / X_BEM."""
    from raft_b200 import grid
    base, z = _base(N)
    if nw is not None:
        base = [grid.regrid(P, nw, 0.005 * nw) for P in base]
    packs, C_arr = [], []
    for f in range(F):
        row = []
        for i in range(N):
            P = base[i] if N == len(base) else _moved(base[i % len(base)], 1600.0 * (i - i % len(base)), 0.0)
            row.append(P if f == 0 else _moved(P, 137.0 * f * (i + 1), -211.0 * f * ((i % 3) + 1)))
        packs.append(row)
        C_arr.append(z["C_array"] if f == 0 and N == len(base) else _spd(6 * N, 1000 * N + f))
    if tables:
        rng = np.random.default_rng(77 + N)
        n_w = len(base[0]["w"])
        for row in packs:
            for i, P in enumerate(row):
                d = np.diag(rng.uniform(0.5, 1.5, size=6))
                row[i] = dict(P, A_w=(np.abs(P["M0"]) * 0.05 * d)[:, :, None] * rng.uniform(0.5, 1.0, size=n_w)[None, None, :],
                              B_w=(np.abs(P["M0"]) * 0.01 * d)[:, :, None] * rng.uniform(0.0, 1.0, size=n_w)[None, None, :],
                              bem_headings=np.array([0.0, 90.0, 180.0, 270.0]), heading_adjust=0.0,
                              X_BEM=(rng.normal(size=(4, 6, n_w)) + 1j * rng.normal(size=(4, 6, n_w))) * 2e5)
    return packs, np.array(C_arr)


def _flat(packs):
    return [P for row in packs for P in row]


def _assert_farms_equal_single(packs, cases_of, C_arr, out, N, kernel, want=PER_FOWT, primary=None):
    """Every farm of the batched ``out`` against solve_dynamics_farm on that farm alone: identical bits.  B_drag belongs to
    the primary cases (a secondary wave train uses its primary's), so it is compared there."""
    from raft_b200 import solver
    for f, row in enumerate(packs):
        one = solver.solve_dynamics_farm(solver.DesignBatch(row), cases_of(f), C_arr=C_arr[f], want=want)
        assert solver.last_dispatch()["kernel"] == kernel
        assert np.array_equal(out["Xi_sys"][f], one["Xi_sys"]), f
        assert np.array_equal(out["info"][f], one["info"]), f
        for k in want:
            a, b = out[k][f * N:(f + 1) * N], one[k]
            if k == "B_drag" and primary is not None:
                a, b = a[:, np.unique(primary)], b[:, np.unique(primary)]
            assert np.array_equal(a, b), (f, k, np.unique(np.nonzero(a != b)[1]))


@gpu
@pytest.mark.parametrize("N,kernel", [(2, "farm-rows12"), (24, "farm-global")])
def test_farm_zero_of_a_batch_vs_reference_run(N, kernel):
    """Being in a batch changes nothing about a reference-pinned farm: farm 0 against the reference's own run."""
    from raft_b200 import solver
    F = 3
    packs, C_arr = _farms(N, F)
    _, z = _base(N)
    out = solver.solve_dynamics_farm_batch(solver.DesignBatch(_flat(packs)), solver.CaseTable(_cases(z["cases"])), N, C_arr=C_arr,
                                           n_iter=int(z["n_iter"]), xi_start=float(z["xi_start"]))
    rec = solver.last_dispatch()
    assert rec["family"] == "farm" and rec["kernel"] == kernel, rec
    nC, nw = len(z["cases"]), len(packs[0][0]["w"])
    assert out["Xi_sys"].shape == (F, nC, 6 * N, nw) and out["info"].shape == (F, nC, nw) and out["Xi"].shape == (F * N, nC, 6, nw)
    assert not np.any(out["info"]) and np.all(out["status"][..., 2] == 0)
    assert np.array_equal(out["status"][:N, :, 0].T, z["ref_run_passes"])
    ref = z["ref_run_Xi"][:, 0]
    err = max(response_err(out["Xi_sys"][0][:, 6 * i:6 * i + 6], ref[:, 6 * i:6 * i + 6]) for i in range(N))
    assert err < RTOL, err
    for f in range(1, F):                                                      # the moved farms are other systems
        assert not np.array_equal(out["Xi_sys"][f], out["Xi_sys"][0])


@gpu
@pytest.mark.parametrize("N,kernel,nw", [
    (2, "farm-rows12", 45),       # 8 systems per CTA: 45 = 5 * 8 + 5
    (2, "farm-rows12", 48),
    (3, "farm-warp", 45),         # FARM_WPC = 4 systems per CTA: 45 = 11 * 4 + 1
    (4, "farm-warp", 45),
    (4, "farm-warp", 13),
    (8, "farm-block", 21),
    (24, "farm-global", 13),
])
def test_every_farm_equals_the_single_farm_entry(N, kernel, nw):
    """Xi_sys[f], info[f] and the per-FOWT outputs of farm f's designs equal solve_dynamics_farm on that farm alone, bit for
    bit, on each kernel; the frequency counts leave a ragged last group of systems next to another farm's."""
    from raft_b200 import solver
    F = 4 if N < 24 else 3
    packs, C_arr = _farms(N, F, nw=nw)
    rows = np.array([[6.0, 12.0, 0.0], [3.5, 9.0, 40.0], [8.0, 14.0, -120.0]])
    ct = solver.CaseTable(_cases(rows))
    out = solver.solve_dynamics_farm_batch(solver.DesignBatch(_flat(packs)), ct, N, C_arr=C_arr, want=PER_FOWT)
    rec = solver.last_dispatch()
    assert rec["family"] == "farm" and rec["kernel"] == kernel and rec["farm_classes"] == (kernel,), rec
    assert not np.any(out["info"])
    _assert_farms_equal_single(packs, lambda f: ct, C_arr, out, N, kernel)
    for f in range(1, F):
        assert not np.array_equal(out["Xi_sys"][f], out["Xi_sys"][0])
    # the single-farm C entry, which solve_dynamics_farm no longer calls (it is the farm-batch entry's batch of one), gives
    # the same bits, launches and dispatch record; a [1, 6N, 6N] array matrix is that batch's own (arr_shared = 0)
    row = solver.DesignBatch(packs[1])
    l0 = solver.launch_count()
    one = solver.solve_dynamics_farm(row, ct, C_arr=C_arr[1], want=PER_FOWT)
    l1, rec = solver.launch_count(), solver.last_dispatch()
    raw = _single_farm_entry(row, ct, C_arr[1], PER_FOWT)
    assert solver.launch_count() - l1 == l1 - l0 and solver.last_dispatch() == rec and rec["kernel"] == kernel
    lead = solver.solve_dynamics_farm(row, ct, C_arr=C_arr[1][None], want=PER_FOWT)
    assert solver.last_dispatch() == rec
    for k in ("Xi_sys", "info") + PER_FOWT:
        assert np.array_equal(raw[k], one[k]) and np.array_equal(lead[k], one[k]), k


def _single_farm_entry(batch, ct, C_arr, want):
    """raftk_solve_dynamics_farm_host called directly on one farm: the per-FOWT outputs plus Xi_sys and info."""
    from raft_b200 import _lib, solver
    N, nC, nw = batch.n_designs, ct.n_cases, batch.nw
    outs = solver._alloc_outputs(N, nC, nw, want)
    xi, info = np.zeros([nC, 6 * N, nw], dtype=complex), np.zeros([nC, nw], dtype=np.int32)
    Cm = np.ascontiguousarray(C_arr, dtype=float)
    f = _lib.RaftkFarm(n_fowt=N, C_arr=Cm.ctypes.data, Xi_sys=xi.ctypes.data, info=info.ctypes.data)
    o = _lib.RaftkSolveOpts(10, 0, 0.01, 0.0, 0, 0)
    _lib.check(_lib.lib.raftk_solve_dynamics_farm_host(C.byref(solver._host_struct(batch)), C.byref(solver._host_struct(ct)), C.byref(o),
                                                       C.byref(solver._out_struct(outs, lambda a: a.ctypes.data)), C.byref(f)))
    return dict(outs, Xi_sys=xi, info=info)


@gpu
@pytest.mark.parametrize("N,kernel", [(2, "farm-rows12"), (4, "farm-warp"), (8, "farm-block"), (24, "farm-global")])
def test_shared_matrices_equal_repeated_matrices(N, kernel):
    """arr_shared = 1 with one set of matrices is arr_shared = 0 with that set repeated for every farm (M_arr, B_arr and C_arr)."""
    from raft_b200 import solver
    F, n = 3, 6 * N
    packs, _ = _farms(N, F, nw=19)
    G = np.random.default_rng(N).normal(size=(n, n))
    mats = dict(C_arr=_spd(n, 5), M_arr=(G @ G.T) * 2e3 / n, B_arr=(G + G.T) * 1e3)
    batch, ct = solver.DesignBatch(_flat(packs)), solver.CaseTable(_cases(np.array([[6.0, 12.0, 0.0], [4.0, 10.0, 75.0]])))
    one = solver.solve_dynamics_farm_batch(batch, ct, N, **mats)
    assert solver.last_dispatch()["kernel"] == kernel
    rep = solver.solve_dynamics_farm_batch(batch, ct, N, **{k: np.repeat(v[None], F, axis=0) for k, v in mats.items()})
    assert solver.last_dispatch()["kernel"] == kernel
    assert np.array_equal(one["Xi_sys"], rep["Xi_sys"]) and np.array_equal(one["info"], rep["info"]) and not np.any(one["info"])
    unc = solver.solve_dynamics_farm_batch(batch, ct, N)                      # no array matrices: the stacked per-FOWT responses
    per = unc["Xi"].reshape(F, N, 2, 6, -1).transpose(0, 2, 1, 3, 4).reshape(F, 2, n, -1)
    assert max(response_err(unc["Xi_sys"][..., 6 * i:6 * i + 6, :], per[..., 6 * i:6 * i + 6, :]) for i in range(N)) < RTOL
    assert not np.array_equal(one["Xi_sys"], unc["Xi_sys"])


@gpu
@pytest.mark.parametrize("N,kernel", [(2, "farm-rows12"), (3, "farm-warp"), (8, "farm-block"), (24, "farm-global")])
def test_wave_trains_second_order_force_and_bem_tables(N, kernel):
    """cases.primary (a secondary train uses its primary's damping), cases.F_2nd (rows of the farm's own designs), and designs
    with A_w / B_w / X_BEM (F_BEM in the load) go through the batch and equal the per-farm calls."""
    from raft_b200 import solver
    F = 3
    packs, C_arr = _farms(N, F, tables=True)
    nw = len(packs[0][0]["w"])
    rows = np.array([[6.0, 12.0, 0.0], [2.0, 7.0, 60.0], [4.0, 10.0, 200.0], [1.5, 6.0, 100.0]])
    cs = _cases(rows, primary=[0, 0, 2, 2])
    F2 = np.random.default_rng(3 * N).normal(size=(F * N, len(rows), 6, nw)) * 5e4
    want = PER_FOWT + ("F_BEM",)
    out = solver.solve_dynamics_farm_batch(solver.DesignBatch(_flat(packs)), solver.CaseTable(cs, F_2nd=F2), N, C_arr=C_arr, want=want)
    assert solver.last_dispatch()["kernel"] == kernel and not np.any(out["info"])
    _assert_farms_equal_single(packs, lambda f: solver.CaseTable(cs, F_2nd=F2[f * N:(f + 1) * N]), C_arr, out, N, kernel, want=want,
                               primary=cs["primary"])
    plain = solver.solve_dynamics_farm_batch(solver.DesignBatch(_flat(packs)), solver.CaseTable(cs), N, C_arr=C_arr)
    assert not np.array_equal(plain["Xi_sys"], out["Xi_sys"])                 # the second-order force is in the load
    assert np.any(out["F_BEM"] != 0)


def _session(packs, cs):
    from raft_b200 import solver
    sess = solver.DeviceSession(solver.DesignBatch(_flat(packs)), solver.CaseTable(cs), device="cuda:0", want=PER_FOWT)
    sess.solve(n_iter=10)
    return sess


@gpu
def test_global_kernel_across_workspace_sizes():
    """The full query, one slab and a size in between: fewer bytes run fewer CTAs over the same (farm, case, frequency) list."""
    import torch
    from raft_b200 import _lib, solver
    N, F, nw = 24, 3, 16
    n = 6 * N
    packs, C_arr = _farms(N, F, nw=nw)
    sess = _session(packs, _cases(np.array([[6.0, 12.0, 0.0], [3.0, 8.0, -70.0]])))
    xi, info = sess.farm_response(C_arr=C_arr, n_fowt=N)
    assert solver.last_dispatch()["kernel"] == "farm-global"
    full_xi, full_info = xi.cpu().numpy().copy(), info.cpu().numpy().copy()
    f, _, _, _, _, wsb = sess._farm_batch
    slab = n * (n + 1) * 16
    assert wsb == solver.farm_batch_workspace_bytes(F, N, 2, nw) == F * 2 * nw * slab         # 96 systems: fewer than a full grid
    buf = torch.empty(wsb, dtype=torch.uint8, device="cuda:0")
    args = (C.byref(sess.d_struct), C.byref(sess.c_struct), C.byref(sess.o_struct), C.byref(f))
    stream = torch.cuda.current_stream().cuda_stream
    for nbytes in (slab, 7 * slab + 100):
        xi.zero_()
        info.fill_(-7)
        assert _lib.lib.raftk_farm_batch_response_ws_dev(*args, buf.data_ptr(), nbytes, stream) == 0
        assert solver.last_dispatch()["kernel"] == "farm-global"
        torch.cuda.synchronize()
        assert np.array_equal(xi.cpu().numpy(), full_xi) and np.array_equal(info.cpu().numpy(), full_info), nbytes
    assert _lib.lib.raftk_farm_batch_response_ws_dev(*args, buf.data_ptr(), slab - 1, stream) == -1
    assert solver.last_dispatch()["kernel"] == "none"


@gpu
@pytest.mark.parametrize("N,kernel", [(2, "farm-rows12"), (4, "farm-warp"), (24, "farm-global")])
def test_device_session_farm_axis(N, kernel):
    """DeviceSession.farm_response(n_fowt=N) equals the host entry; n_fowt=None is one farm of all the session's designs."""
    from raft_b200 import solver
    F = 3
    packs, C_arr = _farms(N, F, nw=20)
    cs = _cases(np.array([[6.0, 12.0, 0.0], [3.0, 8.0, -70.0]]))
    host = solver.solve_dynamics_farm_batch(solver.DesignBatch(_flat(packs)), solver.CaseTable(cs), N, C_arr=C_arr)
    sess = _session(packs, cs)
    xi, info = sess.farm_response(C_arr=C_arr, n_fowt=N)
    assert solver.last_dispatch()["kernel"] == kernel
    assert np.array_equal(xi.cpu().numpy(), host["Xi_sys"]) and np.array_equal(info.cpu().numpy(), host["info"])
    assert np.array_equal(sess.out["Xi"].cpu().numpy(), host["Xi"])
    xi2, _ = sess.farm_response(n_fowt=N)                                      # matrices, outputs and workspace stay with the session
    assert xi2 is xi and np.array_equal(xi2.cpu().numpy(), host["Xi_sys"])
    one = _session(packs[1:2], cs)
    x1, i1 = one.farm_response(C_arr=C_arr[1])
    assert tuple(x1.shape) == (2, 6 * N, 20) and tuple(i1.shape) == (2, 20)
    assert np.array_equal(x1.cpu().numpy(), host["Xi_sys"][1]) and np.array_equal(i1.cpu().numpy(), host["info"][1])


@gpu
@pytest.mark.parametrize("N,kernel", [(2, "farm-rows12"), (4, "farm-warp"), (8, "farm-block"), (24, "farm-global")])
def test_a_zero_pivot_stays_in_its_own_farm(N, kernel):
    """Farm 1's last FOWT has no inertia, damping or stiffness in yaw and the farm's array stiffness leaves that DOF free:
    column 6N - 1 of its systems is exactly zero.  info[1] reports the pivot (6N) at every case and frequency, info of the
    other farms stays 0 and their Xi_sys keeps the bits of the run without the defect."""
    from raft_b200 import solver
    F, n = 3, 6 * N
    packs, C_arr = _farms(N, F, nw=14)
    sess = _session(packs, _cases(np.array([[6.0, 12.0, 0.0], [3.0, 8.0, -70.0]])))
    xi, info = sess.farm_response(C_arr=C_arr, n_fowt=N)
    good = xi.cpu().numpy().copy()
    assert not np.any(info.cpu().numpy())
    d = 2 * N - 1                                                              # design of farm 1's last FOWT
    for t in (sess.dt["M0"], sess.dt["B0"], sess.dt["C0"]):
        t.view(-1, 6, 6)[d, :, 5] = 0.0
    sess.out["B_drag"][d, :, :, 5] = 0.0
    mats = sess._farm_batch[1]
    mats["C_arr"][1, :, n - 1] = 0.0
    xi, info = sess.farm_response(n_fowt=N)
    assert solver.last_dispatch()["kernel"] == kernel
    info, xi = info.cpu().numpy(), xi.cpu().numpy()
    assert np.all(info[1] == n) and not np.any(info[0]) and not np.any(info[2])
    assert np.array_equal(xi[0], good[0]) and np.array_equal(xi[2], good[2])
    assert not np.array_equal(xi[1], good[1], equal_nan=True)
