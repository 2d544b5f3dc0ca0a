"""Ragged farm batches (raftk_farm_ragged, solver.solve_dynamics_farm_ragged, DeviceSession.farm_response(farm_sizes=...)):
farms of different turbine counts in one call.  Without a GPU: the struct layout and prototypes against include/raftk.h,
the CSR helpers, the workspace query, every refusal decided before a device is used, and the shard planner.  On the GPU:
one batch whose sizes cover every kernel class in interleaved order, every farm against solve_dynamics_farm on that farm
alone, bit for bit, with and without operating points, BEM tables, the second-order force and wave trains; equal-N batches
against solve_dynamics_farm_batch; a singular farm; reordering; the device entry; workspace sizes; the reference runs."""
import ctypes as C
import itertools
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT, response_err
from test_farm_batch import _base, _cases, _moved, _prototype, _spd

NEW = ("raftk_farm_ragged_workspace_bytes", "raftk_farm_ragged_response_ws_dev", "raftk_solve_dynamics_farm_ragged_host")
PER_FOWT = ("Xi", "status", "B_drag", "F_drag", "F_iner")
SIZES = (3, 2, 21, 1, 20, 24, 2, 7)          # every kernel class, interleaved: rows12, warp, global, warp, block, global, rows12, block
CLASS = {1: "farm-warp", 2: "farm-rows12", 3: "farm-warp", 4: "farm-warp", 7: "farm-block", 20: "farm-block", 21: "farm-global",
         24: "farm-global"}
gpu = pytest.mark.gpu


# ---- without a GPU --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NEW)
def test_bindings_match_header_prototypes(name):
    from raft_b200 import _lib
    structs = (("raftk_farm_ragged", _lib.RaftkFarmRagged), ("raftk_designs", _lib.RaftkDesigns), ("raftk_cases", _lib.RaftkCases),
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
    checks = [("raftk_farm_ragged", _lib.RaftkFarmRagged), ("raftk_dispatch", _lib.RaftkDispatch)]
    body = ""
    for cname, S in checks:
        fields = [n for n, _ in S._fields_]
        body += 'printf("%%zu %s\\n", sizeof(%s), %s);' % (" ".join(["%zu"] * len(fields)), cname,
                                                       ", ".join("offsetof(%s, %s)" % (cname, n) for n in fields))
    src = tmp_path / "t.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "raftk.h"\nint main(void){%sreturn 0;}\n' % body)
    exe = tmp_path / "t"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    want = []
    for _, S in checks:
        want += [C.sizeof(S)] + [getattr(S, n).offset for n, _ in S._fields_]
    assert got == want


def test_csr_helpers_and_views():
    from raft_b200 import solver
    fowt0, arr = solver.ragged_offsets(SIZES)
    assert fowt0.dtype == np.int32 and arr.dtype == np.int64
    assert fowt0.tolist() == [0, 3, 5, 26, 27, 47, 71, 73, 80]
    assert np.array_equal(np.diff(arr), 36 * np.array(SIZES) ** 2) and arr[0] == 0
    nC, nw = 2, 5
    flat = np.arange(6 * 80 * nC * nw) * (1 + 1j)
    views = solver.ragged_views(flat, SIZES, nC, nw)
    assert [v.shape for v in views] == [(nC, 6 * n, nw) for n in SIZES]
    for v, a in zip(views, fowt0[:-1]):
        assert np.shares_memory(v, flat) and v[0, 0, 0] == flat[6 * nC * nw * a]
    mats, shared = solver._ragged_matrices(SIZES, None, None, [np.eye(6 * n) * (k + 1) for k, n in enumerate(SIZES)])
    assert shared == 0 and mats["C_arr"].shape == (int(arr[-1]),)
    for k, n in enumerate(SIZES):
        assert np.array_equal(mats["C_arr"][arr[k]:arr[k + 1]].reshape(6 * n, 6 * n), np.eye(6 * n) * (k + 1))
    assert solver._ragged_matrices((2, 2), np.eye(12), None, None)[1] == 1
    with pytest.raises(ValueError, match="a list of 2 matrices"):
        solver._ragged_matrices((2, 3), None, None, [np.eye(12), np.eye(12)])
    with pytest.raises(ValueError, match="all be shared"):
        solver._ragged_matrices((2, 2), np.eye(12), None, [np.eye(12), np.eye(12)])


def test_shared_matrix_shapes_are_checked():
    """A matrix that is not a list is one [6N,6N] set or a stacked [F,6N,6N], and only when every N_f equals N: a set of the
    wrong size or a set for unequal sizes is refused (it would be read past its end), a stack is per farm, not shared."""
    from raft_b200 import solver
    for sizes, bad in (((3, 3), np.eye(12)), ((2, 3), np.eye(12)), ((2, 3), np.eye(18)), ((2, 2), np.zeros([3, 12, 12])),
                       ((2, 2), np.zeros([2, 12, 13])), ((2, 2), np.zeros(144))):
        with pytest.raises(ValueError, match="a list of"):
            solver._ragged_matrices(sizes, None, None, bad)
    stack = np.arange(2 * 144, dtype=float).reshape(2, 12, 12)
    mats, shared = solver._ragged_matrices((2, 2), None, None, stack)
    assert shared == 0 and np.array_equal(mats["C_arr"], stack.reshape(-1))
    mats, shared = solver._ragged_matrices((2, 2), stack[0], None, None)
    assert shared == 1 and np.array_equal(mats["M_arr"], stack[0])


def _structs(sizes=(2, 3), nC=2, nw=16):
    """Structs whose device pointers are never followed: every refusal below is decided from counts, the host CSR arrays and
    NULL tests alone.  The CSR arrays are returned to keep them alive."""
    from raft_b200 import _lib, solver
    fowt0, arr = solver.ragged_offsets(sizes)
    d, c = _lib.RaftkDesigns(), _lib.RaftkCases()
    d.n_designs, d.nw, d.max_nodes, d.max_members, c.n_cases = int(fowt0[-1]), nw, 8, 2, nC
    o = _lib.RaftkSolveOpts(10, 0, 0.01, 0.0, 0, 0)
    out = _lib.RaftkOutputs()
    for k in PER_FOWT:
        setattr(out, k, 0x1000)
    f = _lib.RaftkFarmRagged()
    f.n_farms, f.arr_shared, f.farm_fowt0, f.arr_offset = len(sizes), 0, fowt0.ctypes.data, arr.ctypes.data
    f.C_arr, f.Xi_sys = 0x1000, 0x1000
    return d, c, o, out, f, (fowt0, arr)


def test_workspace_query_without_gpu():
    from raft_b200._lib import lib
    table = lambda F: -(-F * 40 // 256) * 256    # noqa: E731  (40-byte descriptors, 256-byte aligned)
    for sizes in ((2, 3), (1, 20, 7), (4,) * 100):
        d, c, _, _, f, keep = _structs(sizes, nC=64, nw=1024)
        assert lib.raftk_farm_ragged_workspace_bytes(C.byref(d), C.byref(c), C.byref(f)) == table(len(sizes))
    slab24, slab21 = 144 * 145 * 16, 126 * 127 * 16
    d, c, _, _, f, keep = _structs((21, 2, 24), nC=2, nw=3)                  # 12 systems in global memory, slabs of the largest N
    assert lib.raftk_farm_ragged_workspace_bytes(C.byref(d), C.byref(c), C.byref(f)) == 256 + 12 * slab24
    d, c, _, _, f, keep = _structs((21, 3), nC=64, nw=1024)                  # a full persistent grid, as the uniform batch's
    from raft_b200 import solver
    assert lib.raftk_farm_ragged_workspace_bytes(C.byref(d), C.byref(c), C.byref(f)) == 256 + solver.farm_batch_workspace_bytes(1, 21, 64, 1024)
    assert solver.farm_batch_workspace_bytes(1, 21, 64, 1024) % slab21 == 0
    d, c, _, _, f, keep = _structs((2, 0, 3))
    assert lib.raftk_farm_ragged_workspace_bytes(C.byref(d), C.byref(c), C.byref(f)) == 0


def _refuse(mutate, msg, sizes=(2, 3), **kw):
    from raft_b200._lib import lib
    d, c, o, out, f, keep = _structs(sizes, **kw)
    keep = (keep, mutate(d, c, out, f))
    before = lib.raftk_launch_count()
    rc = lib.raftk_solve_dynamics_farm_ragged_host(C.byref(d), C.byref(c), C.byref(o), C.byref(out), C.byref(f))
    assert rc == -1 and msg in lib.raftk_last_error().decode(), lib.raftk_last_error()
    rc = lib.raftk_farm_ragged_response_ws_dev(C.byref(d), C.byref(c), C.byref(out), C.byref(f), 0x1000, 1 << 30, None)
    assert rc == -1 and msg in lib.raftk_last_error().decode(), lib.raftk_last_error()
    assert lib.raftk_launch_count() == before


def _set(**kv):
    def m(d, c, out, f):
        for k, v in kv.items():
            setattr(f, k, v)
    return m


def _csr(name, values, dtype):
    def m(d, c, out, f):
        a = np.array(values, dtype=dtype)
        setattr(f, name, a.ctypes.data)
        return a
    return m


@pytest.mark.parametrize("mutate,msg", [
    (_set(n_farms=0), "n_farms must be >= 1"),
    (_set(farm_fowt0=None), "farm_fowt0 is required"),
    (_csr("farm_fowt0", [1, 2, 5], np.int32), "farm_fowt0[0] must be 0"),
    (_csr("farm_fowt0", [0, 2, 2], np.int32), "strictly increasing (farm 1 is empty)"),
    (_csr("farm_fowt0", [0, 3, 2], np.int32), "strictly increasing (farm 1 is empty)"),
    (_csr("farm_fowt0", [0, 2, 4], np.int32), "farm_fowt0[n_farms] must equal designs.n_designs"),
    (_set(arr_shared=2), "arr_shared must be 0 or 1"),
    (_set(arr_shared=1), "arr_shared = 1 needs every farm to have the same N (farm 1 differs)"),
    (_set(arr_offset=None), "arr_offset is required"),
    (_csr("arr_offset", [0, 144, 144 + 323], np.int64), "step by 36 N^2 (farm 1 does not)"),
    (_csr("arr_offset", [8, 152, 152 + 324], np.int64), "arr_offset must start at 0"),
    (_set(Xi_sys=None), "Xi_sys is required"),
])
def test_refusals_before_any_device_use(mutate, msg):
    _refuse(mutate, msg)


def test_device_entry_refusals():
    from raft_b200._lib import lib
    for missing in ("B_drag", "F_drag", "F_iner"):
        d, c, o, out, f, keep = _structs()
        setattr(out, missing, None)
        assert lib.raftk_farm_ragged_response_ws_dev(C.byref(d), C.byref(c), C.byref(out), C.byref(f), 0x1000, 1 << 20, None) == -1
        assert "B_drag, F_drag, F_iner" in lib.raftk_last_error().decode()
    d, c, o, out, f, keep = _structs()
    d.n_bem_head = 4
    assert lib.raftk_farm_ragged_response_ws_dev(C.byref(d), C.byref(c), C.byref(out), C.byref(f), 0x1000, 1 << 20, None) == -1
    assert "F_BEM is required" in lib.raftk_last_error().decode()
    d, c, o, out, f, keep = _structs((2, 24, 3))
    for ws, nbytes in ((None, 1 << 30), (0x1000, 255), (0x1000, 256 + 144 * 145 * 16 - 1)):
        assert lib.raftk_farm_ragged_response_ws_dev(C.byref(d), C.byref(c), C.byref(out), C.byref(f), ws, nbytes, None) == -1
        assert "descriptor table and one [6N][6N+1] slab" in lib.raftk_last_error().decode()
    d, c, o, out, f, keep = _structs((2, 3), nC=65536)
    assert lib.raftk_farm_ragged_response_ws_dev(C.byref(d), C.byref(c), C.byref(out), C.byref(f), 0x1000, 1 << 20, None) == -1
    assert "65535 cases" in lib.raftk_last_error().decode()
    d, c, o, out, f, keep = _structs((1,) * 65536 + (2,))
    assert lib.raftk_farm_ragged_response_ws_dev(C.byref(d), C.byref(c), C.byref(out), C.byref(f), 0x1000, 1 << 30, None) == -1
    assert "65535 farms of one on-chip kernel class" in lib.raftk_last_error().decode()


def _brute_best(cost, world):
    best = sum(cost)
    for cuts in itertools.combinations_with_replacement(range(len(cost) + 1), world - 1):
        b = (0,) + cuts + (len(cost),)
        best = min(best, max(sum(cost[b[r]:b[r + 1]]) for r in range(world)))
    return best


@pytest.mark.parametrize("sizes,world", [(SIZES, 1), (SIZES, 2), (SIZES, 3), (SIZES, 5), ((2, 4, 8, 16, 32, 64) * 2, 4),
                                         ((3,), 4), ((64, 2, 2, 2, 2, 2, 2), 2), ((1, 1, 1, 1), 3)])
def test_ragged_farm_shards(sizes, world):
    """Contiguous runs, every farm exactly once, and the largest rank cost is the optimum over all contiguous splits."""
    from raft_b200 import sweep
    b = sweep.ragged_farm_shards(sizes, world)
    assert len(b) == world and b[0][0] == 0 and b[-1][1] == len(sizes)
    assert all(lo <= hi for lo, hi in b) and all(b[r][1] == b[r + 1][0] for r in range(world - 1))
    cost = [sweep.ragged_farm_cost(n) for n in sizes]
    assert max(sum(cost[lo:hi]) for lo, hi in b) == _brute_best(cost, world)


def _gloo_worker(rank, world, port, sizes, q):
    import torch
    import torch.distributed as dist
    from raft_b200 import solver, sweep
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    bounds = sweep.ragged_farm_shards(sizes, world)
    fowt0, _ = solver.ragged_offsets(sizes)
    lo, hi = bounds[rank]
    a, b = int(fowt0[lo]), int(fowt0[hi])
    U, nC, nw = 6 * 2 * 3, 2, 3
    xi = (torch.arange(a * U, b * U, dtype=torch.float64) + 1j * rank).to(torch.complex128).view(-1, U)
    info = (torch.arange(lo, hi, dtype=torch.int32)[:, None, None] * 100 + rank).repeat(1, nC, nw)
    st = torch.arange(a, b, dtype=torch.int32)[:, None, None].repeat(1, nC, 4)
    X, I, S = sweep.gather_ragged_farm_shards((xi, info, st), bounds, fowt0)
    q.put((rank, bounds, X.numpy(), I.numpy(), S.numpy()))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("sizes", [(3, 2, 21, 1, 20), (64, 2, 2), (5,)])
def test_ragged_gather_on_two_gloo_ranks(sizes):
    """The NCCL exchange of ShardedFarmSolve(farm_sizes=...) on 2 gloo ranks: every farm's flat Xi_sys, info and status rows
    land at their global offsets on both ranks (an uneven split, a rank with one large farm, a rank without farms)."""
    import torch.multiprocessing as mp
    from raft_b200 import solver
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    world, port = 2, 29800 + len(sizes) * 7 + sizes[0]
    procs = [ctx.Process(target=_gloo_worker, args=(r, world, port, sizes, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    fowt0, _ = solver.ragged_offsets(sizes)
    nD, U = int(fowt0[-1]), 36
    for rank, bounds, X, I, S in got:
        owner = np.concatenate([[r] * (int(fowt0[h]) - int(fowt0[l])) for r, (l, h) in enumerate(bounds)]).astype(int)
        assert X.shape == (nD, U) and np.array_equal(X.real.reshape(-1), np.arange(nD * U)), rank
        assert np.array_equal(X.imag[:, 0], owner)
        fo = np.concatenate([[r] * (h - l) for r, (l, h) in enumerate(bounds)]).astype(int)
        assert np.array_equal(I[:, 0, 0], np.arange(len(sizes)) * 100 + fo)
        assert S.shape == (nD, 2, 4) and np.array_equal(S[:, 0, 0], np.arange(nD))


# ---- on the GPU ---------------------------------------------------------------------------------------------------------
def _ragged(sizes, nw=13, tables=False, seed=0):
    """-> (packs [F][N_f], C_arr list of [6N_f,6N_f]): the two-FOWT fixture's FOWTs on 1600 m rows, each farm moved by its own
    offsets and with a seeded SPD array stiffness; ``tables``: seeded A_w / B_w / X_BEM as test_farm_batch's."""
    from raft_b200 import grid
    base, _ = _base(2)
    base = [grid.regrid(P, nw, 0.005 * nw) for P in base]
    rng = np.random.default_rng(11 + seed)
    packs, C_arr = [], []
    for f, N in enumerate(sizes):
        row = []
        for i in range(N):
            P = _moved(base[i % 2], 1600.0 * (i - i % 2), 0.0)
            row.append(_moved(P, 97.0 * (f + seed) * (i % 4 + 1), -173.0 * (f + seed) * (i % 3 + 1)))
        packs.append(row)
        C_arr.append(_spd(6 * N, 700 * N + f + seed))
    if tables:
        for row in packs:
            for i, P in enumerate(row):
                d = np.diag(rng.uniform(0.5, 1.5, size=6))
                row[i] = dict(P, A_w=(np.abs(P["M0"]) * 0.05 * d)[:, :, None] * rng.uniform(0.5, 1.0, size=nw)[None, None, :],
                              B_w=(np.abs(P["M0"]) * 0.01 * d)[:, :, None] * rng.uniform(0.0, 1.0, size=nw)[None, None, :],
                              bem_headings=np.array([0.0, 90.0, 180.0, 270.0]), heading_adjust=0.0,
                              X_BEM=(rng.normal(size=(4, 6, nw)) + 1j * rng.normal(size=(4, 6, nw))) * 2e5)
    return packs, C_arr


def _flat(packs):
    return [P for row in packs for P in row]


ROWS = np.array([[6.0, 12.0, 0.0], [3.5, 9.0, 40.0]])


def _check_against_single(packs, out, C_arr, cases_of, want=PER_FOWT, primary=None):
    from raft_b200 import solver
    d0 = 0
    for f, row in enumerate(packs):
        N = len(row)
        one = solver.solve_dynamics_farm(solver.DesignBatch(row), cases_of(f, d0, d0 + N), C_arr=C_arr[f], want=want)
        assert solver.last_dispatch()["kernel"] == CLASS[N]
        assert out["Xi_sys"][f].shape == one["Xi_sys"].shape
        assert np.array_equal(out["Xi_sys"][f], one["Xi_sys"]), (f, N)
        assert np.array_equal(out["info"][f], one["info"]), (f, N)
        for k in want:
            a, b = out[k][d0:d0 + N], one[k]
            if k == "B_drag" and primary is not None:
                a, b = a[:, np.unique(primary)], b[:, np.unique(primary)]
            assert np.array_equal(a, b), (f, N, k)
        d0 += N


@gpu
def test_every_farm_equals_the_single_farm_entry():
    """Sizes covering every kernel class in interleaved order: each farm's Xi_sys, info and per-FOWT outputs equal
    solve_dynamics_farm on that farm alone, bit for bit; the dispatch record names the four classes."""
    from raft_b200 import solver
    packs, C_arr = _ragged(SIZES)
    ct = solver.CaseTable(_cases(ROWS))
    out = solver.solve_dynamics_farm_ragged(solver.DesignBatch(_flat(packs)), ct, SIZES, C_arr=C_arr, want=PER_FOWT)
    rec = solver.last_dispatch()
    assert rec["family"] == "farm" and rec["kernel"] == "farm-global", rec
    assert set(rec["farm_classes"]) == {"farm-rows12", "farm-warp", "farm-block", "farm-global"}, rec
    assert out["info"].shape == (len(SIZES), 2, 13) and not np.any(out["info"])
    assert all(np.shares_memory(x, out["Xi_sys_flat"]) for x in out["Xi_sys"])
    _check_against_single(packs, out, C_arr, lambda f, a, b: ct)


@gpu
def test_reordering_permutes_the_results():
    from raft_b200 import solver
    packs, C_arr = _ragged(SIZES)
    ct = solver.CaseTable(_cases(ROWS))
    out = solver.solve_dynamics_farm_ragged(solver.DesignBatch(_flat(packs)), ct, SIZES, C_arr=C_arr)
    perm = [5, 1, 7, 3, 0, 6, 2, 4]
    sizes = [SIZES[p] for p in perm]
    alt = solver.solve_dynamics_farm_ragged(solver.DesignBatch(_flat([packs[p] for p in perm])), ct, sizes, C_arr=[C_arr[p] for p in perm])
    assert set(solver.last_dispatch()["farm_classes"]) == {"farm-rows12", "farm-warp", "farm-block", "farm-global"}
    for k, p in enumerate(perm):
        assert np.array_equal(alt["Xi_sys"][k], out["Xi_sys"][p]) and np.array_equal(alt["info"][k], out["info"][p])
    fowt0, _ = solver.ragged_offsets(SIZES)
    order = np.concatenate([np.arange(fowt0[p], fowt0[p + 1]) for p in perm])
    assert np.array_equal(alt["Xi"], out["Xi"][order]) and np.array_equal(alt["status"], out["status"][order])


@gpu
@pytest.mark.parametrize("N", [2, 3, 8, 24])
def test_equal_sizes_equal_the_uniform_batch(N):
    """A ragged batch whose farms all have N FOWTs equals solve_dynamics_farm_batch(n_fowt=N), per-farm and shared matrices."""
    from raft_b200 import solver
    F = 3
    packs, C_arr = _ragged((N,) * F, nw=11, seed=N)
    ct = solver.CaseTable(_cases(ROWS))
    b = solver.DesignBatch(_flat(packs))
    for mats in (C_arr, C_arr[1]):
        uni = solver.solve_dynamics_farm_batch(b, ct, N, C_arr=np.array(mats))
        kernel = solver.last_dispatch()["kernel"]
        rag = solver.solve_dynamics_farm_ragged(b, ct, (N,) * F, C_arr=mats)
        assert solver.last_dispatch()["farm_classes"] == (kernel,)
        for f in range(F):
            assert np.array_equal(rag["Xi_sys"][f], uni["Xi_sys"][f]) and np.array_equal(rag["info"][f], uni["info"][f])
        assert np.array_equal(rag["Xi"], uni["Xi"])


@gpu
@pytest.mark.parametrize("variant", ["ops", "bem", "oc4_wamit", "f2nd_trains"])
def test_operating_points_bem_second_order_and_trains(variant):
    """Per-case operating points, BEM tables (F_BEM in the load), the second-order force and secondary wave trains go
    through a ragged batch and equal the per-farm calls, bit for bit."""
    from raft_b200 import solver
    sizes = (2, 21, 1, 7, 3)
    packs, C_arr = _ragged(sizes, nw=12, tables=variant == "bem", seed=5)
    if variant == "oc4_wamit":                 # the OC4 semi with its WAMIT tables (A_w, B_w, X_BEM), moved copies per farm
        from conftest import GOLDEN
        z = np.load(os.path.join(GOLDEN, "test_OC4semi-WAMIT_Coefs.npz"))
        P = {k[2:]: z[k] for k in z.files if k.startswith("P_")}
        assert "A_w" in P and "X_BEM" in P
        packs = [[_moved(P, 900.0 * i + 61.0 * f, -47.0 * f * (i % 3)) for i in range(N)] for f, N in enumerate(sizes)]
    nD, nw = sum(sizes), len(packs[0][0]["w"])
    rng = np.random.default_rng(9)
    want, primary = PER_FOWT, None
    if variant == "ops":
        rows = np.array([[6.0, 12.0, 0.0], [3.0, 8.0, 30.0], [4.0, 9.0, 60.0]])
        op = np.array([1, 0, 1], dtype=np.int32)
        A = rng.normal(size=(nD, 2, 6, 6, nw)) * 1e4
        B = rng.normal(size=(nD, 2, 6, 6, nw)) * 1e3
        ct = solver.CaseTable(_cases(rows), ops=dict(op=op, A_w=A, B_w=B))
        cases_of = lambda f, a, b: solver.CaseTable(_cases(rows), ops=dict(op=op, A_w=A[a:b], B_w=B[a:b]))   # noqa: E731
    elif variant in ("bem", "oc4_wamit"):
        ct = solver.CaseTable(_cases(ROWS))
        cases_of = lambda f, a, b: ct     # noqa: E731
        want = PER_FOWT + ("F_BEM",)
    else:
        rows = np.array([[6.0, 12.0, 0.0], [2.0, 7.0, 60.0], [4.0, 10.0, 200.0], [1.5, 6.0, 100.0]])
        primary = [0, 0, 2, 2]
        F2 = rng.normal(size=(nD, len(rows), 6, nw)) * 5e4
        ct = solver.CaseTable(_cases(rows, primary=primary), F_2nd=F2)
        cases_of = lambda f, a, b: solver.CaseTable(_cases(rows, primary=primary), F_2nd=F2[a:b])   # noqa: E731
    out = solver.solve_dynamics_farm_ragged(solver.DesignBatch(_flat(packs)), ct, sizes, C_arr=C_arr, want=want)
    assert not np.any(out["info"])
    _check_against_single(packs, out, C_arr, cases_of, want=want, primary=primary)
    if variant in ("bem", "oc4_wamit"):
        assert np.any(out["F_BEM"] != 0)


def _session(packs, rows=ROWS):
    from raft_b200 import solver
    sess = solver.DeviceSession(solver.DesignBatch(_flat(packs)), solver.CaseTable(_cases(rows)), device="cuda:0", want=PER_FOWT)
    sess.solve(n_iter=10)
    return sess


@gpu
def test_device_session_and_workspace_sizes():
    """DeviceSession.farm_response(farm_sizes=...) (the _ws_dev entry) equals the host entry; workspaces below the query that
    hold the table and one slab give the same bits; one byte less is refused."""
    import torch
    from raft_b200 import _lib, solver
    packs, C_arr = _ragged(SIZES)
    host = solver.solve_dynamics_farm_ragged(solver.DesignBatch(_flat(packs)), solver.CaseTable(_cases(ROWS)), SIZES, C_arr=C_arr)
    sess = _session(packs)
    xi, info = sess.farm_response(C_arr=C_arr, farm_sizes=SIZES)
    torch.cuda.synchronize()
    assert len(xi) == len(SIZES) and set(solver.last_dispatch()["farm_classes"]) == {"farm-rows12", "farm-warp", "farm-block", "farm-global"}
    for f in range(len(SIZES)):
        assert np.array_equal(xi[f].cpu().numpy(), host["Xi_sys"][f]) and np.array_equal(info[f].cpu().numpy(), host["info"][f])
    _, fs, _, flat, _, ws, wsb, _ = sess._farm_rag
    slab, table = 144 * 145 * 16, 512                                          # 8 descriptors of 40 bytes, 256-byte aligned
    assert wsb == table + 2 * 13 * (1 + 1) * slab                             # 52 global systems: fewer than a full grid
    args = (C.byref(sess.d_struct), C.byref(sess.c_struct), C.byref(sess.o_struct), C.byref(fs))
    stream = torch.cuda.current_stream().cuda_stream
    for nbytes in (table + slab, table + 5 * slab + 100):
        flat.zero_()
        info.fill_(-7)
        assert _lib.lib.raftk_farm_ragged_response_ws_dev(*args, ws.data_ptr(), nbytes, stream) == 0
        torch.cuda.synchronize()
        for f in range(len(SIZES)):
            assert np.array_equal(xi[f].cpu().numpy(), host["Xi_sys"][f]) and np.array_equal(info[f].cpu().numpy(), host["info"][f]), nbytes
    assert _lib.lib.raftk_farm_ragged_response_ws_dev(*args, ws.data_ptr(), table + slab - 1, stream) == -1
    assert solver.last_dispatch()["kernel"] == "none"


@gpu
def test_a_zero_pivot_stays_in_its_own_farm():
    """Farm 2's (N = 21, global memory) and farm 4's (N = 20, shared memory) last FOWT lose yaw inertia, damping and stiffness
    and their array stiffness leaves that DOF free: info of those farms reports pivot 6N everywhere, every other farm keeps
    info 0 and the bits of the run without the defect."""
    from raft_b200 import solver
    packs, C_arr = _ragged(SIZES)
    sess = _session(packs)
    xi, info = sess.farm_response(C_arr=C_arr, farm_sizes=SIZES)
    good = [x.cpu().numpy().copy() for x in xi]
    fowt0, arr = solver.ragged_offsets(SIZES)
    mats = sess._farm_rag[2][2]["C_arr"]
    for f in (2, 4):
        d, n = int(fowt0[f + 1]) - 1, 6 * SIZES[f]
        for t in (sess.dt["M0"], sess.dt["B0"], sess.dt["C0"]):
            t.view(-1, 6, 6)[d, :, 5] = 0.0
        sess.out["B_drag"][d, :, :, 5] = 0.0
        mats[int(arr[f]):int(arr[f + 1])].view(n, n)[:, n - 1] = 0.0
    xi, info = sess.farm_response(farm_sizes=SIZES)
    info = info.cpu().numpy()
    for f, N in enumerate(SIZES):
        if f in (2, 4):
            assert np.all(info[f] == 6 * N), f
        else:
            assert not np.any(info[f]) and np.array_equal(xi[f].cpu().numpy(), good[f]), f


@gpu
def test_reference_runs_in_a_ragged_batch():
    """The two-FOWT and 24-FOWT reference farms, with synthetic farms between them, reproduce the reference's own runs."""
    from raft_b200 import solver
    p2, z2 = _base(2)
    p24, z24 = _base(24)
    nC = len(z24["cases"])                                                     # the 24-FOWT run's cases are the first of the other's
    assert np.array_equal(z2["cases"][:nC], z24["cases"]) and np.array_equal(p2[0]["w"], p24[0]["w"])
    assert int(z2["n_iter"]) == int(z24["n_iter"]) and float(z2["xi_start"]) == float(z24["xi_start"])
    mid = [[_moved(p2[i % 2], 1600.0 * (i - i % 2) + 50.0 * k, 30.0 * k) for i in range(N)] for k, N in enumerate((3, 7))]
    packs = [p2] + mid + [p24]
    sizes = tuple(len(r) for r in packs)
    C_arr = [z2["C_array"], _spd(18, 1), _spd(42, 2), z24["C_array"]]
    out = solver.solve_dynamics_farm_ragged(solver.DesignBatch(_flat(packs)), solver.CaseTable(_cases(z24["cases"])), sizes, C_arr=C_arr,
                                            n_iter=int(z2["n_iter"]), xi_start=float(z2["xi_start"]))
    assert set(solver.last_dispatch()["farm_classes"]) == {"farm-rows12", "farm-warp", "farm-block", "farm-global"}
    assert not np.any(out["info"])
    for f, z in ((0, z2), (3, z24)):
        N = sizes[f]
        ref = z["ref_run_Xi"][:nC, 0]
        err = max(response_err(out["Xi_sys"][f][:, 6 * i:6 * i + 6], ref[:, 6 * i:6 * i + 6]) for i in range(N))
        assert err < 1e-10, (f, err)


@gpu
@pytest.mark.parametrize("tile_w", [0, 5, -1])
def test_channel_statistics_of_a_ragged_batch(tile_w):
    """raftk_farm_ragged_channel_stats on the flat Xi_sys (R_f packed, channels per farm, mixed wpow) against
    raftk_farm_channel_stats on each farm alone, bit for bit; host buffers, the resident views, and views that are not one
    buffer (packed by the wrapper) give the same bits."""
    import torch
    from raft_b200 import solver
    sizes = (2, 21, 3)
    packs, C_arr = _ragged(sizes, nw=12, seed=8)
    out = solver.solve_dynamics_farm_ragged(solver.DesignBatch(_flat(packs)), solver.CaseTable(_cases(ROWS)), sizes, C_arr=C_arr)
    rng = np.random.default_rng(4)
    R = [rng.normal(size=(3 * N + 1, 6 * N)) * 1e3 for N in sizes]
    wpow = [rng.integers(0, 3, size=3 * N + 1) for N in sizes]
    w = packs[0][0]["w"]
    l0 = solver.launch_count()
    sd, P, A = solver.farm_channel_stats(R, out["Xi_sys"], float(w[0]), w=w, wpow=wpow, psd=True, amp=True, tile_w=tile_w)
    assert solver.launch_count() - l0 == 2                                     # one tile pass and one reduction for every farm
    for f in range(len(sizes)):
        s1, p1, a1 = solver.farm_channel_stats(R[f], np.ascontiguousarray(out["Xi_sys"][f]), float(w[0]), w=w, wpow=wpow[f], psd=True,
                                               amp=True)
        assert sd[f].shape == s1.shape == (2, 3 * sizes[f] + 1)
        assert np.array_equal(sd[f], s1) and np.array_equal(P[f], p1) and np.array_equal(A[f], a1), f
    dev = [torch.from_numpy(out["Xi_sys_flat"]).cuda()]
    views = solver.ragged_views(dev[0], sizes, 2, 12)
    for xs in (views, [v.clone() for v in views]):
        sd2, _, _ = solver.farm_channel_stats(R, xs, float(w[0]), w=w, wpow=wpow, psd=False, tile_w=tile_w)
        torch.cuda.synchronize()
        for f in range(len(sizes)):
            assert np.array_equal(sd2[f].cpu().numpy(), sd[f])


def _same_ragged(got, ref):
    X, I, S = got
    for f, x in enumerate(X):
        assert np.array_equal(x.cpu().numpy(), ref["Xi_sys"][f]), f
    assert np.array_equal(I.cpu().numpy(), ref["info"]) and np.array_equal(S.cpu().numpy(), ref["status"])


@gpu
@pytest.mark.parametrize("exchange", ["peer", "nccl"])
def test_single_rank_sharded_ragged_solve(exchange):
    """ShardedFarmSolve(farm_sizes=...) without a process group, both exchanges, two steps (alternating copies): the one-call
    ragged batch's Xi_sys, info and status, bit for bit."""
    import torch
    from raft_b200 import solver, sweep
    packs, C_arr = _ragged(SIZES)
    ct = solver.CaseTable(_cases(ROWS))
    ref = solver.solve_dynamics_farm_ragged(solver.DesignBatch(_flat(packs)), ct, SIZES, C_arr=C_arr)
    sh = sweep.ShardedFarmSolve(solver.DesignBatch(_flat(packs)), ct, C_arr=C_arr, exchange=exchange, farm_sizes=SIZES)
    assert sh.exchange == exchange and sh.world == 1 and sh.bounds == [(0, len(SIZES))]
    for _ in range(2):
        got = sh.step(n_iter=10)
        torch.cuda.synchronize()
        _same_ragged(got, ref)
    sh.close()


@gpu
@pytest.mark.parametrize("world", [2, 3])
def test_emulated_ranks_of_the_ragged_gather(world):
    """``world`` ranks on one device, each with its own copy: rank r solves its farms of ragged_farm_shards and
    raftk_farm_ragged_response_gather_dev stores them at their global offsets of every copy; every copy then holds the
    one-call batch, bit for bit.  (Ranks run in turn on one stream, so no barrier is needed.)"""
    import torch
    from raft_b200 import _lib, solver, sweep
    packs, C_arr = _ragged(SIZES)
    ct = solver.CaseTable(_cases(ROWS))
    batch = solver.DesignBatch(_flat(packs))
    ref = solver.solve_dynamics_farm_ragged(batch, ct, SIZES, C_arr=C_arr)
    fowt0, _ = solver.ragged_offsets(SIZES)
    F, nD, nC, nw = len(SIZES), int(fowt0[-1]), 2, 13
    U = 6 * nC * nw
    bounds = sweep.ragged_farm_shards(SIZES, world)
    copies = [(torch.full([nD * U], complex("nan"), dtype=torch.complex128, device="cuda:0"),
               torch.full([F * nC * nw + nD * nC * 4], -9, dtype=torch.int32, device="cuda:0"),
               torch.zeros(64, dtype=torch.int32, device="cuda:0")) for _ in range(world)]
    block = -(-nD * U // world)
    for r, (lo, hi) in enumerate(bounds):
        if hi == lo:
            continue
        a, b = int(fowt0[lo]), int(fowt0[hi])
        sess = solver.DeviceSession(batch.take(a, b), sweep.shard_design_cases(ct, a, b), device="cuda:0", want=PER_FOWT)
        sess.solve(n_iter=10)
        pr = _lib.RaftkPeers()
        pr.n_ranks, pr.rank, pr.epoch, pr.block_elems = world, r, 1, block
        for q, (X, I, Fl) in enumerate(copies):
            pr.gathered[q], pr.status[q], pr.flags[q] = X.data_ptr(), I.data_ptr(), Fl.data_ptr()
        X, I, _ = copies[r]
        sess.farm_response_ragged_gather(pr, lo, a, F, X[a * U:b * U], I[lo * nC * nw:hi * nC * nw], SIZES[lo:hi], C_arr=C_arr[lo:hi])
    torch.cuda.synchronize()
    for X, I, _ in copies:
        got = (solver.ragged_views(X, SIZES, nC, nw), I[:F * nC * nw].view(F, nC, nw), I[F * nC * nw:].view(nD, nC, 4))
        _same_ragged(got, ref)


def _nccl_worker(rank, world, port, exchange, q):
    import torch
    import torch.distributed as dist
    from raft_b200 import solver, sweep
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    packs, C_arr = _ragged(SIZES)
    sh = sweep.ShardedFarmSolve(solver.DesignBatch(_flat(packs)), solver.CaseTable(_cases(ROWS)), C_arr=C_arr, exchange=exchange,
                                farm_sizes=SIZES)
    X, I, S = sh.step(n_iter=10)
    torch.cuda.synchronize()
    q.put((rank, sh.exchange, [x.cpu().numpy() for x in X], I.cpu().numpy(), S.cpu().numpy()))
    sh.close()
    dist.barrier()
    dist.destroy_process_group()


@gpu
@pytest.mark.parametrize("exchange", ["peer", "nccl"])
def test_ragged_batch_sharded_over_two_gpus(exchange):
    """Two processes on two GPUs (NCCL group): ShardedFarmSolve(farm_sizes=...) returns the whole batch on every rank, bit
    for bit what the one-GPU call returns, with both exchanges."""
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two visible GPUs")
    from raft_b200 import solver
    packs, C_arr = _ragged(SIZES)
    ref = solver.solve_dynamics_farm_ragged(solver.DesignBatch(_flat(packs)), solver.CaseTable(_cases(ROWS)), SIZES, C_arr=C_arr)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29900 + (exchange == "peer")
    procs = [ctx.Process(target=_nccl_worker, args=(r, 2, port, exchange, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = [q.get(timeout=600) for _ in procs]
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    for rank, used, X, I, S in got:
        for f, x in enumerate(X):
            assert np.array_equal(x, ref["Xi_sys"][f]), (rank, used, f)
        assert np.array_equal(I, ref["info"]) and np.array_equal(S, ref["status"]), (rank, used)
