"""Farm batches sharded over GPUs (raftk_farm_batch_response_gather_dev, sweep.farm_shards, sweep.ShardedFarmSolve).

Without a GPU: the shard plan, the binding against include/raftk.h, every refusal of the gather entry (before any launch),
DesignBatch.take and the per-design case rows of a shard, and the NCCL-path gather of padded shards on two gloo ranks.
On the GPU: emulated ranks on separate streams of one device, each with its own gathered copy (plain raftk_peer_alloc memory,
as tests/test_exchange.py): every rank's gathered Xi_sys, info and status equal one solve_dynamics_farm_batch call over all
farms, bit for bit, on every farm kernel, with even and uneven shards and a rank without farms."""
import ctypes as C
import os

import numpy as np
import pytest

from test_farm_batch import _cases, _farms, _flat, _prototype, _refusal_structs

gpu = pytest.mark.gpu
WANT = ("Xi", "status", "B_drag", "F_drag", "F_iner")


# ---- without a GPU --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("F,world", [(4, 2), (5, 2), (5, 3), (16, 8), (7, 4), (2, 3), (1, 4), (0, 2)])
def test_farm_shards(F, world):
    from raft_b200 import sweep
    b = sweep.farm_shards(F, world)
    assert len(b) == world and b[0][0] == 0 and b[-1][1] == F
    assert all(b[r][1] == b[r + 1][0] for r in range(world - 1))               # contiguous, every farm once, in order
    sizes = [h - l for l, h in b]
    assert max(sizes) - min(sizes) <= 1 and sizes == sorted(sizes, reverse=True)
    assert max(sizes) == -(-F // world)                                         # F_max: the padded slot count per rank
    if world > F:
        assert sizes[F:] == [0] * (world - F)
    rows = max(1, max(sizes))
    for per in (1, 3):                                                          # the farms' rows of a padded gathered array
        keep = sweep.farm_rows(b, per).numpy()
        want = [(r * rows + (f - lo)) * per + j for r, (lo, hi) in enumerate(b) for f in range(lo, hi) for j in range(per)]
        assert keep.tolist() == want and (F == 0 or keep.max() < world * rows * per)


def test_binding_matches_header_prototype():
    from raft_b200 import _lib
    name = "raftk_farm_batch_response_gather_dev"
    structs = (("raftk_farm_batch", _lib.RaftkFarmBatch), ("raftk_designs", _lib.RaftkDesigns), ("raftk_cases", _lib.RaftkCases),
               ("raftk_outputs", _lib.RaftkOutputs), ("raftk_peers", _lib.RaftkPeers))
    ret, params = _prototype(name)
    fn = getattr(_lib.lib, name)
    assert name in _lib.SYMBOLS and len(fn.argtypes) == len(params) and ret == "int" and fn.restype is C.c_int
    for decl, ct in zip(params, fn.argtypes):
        want = next((C.POINTER(t) for s, t in structs if s in decl),
                    C.c_void_p if "*" in decl else C.c_int32 if "int32_t" in decl else C.c_size_t)
        assert ct is want, (decl, ct)


def test_peers_struct_layout_matches_header(tmp_path):
    import subprocess
    from conftest import ROOT
    from raft_b200 import _lib
    S = _lib.RaftkPeers
    fields = [n for n, _ in S._fields_]
    src = tmp_path / "t.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "raftk.h"\nint main(void){printf("%%zu %s\\n", sizeof(raftk_peers), %s);'
                   'return 0;}\n' % (" ".join(["%zu"] * len(fields)), ", ".join("offsetof(raftk_peers, %s)" % n for n in fields)))
    exe = tmp_path / "t"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert got == [C.sizeof(S)] + [getattr(S, n).offset for n in fields]


def _gather_args(world=2, rank=1, F_max=3, nD=6, nC=2, nw=16, N=2):
    """Structs of a rank holding farms [rank * F_max, + 3) of 2 FOWTs in a consistent copy; pointers are never followed."""
    from raft_b200 import _lib
    d, c, o, out, f = _refusal_structs(nD, nC, nw)
    per_farm = nC * 6 * N * nw
    pr = _lib.RaftkPeers()
    pr.n_ranks, pr.rank, pr.epoch, pr.block_elems = world, rank, 1, F_max * per_farm
    for r in range(world):
        base = 0x10000000 * (r + 1)
        pr.gathered[r], pr.flags[r], pr.status[r] = base, base + 0x8000000, base + 0x9000000
    f.Xi_sys = pr.gathered[rank] + rank * F_max * per_farm * 16
    f.info = pr.status[rank] + rank * F_max * nC * nw * 4
    return d, c, out, f, pr, rank * F_max


def _gather(d, c, out, f, pr, row0, peers=True):
    from raft_b200._lib import lib
    return lib.raftk_farm_batch_response_gather_dev(C.byref(d), C.byref(c), C.byref(out), C.byref(f), C.byref(pr) if peers else None,
                                                    row0, None, 0, None)


def _bad(what):
    d, c, out, f, pr, row0 = _gather_args()
    peers = True
    if what == "null peers":
        peers = False
    elif what == "rank":
        pr.rank = 2
    elif what == "negative rank":
        pr.rank = -1
    elif what == "n_ranks":
        pr.n_ranks = 17
    elif what == "flags":
        pr.flags[0] = None
    elif what == "status copy":
        pr.status[0] = None
    elif what == "info":
        f.info = None
    elif what == "per-FOWT status":
        out.status = None
    elif what == "block not farm-shaped":
        pr.block_elems += 1
    elif what == "copy smaller than one farm":
        pr.block_elems = 0
    elif what == "F_local > F_max":
        pr.block_elems //= 3                                                   # F_max = 1 for a rank with 3 farms
        f.Xi_sys, f.info = pr.gathered[1] + 1 * 768 * 16, pr.status[1] + 32 * 4
        row0 = 1
    elif what == "row0 past the copy":
        row0 = 4
    elif what == "negative row0":
        row0 = -1
    elif what == "another rank's rows":
        row0 = 0                                                                # rank 0's farms, with pointers that match them
        f.Xi_sys, f.info = pr.gathered[1], pr.status[1]
    elif what == "Xi_sys elsewhere":
        f.Xi_sys += 16
    elif what == "info elsewhere":
        f.info = pr.status[0] + row0 * 32 * 4
    elif what == "farm shape":
        f.n_fowt = 3
    return _gather(d, c, out, f, pr, row0, peers)


@pytest.mark.parametrize("what,msg", [
    ("null peers", "null peers"), ("rank", "0 <= rank < n_ranks"), ("negative rank", "0 <= rank < n_ranks"),
    ("n_ranks", "n_ranks <= RAFTK_MAX_PEERS"), ("flags", "gathered / flags pointer missing"),
    ("status copy", "gathered info and status (peers.status) is missing"), ("info", "farm_batch.info and the per-FOWT status"),
    ("per-FOWT status", "farm_batch.info and the per-FOWT status"), ("block not farm-shaped", "F_max * nC * 6N * nw"),
    ("copy smaller than one farm", "F_max * nC * 6N * nw"), ("F_local > F_max", "n_farms exceeds F_max"),
    ("row0 past the copy", "farm_row0 must be rank * F_max"), ("negative row0", "farm_row0 must be rank * F_max"),
    ("another rank's rows", "farm_row0 must be rank * F_max"),
    ("Xi_sys elsewhere", "this rank's farms in its own gathered copy"), ("info elsewhere", "this rank's farms in its own gathered copy"),
    ("farm shape", "n_farms * n_fowt"),
])
def test_gather_entry_refuses_before_any_launch(what, msg):
    from raft_b200._lib import lib
    before = lib.raftk_launch_count()
    assert _bad(what) == -1
    assert msg in lib.raftk_last_error().decode(), (what, lib.raftk_last_error())
    assert lib.raftk_launch_count() == before


def test_take_and_case_rows_of_a_shard():
    """DesignBatch.take(lo, hi) holds exactly the tables of DesignBatch(packs[lo:hi]) and keeps the whole batch's hints;
    shard_design_cases keeps every case and the designs' rows of F_2nd and of per-design operating-point tables."""
    from raft_b200 import solver, sweep
    packs, _ = _farms(3, 3, nw=20, tables=True)
    flat = _flat(packs)
    whole = solver.DesignBatch(flat)
    for lo, hi in ((0, 3), (3, 9), (6, 9), (4, 5)):
        part, own = whole.take(lo, hi), solver.DesignBatch(flat[lo:hi])
        assert part.n_designs == hi - lo and sorted(part.arrays) == sorted(own.arrays)
        for k in own.arrays:
            assert np.array_equal(part.arrays[k], own.arrays[k]), (lo, hi, k)
        assert (part.n_members_total, part.n_nodes_total) == (own.n_members_total, own.n_nodes_total)
        assert (part.max_nodes, part.max_members, part.max_w_classes, part.walk_exact) == \
            (whole.max_nodes, whole.max_members, whole.max_w_classes, whole.walk_exact)
    assert whole.n_designs == 9 and whole.arrays["M0"].shape == (9, 36)
    with pytest.raises(ValueError, match="non-empty range"):
        whole.take(4, 4)
    nw, nC = whole.nw, 4
    rng = np.random.default_rng(1)
    F2 = rng.normal(size=(9, nC, 6, nw))
    ops = dict(op=np.array([0, 1, 1, 0], dtype=np.int32), A_w=rng.normal(size=(9, 2, 6, 6, nw)), B_w=rng.normal(size=(9, 2, 6, 6, nw)))
    cs = _cases(np.array([[6.0, 12.0, 0.0], [3.0, 8.0, 30.0], [4.0, 9.0, 60.0], [2.0, 7.0, 90.0]]), primary=[0, 1, 1, 3])
    ct = solver.CaseTable(cs, F_2nd=F2, ops=ops)
    sub = sweep.shard_design_cases(ct, 3, 6)
    sub.check_ops(whole.take(3, 6))
    assert sub.n_cases == nC and np.array_equal(sub.arrays["primary"], cs["primary"]) and np.array_equal(sub.arrays["F_2nd"], F2[3:6])
    assert np.array_equal(sub.ops["A_w"], ops["A_w"][3:6]) and np.array_equal(sub.arrays["op"], ops["op"])
    shared = sweep.shard_design_cases(solver.CaseTable(cs, ops=dict(ops, A_w=ops["A_w"][0], B_w=ops["B_w"][0])), 3, 6)
    assert shared.op_shared and np.array_equal(shared.ops["A_w"], ops["A_w"][0])


def _gloo_worker(rank, world, port, F, N, q):
    import torch
    import torch.distributed as dist
    from raft_b200 import sweep
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    bounds = sweep.farm_shards(F, world)
    lo, hi = bounds[rank]
    f = torch.arange(lo, hi, dtype=torch.float64)
    xi = (f[:, None, None, None] * 100 + torch.arange(2.0)[None, :, None, None] * 10 + torch.arange(6.0 * N)[None, None, :, None]
          + 1j * torch.arange(3.0)[None, None, None, :]).to(torch.complex128)
    info = (f[:, None, None] * 10 + torch.arange(3.0)[None, None, :]).repeat(1, 2, 1).to(torch.int32)
    st = torch.arange(lo * N, hi * N, dtype=torch.int32)[:, None, None].repeat(1, 2, 4)
    X, I, S = sweep.gather_farm_shards((xi, info, st), bounds, N)
    q.put((rank, X.numpy(), I.numpy(), S.numpy()))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("F,world", [(4, 2), (5, 2), (1, 2)])
def test_padded_gather_on_two_gloo_ranks(F, world):
    """The NCCL exchange of ShardedFarmSolve (padded shards, one all-gather per tensor, padding dropped) on 2 gloo ranks,
    with an even split, an uneven one and a rank without farms."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port, N = 29700 + 10 * F + world, 2
    procs = [ctx.Process(target=_gloo_worker, args=(r, world, port, F, N, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    f = np.arange(F, dtype=float)
    want_x = f[:, None, None, None] * 100 + np.arange(2)[None, :, None, None] * 10 + np.arange(6 * N)[None, None, :, None] + 1j * np.arange(3)
    for rank, X, I, S in got:
        assert X.shape == (F, 2, 6 * N, 3) and np.array_equal(X, want_x), rank
        assert np.array_equal(I, np.repeat((f[:, None, None] * 10 + np.arange(3)).astype(np.int32), 2, axis=1))
        assert S.shape == (F * N, 2, 4) and np.array_equal(S[:, 0, 0], np.arange(F * N))


def _agree_worker(rank, world, port, q):
    import torch.distributed as dist
    from raft_b200 import sweep
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    px = sweep.PeerExchange.__new__(sweep.PeerExchange)                       # the setup state _agree needs, without a GPU
    px.world, px.rank, px.dist, px.group, px.local, px.remote = world, rank, dist, None, [], []
    px.gathered, px.status = [], []
    px._agree(None, "allocation")                                             # every rank fine: nobody raises
    try:
        px._agree("RaftkError: cudaIpcOpenMemHandle failed" if rank == 1 else None, "peer mapping")
        q.put((rank, None))
    except sweep.PeerSetupError as e:
        q.put((rank, str(e)))
    dist.barrier()                                                            # both ranks reach the next collective
    dist.destroy_process_group()


def test_peer_setup_failure_is_raised_on_every_rank():
    """A setup stage of PeerExchange that fails on one rank (here rank 1's peer mapping) raises PeerSetupError on both gloo
    ranks, so ShardedFarmSolve falls back to NCCL everywhere instead of leaving a rank alone in a collective."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_agree_worker, args=(r, 2, 29790, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=120) for _ in procs)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert got[0] == got[1] == "peer exchange peer mapping failed on rank 1: RaftkError: cudaIpcOpenMemHandle failed"


# ---- on the GPU: emulated ranks ------------------------------------------------------------------------------------
class _Emulated:
    """``world`` ranks on one device: rank r's session over its farms' FOWTs, its own gathered copy and its own stream."""

    def __init__(self, batch, ct, N, mats, world, shared):
        import torch
        from raft_b200 import solver, sweep
        from raft_b200._lib import check, lib
        self.torch, self.check, self.lib = torch, check, lib
        self.N, self.world, self.nC, self.nw, n = N, world, ct.n_cases, batch.nw, 6 * N
        F = batch.n_designs // N
        self.bounds = sweep.farm_shards(F, world)
        self.rows = rows = max(h - l for l, h in self.bounds)
        self.dev = torch.device("cuda", 0)
        self.block = rows * self.nC * n * self.nw
        R = world * rows
        xi_bytes = world * self.block * 16
        self.off_flags = (xi_bytes + 255) // 256 * 256
        self.off_status = self.off_flags + 256
        total = self.off_status + R * self.nC * (self.nw + 4 * N) * 4
        self.ptrs = []
        for _ in range(world):
            p, h = C.c_void_p(), C.create_string_buffer(64)
            check(lib.raftk_peer_alloc(total, C.byref(p), h))
            self.ptrs.append(p.value)
        self.streams = [torch.cuda.Stream(device=self.dev) for _ in range(world)]
        self.timeout = torch.zeros(1, dtype=torch.int32, device=self.dev)
        self.sessions, self.mats, self.views = [], [], []
        for r, (lo, hi) in enumerate(self.bounds):
            s = None
            if hi > lo:
                s = solver.DeviceSession(batch.take(lo * N, hi * N), sweep.shard_design_cases(ct, lo * N, hi * N), device=self.dev,
                                         want=WANT + (("F_BEM",) if batch.n_bem_head else ()))
            self.sessions.append(s)
            self.mats.append({k: v if shared else v[lo:hi] for k, v in mats.items()})
            raw = torch.as_tensor(sweep._DevMem(self.ptrs[r], total), device=self.dev)
            ints = raw[self.off_status:total].view(torch.int32)
            self.views.append((torch.view_as_complex(raw[:xi_bytes].view(torch.float64).view(-1, 2)).view(R, self.nC, n, self.nw),
                               ints[:R * self.nC * self.nw].view(R, self.nC, self.nw), ints[R * self.nC * self.nw:].view(R * N, self.nC, 4)))
        self.fk, self.sk = sweep.farm_rows(self.bounds).to(self.dev), sweep.farm_rows(self.bounds, N).to(self.dev)
        self.kernels = set()

    def step(self, epoch, device=False):
        """One step of every rank -> [(Xi_sys, info, status) of every rank's copy], padding removed: numpy, or with ``device``
        torch tensors on the GPU (copies: the views are cleared for the next step)."""
        from raft_b200 import solver
        from raft_b200._lib import RaftkPeers
        torch = self.torch
        torch.cuda.synchronize()
        for r, (lo, hi) in enumerate(self.bounds):
            pr = RaftkPeers()
            pr.n_ranks, pr.rank, pr.epoch, pr.block_elems = self.world, r, epoch, self.block
            for q in range(self.world):
                pr.gathered[q], pr.flags[q], pr.status[q] = self.ptrs[q], self.ptrs[q] + self.off_flags, self.ptrs[q] + self.off_status
            with torch.cuda.stream(self.streams[r]):
                s, (X, I, _) = self.sessions[r], self.views[r]
                if s is not None:
                    s.solve(n_iter=10)
                    r0 = r * self.rows
                    s.farm_response_gather(pr, r0, X[r0:r0 + hi - lo], I[r0:r0 + hi - lo], self.N, **self.mats[r])
                    self.kernels.add(solver.last_dispatch()["kernel"])
                self.check(self.lib.raftk_peer_barrier_dev(C.byref(pr), self.timeout.data_ptr(), self.streams[r].cuda_stream))
        torch.cuda.synchronize()
        assert self.timeout.item() == 0
        got = [tuple(t.index_select(0, k) if device else t.index_select(0, k).cpu().numpy() for t, k in zip(v, (self.fk, self.fk, self.sk)))
               for v in self.views]
        for v in self.views:
            for t in v:
                t.zero_()
        torch.cuda.synchronize()
        return got

    def close(self):
        self.views, self.sessions = [], []
        for p in self.ptrs:
            self.check(self.lib.raftk_peer_free(p))


def _check_emulated(batch, ct, N, mats, world, kernel, shared=False):
    from raft_b200 import solver
    ref = solver.solve_dynamics_farm_batch(batch, ct, N, n_iter=10, **mats)
    assert solver.last_dispatch()["kernel"] == kernel
    em = _Emulated(batch, ct, N, mats, world, shared)
    try:
        for epoch in (1, 2):                                                   # the flags count epochs
            for r, (X, I, S) in enumerate(em.step(epoch)):
                assert np.array_equal(X, ref["Xi_sys"]), "Xi_sys in the copy of rank %d" % r
                assert np.array_equal(I, ref["info"]), r
                assert np.array_equal(S, ref["status"]), r
        assert em.kernels == {kernel}, em.kernels
    finally:
        em.close()
    return ref


KERNELS = [(1, "farm-warp"), (3, "farm-warp"), (4, "farm-warp"), (2, "farm-rows12"), (5, "farm-block"), (21, "farm-global")]


@gpu
@pytest.mark.parametrize("world,F", [(2, 4), (3, 5), (3, 2)], ids=["2ranks-even", "3ranks-uneven", "3ranks-2farms"])
@pytest.mark.parametrize("N,kernel", KERNELS, ids=[k + "-N%d" % n for n, k in KERNELS])
def test_emulated_ranks_gather_the_single_gpu_batch(N, kernel, world, F):
    """Every rank's copy of Xi_sys, info and the per-FOWT status equals one solve_dynamics_farm_batch call over all farms, bit
    for bit; [F,6N,6N] array stiffness; 3 ranks over 2 farms leave the last rank without farms (it only arrives at the barrier)."""
    from raft_b200 import solver
    packs, C_arr = _farms(N, F, nw=13 if N >= 21 else 21)
    ct = solver.CaseTable(_cases(np.array([[6.0, 12.0, 0.0], [3.5, 9.0, 40.0], [8.0, 14.0, -120.0]])))
    ref = _check_emulated(solver.DesignBatch(_flat(packs)), ct, N, dict(C_arr=C_arr), world, kernel)
    assert not np.any(ref["info"]) and not np.array_equal(ref["Xi_sys"][0], ref["Xi_sys"][-1])


OPS_KERNELS = [(2, "farm-rows12"), (3, "farm-warp"), (5, "farm-block"), (21, "farm-global")]


@gpu
@pytest.mark.parametrize("N,kernel", OPS_KERNELS, ids=[k for _, k in OPS_KERNELS])
def test_emulated_ranks_with_operating_points_trains_second_order_force_and_matrices(N, kernel):
    """Per-case operating points (per-design tables), wave trains, F_2nd, BEM tables and [F,6N,6N] M_arr / B_arr / C_arr, over
    3 ranks and 5 farms; then one shared set of matrices and of operating points."""
    from raft_b200 import solver
    from test_operating_points import _op_tables
    F, n = 5, 6 * N
    packs, C_arr = _farms(N, F, nw=13 if N >= 21 else 17, tables=True)
    flat = _flat(packs)
    nw = len(flat[0]["w"])
    rows = np.array([[6.0, 12.0, 0.0], [2.0, 7.0, 60.0], [4.0, 10.0, 200.0], [1.5, 6.0, 100.0]])
    cs = _cases(rows, primary=[0, 0, 2, 2])
    rng = np.random.default_rng(5 * N)
    A, B = _op_tables(rng, flat[0], 2, F * N)
    op = np.array([1, 1, 0, 0], dtype=np.int32)
    F2 = rng.normal(size=(F * N, len(rows), 6, nw)) * 5e4
    G = rng.normal(size=(F, n, n))
    mats = dict(C_arr=C_arr, M_arr=np.einsum("fij,fkj->fik", G, G) * 2e3 / n, B_arr=(G + np.swapaxes(G, 1, 2)) * 1e3)
    batch = solver.DesignBatch(flat)
    ct = solver.CaseTable(cs, F_2nd=F2, ops=dict(op=op, A_w=A, B_w=B))
    ref = _check_emulated(batch, ct, N, mats, 3, kernel)
    plain = solver.solve_dynamics_farm_batch(batch, solver.CaseTable(cs), N, C_arr=C_arr)
    assert not np.array_equal(plain["Xi_sys"], ref["Xi_sys"])                    # the extra terms are in the systems
    one = {k: v[2] for k, v in mats.items()}
    _check_emulated(batch, solver.CaseTable(cs, F_2nd=F2, ops=dict(op=op, A_w=A[0], B_w=B[0])), N, one, 3, kernel, shared=True)


@gpu
@pytest.mark.parametrize("exchange", ["peer", "nccl"])
@pytest.mark.parametrize("N,kernel", [(2, "farm-rows12"), (4, "farm-warp"), (21, "farm-global")])
def test_single_rank_sharded_farm_solve_equals_the_session(N, kernel, exchange):
    """Without a process group ShardedFarmSolve is DeviceSession.farm_response(n_fowt=N) delivered through the exchange's
    copies, for both exchanges and over two steps (alternating copies)."""
    import torch
    from raft_b200 import solver, sweep
    F = 3
    packs, C_arr = _farms(N, F, nw=11 if N >= 21 else 20)
    cs = _cases(np.array([[6.0, 12.0, 0.0], [3.0, 8.0, -70.0]]))
    sess = solver.DeviceSession(solver.DesignBatch(_flat(packs)), solver.CaseTable(cs), device="cuda:0", want=WANT)
    sess.solve(n_iter=10)
    xi, info = sess.farm_response(C_arr=C_arr, n_fowt=N)
    ref = (xi.cpu().numpy(), info.cpu().numpy(), sess.out["status"].cpu().numpy())
    sh = sweep.ShardedFarmSolve(solver.DesignBatch(_flat(packs)), solver.CaseTable(cs), N, C_arr=C_arr, exchange=exchange)
    assert sh.exchange == exchange and sh.world == 1 and sh.bounds == [(0, F)]
    for _ in range(2):
        got = sh.step(n_iter=10)
        assert solver.last_dispatch()["kernel"] == kernel
        torch.cuda.synchronize()
        for a, b in zip(got, ref):
            assert np.array_equal(a.cpu().numpy(), b)
    assert not sh.timed_out()
    sh.close()


def _host(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else x


def _same_results(dev, host):
    if isinstance(host, dict):
        assert dev.keys() == host.keys()
        pairs = [(dev[k], host[k]) for k in host]
    else:
        pairs = list(zip(dev, host))
    for a, b in pairs:
        assert (a is None and b is None) or np.array_equal(_host(a), b)


def _reductions(Xi, w, dw, N, seed=2):
    """farm_channel_stats, rotor_stats, fatigue and stress_ring of a farm batch's Xi_sys [F, nC, 6N, nw] (FOWT i's hub and
    tower at column 6 i), on whatever buffers Xi is in."""
    from raft_b200 import solver
    rng = np.random.default_rng(seed)
    nC, n, nw = Xi.shape[1], 6 * N, len(w)
    R = rng.normal(size=(4, n)) * 1e5
    col0 = [6 * i for i in range(N)]
    out = [solver.farm_channel_stats(R, Xi, dw, w=w, wpow=np.array([0, 1, 2, 0]))]
    out.append(solver.rotor_stats(rng.normal(size=(N, 6)), rng.normal(size=(nC, N, nw)) + 1j * rng.normal(size=(nC, N, nw)),
                                  rng.normal(size=(nC, N, nw)) + 0j, rng.normal(size=(nC, N, 4)), w, Xi, dw, col0=col0))
    out.append(solver.fatigue(Xi, w, 4.0, R=R))
    out.append(solver.stress_ring(Xi, w, rng.normal(size=(N, 6)), rng.normal(size=(N, 6)), m=3.0, col0=col0, dw=dw))
    return out


@gpu
def test_reductions_take_the_gathered_tensor():
    """The module-level reductions take the gathered Xi_sys as the exchange returns it -- a CUDA tensor, reduced on the device
    into torch tensors -- from 3 emulated ranks' copies and from ShardedFarmSolve.step, and give the host path's results on
    the single-GPU batch's Xi_sys, bit for bit."""
    import torch
    from raft_b200 import solver, sweep
    N, F = 3, 5
    packs, C_arr = _farms(N, F, nw=24)
    batch = solver.DesignBatch(_flat(packs))
    ct = solver.CaseTable(_cases(np.array([[6.0, 12.0, 0.0], [3.0, 8.0, -70.0]])))
    ref = solver.solve_dynamics_farm_batch(batch, ct, N, C_arr=C_arr, n_iter=10)["Xi_sys"]
    w, dw = batch.w, batch.dw
    want = _reductions(ref, w, dw, N)
    em = _Emulated(batch, ct, N, dict(C_arr=C_arr), 3, False)
    try:
        copies = [X for X, _, _ in em.step(1, device=True)]
    finally:
        em.close()
    sh = sweep.ShardedFarmSolve(batch, ct, N, C_arr=C_arr)
    copies.append(sh.step(n_iter=10)[0])
    for X in copies:
        assert X.is_cuda and np.array_equal(X.cpu().numpy(), ref)
        got = _reductions(X, w, dw, N)
        torch.cuda.synchronize()
        assert all(isinstance(t, torch.Tensor) and t.is_cuda for t in got[0] if t is not None)
        for g, h in zip(got, want):
            _same_results(g, h)
    sh.close()
