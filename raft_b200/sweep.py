"""Design sweeps sharded over GPUs (SURVEY.md section 8e; pattern of the reference's parametersweep.py:29-95).

(design) units are independent, so a sweep is an embarrassingly parallel shard: one process per GPU
(``torchrun``), rank r owns a contiguous block of designs, runs the fused solver on it, and the RAO blocks are
exchanged with ONE ``all_gather_into_tensor`` at the end -- the only collective on the path.  The helpers are
backend-agnostic (NCCL on GPUs; gloo on CPU tensors in the unit tests of the sharding logic).
"""
import copy

import numpy as np

from . import grid


def shard_bounds(n_items, rank, world):
    """Contiguous, balanced [lo, hi) of rank ``rank``: the first ``n_items % world`` ranks get one extra item."""
    base, extra = divmod(int(n_items), int(world))
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def all_gather_blocks(local, n_items, group=None):
    """All-gather per-rank blocks [n_local, ...] of a sharded array into [n_items, ...] (order = design index).

    Shards may be ragged by one item; every rank pads to the largest shard so a single
    ``all_gather_into_tensor`` suffices, then the padding is dropped."""
    import torch
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return local
    world = dist.get_world_size(group)
    n_max = -(-int(n_items) // world)
    pad = n_max - local.shape[0]
    buf = local if pad == 0 else torch.cat([local, local.new_zeros((pad,) + tuple(local.shape[1:]))], dim=0)
    out = local.new_empty((world * n_max,) + tuple(local.shape[1:]))
    dist.all_gather_into_tensor(out, buf.contiguous(), group=group)
    if n_max * world == n_items:
        return out
    keep = []
    for r in range(world):
        lo, hi = shard_bounds(n_items, r, world)
        keep.append(out[r * n_max:r * n_max + (hi - lo)])
    return torch.cat(keep, dim=0)


# ---- synthetic VolturnUS-S geometry variants (BASELINE.json configs[3]) ---------------------------------------

PARAMS = ("center_column_d", "outer_column_d", "draft", "outer_column_radius", "pontoon_height")


def sample_factors(n, seed=40, lower=0.75, upper=1.25):
    """[n,5] multiplicative factors ~ U[lower, upper] on the five parameters of parametersweep.py:29-44."""
    return np.random.default_rng(seed).uniform(lower, upper, size=(n, len(PARAMS)))


def apply_factors(base_design, f):
    """VolturnUS-S-like platform (center column, 3 outer columns, 3 pontoons, [upper supports]) with scaled
    centre-column diameter, outer-column diameter, draft, outer-column radius and pontoon height."""
    d = copy.deepcopy(base_design)
    mem = {m["name"]: m for m in d["platform"]["members"]}
    cc, oc, po = mem["center_column"], mem["outer_column"], mem["pontoon"]
    ccD, ocD = float(np.atleast_1d(cc["d"])[0]) * f[0], float(np.atleast_1d(oc["d"])[0]) * f[1]
    T = float(cc["rA"][2]) * f[2]
    ocR = float(oc["rA"][0]) * f[3]
    pH = float(po["d"][1]) * f[4]
    cc["d"], oc["d"] = ccD, ocD
    cc["rA"] = [cc["rA"][0], cc["rA"][1], T]
    oc["rA"] = [ocR, oc["rA"][1], T]
    oc["rB"] = [ocR, oc["rB"][1], oc["rB"][2]]
    po["d"] = [po["d"][0], pH]
    zp = T + pH / 2
    po["rA"] = [ccD / 2, po["rA"][1], zp]
    po["rB"] = [ocR - ocD / 2, po["rB"][1], zp]
    if "upper_support" in mem:
        us = mem["upper_support"]
        us["rA"] = [ccD / 2, us["rA"][1], us["rA"][2]]
        us["rB"] = [ocR - ocD / 2, us["rB"][1], us["rB"][2]]
    return d


def build_variants(base_design, base_matrices, factors, nw, max_freq, depth):
    """Packed designs (``packer.pack_fowt`` dicts) for every row of ``factors`` on a grid of nw bins.

    Node tables and the Morison added mass follow the geometry (``raft_b200.member``); structural mass,
    hydrostatic and mooring stiffness are statics (out of scope) and stay at ``base_matrices``."""
    from .fowt import FOWT
    w = grid.make_w(max_freq / nw, max_freq)
    k = grid.wave_number(w, depth)
    out = []
    for f in np.atleast_2d(factors):
        fw = FOWT(apply_factors(base_design, f), w, depth=depth, matrices=base_matrices, k=k)
        fw.calcHydroConstants()
        out.append(fw.pack())
    return out


def family_from_factors(base_design, factors):
    """``apply_factors`` for every row of ``factors`` at once: the per-design member geometry as arrays
    (``batch_builder.DesignFamily``), same arithmetic per element."""
    from .batch_builder import DesignFamily
    f = np.atleast_2d(np.asarray(factors, dtype=float))
    nD = len(f)
    mem = {m["name"]: m for m in base_design["platform"]["members"]}
    cc, oc, po = mem["center_column"], mem["outer_column"], mem["pontoon"]
    ccD, ocD = float(np.atleast_1d(cc["d"])[0]) * f[:, 0], float(np.atleast_1d(oc["d"])[0]) * f[:, 1]
    T = float(cc["rA"][2]) * f[:, 2]
    ocR = float(oc["rA"][0]) * f[:, 3]
    pH = float(po["d"][1]) * f[:, 4]
    col = lambda *xs: np.stack([np.broadcast_to(np.asarray(x, dtype=float), (nD,)) for x in xs], axis=1)
    zp = T + pH / 2
    geom = dict(center_column=dict(d=ccD, rA=col(cc["rA"][0], cc["rA"][1], T)),
                outer_column=dict(d=ocD, rA=col(ocR, oc["rA"][1], T), rB=col(ocR, oc["rB"][1], oc["rB"][2])),
                pontoon=dict(d=col(po["d"][0], pH), rA=col(ccD / 2, po["rA"][1], zp), rB=col(ocR - ocD / 2, po["rB"][1], zp)))
    if "upper_support" in mem:
        us = mem["upper_support"]
        geom["upper_support"] = dict(rA=col(ccD / 2, us["rA"][1], us["rA"][2]), rB=col(ocR - ocD / 2, us["rB"][1], us["rB"][2]))
    return DesignFamily(base_design, geom, nD)


def build_variants_batched(base_design, base_matrices, factors, nw, max_freq, depth, native=None):
    """``build_variants`` without per-design Python: -> ``solver.DesignBatch`` of all variants.  ``native`` (default: on unless
    RAFTK_NO_NATIVE_BUILDER is set) uses the library's C++ builder (``batch_builder.build_family_native``, ~12 ms per 1250
    designs); otherwise the vectorised NumPy one (``batch_builder.build_family``, ~80 ms), which needs no shared library."""
    import os
    from . import batch_builder
    w = grid.make_w(max_freq / nw, max_freq)
    k = grid.wave_number(w, depth)
    if native is None:
        native = not os.environ.get("RAFTK_NO_NATIVE_BUILDER")
    fam = family_from_factors(base_design, factors)
    if native:
        return batch_builder.build_family_native(fam, w, k, depth, base_matrices)
    return batch_builder.build_family(fam, w, k, depth, base_matrices)


def solve_sweep(packed_designs, cases, n_iter=10, tol=0.01, xi_start=0.0, device=None, group=None, n_total=None):
    """Solve this rank's designs on its GPU and all-gather the RAOs: -> (Xi [n_total,nC,6,nw], status [n_total,nC,4])."""
    from . import solver
    batch, ct = solver.DesignBatch(packed_designs), solver.CaseTable(cases)
    out = solver.DeviceSession(batch, ct, device=device).solve(n_iter=n_iter, tol=tol, xi_start=xi_start)
    if bool(((out["status"][..., 2] & solver.FLAG_PLAN) != 0).any()):
        # units whose step classes overflowed the hints ran no pass and hold zeros: solve again with worst-case tables
        out = solver.DeviceSession(solver.worst_case_hints(batch), ct, device=device).solve(n_iter=n_iter, tol=tol, xi_start=xi_start)
        if bool(((out["status"][..., 2] & solver.FLAG_PLAN) != 0).any()):
            raise solver._lib.RaftkError("step-class tables overflowed even with worst-case sizes")
    n_total = len(packed_designs) if n_total is None else n_total
    return all_gather_blocks(out["Xi"], n_total, group), all_gather_blocks(out["status"], n_total, group)


def solve_sweep_slender(packed_designs, cases, n_iter=10, tol=0.01, xi_start=0.0, device=None, group=None, n_total=None, qtf_chunk=0):
    """``solve_sweep`` for designs with potSecOrder 1 (``build_variants`` emits their ``qs_*`` tables): this rank's designs
    through ``solver.SlenderSession`` on its GPU, then the all-gather -> (Xi [n_total,nC,6,nw], status [n_total,nC,4]).
    ``qtf_chunk``: units whose QTF tables are built at once (0: all)."""
    from . import solver
    out = solver.SlenderSession(packed_designs, solver.CaseTable(cases), device=device, qtf_chunk=qtf_chunk).solve(n_iter=n_iter, tol=tol,
                                                                                                                  xi_start=xi_start)
    if bool(((out["status"][..., 2] & solver.FLAG_PLAN) != 0).any()):
        raise solver._lib.RaftkError("step-class tables overflowed the hints of the design batch")
    n_total = len(packed_designs) if n_total is None else n_total
    return all_gather_blocks(out["Xi"], n_total, group), all_gather_blocks(out["status"], n_total, group)


class _DevMem:
    """Raw device allocation exposed through __cuda_array_interface__ so torch can view it without owning it."""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = dict(shape=(int(nbytes),), typestr="|u1", data=(int(ptr), False), version=3)


def _align(n, a=256):
    return (int(n) + a - 1) // a * a


class PeerExchange:
    """Peer-shared gathered arrays for the exchange fused into the solve kernel (include/raftk.h ``raftk_peers``).

    Every rank owns ``n_buffers`` copies of ``Xi [world, units_per_rank, 6, nw]`` (+ arrival flags + status words),
    allocated by the library (cudaMalloc + CUDA IPC handle).  Handles are exchanged once with ``all_gather_object``
    and opened, so rank r's kernel can store its finished units straight into every rank's copy over NVLink -- the
    step has no separate collective.  Two copies alternate between steps because a rank may start the next step
    (and overwrite its block in a peer's copy) while that peer still reads the previous one."""

    def __init__(self, units_per_rank, nw, device, group=None, n_buffers=2):
        import ctypes as C
        import torch
        import torch.distributed as dist
        from ._lib import MAX_PEERS, RaftkPeers, check, lib
        self.torch, self.lib, self.check = torch, lib, check
        on = dist.is_available() and dist.is_initialized()
        self.world = dist.get_world_size(group) if on else 1
        self.rank = dist.get_rank(group) if on else 0
        if self.world > MAX_PEERS:
            raise ValueError("PeerExchange supports at most %d ranks" % MAX_PEERS)
        self.device = torch.device(device)
        self.units, self.nw = int(units_per_rank), int(nw)
        self.block_elems = self.units * 6 * self.nw
        self.xi_bytes = self.world * self.block_elems * 16
        self.off_flags = _align(self.xi_bytes)
        self.off_status = self.off_flags + 256
        self.total = _align(self.off_status + self.world * self.units * 16)
        self.local, self.remote, self.peers, self.gathered, self.status = [], [], [], [], []
        with torch.cuda.device(self.device):
            handles = []
            for _ in range(n_buffers):
                ptr, h = C.c_void_p(), C.create_string_buffer(64)
                check(lib.raftk_peer_alloc(self.total, C.byref(ptr), h))
                self.local.append(ptr.value)
                handles.append(h.raw)
            allh = [None] * self.world
            if self.world > 1:
                dist.all_gather_object(allh, handles, group=group)
            else:
                allh = [handles]
            for b in range(n_buffers):
                base = []
                for r in range(self.world):
                    if r == self.rank:
                        base.append(self.local[b])
                    else:
                        ptr = C.c_void_p()
                        check(lib.raftk_peer_open(allh[r][b], C.byref(ptr)))
                        self.remote.append(ptr.value)
                        base.append(ptr.value)
                pr = RaftkPeers()
                pr.n_ranks, pr.rank, pr.epoch, pr.block_elems = self.world, self.rank, 0, self.block_elems
                for r in range(self.world):
                    pr.gathered[r] = base[r]
                    pr.flags[r] = base[r] + self.off_flags
                    pr.status[r] = base[r] + self.off_status
                self.peers.append(pr)
                raw = torch.as_tensor(_DevMem(self.local[b], self.total), device=self.device)
                self.gathered.append(torch.view_as_complex(raw[:self.xi_bytes].view(torch.float64).view(-1, 2))
                                     .view(self.world, self.units, 6, self.nw))
                self.status.append(raw[self.off_status:self.off_status + self.world * self.units * 16].view(torch.int32)
                                   .view(self.world, self.units, 4))
            self.timeout = torch.zeros(1, dtype=torch.int32, device=self.device)
        if self.world > 1:
            dist.barrier(group=group)          # every rank has opened every handle before anyone stores into a peer
        self.n_steps = 0

    def next(self):
        """-> (buffer index, peers struct) for the next exchange; epochs count steps across both buffers."""
        b = self.n_steps % len(self.peers)
        self.n_steps += 1
        self.peers[b].epoch = self.n_steps
        return b, self.peers[b]

    def close(self):
        for p in self.remote:
            self.lib.raftk_peer_close(p)
        self.remote = []
        self.gathered, self.status = [], []
        for p in self.local:
            self.lib.raftk_peer_free(p)
        self.local = []


class ShardedSolve:
    """This rank's shard of (design, case) units on its GPU with the RAO exchange fused into the solve kernel.

    ``step()`` enqueues one solve of the shard; when the stream reaches the end of it, ``gathered`` [world, nD, nC, 6, nw]
    and ``status`` [world, nD, nC, 4] of the returned buffer hold EVERY rank's results (SURVEY.md 8e: the one exchange of
    the path).  ``step_host()`` is the same through host buffers: pinned inputs -> H2D -> solve + exchange -> D2H of this
    rank's block (what bench.py times as e2e at N > 1).  With one rank it degenerates to the plain solve."""

    def __init__(self, packed_designs, cases, device=None, group=None, want=("Xi", "status")):
        import torch
        from . import solver
        self.torch = torch
        if isinstance(packed_designs, solver.DesignBatch):
            self.batch = packed_designs
        else:
            self.batch = solver.DesignBatch([packed_designs] if isinstance(packed_designs, dict) else list(packed_designs))
        self.cases = cases if isinstance(cases, solver.CaseTable) else solver.CaseTable(cases)
        nD, nC, nw = self.batch.n_designs, self.cases.n_cases, self.batch.nw
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.px = PeerExchange(nD * nC, nw, dev, group=group)
        self.world, self.rank = self.px.world, self.px.rank
        g0 = self.px.gathered[0][self.rank].view(nD, nC, 6, nw)
        s0 = self.px.status[0][self.rank].view(nD, nC, 4)
        self.sess = solver.DeviceSession(self.batch, self.cases, device=dev, want=want, out_tensors=dict(Xi=g0, status=s0))
        self.o_structs = []
        for b in range(len(self.px.peers)):
            outs = dict(self.sess.out)
            outs["Xi"] = self.px.gathered[b][self.rank].view(nD, nC, 6, nw)
            outs["status"] = self.px.status[b][self.rank].view(nD, nC, 4)
            self.o_structs.append((solver._out_struct(outs, lambda t: t.data_ptr()), outs))
        self.shape = (nD, nC, 6, nw)
        self.units = nD * nC * nw
        self._pin = None

    def step(self, n_iter=10, tol=0.01, xi_start=0.0, cluster_size=0):
        """-> (gathered Xi [world,nD,nC,6,nw], status [world,nD,nC,4]) of this step's buffer (valid in stream order)."""
        nD, nC, _, nw = self.shape
        b, peers = self.px.next()
        o_struct, outs = self.o_structs[b]
        if self.world == 1:
            saved = self.sess.o_struct
            self.sess.o_struct = o_struct
            self.sess.solve(n_iter=n_iter, tol=tol, xi_start=xi_start, cluster_size=cluster_size)
            self.sess.o_struct = saved
        else:
            self.sess.solve_gather(peers, o_struct, n_iter=n_iter, tol=tol, xi_start=xi_start, cluster_size=cluster_size,
                                   timeout_flag=self.px.timeout.data_ptr())
        self.last = b
        return self.px.gathered[b].view(self.world, nD, nC, 6, nw), self.px.status[b].view(self.world, nD, nC, 4)

    def host_buffers(self):
        """Pinned host mirrors of the input block (all tables, ``DeviceSession.tables``) and of this rank's output block
        (allocated once)."""
        if self._pin is None:
            torch = self.torch
            pin_in = torch.empty(self.sess.tables.shape, dtype=torch.uint8, pin_memory=True)
            pin_in.copy_(self.sess.tables)
            nD, nC, _, nw = self.shape
            self._pin = (pin_in, torch.empty(self.shape, dtype=torch.complex128, pin_memory=True),
                         torch.empty((nD, nC, 4), dtype=torch.int32, pin_memory=True))
        return self._pin

    def step_host(self, **kw):
        """Host buffers in and out: H2D of every table and the case columns (one copy of the session's table block), solve +
        fused exchange + arrival barrier, D2H of this rank's responses and status; synchronises.
        -> (Xi host, status host, h2d bytes, d2h bytes)."""
        pin_in, xi_h, st_h = self.host_buffers()
        self.sess.tables.copy_(pin_in, non_blocking=True)
        h2d = self.sess.table_bytes
        self.sess._plan_key = None                     # fresh tables from the host: the per-design plan is rebuilt
        g, s = self.step(**kw)
        xi_h.copy_(g[self.rank], non_blocking=True)
        st_h.copy_(s[self.rank], non_blocking=True)
        self.torch.cuda.current_stream(self.sess.device).synchronize()
        return xi_h, st_h, h2d, xi_h.numel() * 16 + st_h.numel() * 4

    def timed_out(self):
        return bool(self.px.timeout.item())

    def close(self):
        self.px.close()


class PipelinedSolve:
    """Solve this rank's units in ``n_chunks`` launches and overlap each chunk's all-gather (NCCL, side stream)
    with the next chunk's kernels -- the transfer of chunk i hides behind the compute of chunk i+1.

    ``split="designs"`` chunks the design list (sweeps), ``split="cases"`` the case table (one design, many sea
    states).  ``gathered[i]`` is [world, ...] for chunk i; with one rank nothing is gathered."""

    def __init__(self, packed_designs, cases, n_chunks=2, split="designs", device=None, group=None, want=("Xi", "status")):
        import torch
        import torch.distributed as dist
        from . import solver
        self.torch, self.dist, self.group = torch, dist, group
        self.world = dist.get_world_size(group) if (dist.is_available() and dist.is_initialized()) else 1
        designs = [packed_designs] if isinstance(packed_designs, dict) else list(packed_designs)
        n = len(designs) if split == "designs" else len(cases["Hs"])
        n_chunks = max(1, min(n_chunks, n))
        self.sessions = []
        for i in range(n_chunks):
            lo, hi = shard_bounds(n, i, n_chunks)
            if split == "designs":
                sess = solver.DeviceSession(solver.DesignBatch(designs[lo:hi]), solver.CaseTable(cases), device=device, want=want)
            else:
                sub = {k: np.asarray(v)[lo:hi] for k, v in cases.items()}
                sess = solver.DeviceSession(solver.DesignBatch(designs), solver.CaseTable(sub), device=device, want=want)
            self.sessions.append(sess)
        dev = self.sessions[0].device
        self.comm = torch.cuda.Stream(device=dev) if self.world > 1 else None
        self.gathered = [torch.empty((self.world,) + tuple(s.out["Xi"].shape), dtype=s.out["Xi"].dtype, device=dev)
                         if self.world > 1 else None for s in self.sessions]
        self._ag_done = [None] * len(self.sessions)
        self.units = sum(s.batch.n_designs * s.cases.n_cases * s.batch.nw for s in self.sessions)

    def step(self, **solve_kw):
        """Enqueue one step.  Software pipeline: chunk i's kernels only wait for the all-gather that last read chunk
        i's output buffer (issued one step ago), so gathers also overlap the NEXT step's kernels; call ``drain()``
        before reading ``gathered`` or stopping a timer."""
        torch = self.torch
        cur = torch.cuda.current_stream(self.sessions[0].device)
        for i, (sess, g) in enumerate(zip(self.sessions, self.gathered)):
            if self.world > 1 and self._ag_done[i] is not None:
                cur.wait_event(self._ag_done[i])            # the previous gather of this buffer has consumed it
            sess.solve(**solve_kw)
            if self.world > 1:
                ev = torch.cuda.Event()
                ev.record(cur)
                with torch.cuda.stream(self.comm):
                    self.comm.wait_event(ev)
                    self.dist.all_gather_into_tensor(g, sess.out["Xi"], group=self.group)
                    done = torch.cuda.Event()
                    done.record(self.comm)
                self._ag_done[i] = done

    def drain(self):
        """Make the current stream wait for every outstanding all-gather."""
        if self.world > 1:
            self.torch.cuda.current_stream(self.sessions[0].device).wait_stream(self.comm)

    def status(self):
        return np.concatenate([s.out["status"].cpu().numpy().reshape(-1, 4) for s in self.sessions], axis=0)
