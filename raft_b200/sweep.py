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
    out = solver._retry_on_plan(batch, lambda b: solver.DeviceSession(b, ct, device=device).solve(n_iter=n_iter, tol=tol, xi_start=xi_start))
    n_total = len(packed_designs) if n_total is None else n_total
    return all_gather_blocks(out["Xi"], n_total, group), all_gather_blocks(out["status"], n_total, group)


def solve_sweep_slender(packed_designs, cases, n_iter=10, tol=0.01, xi_start=0.0, device=None, group=None, n_total=None, qtf_chunk=0):
    """``solve_sweep`` for designs with potSecOrder 1 (``build_variants`` emits their ``qs_*`` tables): this rank's designs
    through ``solver.SlenderSession`` on its GPU, then the all-gather -> (Xi [n_total,nC,6,nw], status [n_total,nC,4]).
    ``qtf_chunk``: units whose QTF tables are built at once (0: all)."""
    from . import solver
    out = solver.SlenderSession(packed_designs, solver.CaseTable(cases), device=device, qtf_chunk=qtf_chunk).solve(n_iter=n_iter, tol=tol,
                                                                                                                  xi_start=xi_start)
    if solver._plan_overflowed(out["status"]):
        raise solver._lib.RaftkError("step-class tables overflowed the hints of the design batch")
    n_total = len(packed_designs) if n_total is None else n_total
    return all_gather_blocks(out["Xi"], n_total, group), all_gather_blocks(out["status"], n_total, group)


class _DevMem:
    """Raw device allocation exposed through __cuda_array_interface__ so torch can view it without owning it."""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = dict(shape=(int(nbytes),), typestr="|u1", data=(int(ptr), False), version=3)


def _align(n, a=256):
    return (int(n) + a - 1) // a * a


class PeerSetupError(RuntimeError):
    """The peer-mapped copies of a ``PeerExchange`` could not be set up on some rank (e.g. no CUDA IPC); raised on every rank."""


class PeerExchange:
    """Peer-shared gathered arrays for the exchange fused into the solve kernel (include/raftk.h ``raftk_peers``).

    Every rank owns ``n_buffers`` copies of ``Xi [world, units_per_rank, dof, nw]`` (+ arrival flags + status words; ``dof``
    is 6 for rigid units, n_dof for the rows of a generalised-DOF shard, ``ShardedGeneralSolve``),
    allocated by the library (cudaMalloc + CUDA IPC handle).  Handles are exchanged once with ``all_gather_object``
    and opened, so rank r's kernel can store its finished units straight into every rank's copy over NVLink -- the
    step has no separate collective.  Two copies alternate between steps because a rank may start the next step
    (and overwrite its block in a peer's copy) while that peer still reads the previous one.  ``status_elems``: int32 elements
    per rank of the status region, viewed flat ([world * status_elems]); default 4 per unit, viewed [world, units, 4]."""

    def __init__(self, units_per_rank, nw, device, group=None, n_buffers=2, dof=6, status_elems=None):
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
        self.units, self.nw, self.dof = int(units_per_rank), int(nw), int(dof)
        self.block_elems = self.units * self.dof * self.nw
        self.xi_bytes = self.world * self.block_elems * 16
        self.off_flags = _align(self.xi_bytes)
        self.off_status = self.off_flags + 256
        self.status_elems = self.units * 4 if status_elems is None else int(status_elems)
        self.total = _align(self.off_status + self.world * self.status_elems * 4)
        self.local, self.remote, self.peers, self.gathered, self.status = [], [], [], [], []
        self.dist, self.group = dist, group
        with torch.cuda.device(self.device):
            handles, err = [], None
            try:
                for _ in range(n_buffers):
                    ptr, h = C.c_void_p(), C.create_string_buffer(64)
                    check(lib.raftk_peer_alloc(self.total, C.byref(ptr), h))
                    self.local.append(ptr.value)
                    handles.append(h.raw)
            except Exception as e:                    # noqa: BLE001  (agreed on below, then raised on every rank)
                err = "%s: %s" % (type(e).__name__, e)
            self._agree(err, "allocation")
            allh = [None] * self.world
            if self.world > 1:
                dist.all_gather_object(allh, handles, group=group)
            else:
                allh = [handles]
            bases = [[None] * self.world for _ in range(n_buffers)]
            try:
                for b in range(n_buffers):
                    for r in range(self.world):
                        if r == self.rank:
                            bases[b][r] = self.local[b]
                        else:
                            ptr = C.c_void_p()
                            check(lib.raftk_peer_open(allh[r][b], C.byref(ptr)))
                            self.remote.append(ptr.value)
                            bases[b][r] = ptr.value
            except Exception as e:                    # noqa: BLE001
                err = "%s: %s" % (type(e).__name__, e)
            self._agree(err, "peer mapping")
            for b in range(n_buffers):
                base = bases[b]
                pr = RaftkPeers()
                pr.n_ranks, pr.rank, pr.epoch, pr.block_elems = self.world, self.rank, 0, self.block_elems
                for r in range(self.world):
                    pr.gathered[r] = base[r]
                    pr.flags[r] = base[r] + self.off_flags
                    pr.status[r] = base[r] + self.off_status
                self.peers.append(pr)
                raw = torch.as_tensor(_DevMem(self.local[b], self.total), device=self.device)
                self.gathered.append(torch.view_as_complex(raw[:self.xi_bytes].view(torch.float64).view(-1, 2))
                                     .view(self.world, self.units, self.dof, self.nw))
                st = raw[self.off_status:self.off_status + self.world * self.status_elems * 4].view(torch.int32)
                self.status.append(st.view(self.world, self.units, 4) if status_elems is None else st)
            self.timeout = torch.zeros(1, dtype=torch.int32, device=self.device)
        if self.world > 1:
            dist.barrier(group=group)          # every rank has opened every handle before anyone stores into a peer
        self.n_steps = 0

    def _agree(self, err, stage):
        """Every rank learns every rank's outcome of a setup stage (one all_gather_object); if any failed, all free what they
        hold and raise PeerSetupError together, so no rank enters the next collective alone."""
        errs = [err]
        if self.world > 1:
            errs = [None] * self.world
            self.dist.all_gather_object(errs, err, group=self.group)
        bad = [(r, e) for r, e in enumerate(errs) if e is not None]
        if bad:
            self.close()
            raise PeerSetupError("peer exchange %s failed on rank %d: %s" % ((stage,) + bad[0]))

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


def general_groups(primary, n_cases):
    """Start of every train group (the cases that share a primary) of a case table, plus ``n_cases``: the units the
    generalised-DOF path never splits.  ``primary`` None: every case is a group.  ValueError when a group is not contiguous
    in the table (``packer.pack_case_trains`` never builds one)."""
    n = int(n_cases)
    if primary is None:
        return np.arange(n + 1)
    pr = np.asarray(primary, dtype=np.int64)
    starts = np.flatnonzero(np.r_[True, pr[1:] != pr[:-1]])
    if len(np.unique(pr[starts])) != len(starts):
        raise ValueError("the train groups of cases.primary interleave: every group must be contiguous in the table")
    return np.r_[starts, n]


def general_shards(primary, n_cases, world):
    """[lo, hi) of every rank: contiguous runs of whole train groups, balanced by case count (each cut at the group start
    nearest to r * n_cases / world, the later one on a tie).  A rank may get no cases when groups are large."""
    g = general_groups(primary, n_cases)
    cuts = [0]
    for r in range(1, int(world)):
        t = r * int(n_cases) / int(world)
        i = int(np.searchsorted(g, t))
        best = min((c for c in (g[max(i - 1, 0)], g[min(i, len(g) - 1)])), key=lambda c: (abs(c - t), -c))
        cuts.append(max(int(best), cuts[-1]))
    cuts.append(int(n_cases))
    return [(cuts[r], cuts[r + 1]) for r in range(int(world))]


def shard_case_table(cases, lo, hi):
    """Rows [lo, hi) of a ``solver.CaseTable`` as a table of their own (whole train groups: primaries rebased to lo).  Per-case
    operating points keep their rows of ``op`` and the whole tables."""
    from . import solver
    a = cases.arrays
    sub = {k: a[k][lo:hi] for k in ("Hs", "Tp", "gamma", "beta_deg", "spec")}
    if "primary" in a:
        sub["primary"] = a["primary"][lo:hi] - lo
    ops = None if cases.ops is None else dict(cases.ops, op=cases.ops["op"][lo:hi])
    return solver.CaseTable(sub, zeta=a["zeta"][lo:hi] if "zeta" in a else None, ops=ops)


class ShardedGeneralSolve:
    """A generalised-DOF case table (flexible FOWT, ``solver.GeneralSession``) sharded over GPUs: rank r takes a contiguous,
    count-balanced run of whole train groups (``general_shards``) and streams it through ``max_chunk_cases`` as
    ``GeneralSession`` does.  ``step()`` enqueues the solve, then the exchange, and returns (Xi complex [nC, n_dof, nw],
    status [nC, 4]) of the WHOLE table in table order, valid in stream order on every rank.

    ``exchange="peer"``: the shard's rows are stored into every rank's gathered copy through CUDA IPC peer pointers
    (raftk_general_publish_dev, ``PeerExchange`` with dof = n_dof, rows padded to the largest shard), then
    raftk_peer_barrier_dev.  ``exchange="nccl"``: one ``all_gather_into_tensor`` of the padded shards instead.  Status word 3
    of a secondary train holds its primary's index in the whole table + 1 either way.  With one rank it is the plain solve."""

    def __init__(self, P, M, B, Cm, cases, fd=None, qtf=None, max_chunk_cases=None, group=None, device=None, exchange="peer"):
        import torch
        import torch.distributed as dist
        from . import solver
        if exchange not in ("peer", "nccl"):
            raise ValueError("exchange must be 'peer' or 'nccl'")
        self.torch, self.dist, self.group, self.exchange = torch, dist, group, exchange
        on = dist.is_available() and dist.is_initialized()
        self.world = dist.get_world_size(group) if on else 1
        self.rank = dist.get_rank(group) if on else 0
        ct = cases if isinstance(cases, solver.CaseTable) else solver.CaseTable(cases)
        self.n_cases, self.n, self.nw = ct.n_cases, int(P["gen_nDOF"]), len(P["w"])
        self.bounds = general_shards(ct.arrays.get("primary"), ct.n_cases, self.world)
        self.lo, self.hi = self.bounds[self.rank]
        self.rows = max(1, max(h - l for l, h in self.bounds))
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.sess = None
        if self.hi > self.lo:
            self.sess = solver.GeneralSession(P, M, B, Cm, shard_case_table(ct, self.lo, self.hi), device=self.device, fd=fd, qtf=qtf,
                                              max_chunk_cases=max_chunk_cases)
        self.index = torch.cat([torch.arange(h - l) + r * self.rows for r, (l, h) in enumerate(self.bounds)]).to(self.device)
        self.px = None
        if exchange == "peer":
            self.px = PeerExchange(self.rows, self.nw, self.device, group=group, dof=self.n)
        else:
            with torch.cuda.device(self.device):
                self.x_pad = torch.zeros([self.rows, self.n, self.nw], dtype=torch.complex128, device=self.device)
                self.s_pad = torch.zeros([self.rows, 4], dtype=torch.int32, device=self.device)
                self.x_all = torch.empty([self.world * self.rows, self.n, self.nw], dtype=torch.complex128, device=self.device)
                self.s_all = torch.empty([self.world * self.rows, 4], dtype=torch.int32, device=self.device)

    def step(self, n_iter=10, tol=0.01, xi_start=0.0):
        import ctypes as C
        from ._lib import check, lib
        torch = self.torch
        m = self.hi - self.lo
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream(self.device)
            if self.sess is not None:
                self.sess.solve(n_iter=n_iter, tol=tol, xi_start=xi_start)
            if self.px is not None:
                b, peers = self.px.next()
                if m:
                    check(lib.raftk_general_publish_dev(C.byref(peers), self.sess.Xi.data_ptr(), self.sess.status.data_ptr(), self.rank * self.rows,
                                                        m, self.n, self.nw, self.lo, stream.cuda_stream))
                check(lib.raftk_peer_barrier_dev(C.byref(peers), self.px.timeout.data_ptr(), stream.cuda_stream))
                X = self.px.gathered[b].view(self.world * self.rows, self.n, self.nw)
                S = self.px.status[b].view(self.world * self.rows, 4)
            else:
                if m:
                    self.x_pad[:m].copy_(self.sess.Xi)
                    st = self.sess.status
                    self.s_pad[:m].copy_(st)
                    self.s_pad[:m, 3] = torch.where(st[:, 3] != 0, st[:, 3] + self.lo, st[:, 3])
                if self.world > 1:
                    self.dist.all_gather_into_tensor(self.x_all, self.x_pad, group=self.group)
                    self.dist.all_gather_into_tensor(self.s_all, self.s_pad, group=self.group)
                    X, S = self.x_all, self.s_all
                else:
                    X, S = self.x_pad, self.s_pad
            return X.index_select(0, self.index), S.index_select(0, self.index)

    def timed_out(self):
        return bool(self.px.timeout.item()) if self.px is not None else False

    def close(self):
        if self.px is not None:
            self.px.close()


def farm_shards(n_farms, world):
    """[lo, hi) farms of every rank: contiguous runs of whole farms whose sizes differ by at most one (``shard_bounds``); with
    more ranks than farms the last ranks get none."""
    return [shard_bounds(n_farms, r, world) for r in range(int(world))]


def shard_design_cases(cases, lo, hi):
    """A ``solver.CaseTable`` for designs [lo, hi) of its batch: every case, with those designs' rows of F_2nd, Xi_init and
    per-design operating-point tables (a shared operating-point set stays whole)."""
    from . import solver
    a = cases.arrays
    sub = {k: a[k] for k in ("Hs", "Tp", "gamma", "beta_deg", "spec", "primary") if k in a}
    ops = cases.ops
    if ops is not None and not cases.op_shared:
        ops = dict(ops, A_w=ops["A_w"][lo:hi], B_w=ops["B_w"][lo:hi])
    rows = {k: a[k][lo:hi] for k in ("F_2nd", "Xi_init") if k in a}
    return solver.CaseTable(sub, zeta=a.get("zeta"), ops=ops, **rows)


def farm_rows(bounds, per=1):
    """Rows of a gathered array [world * F_max * per, ...] (rank r's block at r * F_max * per, ``per`` rows per farm) that hold
    farms 0..F-1 in order, F_max the largest shard of ``bounds`` (``farm_shards``): the index that drops the padding."""
    import torch
    rows = max(1, max(h - l for l, h in bounds))
    return torch.cat([torch.arange((h - l) * per) + r * rows * per for r, (l, h) in enumerate(bounds)])


def gather_farm_shards(blocks, bounds, n_fowt, group=None):
    """The ``exchange="nccl"`` path of ``ShardedFarmSolve``: this rank's (Xi_sys [F_r,nC,6N,nw], info [F_r,nC,nw], status
    [F_r*N,nC,4]) -> the whole batch's three tensors in farm order (``_gather_rows``: padded to the largest shard, one
    ``all_gather_into_tensor`` each, padding dropped).  Backend-agnostic (NCCL on GPUs, gloo on CPU tensors)."""
    N = int(n_fowt)
    spans = (list(bounds), list(bounds), [(lo * N, hi * N) for lo, hi in bounds])
    return tuple(_gather_rows(t, sp, group) for t, sp in zip(blocks, spans))


def ragged_farm_cost(N):
    """Estimated work of one farm of N FOWTs, per (case, bin): N per-FOWT solves plus one dense (6N)^3 factorisation."""
    N = int(N)
    return N + (6 * N) ** 3


def ragged_farm_shards(sizes, world):
    """Contiguous runs of whole farms of a ragged batch (farm f: ``sizes[f]`` FOWTs), one [lo, hi) per rank, that minimise the
    largest rank's estimated work (``ragged_farm_cost``; every farm shares the case table and grid, so nC * nw drops out).
    The bottleneck is found exactly: bisection over integer loads with a greedy fill, which is optimal for contiguous runs.
    Ranks past the last farm get empty runs."""
    cost = [ragged_farm_cost(n) for n in sizes]
    world = int(world)
    if world < 1:
        raise ValueError("world must be >= 1")

    def fill(cap):
        bounds, lo, load = [], 0, 0
        for f, c in enumerate(cost):
            if load + c > cap and f > lo:
                bounds.append((lo, f))
                lo, load = f, 0
            load += c
        bounds.append((lo, len(cost)))
        return bounds

    lo, hi = max(cost, default=0), sum(cost)
    while lo < hi:
        mid = (lo + hi) // 2
        if len(fill(mid)) <= world:
            hi = mid
        else:
            lo = mid + 1
    bounds = fill(lo) if cost else []
    return bounds + [(len(cost), len(cost))] * (world - len(bounds))


def _gather_rows(t, spans, group=None):
    """Rows [a_r, b_r) of a tensor sharded by rank (``t``: this rank's rows) -> every rank's rows in order: padded to the
    largest span, one ``all_gather_into_tensor``, padding dropped."""
    import torch
    import torch.distributed as dist
    world, rmax = len(spans), max(1, max(b - a for a, b in spans))
    pad = t.new_zeros((rmax,) + tuple(t.shape[1:]))
    pad[:t.shape[0]].copy_(t)
    if world > 1:
        full = t.new_empty((world * rmax,) + tuple(t.shape[1:]))
        dist.all_gather_into_tensor(full, pad, group=group)
    else:
        full = pad
    idx = torch.cat([torch.arange(b - a) + r * rmax for r, (a, b) in enumerate(spans)])
    return full.index_select(0, idx.to(full.device))


def gather_ragged_farm_shards(blocks, bounds, farm_fowt0, group=None):
    """The ``exchange="nccl"`` path of ``ShardedFarmSolve(farm_sizes=...)``: this rank's (Xi_sys [D_r, 6 nC nw] -- its farms'
    flat Xi_sys in rows of one FOWT's length --, info [F_r,nC,nw], status [D_r,nC,4]) -> the whole batch's ([nD, 6 nC nw],
    [F,nC,nw], [nD,nC,4]), every rank's rows at their global offsets.  ``bounds``: [lo, hi) farms of every rank
    (``ragged_farm_shards``); ``farm_fowt0``: the batch's CSR of designs.  Backend-agnostic (NCCL on GPUs, gloo on CPU)."""
    fowt0 = [int(v) for v in farm_fowt0]
    dspans = [(fowt0[lo], fowt0[hi]) for lo, hi in bounds]
    xi, info, st = blocks
    return _gather_rows(xi, dspans, group), _gather_rows(info, list(bounds), group), _gather_rows(st, dspans, group)


class ShardedFarmSolve:
    """A farm batch (``solver.solve_dynamics_farm_batch``) sharded over GPUs: rank r takes the whole farms
    ``farm_shards(F, world)[r]`` (a farm's coupled system stays on one GPU), runs its FOWTs' drag linearisation and its farms'
    coupled 6N-DOF solves in a ``solver.DeviceSession`` of its own, and ``step()`` returns (Xi_sys [F,nC,6N,nw], info [F,nC,nw],
    status [F*N,nC,4]) of the WHOLE batch as device tensors, valid in stream order on every rank: bit for bit what one
    ``solve_dynamics_farm_batch`` call over all F farms returns.

    ``designs``: ``solver.DesignBatch`` of F * n_fowt FOWTs in the farm batch's order (design f * N + i is FOWT i of farm f), or
    the packed designs; ``cases``: ``solver.CaseTable`` as for the single-GPU entry (operating points, wave trains, F_2nd);
    array matrices [6N,6N] for every farm or [F,6N,6N], sliced to each rank's farms.
    ``exchange="peer"``: each rank solves its farms, then k_farm_publish copies its results into every rank's gathered copy
    through CUDA IPC peer pointers (raftk_farm_batch_response_gather_dev), then raftk_peer_barrier_dev; the copies hold F_max = the largest shard's farm count per rank.  ``exchange="nccl"``:
    ``gather_farm_shards`` instead; a peer exchange that cannot be set up (CUDA IPC unavailable) falls back to it on every
    rank.  With one rank it is ``DeviceSession.farm_response(n_fowt=N)`` with the exchange's copies as outputs.

    ``farm_sizes`` instead of ``n_fowt``: a ragged batch (``solver.solve_dynamics_farm_ragged``), farm f of farm_sizes[f]
    FOWTs, array matrices as that function takes them.  Rank r takes the whole farms ``ragged_farm_shards(farm_sizes,
    world)[r]`` (balanced by estimated work), and every farm is stored at its global offset of every rank's copy, no padding:
    ``exchange="peer"`` through raftk_farm_ragged_response_gather_dev (solve, then k_farm_publish), ``"nccl"`` through
    ``gather_ragged_farm_shards``.  ``step()`` -> (Xi_sys: per-farm [nC,6N_f,nw] views of one flat tensor, info [F,nC,nw],
    status [nD,nC,4]), bit for bit what one ``solve_dynamics_farm_ragged`` call returns."""

    WANT = ("Xi", "status", "B_drag", "F_drag", "F_iner")

    def __init__(self, designs, cases, n_fowt=None, C_arr=None, M_arr=None, B_arr=None, device=None, group=None, exchange="peer",
                 farm_sizes=None):
        import torch
        import torch.distributed as dist
        from . import solver
        if exchange not in ("peer", "nccl"):
            raise ValueError("exchange must be 'peer' or 'nccl'")
        self.torch, self.dist, self.group = torch, dist, group
        batch = designs if isinstance(designs, solver.DesignBatch) else solver.DesignBatch(designs)
        ct = cases if isinstance(cases, solver.CaseTable) else solver.CaseTable(cases)
        self.sizes = None
        if farm_sizes is not None:
            if n_fowt is not None:
                raise ValueError("give n_fowt or farm_sizes, not both")
            return self._init_ragged(batch, ct, farm_sizes, M_arr, B_arr, C_arr, device, group, exchange)
        N = self.N = int(n_fowt)
        if N < 1 or batch.n_designs % N:
            raise ValueError("n_fowt must divide the batch's %d designs" % batch.n_designs)
        ct.check_ops(batch)
        on = dist.is_available() and dist.is_initialized()
        self.world = dist.get_world_size(group) if on else 1
        self.rank = dist.get_rank(group) if on else 0
        self.F, self.nC, self.nw, n = batch.n_designs // N, ct.n_cases, batch.nw, 6 * N
        mats, shared = solver._farm_batch_matrices(self.F, n, M_arr, B_arr, C_arr)
        self.bounds = farm_shards(self.F, self.world)
        self.lo, self.hi = self.bounds[self.rank]
        self.rows = max(1, max(h - l for l, h in self.bounds))
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.sess, self.mats = None, {}
        if self.hi > self.lo:
            want = self.WANT + (("F_BEM",) if batch.n_bem_head else ())
            self.sess = solver.DeviceSession(batch.take(self.lo * N, self.hi * N), shard_design_cases(ct, self.lo * N, self.hi * N),
                                             device=self.device, want=want)
            self.mats = {k: v if shared else v[self.lo:self.hi] for k, v in mats.items()}
        self.px, self.exchange, self.fallback = None, exchange, None
        if exchange == "peer":
            # PeerExchange raises on every rank together when the IPC allocation or mapping fails on any (PeerSetupError), so
            # all ranks fall back to NCCL and none is left alone in a collective of the setup
            try:
                self.px = PeerExchange(self.rows * self.nC, self.nw, self.device, group=group, dof=n,
                                       status_elems=self.rows * self.nC * (self.nw + 4 * N))
            except PeerSetupError as e:
                self.fallback, self.exchange = str(e), "nccl"
        if self.px is not None:
            R = self.world * self.rows
            self.views = []
            for b in range(len(self.px.peers)):
                ints = self.px.status[b]
                self.views.append((self.px.gathered[b].view(R, self.nC, n, self.nw), ints[:R * self.nC * self.nw].view(R, self.nC, self.nw),
                                   ints[R * self.nC * self.nw:].view(R * N, self.nC, 4)))
            self.keep = [farm_rows(self.bounds).to(self.device), farm_rows(self.bounds, N).to(self.device)]

    def _init_ragged(self, batch, ct, farm_sizes, M_arr, B_arr, C_arr, device, group, exchange):
        torch, dist = self.torch, self.dist
        from . import solver
        sizes = self.sizes = tuple(int(n) for n in farm_sizes)
        fowt0 = self.fowt0 = [int(v) for v in solver.ragged_offsets(sizes)[0]]
        if min(sizes, default=0) < 1 or fowt0[-1] != batch.n_designs:
            raise ValueError("farm_sizes must be >= 1 and add up to the batch's %d designs" % batch.n_designs)
        solver._ragged_matrices(sizes, M_arr, B_arr, C_arr)                  # the whole batch's matrices, checked once
        ct.check_ops(batch)
        on = dist.is_available() and dist.is_initialized()
        self.world = dist.get_world_size(group) if on else 1
        self.rank = dist.get_rank(group) if on else 0
        self.F, self.nC, self.nw = len(sizes), ct.n_cases, batch.nw
        self.bounds = ragged_farm_shards(sizes, self.world)
        self.lo, self.hi = self.bounds[self.rank]
        self.d_lo, self.d_hi = fowt0[self.lo], fowt0[self.hi]
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.sess, self.mats = None, {}
        if self.hi > self.lo:
            want = self.WANT + (("F_BEM",) if batch.n_bem_head else ())
            self.sess = solver.DeviceSession(batch.take(self.d_lo, self.d_hi), shard_design_cases(ct, self.d_lo, self.d_hi),
                                             device=self.device, want=want)
            for k, v in (("M_arr", M_arr), ("B_arr", B_arr), ("C_arr", C_arr)):
                if v is not None:                                              # a shared [6N,6N] set stays whole
                    self.mats[k] = v if (not isinstance(v, (list, tuple)) and np.ndim(v) == 2) else list(v)[self.lo:self.hi]
        self.px, self.exchange, self.fallback = None, exchange, None
        nD, U = batch.n_designs, 6 * self.nC * self.nw
        if exchange == "peer":
            try:
                self.px = PeerExchange(-(-nD // self.world), self.nw, self.device, group=group, dof=6 * self.nC,
                                       status_elems=-(-(self.F * self.nC * self.nw + nD * self.nC * 4) // self.world))
            except PeerSetupError as e:
                self.fallback, self.exchange = str(e), "nccl"
        if self.px is not None:
            ni = self.F * self.nC * self.nw
            self.views = [(self.px.gathered[b].reshape(-1)[:nD * U], self.px.status[b].reshape(-1)[:ni].view(self.F, self.nC, self.nw),
                           self.px.status[b].reshape(-1)[ni:ni + nD * self.nC * 4].view(nD, self.nC, 4)) for b in range(len(self.px.peers))]

    def _step_ragged(self, n_iter, tol, xi_start):
        import ctypes as C
        from . import solver
        from ._lib import check, lib
        torch, U = self.torch, 6 * self.nC * self.nw
        m = self.hi - self.lo
        with torch.cuda.device(self.device):
            if self.sess is not None:
                self.sess.solve(n_iter=n_iter, tol=tol, xi_start=xi_start)
            if self.px is not None:
                b, peers = self.px.next()
                X, I, S = self.views[b]
                if m:
                    self.sess.farm_response_ragged_gather(peers, self.lo, self.d_lo, self.F, X[self.d_lo * U:self.d_hi * U], I[self.lo:self.hi],
                                                          self.sizes[self.lo:self.hi], **self.mats)
                check(lib.raftk_peer_barrier_dev(C.byref(peers), self.px.timeout.data_ptr(), torch.cuda.current_stream(self.device).cuda_stream))
                X, I, S = X.clone(), I.clone(), S.clone()                  # the copy is rewritten two steps on
            else:
                if m:
                    _, info = self.sess.farm_response(farm_sizes=self.sizes[self.lo:self.hi], **self.mats)
                    blocks = (self.sess._farm_rag[3].view(-1, U), info, self.sess.out["status"])
                else:
                    blocks = (torch.zeros([0, U], dtype=torch.complex128, device=self.device),
                              torch.zeros([0, self.nC, self.nw], dtype=torch.int32, device=self.device),
                              torch.zeros([0, self.nC, 4], dtype=torch.int32, device=self.device))
                X, I, S = gather_ragged_farm_shards(blocks, self.bounds, self.fowt0, self.group)
                X = X.reshape(-1)
            return solver.ragged_views(X, self.sizes, self.nC, self.nw), I, S

    def step(self, n_iter=10, tol=0.01, xi_start=0.0):
        """Enqueue the per-FOWT solve, the coupled solve and the exchange of this rank's farms on the current stream
        -> (Xi_sys [F,nC,6N,nw], info [F,nC,nw], status [F*N,nC,4]) of the whole batch (device tensors, stream order); a
        ragged batch (``farm_sizes``): (Xi_sys per-farm views, info, status) as the class documents."""
        if self.sizes is not None:
            return self._step_ragged(n_iter, tol, xi_start)
        import ctypes as C
        from ._lib import check, lib
        torch, N, m = self.torch, self.N, self.hi - self.lo
        with torch.cuda.device(self.device):
            if self.sess is not None:
                self.sess.solve(n_iter=n_iter, tol=tol, xi_start=xi_start)
            if self.px is not None:
                b, peers = self.px.next()
                X, I, S = self.views[b]
                if m:
                    r0 = self.rank * self.rows
                    self.sess.farm_response_gather(peers, r0, X[r0:r0 + m], I[r0:r0 + m], N, **self.mats)
                check(lib.raftk_peer_barrier_dev(C.byref(peers), self.px.timeout.data_ptr(), torch.cuda.current_stream(self.device).cuda_stream))
                fk, sk = self.keep
                return X.index_select(0, fk), I.index_select(0, fk), S.index_select(0, sk)
            if m:
                xi, info = self.sess.farm_response(n_fowt=N, **self.mats)
                blocks = (xi, info, self.sess.out["status"])
            else:
                n = 6 * N
                blocks = (torch.zeros([0, self.nC, n, self.nw], dtype=torch.complex128, device=self.device),
                          torch.zeros([0, self.nC, self.nw], dtype=torch.int32, device=self.device),
                          torch.zeros([0, self.nC, 4], dtype=torch.int32, device=self.device))
            return gather_farm_shards(blocks, self.bounds, N, self.group)

    def timed_out(self):
        return bool(self.px.timeout.item()) if self.px is not None else False

    def close(self):
        if self.px is not None:
            self.px.close()
            self.px = None


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
