"""Cost of the sharded farm batch's exchange on one GPU (profiles/h100_farm_shard.txt, profiles/h100_farm_one_path.txt).

* The gather: the coupled farm solve of a DeviceSession through raftk_farm_batch_response_gather_dev with one emulated peer
  (a second gathered copy on the same device, so every result is stored twice: the solve, then k_farm_publish's copy)
  against the plain solve (raftk_farm_batch_response_ws_dev), alternated, CUDA events around a run of calls per sample.
  One shape per kernel class: 16 farms of 2 (rows12), 4 (warp) and 8 (block) FOWTs, 4 farms of 64 (global).
* k_farm_publish: its kernel time and the solve's from torch.profiler, in a run of its own after the timed one.
The multi-GPU speed-up needs several GPUs and is not measured here.  Usage: python tools/farm_shard_timing.py [--out FILE]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WANT = ("Xi", "status", "B_drag", "F_drag", "F_iner")


def farm_designs(F, N, nw):
    """F farms of N FOWTs from the two-FOWT fixture on an nw-bin grid: FOWTs on 1600 m rows, every farm shifted."""
    from raft_b200 import grid
    z = np.load(os.path.join(ROOT, "tests", "golden", "farm_VolturnUS-S_farm_nw48.npz"))
    base = [grid.regrid({k[3:]: z[k] for k in z.files if k.startswith("P%d_" % i)}, nw, 0.005 * nw) for i in range(int(z["n_fowt"]))]
    out = []
    for f in range(F):
        for i in range(N):
            P = dict(base[i % 2])
            r = np.array([1600.0 * (i // 2) + 137.0 * f, 800.0 * (i % 2) - 211.0 * f, 0.0])
            for k in ("mem_rA", "node_r", "prp"):
                P[k] = np.asarray(P[k], dtype=float) + r
            P["x_ref"], P["y_ref"] = float(P["x_ref"]) + r[0], float(P["y_ref"]) + r[1]
            out.append(P)
    return out


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "nvidia-smi unavailable"


class Shape:
    def __init__(self, F, N, nC, nw):
        import torch
        from raft_b200 import solver, sweep
        from raft_b200._lib import RaftkPeers, check, lib
        self.F, self.N, self.torch = F, N, torch
        n = 6 * N
        rng = np.random.default_rng(N)
        K = rng.normal(size=(n, n)) * 2e4
        self.C_arr = K @ K.T / n + np.diag([5e4] * n)
        cs = dict(Hs=rng.uniform(1, 9, nC), Tp=rng.uniform(6, 16, nC), gamma=np.zeros(nC), beta_deg=rng.uniform(-180, 180, nC),
                  spec=np.zeros(nC, dtype=np.int32))
        self.sess = solver.DeviceSession(solver.DesignBatch(farm_designs(F, N, nw)), solver.CaseTable(cs), device="cuda:0", want=WANT)
        self.sess.solve(n_iter=10)
        self.xi, self.info = self.sess.farm_response(C_arr=self.C_arr, n_fowt=N)
        self.kernel = solver.last_dispatch()["kernel"]
        # two gathered copies on this device: rank 0's own and its one emulated peer's
        self.block = F * nC * n * nw
        xi_bytes = 2 * self.block * 16
        off_flags = (xi_bytes + 255) // 256 * 256
        off_status = off_flags + 256
        total = off_status + 2 * F * nC * (nw + 4 * N) * 4
        self.ptrs = []
        for _ in range(2):
            p, h = C.c_void_p(), C.create_string_buffer(64)
            check(lib.raftk_peer_alloc(total, C.byref(p), h))
            self.ptrs.append(p.value)
        self.peers = RaftkPeers()
        self.peers.n_ranks, self.peers.rank, self.peers.epoch, self.peers.block_elems = 2, 0, 1, self.block
        for q in range(2):
            self.peers.gathered[q], self.peers.flags[q], self.peers.status[q] = self.ptrs[q], self.ptrs[q] + off_flags, self.ptrs[q] + off_status
        raw = torch.as_tensor(sweep._DevMem(self.ptrs[0], total), device="cuda:0")
        self.gx = torch.view_as_complex(raw[:xi_bytes].view(torch.float64).view(-1, 2)).view(2 * F, nC, n, nw)
        self.gi = raw[off_status:off_status + 2 * F * nC * nw * 4].view(torch.int32).view(2 * F, nC, nw)

    def plain(self):
        self.sess.farm_response(C_arr=self.C_arr, n_fowt=self.N)

    def peer(self):
        self.sess.farm_response_gather(self.peers, 0, self.gx[:self.F], self.gi[:self.F], self.N, C_arr=self.C_arr)

    def same_bits(self):
        """The peer call's local rows and the emulated peer's copy against the plain call's output."""
        torch = self.torch
        self.plain()
        self.peer()
        torch.cuda.synchronize()
        from raft_b200 import sweep
        peer = torch.as_tensor(sweep._DevMem(self.ptrs[1], self.block * 16), device="cuda:0")
        px = torch.view_as_complex(peer.view(torch.float64).view(-1, 2)).view(self.xi.shape)
        return bool(torch.equal(self.gx[:self.F], self.xi) and torch.equal(px, self.xi) and torch.equal(self.gi[:self.F], self.info))

    def close(self):
        from raft_b200._lib import check, lib
        self.gx = self.gi = None
        for p in self.ptrs:
            check(lib.raftk_peer_free(p))


def timed(fn, calls):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(calls):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nC", type=int, default=8)
    ap.add_argument("--nw", type=int, default=256)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("farm_shard_timing needs a CUDA device")
    info = gpu_info()
    lines = ["GPU (name, power limit, max SM clock): %s" % info,
             "shape: %d cases x %d bins; per sample: CUDA events around a run of calls on one stream, after 3 warm-up calls of each;"
             " plain and peer alternated, %d samples each, median and spread (min..max) reported" % (args.nC, args.nw, args.reps)]
    rec = dict(gpu=info, nC=args.nC, nw=args.nw, shapes=[])
    for F, N, calls in ((16, 2, 100), (16, 4, 100), (16, 8, 40), (4, 64, 3)):
        s = Shape(F, N, args.nC, args.nw)
        for _ in range(3):
            s.plain()
            s.peer()
        torch.cuda.synchronize()
        t = {"plain": [], "peer": []}
        for _ in range(args.reps):
            t["plain"].append(timed(s.plain, calls))
            t["peer"].append(timed(s.peer, calls))
        same = s.same_bits()
        med = {k: float(np.median(v)) for k, v in t.items()}
        r = dict(F=F, N=N, kernel=s.kernel, calls_per_sample=calls, same_bits=same,
                 plain_ms=med["plain"], peer_ms=med["peer"], plain_range=[min(t["plain"]), max(t["plain"])],
                 peer_range=[min(t["peer"]), max(t["peer"])], peer_over_plain=med["peer"] / med["plain"])
        lines.append("%2d farms x %2d FOWTs (%s): plain %.3f ms [%.3f..%.3f], peer (one emulated peer) %.3f ms [%.3f..%.3f], "
                     "ratio %.3f; peer results == plain results: %s"
                     % (F, N, s.kernel, med["plain"], *r["plain_range"], med["peer"], *r["peer_range"], r["peer_over_plain"], same))
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(calls):
                s.peer()
            torch.cuda.synchronize()
        ker = {}
        for e in prof.key_averages():
            nm = "k_farm_publish" if "k_farm_publish" in e.key else "solve" if ("k_farm_r" in e.key) else None
            if nm:
                ker[nm] = ker.get(nm, 0.0) + e.device_time_total / 1e3 / calls
        r["profiler_ms"] = ker
        pub_bytes = F * args.nC * (6 * N * args.nw * 16 + args.nw * 4 + N * 4 * 4)
        pub = ker.get("k_farm_publish", float("nan"))
        lines.append("   torch.profiler, %d peer calls: solve kernel %.3f ms/call, k_farm_publish %.4f ms/call "
                     "(%.1f MB to the one peer copy + status rows: %.0f GB/s device-to-device on one GPU)"
                     % (calls, ker.get("solve", float("nan")), pub, pub_bytes / 1e6, pub_bytes / (pub * 1e-3) / 1e9))
        rec["shapes"].append(r)
        s.close()
    lines.append("multi-GPU speed-up of ShardedFarmSolve: not measured (one GPU)")
    text = "\n".join(lines)
    print(text)
    print(json.dumps(rec))
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(text + "\n" + json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
