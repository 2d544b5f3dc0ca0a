#!/usr/bin/env python
"""Cost of second-order wave loads on the generalised-DOF solve.

1. The bench's flex workload shape (bench_extra.flex_design: 150 DOFs, 200 bins, 64 cases) solved through GeneralSession
   without and with the marin_semi QTF (tests/golden/wamit_marin_semi.npz's .12d rows read by bem.read_qtf: 56 frequencies,
   one heading), alternated within one run, CUDA events around each solve.
2. With ``--parent DIR``: ``bench.py --workload flex`` run alternately from this tree and from DIR, a checkout of the parent
   commit that its own build() has built, to show that the solve without a table is unchanged.

The card's name, power limit and SM clocks are printed with the numbers.

Usage:  python tools/general_qtf_timing.py [--reps 7] [--nw 200] [--cases 64] [--parent DIR --rounds 3 --steps 10]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def marin_qtf():
    from raft_b200 import bem
    rows = np.load(os.path.join(ROOT, "tests", "golden", "wamit_marin_semi.npz"))["qtf_rows"]
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "semi.12d")
        np.savetxt(path, rows, fmt="%.5e")
        q, w, heads = bem.read_qtf(path)
    return dict(qtf=q, qtf_w=w, qtf_heads=heads)


def device_line():
    import torch
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                            # pragma: no cover
        smi = "nvidia-smi unavailable (%s)" % e
    return "device: %s | %s" % (torch.cuda.get_device_name(0), smi)


def session_timing(args):
    import torch
    import bench_extra
    from raft_b200 import solver
    dev = torch.device("cuda", 0)
    P, M, B, Cm = bench_extra.flex_design(args.nw)
    nC = args.cases
    rng = np.random.default_rng(6)
    cs = solver.CaseTable(dict(Hs=rng.uniform(1, 10, nC), Tp=rng.uniform(5, 18, nC), gamma=np.zeros(nC), beta_deg=rng.uniform(-180, 180, nC),
                               spec=np.zeros(nC, dtype=np.int32)))
    sess = {"no qtf": solver.GeneralSession(P, M, B, Cm, cs, device=dev),
            "qtf": solver.GeneralSession(P, M, B, Cm, cs, device=dev, qtf=marin_qtf())}
    for s in sess.values():
        s.solve(n_iter=10)
    torch.cuda.synchronize()
    times = {k: [] for k in sess}
    for _ in range(args.reps):
        for k, s in sess.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            s.solve(n_iter=10)
            b.record()
            b.synchronize()
            times[k].append(a.elapsed_time(b))
    passes = {k: s.status[:, 0].cpu().numpy() for k, s in sess.items()}
    q = sess["qtf"].qtf
    print(device_line())
    print("shape: %d DOFs, %d bins, %d cases, n_iter 10, QTF %d frequencies x %d heading(s)" % (int(P["gen_nDOF"]), args.nw, nC, q.n_qtf_w, q.n_qtf_head))
    for k, t in times.items():
        t = np.array(t)
        print("%-7s median %.2f ms  min %.2f  max %.2f  (%d reps)  passes: mean %.2f" % (k, np.median(t), t.min(), t.max(), len(t), passes[k].mean()))
    r = np.array(times["qtf"]) / np.array(times["no qtf"])
    print("qtf / no qtf per alternation: median %.4f  min %.4f  max %.4f" % (np.median(r), r.min(), r.max()))
    print("F_2nd max over cases: %.3e" % float(sess["qtf"].F_2nd.abs().max()))


def bench_ab(args):
    env = dict(os.environ)
    env.pop("RAFTK_LIB", None)
    opts = ["--workload", "flex", "--gpus", "1", "--steps", str(args.steps), "--warmup", str(args.warmup)]
    trees = (("this", ROOT), ("parent", os.path.abspath(args.parent)))
    rows = {"this": [], "parent": []}
    for _ in range(args.rounds):
        for name, tree in trees:
            out = subprocess.run([sys.executable, os.path.join(tree, "bench.py")] + opts, cwd=tree, env=env, capture_output=True, text=True,
                                 timeout=1200)
            line = [l for l in out.stdout.splitlines() if l.startswith("{")]
            if out.returncode or not line:
                print("bench.py failed (%s):" % name, out.stdout[-2000:], out.stderr[-2000:])
                return
            rows[name].append(json.loads(line[-1]))
    print(device_line())
    for name, rs in rows.items():
        ms = [r.get("ms_per_step") for r in rs]
        e2e = [r.get("e2e", {}).get("ms_per_step") for r in rs]
        print("bench flex %-6s ms_per_step: %s   e2e.ms_per_step: %s" % (name, ", ".join("%.2f" % m for m in ms if m is not None),
                                                                          ", ".join("%.2f" % m for m in e2e if m is not None)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--nw", type=int, default=200)
    ap.add_argument("--cases", type=int, default=64)
    ap.add_argument("--parent", default=None, help="checkout of the parent commit, built, for the bench.py A/B")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    session_timing(args)
    if args.parent:
        bench_ab(args)


if __name__ == "__main__":
    main()
