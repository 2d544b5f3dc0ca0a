"""Bit-for-bit A/B of every dense complex LU the library runs (raftk_lu.cuh): system_solve, the farm kernels and the
generalised-DOF solve with its trains, between two builds of the same ABI.

  python tools/lu_ab.py dump OUT.npz          # with the build RAFTK_LIB names (default: the tree's own)
  python tools/lu_ab.py compare A.npz B.npz   # every array byte for byte, every dispatch name and workspace answer equal

dump runs, on seeded inputs:
  * system_solve at n in {6, 24, 25, 64, 120, 121, 300} x nrhs in {1, 3} (Z with ties and a zero column in one bin);
  * farm batches of two farms, N in {1, 3, 4, 5, 20, 21, 32}, with and without per-case operating points and trains;
  * generalised solves at n in {9, 40, 150, 256}: the planted inputs of test_general_solve_edges with trains, the same
    tables as an operating point, a two-design batch, and general_synth's rows a (FD, trains), c (BEM only), e (256 DOFs) and f (QTF, through k_qtf_force);
  * raftk_farm_batch_workspace_bytes for N = 1..64;
and records solver.last_dispatch() of each call.  Prints one JSON line.
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _arrays(tag, out, res):
    if isinstance(out, dict):
        for k, v in out.items():
            _arrays("%s.%s" % (tag, k), v, res)
    elif isinstance(out, (tuple, list)):
        for i, v in enumerate(out):
            _arrays("%s.%d" % (tag, i), v, res)
    elif out is not None:
        res[tag] = np.ascontiguousarray(np.asarray(out))


def dump(path):
    from raft_b200 import solver
    import general_synth as gs
    import test_farm_edges as tf
    import test_general_solve_edges as tg
    from test_operating_points import _op_tables
    res, disp = {}, {}

    def rec(tag, out):
        _arrays(tag, out, res)
        d = solver.last_dispatch()
        disp[tag] = "%s/%s" % (d["family"], d["kernel"])

    rng = np.random.default_rng(1)
    for n in (6, 24, 25, 64, 120, 121, 300):
        for nrhs in (1, 3):
            nw = 6
            Z = rng.normal(size=(nw, n, n)) + 1j * rng.normal(size=(nw, n, n))
            Z[1, :, 0] = np.round(Z[1, :, 0].real) + 1j * np.round(Z[1, :, 0].imag)     # ties in the first column
            Z[2, :, n // 2] = 0.0                                                       # a zero pivot
            F = rng.normal(size=(nw, n, nrhs)) + 1j * rng.normal(size=(nw, n, nrhs))
            rec("sys_n%d_r%d" % (n, nrhs), solver.system_solve(Z, F))

    for N in (1, 3, 4, 5, 20, 21, 32):
        Fm, n = 2, 6 * N
        packs = [P for f in range(Fm) for P in tf._packs(N, tables=True, seed=10 * N + f)]
        C_arr = tf._link(N, 10.0, packs[0]["C0"][0, 0]) + np.diag([5e4] * n)
        rows = np.array([[6.0, 12.0, 0.0], [2.0, 7.0, 60.0], [4.0, 10.0, 200.0]])
        r = np.random.default_rng(N)
        A, B = _op_tables(r, packs[0], 2, Fm * N)
        for op in (False, True):
            ops = dict(op=np.array([0, 0, 1], dtype=np.int32), A_w=A, B_w=B) if op else None
            cs = solver.CaseTable(tf._cases(rows, primary=[0, 0, 2]), zeta=np.full((3, tf.NW), 0.5), ops=ops)
            out = solver.solve_dynamics_farm_batch(solver.DesignBatch(packs), cs, N, C_arr=C_arr, n_iter=6)
            rec("farm_N%d_op%d" % (N, op), {k: out[k] for k in ("Xi_sys", "info", "Xi", "status")})
    res["farm_ws"] = np.array([solver.farm_batch_workspace_bytes(2, N, 8, 256) for N in range(1, 65)], dtype=np.int64)

    for n in tg.SIZES:
        D, _, _ = tg._design(n)
        nw = tg._nw(n)
        table = tg._trains()
        rec("gen_n%d_trains" % n, tg._solve(D, solver.CaseTable(table, zeta=tg._zeta(3, nw)), "gen-blocked"))
        fd = D["fd"]
        ops = dict(op=np.zeros(3, dtype=np.int32), A_w=fd["A_w"][None], B_w=fd["B_w"][None])
        fd0 = dict(fd, A_w=np.zeros_like(fd["A_w"]), B_w=np.zeros_like(fd["B_w"]))
        rec("gen_n%d_op" % n, tg._solve(D, solver.CaseTable(table, zeta=tg._zeta(3, nw), ops=ops), "gen-blocked", fd=fd0))
        designs = [tg._design(n, seed=s)[0] for s in (1, 2)]
        rec("gen_n%d_batch" % n, solver.general_solve_dynamics_batch(designs, solver.CaseTable(tg._sea(2), zeta=tg._zeta(2, nw)),
                                                                    n_iter=10, F_BEM=True))
    os.environ["RAFTK_QTF_DIAG"] = "1"          # the second-order force without k_qtf_tiles' atomic sums, so that F_2nd repeats
    for name, arg in (("a", 9), ("a", 17), ("c", 129), ("f", (9, 129)), ("e", "stride")):
        r = gs.row(name, arg)
        table = r["ct"][0]
        out = solver.general_solve_dynamics(r["P"], r["M"], r["B"], r["Cm"], solver.CaseTable(table), n_iter=r["n_iter"], fd=r["fd"],
                                            F_BEM=True, qtf=r["qtf"], F_2nd=r["qtf"] is not None)
        rec("gen_row_%s_%s" % (name, arg), out)
    np.savez(path, __dispatch__=np.array(json.dumps(disp)), **res)
    print(json.dumps(dict(dumped=path, arrays=len(res), calls=len(disp), lib=os.environ.get("RAFTK_LIB", "tree"))))


def compare(a, b):
    A, B = np.load(a), np.load(b)
    diff = []
    for k in sorted(set(A.files) | set(B.files)):
        if k not in A.files or k not in B.files:
            diff.append("%s: missing" % k)
        elif A[k].dtype != B[k].dtype or A[k].shape != B[k].shape or A[k].tobytes() != B[k].tobytes():
            diff.append(k)
    da, db = json.loads(str(A["__dispatch__"])), json.loads(str(B["__dispatch__"]))
    diff += ["dispatch %s: %s / %s" % (k, da.get(k), db.get(k)) for k in sorted(set(da) | set(db)) if da.get(k) != db.get(k)]
    print(json.dumps(dict(arrays=len(A.files), differ=diff, dispatch=da)))
    return 1 if diff else 0


if __name__ == "__main__":
    if sys.argv[1] == "dump":
        dump(sys.argv[2])
    else:
        sys.exit(compare(sys.argv[2], sys.argv[3]))
