"""Bit-for-bit A/B of every rigid FOWT solve kernel (k_drag_solve, k_rao_fused<128/256>, k_fused_plan + k_rao_fused2 on
clusters and on the grid) and of the flows built on them, between two builds of the same ABI.

  python tools/rigid_ab.py dump OUT.npz          # with the build RAFTK_LIB names (default: the tree's own)
  python tools/rigid_ab.py compare A.npz B.npz   # every array byte for byte, every dispatch name and workspace answer equal

dump runs, on the seeded inputs of tests/test_dispatch_solve.py (SHAPES, _design, _train_table):
  * every SHAPES variant with Xi, status, B_drag, F_drag, F_iner, F_BEM, zeta (and Xi_last on the fused kernels);
  * per fused variant of cfg2 and cfg3 (BEM): wave trains, Xi_init, per-case operating points (k_rao_fused2's OP and
    non-OP instantiations both run) and the potSecOrder 2 QTF force in the loop (F_2nd, F_2nd_mean);
  * hydro_excitation, hydro_linearization and DeviceSession.excitation / linearization;
  * a sweep.solve_sweep shard of three designs, the potSecOrder 1 slender flow, and a two-FOWT farm solve;
  * the workspace each DeviceSession sizes, with and without the global wave tables;
and records solver.last_dispatch() of each call.  The second-order forces go through k_qtf_force (RAFTK_QTF_DIAG=1):
k_qtf_tiles' atomic sums make F_2nd differ from run to run upstream of the solve.  Prints one JSON line.
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

ENV = ("RAFTK_FORCE_V1", "RAFTK_FUSED2_XCHG", "RAFTK_NO_DIRECT_D2H")


def _arrays(tag, out, res):
    if isinstance(out, dict):
        for k, v in out.items():
            _arrays("%s.%s" % (tag, k), v, res)
    elif isinstance(out, (tuple, list)):
        for i, v in enumerate(out):
            _arrays("%s.%d" % (tag, i), v, res)
    elif out is not None:
        if hasattr(out, "cpu"):
            out = out.cpu().numpy()
        res[tag] = np.ascontiguousarray(np.asarray(out))


def _env(env):
    for k in ENV:
        os.environ.pop(k, None)
    os.environ.update(env)


def dump(path):
    import torch
    from raft_b200 import solver, sweep
    from conftest import QTF_GOLDEN, load_golden
    import test_dispatch_solve as ts
    import test_slender_flow_device as tsf
    from test_operating_points import _op_tables
    res, disp = {}, {}

    def rec(tag, out):
        torch.cuda.synchronize()
        _arrays(tag, out, res)
        d = solver.last_dispatch()
        disp[tag] = "%s/%s" % (d.get("family"), d.get("kernel"))

    os.environ["RAFTK_QTF_DIAG"] = "1"
    full = ("Xi", "status", "B_drag", "F_drag", "F_iner", "F_BEM", "zeta")
    _, Pq = load_golden(QTF_GOLDEN)
    for shape in ts.SHAPES:
        name, nw, cs, env, kernel, _ = shape
        sid = ts._shape_id(shape)
        _env(env)
        P = ts._design(name, nw)
        sea = ts._sea_states(ts.SEEDS[name])
        fused = kernel != "v1"
        want = full + (("Xi_last",) if fused else ())

        def run(cases, packed=P, want=want):
            return solver.solve_dynamics(solver.DesignBatch(packed), cases, n_iter=10, cluster_size=cs, want=want)
        first = run(solver.CaseTable(sea))
        rec(sid, first)
        if not fused or name not in ("cfg2", "cfg3"):
            continue
        rec(sid + ".trains", run(solver.CaseTable(ts._train_table())))
        rec(sid + ".xi_init", run(solver.CaseTable(sea, Xi_init=first["Xi"] * (0.9 + 0.05j))))
        A, B = _op_tables(np.random.default_rng(nw), P, 2, 1)
        rec(sid + ".ops", run(solver.CaseTable(sea, ops=dict(op=np.array([1, 0, 1], dtype=np.int32), A_w=A, B_w=B))))
        if name == "cfg2":
            Q = dict(P, qtf=Pq["qtf"], qtf_w=Pq["qtf_w"], qtf_heads=Pq["qtf_heads"])
            rec(sid + ".qtf", run(solver.CaseTable(sea), packed=Q, want=("Xi", "status", "F_2nd", "F_2nd_mean", "B_drag")))
    _env({})

    for name, nw in (("cfg2", 201), ("cfg3", 201), ("rand2", 151)):
        P = ts._design(name, nw)
        sea = ts._sea_states(ts.SEEDS[name])
        batch, ct = solver.DesignBatch(P), solver.CaseTable(sea)
        rec("exc_%s" % name, solver.hydro_excitation(batch, ct))
        Xi = solver.solve_dynamics(batch, ct, n_iter=10)["Xi"]
        rec("lin_%s" % name, solver.hydro_linearization(batch, ct, Xi))
        sess = solver.DeviceSession(batch, ct, want=("Xi", "status", "B_drag", "F_drag", "F_iner", "F_BEM", "zeta"), tables=True)
        rec("sess_exc_%s" % name, {k: v.clone() for k, v in sess.excitation().items() if k in ("F_iner", "F_BEM", "zeta")})
        rec("sess_lin_%s" % name, {k: v.clone() for k, v in sess.linearization(torch.as_tensor(Xi, device="cuda")).items()
                                   if k in ("B_drag", "F_drag")})
        res["ws_%s" % name] = np.array([sess.workspace_bytes, solver.DeviceSession(batch, ct).workspace_bytes], dtype=np.int64)

    Pa = ts._design("cfg2", 201)
    designs = [Pa, dict(Pa, C0=Pa["C0"] * 1.3), dict(Pa, M0=Pa["M0"] * 0.9)]
    rec("sweep", sweep.solve_sweep(designs, ts._sea_states(41)))

    _, Ps = tsf._golden("slender_VolturnUS-S")
    slender = [Ps, tsf._random_design(Ps, 9)]
    rec("slender", solver.slender_flow_host(slender, solver.CaseTable(tsf._cases(7, 6)), n_iter=4, want=tsf.OUTS))

    zf = np.load(os.path.join(ROOT, "tests", "golden", "farm_VolturnUS-S_farm_nw48.npz"))
    packs = [{k[3:]: zf[k] for k in zf.files if k.startswith("P%d_" % i)} for i in range(int(zf["n_fowt"]))]
    cf = zf["cases"]
    cases = dict(Hs=cf[:, 0], Tp=cf[:, 1], gamma=np.zeros(len(cf)), beta_deg=cf[:, 2], spec=np.zeros(len(cf), dtype=np.int32))
    rec("farm", solver.solve_dynamics_farm(solver.DesignBatch(packs), solver.CaseTable(cases), C_arr=zf["C_array"],
                                           n_iter=int(zf["n_iter"]), xi_start=float(zf["xi_start"])))
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
    print(json.dumps(dict(arrays=len(A.files), differ=diff, kernels=sorted(set(da.values())))))
    return 1 if diff else 0


if __name__ == "__main__":
    if sys.argv[1] == "dump":
        dump(sys.argv[2])
    else:
        sys.exit(compare(sys.argv[2], sys.argv[3]))
