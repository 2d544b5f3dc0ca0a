"""bench.py support (measurement code, not product): workloads beyond the single-FOWT solve: the coupled farm (BASELINE.json configs[4]) and the flexible
(generalised-DOF) platform.  Each prints ONE JSON line in bench.py's format on rank 0.

farm: N copies of the VolturnUS-S farm platform (designs/VolturnUS-S_farm.yaml, fixture farm_VolturnUS-S_farm_nw48) on a
    1600 m grid, 1024 bins (min_freq 0.0001, max_freq 0.1024 Hz), array mooring = seeded SPD 6N x 6N stiffness; a step is
    the per-FOWT drag-linearisation solve of all N FOWTs + the 6N x 6N system response for every (case, frequency).
    One RAO solve = one 6N-DOF response for one (case, frequency).  Default: the file's case (JONSWAP Hs 6 m, Tp 12 s) as
    configs[4] states, plus a 64-sea-state batch as the throughput figure; N in {2, 4, 8, 16} summarised in `farm_sizes`.
"""
import json
import os
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
METRIC = "RAO solves/sec (freq-bins x cases x designs)"
UNIT = "solves/s"


def farm_designs(N, nw=1024, max_freq=0.1024):
    """-> (packed FOWT tables of N units on a 1600 m grid, seeded SPD array stiffness [6N,6N], fixture)."""
    from raft_b200 import grid
    from raft_b200.fowt import FOWT
    z = np.load(os.path.join(ROOT, "tests", "golden", "farm_VolturnUS-S_farm_nw48.npz"))
    D = json.load(open(os.path.join(ROOT, "tests", "golden", "designs.json")))["farm_VolturnUS-S_farm_nw48"]
    P1 = {k[3:]: z[k] for k in z.files if k.startswith("P1_")}                     # the unit with heading_adjust 0
    mats = dict(M_struc=P1["M0"] - z["A_hydro_morison1"], C_struc=P1["C0"] - z["C_moor1"], C_moor=z["C_moor1"])
    w = grid.make_w(max_freq / nw, max_freq)
    depth = float(P1["depth"])
    k = grid.wave_number(w, depth)
    side = int(np.ceil(np.sqrt(N)))
    packs = []
    for i in range(N):
        f = FOWT(dict(site=D["site"], platform=D["platform"]), w, depth=depth, x_ref=1600.0 * (i % side), y_ref=1600.0 * (i // side),
                 matrices=mats, k=k)
        f.calcHydroConstants()
        packs.append(f.pack())
    rng = np.random.default_rng(5)
    A = rng.normal(size=(6 * N, 6 * N)) * 2e4
    return packs, A @ A.T / (6 * N) + np.diag([5e4] * (6 * N)), z


def _oracle_farm(packs, C_arr, cs):
    from oracle import oracle as orc
    orc.build()
    nC, N, nw = len(cs["Hs"]), len(packs), len(packs[0]["w"])
    Xo = np.zeros([nC, 6 * N, nw], dtype=complex)
    passes = np.zeros([N, nC], dtype=int)
    ods = [orc.OracleDesign(P) for P in packs]
    for c in range(nC):
        Z = np.zeros([nw, 6 * N, 6 * N], dtype=complex)
        F = np.zeros([nw, 6 * N], dtype=complex)
        for i, od in enumerate(ods):
            Xi_i, st, Z_i, _ = orc.solve_dynamics(od, 0, cs["Hs"][c], cs["Tp"][c], 0.0, cs["beta_deg"][c], nIter=10, want_Z=True)
            passes[i, c] = st[0]
            Z[:, 6 * i:6 * i + 6, 6 * i:6 * i + 6] = Z_i
            F[:, 6 * i:6 * i + 6] = np.einsum("wab,bw->wa", Z_i, Xi_i)
        Xo[c] = orc.system_response(Z + C_arr[None], F).T
    return Xo, passes


def _time_farm(N, cs, dev, steps, warmup, parity=False, dump=None):
    """-> dict: device-timed step (solve of N FOWTs + system response), e2e through the host call, optional parity."""
    import torch
    from raft_b200 import solver
    packs, C_arr, _ = farm_designs(N)
    batch, cases = solver.DesignBatch(packs), solver.CaseTable(cs)
    nC, nw, n = cases.n_cases, batch.nw, 6 * N
    sess = solver.DeviceSession(batch, cases, device=dev, want=("Xi", "status", "B_drag", "F_drag", "F_iner"))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def step():
        sess.solve(n_iter=10, tol=0.01, xi_start=0.0)
        return sess.farm_response(C_arr=C_arr)

    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    l0 = solver.launch_count()
    for a, b in ev:
        flush.fill_(1)
        a.record()
        xi, info = step()
        b.record()
    torch.cuda.synchronize()
    launches = solver.launch_count() - l0
    if dump:
        import bench
        bench.dump_outputs(dump, dict(Xi_sys=xi, info=info), lead=1)
    ms = sum(a.elapsed_time(b) for a, b in ev) / steps
    solver.profile_enable(True)
    flush.fill_(1)
    sess.solve(n_iter=10, tol=0.01, xi_start=0.0)
    m1, _ = solver.profile_read()
    sess.farm_response(C_arr=C_arr)
    kernel = solver.last_dispatch()["kernel"]
    m2, _ = solver.profile_read()
    solver.profile_enable(False)
    torch.cuda.synchronize()
    # e2e: page-locked host buffers through the one-call C-ABI entry (H2D of tables + D2H of Xi_sys, per-FOWT Xi, status inside)
    for k_, v in list(batch.arrays.items()):
        p_ = solver.pinned_empty(v.shape, v.dtype); p_[...] = v; batch.arrays[k_] = p_
    for k_, v in list(cases.arrays.items()):
        p_ = solver.pinned_empty(v.shape, v.dtype); p_[...] = v; cases.arrays[k_] = p_
    pin = dict(Xi=solver.pinned_empty([N, nC, 6, nw], np.complex128), status=solver.pinned_empty([N, nC, 4], np.int32),
               B_drag=solver.pinned_empty([N, nC, 6, 6], np.float64), Xi_sys=solver.pinned_empty([nC, n, nw], np.complex128),
               info=solver.pinned_empty([nC, nw], np.int32))
    for _ in range(warmup):
        out = solver.solve_dynamics_farm(batch, cases, C_arr=C_arr, n_iter=10, out=pin)
    t0 = time.perf_counter()
    for _ in range(steps):
        out = solver.solve_dynamics_farm(batch, cases, C_arr=C_arr, n_iter=10, out=pin)
    e2e_ms = 1e3 * (time.perf_counter() - t0) / steps
    assert np.array_equal(out["Xi_sys"], xi.cpu().numpy()), "e2e and resident farm paths disagree"
    units = nC * nw
    res = dict(n_fowt=N, n_dof=n, cases=nC, nw=nw, ms_per_step=ms, value=units / (ms * 1e-3), e2e_ms_per_step=e2e_ms, e2e_value=units / (e2e_ms * 1e-3),
               launches_per_step=launches / steps, solve_kernels_ms=float(sum(m1)), system_kernel_ms=float(m2[1]), kernel=kernel,
               h2d=int(batch.input_bytes() + cases.input_bytes() + C_arr.nbytes),
               d2h=int(out["Xi_sys"].nbytes + out["Xi"].nbytes + out["status"].nbytes + out["info"].nbytes + out["B_drag"].nbytes))
    if parity:
        import sys
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        from conftest import response_err
        Xo, passes = _oracle_farm(packs, C_arr, cs)
        res["parity"] = dict(max_rel_err=max(response_err(out["Xi_sys"][:, 6 * i:6 * i + 6], Xo[:, 6 * i:6 * i + 6]) for i in range(N)),
                             pass_mismatch_units=int(np.sum(passes != out["status"][:, :, 0])), units_checked=int(N * nC), rtol=1e-9,
                             metric="response_err per FOWT block of Xi_sys vs the oracle's per-FOWT solves + explicit-inverse system response "
                                    "(raft_model.py:1189-1216); pinned against the reference's own farm run in tests/test_farm.py")
    del sess, flush
    torch.cuda.empty_cache()
    return res


def bench_special(args, rank, world, dev):
    import torch
    from raft_b200 import solver
    if args.workload != "farm":
        return bench_flex(args, rank, world, dev)
    if rank != 0:
        return                                          # the coupled system stays on one GPU (SURVEY.md 8e): replicas only
    N = args.turbines or 2
    file_case = dict(Hs=np.array([6.0]), Tp=np.array([12.0]), gamma=np.zeros(1), beta_deg=np.array([0.0]), spec=np.zeros(1, dtype=np.int32))
    rng = np.random.default_rng(5)
    nC = args.cases or 64
    batch_cs = dict(Hs=rng.uniform(1, 10, nC), Tp=rng.uniform(5, 18, nC), gamma=np.zeros(nC), beta_deg=rng.uniform(-180, 180, nC),
                    spec=np.zeros(nC, dtype=np.int32))
    one = _time_farm(N, file_case, dev, args.steps, args.warmup, parity=not args.no_parity)
    many = _time_farm(N, batch_cs, dev, args.steps, args.warmup, parity=(not args.no_parity) and N <= 4, dump=args.dump_outputs)
    sizes = {}
    if not args.no_extras:
        for n_ in (2, 4, 8, 16):
            r = many if n_ == N else _time_farm(n_, batch_cs, dev, max(3, args.steps // 2), 3)
            sizes[str(n_)] = dict(value=r["value"], ms_per_step=r["ms_per_step"], system_kernel_ms=r["system_kernel_ms"], solve_kernels_ms=r["solve_kernels_ms"],
                                  e2e_value=r["e2e_value"])
    n = 6 * N
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        pass
    hbm = float(peaks.get("hbm_gbs", 3350.0))
    # SURVEY.md 8(d): farm bytes per solve = 16 n (Xi out) + 8 (zeta) + per-FOWT loads read by the system kernel (3 x 96 N) + ...
    b_alg = 16 * n + 8 + 3 * 96 * N + 288 * N / 1024.0
    ach = b_alg * many["cases"] * many["nw"] / (many["system_kernel_ms"] * 1e-3) / 1e9
    fl = (8.0 / 3.0) * n ** 3 + 8.0 * n * n
    line = dict(metric=METRIC, value=many["value"], unit=UNIT, n_gpus=1, steps=args.steps, warmup=args.warmup, ms_per_step=many["ms_per_step"],
                higher_is_better=True, scaling="weak", vs_baseline=None, dtype="f64", data="synthetic",
                config=dict(workload="farm: designs/VolturnUS-S_farm.yaml platform x %d FOWTs on a 1600 m grid, coupled %d-DOF system, %d bins x %d sea "
                                     "states, seeded SPD array-mooring stiffness, fp64" % (N, n, many["nw"], many["cases"]),
                            n_fowt=N, n_dof=n, nw=many["nw"], cases=many["cases"], l2="flushed between timed steps (256 MiB write)"),
                e2e=dict(value=many["e2e_value"], unit=UNIT, ms_per_step=many["e2e_ms_per_step"], h2d_bytes_per_step=many["h2d"], d2h_bytes_per_step=many["d2h"]),
                gpu_launches=int(round(many["launches_per_step"] * args.steps)),
                roofline=dict(bound="hbm", kernel=("k_farm_response_global (block assembly + %dx%d complex LU per (case, bin), matrix in a global-memory "
                                                   "workspace slab)" if many["kernel"] == "farm-global" else
                                                   "k_farm_response (block assembly + %dx%d complex LU per (case, bin), matrix in shared memory)") % (n, n),
                              achieved=ach, peak=hbm, unit="GB/s", frac=ach / hbm, traffic=None, kernel_ms=many["system_kernel_ms"],
                              algorithmic_bytes_per_solve=b_alg, lu_gflops=fl * many["cases"] * many["nw"] / (many["system_kernel_ms"] * 1e-3) / 1e9,
                              share_of_step=many["system_kernel_ms"] / (many["system_kernel_ms"] + many["solve_kernels_ms"])),
                parity=many.get("parity") or one.get("parity"),
                file_case=dict(note="configs[4] as stated: the design file's single case (JONSWAP Hs 6 m, Tp 12 s, heading 0)", value=one["value"],
                               ms_per_step=one["ms_per_step"], e2e_value=one["e2e_value"], parity=one.get("parity")),
                farm_sizes=sizes)
    print(json.dumps(line))


# ---- flexible platform (generalised DOFs, SURVEY.md 8f row 4) ---------------------------------------------------------------
def flex_design(nw=200, max_freq=0.40):
    """VolturnUS-S-flexible (fixture flex_VolturnUS-S-flexible: 150 DOFs, 33 submerged strip nodes with their fowt.T blocks) on
    a grid of ``nw`` bins.  The fixture's MacCamy-Fuchs tables exist for its own 40 bins only, so the bench variant uses the
    constant Imat (MCF off); parity with MCF on is pinned at the fixture's grid in tests/test_general_dofs.py."""
    from raft_b200 import grid
    z = np.load(os.path.join(ROOT, "tests", "golden", "flex_VolturnUS-S-flexible.npz"))
    P = {k[2:]: z[k] for k in z.files if k.startswith("P_") and not k.endswith("_w")}
    w = grid.make_w(max_freq / nw, max_freq)
    P.update(w=w, k=grid.wave_number(w, float(P["depth"])), dw=np.float64(w[1] - w[0]))
    return P, z["gen_M"], z["gen_B"], z["gen_C"]


def bench_flex(args, rank, world, dev):
    import torch
    from raft_b200 import solver
    if rank != 0:
        return
    nw, nC = args.nw or 200, args.cases or 64
    P, M, B, Cm = flex_design(nw)
    n = int(P["gen_nDOF"])
    rng = np.random.default_rng(6)
    cs = dict(Hs=rng.uniform(1, 10, nC), Tp=rng.uniform(5, 18, nC), gamma=np.zeros(nC), beta_deg=rng.uniform(-180, 180, nC), spec=np.zeros(nC, dtype=np.int32))
    cases = solver.CaseTable(cs)
    sess = solver.GeneralSession(P, M, B, Cm, cases, device=dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    for _ in range(max(args.warmup, 1)):
        sess.solve(n_iter=10)
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
    l0 = solver.launch_count()
    for a, b in ev:
        flush.fill_(1)
        a.record()
        xi, st_ = sess.solve(n_iter=10)
        b.record()
    torch.cuda.synchronize()
    launches = solver.launch_count() - l0
    if args.dump_outputs:
        import bench
        bench.dump_outputs(args.dump_outputs, dict(Xi=xi, status=st_), lead=1)
    ms = sum(a.elapsed_time(b) for a, b in ev) / args.steps
    solver.profile_enable(True)
    sess.solve(n_iter=10)
    kms, kn = solver.profile_read()
    solver.profile_enable(False)
    st = sess.status.cpu().numpy()
    passes = float(st[:, 0].mean())
    units = nC * nw
    t0 = time.perf_counter()
    Xi_h, st_h = solver.general_solve_dynamics(P, M, B, Cm, cases, n_iter=10)
    e2e_ms = 1e3 * (time.perf_counter() - t0)
    assert np.array_equal(st_h, st)
    lu_ms = kms[2] / max(kn[2], 1)                       # one launch = the LUs of every (case, bin) of one pass
    flops_lu = (8.0 / 3.0) * n ** 3 + 8.0 * n * n        # complex LU + solve, real flops per system
    fp64_peak = solver.fp64_peak_gflops(20000)
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        pass
    hbm = float(peaks.get("hbm_gbs", 3350.0))
    b_alg = 16.0 * n + 8 + 16.0 * n * n / nC            # Xi out + zeta + the constant matrices shared by the cases of a bin
    ach = b_alg * units / (lu_ms * 1e-3) / 1e9
    parity = None
    if not args.no_parity:
        from oracle import oracle as orc
        orc.build()
        gd = orc.GeneralDesign(P)
        worst, mism = 0.0, 0
        for c in range(min(nC, 4)):
            Xo, so = orc.general_solve_dynamics(gd, M, B, Cm, 0, cs["Hs"][c], cs["Tp"][c], 0.0, cs["beta_deg"][c], nIter=10)
            worst = max(worst, float(np.abs(Xi_h[c] - Xo).max() / np.abs(Xo).max()))
            mism += int(so[0] != st_h[c, 0])
        parity = dict(max_rel_err=worst, pass_mismatch_units=mism, units_checked=min(nC, 4), rtol=1e-9,
                      metric="max |Xi - Xi_oracle| / max |Xi_oracle| per case (150 DOFs mix translations, rotations and modal amplitudes); the impedance has "
                             "cond ~1e6, two LUs agree to ~1e-11; pinned to the reference's own 150-DOF run in tests/test_general_dofs.py")
    line = dict(metric=METRIC, value=units / (ms * 1e-3), unit=UNIT, n_gpus=1, steps=args.steps, warmup=args.warmup, ms_per_step=ms, higher_is_better=True,
                scaling="weak", vs_baseline=None, dtype="f64", data="synthetic",
                config=dict(workload="flex: VolturnUS-S-flexible (%d generalised DOFs, %d strip nodes, MacCamy-Fuchs off), %d bins x %d sea states, fp64" % (n, len(P["node_ls"]), nw, nC),
                            n_dof=n, nw=nw, cases=nC, mean_passes=passes, l2="flushed between timed steps (256 MiB write)"),
                e2e=dict(value=units / (e2e_ms * 1e-3), unit=UNIT, ms_per_step=e2e_ms, h2d_bytes_per_step=int(P["gen_Tn"].nbytes + 3 * M.nbytes), d2h_bytes_per_step=int(Xi_h.nbytes + st_h.nbytes)),
                gpu_launches=int(launches),
                roofline=dict(bound="hbm", kernel="k_gen_solve_blocked (150x150 complex LU per (case, bin): panel + row block in shared memory, 4x2 register tiles)",
                              achieved=ach, peak=hbm, unit="GB/s", frac=ach / hbm, traffic=None, kernel_ms=lu_ms, launches_per_step=kn[2],
                              algorithmic_bytes_per_solve=b_alg, share_of_step=kms[2] / max(sum(kms), 1e-30)),
                roofline_fp64=dict(bound="fp64", achieved=flops_lu * units / (lu_ms * 1e-3) / 1e12, peak=fp64_peak / 1e3, unit="TFLOP/s",
                                   frac=flops_lu * units / (lu_ms * 1e-3) / 1e9 / fp64_peak, flops_per_system=flops_lu),
                parity=parity)
    del sess
    line["trains"] = _flex_trains(args, P, M, B, Cm, cs, ms, flush, dev)
    print(json.dumps(line))


def _flex_trains(args, P, M, B, Cm, cs, ms_single, flush, dev):
    """The same sea states, each with a second seeded wave train (cases.primary): train 0 drives the linearisation, the
    second is solved from the primary's LU factors.  The primaries repeat the single-train step's work exactly, so the
    secondaries' share of the step is (ms_trains - ms_single) / ms_trains."""
    import torch
    from raft_b200 import solver
    nC, nw = len(cs["Hs"]), len(P["w"])
    rng = np.random.default_rng(7)
    Hs2, Tp2, b2 = rng.uniform(1, 10, nC), rng.uniform(5, 18, nC), rng.uniform(-180, 180, nC)
    rows = lambda a, b: np.stack([a, b], axis=1).reshape(-1)             # noqa: E731  case c -> trains 2c, 2c + 1
    tab = dict(Hs=rows(cs["Hs"], Hs2), Tp=rows(cs["Tp"], Tp2), gamma=np.zeros(2 * nC), beta_deg=rows(cs["beta_deg"], b2),
               spec=np.zeros(2 * nC, dtype=np.int32), primary=np.repeat(np.arange(0, 2 * nC, 2), 2).astype(np.int32))
    ct = solver.CaseTable(tab)
    sess = solver.GeneralSession(P, M, B, Cm, ct, device=dev)
    for _ in range(max(args.warmup, 1)):
        sess.solve(n_iter=10)
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
    for a, b in ev:
        flush.fill_(1)
        a.record()
        sess.solve(n_iter=10)
        b.record()
    torch.cuda.synchronize()
    ms = sum(a.elapsed_time(b) for a, b in ev) / args.steps
    out = dict(trains_per_case=2, ms_per_step=ms, value=2 * nC * nw / (ms * 1e-3), unit="train RAO solves/s",
               secondary_share_of_step=(ms - ms_single) / ms, parity=None)
    if not args.no_parity:
        import sys
        from oracle import oracle as orc
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        import general_trains_checker as gtc
        Xi_h, st_h = solver.general_solve_dynamics(P, M, B, Cm, ct, n_iter=10)
        worst, mism = 0.0, 0
        for c in range(min(nC, 2)):
            tr = np.array([[tab["Hs"][2 * c + h], tab["Tp"][2 * c + h], tab["beta_deg"][2 * c + h]] for h in range(2)])
            Xo, so, _ = gtc.solve_trains(orc, P, M, B, Cm, tr, nIter=10)
            for h in range(2):
                worst = max(worst, float(np.abs(Xi_h[2 * c + h] - Xo[h]).max() / np.abs(Xo[h]).max()))
            mism += int(so[0] != st_h[2 * c, 0])
        out["parity"] = dict(max_rel_err=worst, pass_mismatch_cases=mism, cases_checked=min(nC, 2), rtol=1e-9,
                             metric="max |Xi - Xi_oracle| / max |Xi_oracle| per train, both trains of each checked case")
    return out
