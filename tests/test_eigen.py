"""Natural frequencies and mode shapes (raftk_eigen_*, solver.solve_eigen, DeviceSession.eigen, GeneralBatchSession.eigen,
Model.solveEigen, FOWT.solveEigen).  Without a GPU: the struct layout and prototypes against include/raftk.h, the workspace
query, every refusal, packer.pack_eigen against the reference's own M_tot / C_tot, the numpy conventions of the outputs and the
flag -> exception mapping, and k_eig_small's registers.  On the GPU: every eigen_* fixture (the reference's own runs), seeded
systems against numpy on each kernel variant, complex-conjugate pairs, batch isolation and the entry points."""
import ctypes as C
import json
import os
import re
import shutil
import subprocess
import types

import numpy as np
import pytest

from conftest import GOLDEN, ROOT

HEADER = os.path.join(ROOT, "include", "raftk.h")
NEW = ("raftk_eigen_workspace_bytes", "raftk_eigen_dev", "raftk_eigen_host")
FIXTURES = ("OC3spar", "VolturnUS-S", "VolturnUS-S-pointInertia", "OC4semi-WAMIT", "farm", "farm24", "VolturnUS-S-flexible")
RIGID = FIXTURES[:4]
gpu = pytest.mark.gpu


def fixture(name):
    return dict(np.load(os.path.join(GOLDEN, "eigen_%s.npz" % name)))


def seeded(n, nS, seed):
    """nS seeded systems with a SPD mass and a stiffness with real positive spectrum (a FOWT-like pair of scales)."""
    rng = np.random.default_rng(seed)
    A = rng.normal(size=(nS, n, n))
    M = A @ np.swapaxes(A, 1, 2) / n + np.eye(n) * 2.0
    B = rng.normal(size=(nS, n, n))
    K = (B @ np.swapaxes(B, 1, 2) / n + np.eye(n)) * 10.0 ** rng.uniform(0, 3, size=(nS, 1, 1))
    K = K + 0.05 * rng.normal(size=(nS, n, n)) * np.abs(K).max(axis=(1, 2), keepdims=True) / n
    return M, K


# ---- without a GPU --------------------------------------------------------------------------------------------------
def _prototype(name):
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    m = re.search(r"\b(\w+\s*\*?)\s*\b%s\s*\(([^)]*)\)\s*;" % name, src)
    assert m, name
    return m.group(1).strip(), [a.strip() for a in m.group(2).split(",")]


@pytest.mark.parametrize("name", NEW)
def test_bindings_match_header_prototypes(name):
    from raft_b200 import _lib
    ret, params = _prototype(name)
    fn = getattr(_lib.lib, name)
    assert name in _lib.SYMBOLS and len(fn.argtypes) == len(params), (name, params)
    for decl, ct in zip(params, fn.argtypes):
        want = C.POINTER(_lib.RaftkEigen) if "raftk_eigen" in decl else (C.c_void_p if "*" in decl else C.c_size_t)
        assert ct is want, (name, decl, ct)
    assert fn.restype is (C.c_size_t if ret == "size_t" else C.c_int)


def test_struct_layout_and_flags_match_header(tmp_path):
    from raft_b200 import _lib, solver
    fields = [n for n, _ in _lib.RaftkEigen._fields_]
    flags = ("RAFTK_EIG_SMALL_DIAG", "RAFTK_EIG_NONPOSITIVE", "RAFTK_EIG_COMPLEX", "RAFTK_EIG_SINGULAR", "RAFTK_EIG_NOCONV",
             "RAFTK_EIG_SORT_DOF", "RAFTK_EIG_SORT_ASCENDING")
    src = tmp_path / "t.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "raftk.h"\nint main(void){printf("%%zu %s %s\\n", sizeof(raftk_eigen), %s, %s);'
                   'return 0;}\n' % (" ".join(["%zu"] * len(fields)), " ".join(["%d"] * len(flags)),
                                     ", ".join("offsetof(raftk_eigen, %s)" % n for n in fields), ", ".join(flags)))
    exe = tmp_path / "t"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    E = _lib.RaftkEigen
    assert got == [C.sizeof(E)] + [getattr(E, n).offset for n in fields] + [
        solver.EIG_SMALL_DIAG, solver.EIG_NONPOSITIVE, solver.EIG_COMPLEX, solver.EIG_SINGULAR, solver.EIG_NOCONV, 0, 1]


def test_workspace_query_without_gpu():
    from raft_b200 import solver
    for n in (1, 6, 12):
        for nS in (1, 7, 100000):
            assert solver.eigen_workspace_bytes(nS, n) == 0
    for n in (13, 144, 150, 300):
        slab = solver.eigen_workspace_bytes(1, n)
        mats = 2 if n <= 160 else 3                              # H in shared memory up to ~165 DOFs on an H100, else in the slab
        assert slab == (mats * n * (n | 1) * 8 + 255) // 256 * 256, n
        assert solver.eigen_workspace_bytes(5, n) == 5 * slab
        full = solver.eigen_workspace_bytes(100000, n)
        assert full % slab == 0 and 132 <= full // slab <= 132 * 16 and solver.eigen_workspace_bytes(200000, n) == full
    assert solver.eigen_workspace_bytes(0, 20) == 0 and solver.eigen_workspace_bytes(3, 0) == 0


def _eig(n=20, nS=2, sort=0):
    from raft_b200 import _lib
    e = _lib.RaftkEigen()
    e.n_systems, e.n, e.sort = nS, n, sort
    e.M, e.C, e.lam, e.info = 0x1000, 0x1000, 0x1000, 0x1000
    return e


@pytest.mark.parametrize("field,value,msg", [
    ("n", 0, "n and n_systems"), ("n", -4, "n and n_systems"), ("n_systems", 0, "n and n_systems"), ("sort", 2, "sort must"),
    ("sort", -1, "sort must"), ("M", None, "are required"), ("C", None, "are required"), ("lam", None, "are required"),
    ("info", None, "are required"), ("n", 100000, "too large"),
])
def test_entries_refuse_before_any_launch(field, value, msg):
    from raft_b200._lib import lib
    e = _eig()
    setattr(e, field, value)
    before = lib.raftk_launch_count()
    for rc in (lib.raftk_eigen_host(C.byref(e)), lib.raftk_eigen_dev(C.byref(e), 0x1000, 1 << 30, None)):
        assert rc == -1 and msg in lib.raftk_last_error().decode()
    assert lib.raftk_launch_count() == before
    assert lib.raftk_eigen_host(None) == -1 and lib.raftk_eigen_dev(None, None, 0, None) == -1


def test_device_entry_refuses_less_than_one_slab():
    from raft_b200 import solver
    from raft_b200._lib import lib
    before = lib.raftk_launch_count()
    for n in (20, 300):
        e = _eig(n=n)
        slab = solver.eigen_workspace_bytes(1, n)
        for ws, wsb in ((0x1000, slab - 8), (None, 1 << 30), (0x1000, 0)):
            assert lib.raftk_eigen_dev(C.byref(e), ws, wsb, None) == -1
            assert "less than one slab" in lib.raftk_last_error().decode()
    assert lib.raftk_launch_count() == before


def test_pack_eigen_reproduces_the_references_matrices():
    """Bit for bit from the attributes the reference's FOWT carries (getStiffness's summation order)."""
    from raft_b200 import packer
    for name in RIGID + ("VolturnUS-S-flexible",):
        z = fixture(name)
        f = types.SimpleNamespace(nDOF=len(z["M_tot"]), yawstiff=float(z["fowt_yawstiff"]), body=None,
                                  **{k[5:]: z[k] for k in z if k.startswith("fowt_") and k != "fowt_yawstiff"})
        E = packer.pack_eigen(f)
        assert np.array_equal(E["M"], z["M_tot"]) and np.array_equal(E["C"], z["C_tot"]), name


def test_pack_eigen_on_live_reference_objects():
    import sys
    sys.path.insert(0, ROOT)
    from oracle import ref_harness as rh
    if not rh.reference_available():
        pytest.skip("reference tree not present")
    from raft_b200 import packer
    td = os.path.join(rh.REF_ROOT, "tests", "test_data")
    for name, path in (("OC3spar", os.path.join(td, "OC3spar.yaml")), ("VolturnUS-S", os.path.join(td, "VolturnUS-S.yaml")),
                       ("OC4semi-WAMIT", os.path.join(rh.REF_ROOT, "examples", "OC4semi-WAMIT_Coefs.yaml"))):
        f = rh.build_model(rh.load_design(path)).fowtList[0]
        E, z = packer.pack_eigen(f), fixture(name)
        assert np.array_equal(E["M"], z["M_tot"]) and np.array_equal(E["C"], z["C_tot"]), name


def test_output_conventions_and_exceptions():
    from raft_b200 import solver
    lam = np.array([[4.0 + 0j, -1.0 + 0j, np.nan + 1j * np.nan]])
    with np.errstate(invalid="ignore"):
        want = np.sqrt(np.array([4.0, -1.0, np.nan])) / 2.0 / np.pi
    o = solver.eigen_outputs(lam, np.ones([1, 3, 3], dtype=complex), np.zeros(1, dtype=np.int32))
    assert o["lam"].dtype == np.float64 and o["modes"].dtype == np.float64
    np.testing.assert_array_equal(o["fns"][0], want)
    lam2 = np.array([[4.0 + 1j, 4.0 - 1j]])
    o = solver.eigen_outputs(lam2, None, np.zeros(1, dtype=np.int32))
    assert o["lam"].dtype == np.complex128 and np.array_equal(o["fns"], np.sqrt(lam2) / 2.0 / np.pi)
    M, K = np.eye(3), np.diag([2.0, 0.5, 3.0])
    M[1, 1] = 0.25
    with pytest.raises(RuntimeError, match=re.escape("Diagonal entry 1 of system mass matrix is less than 1 (0.25). "
                                                     "Diagonal entry 1 of system stiffness matrix is less than 1 (0.5).")):
        solver.eigen_raise(M, K, solver.EIG_SMALL_DIAG | solver.EIG_SINGULAR, "dof")
    for f in (solver.EIG_SINGULAR, solver.EIG_NOCONV):
        with pytest.raises(np.linalg.LinAlgError):
            solver.eigen_raise(M, K, f | solver.EIG_NONPOSITIVE, "dof")
    with pytest.raises(RuntimeError, match="zero or negative system eigenvalues"):
        solver.eigen_raise(M, K, solver.EIG_NONPOSITIVE | solver.EIG_COMPLEX, "dof")
    solver.eigen_raise(M, K, solver.EIG_NONPOSITIVE | solver.EIG_COMPLEX, "ascending")


def test_small_kernel_does_not_spill(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not shutil.which(nvcc):
        pytest.skip("nvcc not available")
    src = tmp_path / "k.cu"
    src.write_text('#include <cuda_runtime.h>\n#include <math_constants.h>\n#include "raftk.h"\n#include "raftk_eigen.cuh"\n')
    out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-c", "-Xptxas", "-v",
                          "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "raft_b200", "csrc"), "-o", str(tmp_path / "k.o"), str(src)],
                         capture_output=True, text=True, check=True).stderr
    m = re.search(r"Function properties for \w*k_eig_small\w*\s*\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", out)
    assert m, out
    assert m.group(1) == "0" and m.group(2) == "0", out


# ---- on the GPU -----------------------------------------------------------------------------------------------------
def _clusters(lam, tol):
    """Groups of indices whose eigenvalues lie within tol of each other (transitively)."""
    order = np.argsort(lam.real)
    groups, cur = [], [order[0]]
    for a, b in zip(order[:-1], order[1:]):
        if abs(lam[b] - lam[a]) <= tol:
            cur.append(b)
        else:
            groups.append(cur)
            cur = [b]
    groups.append(cur)
    return groups


def check_against(lam, V, M, K, lam_ref, V_ref, order_ok=True):
    """The issue's fixture checks -> (worst eigenvalue error / max|lam|, worst residual, worst mode sin-angle scaled)."""
    lam, lam_ref = np.asarray(lam, dtype=complex), np.asarray(lam_ref, dtype=complex)
    V, V_ref = np.asarray(V, dtype=complex), np.asarray(V_ref, dtype=complex)
    big = np.abs(lam_ref).max()
    gap_rel = 1e-8 * big
    n = len(lam)
    e_lam = np.abs(lam - lam_ref).max() / big
    nC, nM = np.linalg.norm(K, 2), np.linalg.norm(M, 2)
    res = max(np.linalg.norm(K @ V[:, j] - lam[j] * (M @ V[:, j])) / ((nC + abs(lam[j]) * nM) * np.linalg.norm(V[:, j])) for j in range(n))
    assert e_lam <= 1e-12, e_lam
    assert res <= 1e-13, res
    worst_mode = 0.0
    for g in _clusters(lam_ref, gap_rel):
        if len(g) == 1:
            j = g[0]
            others = np.delete(lam_ref, j)
            gap = np.abs(others - lam_ref[j]).min() if len(others) else big
            a, b = V[:, j] / np.linalg.norm(V[:, j]), V_ref[:, j] / np.linalg.norm(V_ref[:, j])
            s = np.linalg.norm(a - b * np.vdot(b, a))                 # sin of the angle, without cancellation
            bound = 1e-12 * big / gap
            worst_mode = max(worst_mode, s / bound)
            assert s <= max(bound, 1e-15), (j, s, bound)
        else:                                                  # a cluster: the spanned subspaces agree
            Qa, _ = np.linalg.qr(V[:, g])
            Qb, _ = np.linalg.qr(V_ref[:, g])
            sv = np.linalg.svd(Qa.conj().T @ Qb, compute_uv=False)
            assert sv.min() >= 1.0 - 1e-6, (g, sv)
    return e_lam, res, worst_mode


@gpu
@pytest.mark.parametrize("name", FIXTURES)
def test_fixtures_against_the_reference(name):
    from raft_b200 import solver
    z = fixture(name)
    sort = "dof" if int(z["sort"]) == 0 else "ascending"
    r = solver.solve_eigen(z["M_tot"], z["C_tot"], sort=sort)
    assert r["info"] & ~solver.EIG_COMPLEX == 0, r["info"]
    lam_ref = np.asarray(z["eigenvals"])[z["order"]]
    lam = r["lam"]
    # the order is the reference's; inside a cluster (the degenerate surge/sway pairs) a permutation is allowed, and there
    # check_against compares eigenvalues to the tolerance and the spanned subspaces
    e_lam, res, mode = check_against(lam, r["modes"], z["M_tot"], z["C_tot"], lam_ref, z["modes"])
    print("eigen %s: n=%d  |dlam|/max|lam| %.2e  residual %.2e  mode angle / bound %.2e  kernel %s"
          % (name, len(lam), e_lam, res, mode, solver.last_dispatch()["kernel"]))


@gpu
@pytest.mark.parametrize("n,kernel", [(6, "eig-small"), (12, "eig-small"), (144, "eig-cta-smem"), (150, "eig-cta-smem"), (300, "eig-cta-slab")])
def test_seeded_systems_against_numpy(n, kernel):
    from raft_b200 import solver
    nS = 64 if n <= 12 else (8 if n < 300 else 3)
    M, K = seeded(n, nS, seed=n)
    r = solver.solve_eigen(M, K, sort="ascending")
    assert solver.last_dispatch()["family"] == "eigen" and solver.last_dispatch()["kernel"] == kernel
    worst = [0.0, 0.0]
    for s in range(nS):
        w, v = np.linalg.eig(np.linalg.solve(M[s], K[s]))
        o = np.argsort(w)
        e, res, _ = check_against(r["lam"][s], r["modes"][s], M[s], K[s], w[o], v[:, o])
        worst = [max(worst[0], e), max(worst[1], res)]
    assert np.all(r["info"] & ~solver.EIG_COMPLEX == 0)
    print("eigen seeded n=%d (%s): |dlam|/max|lam| %.2e residual %.2e" % (n, kernel, *worst))


@gpu
@pytest.mark.parametrize("n", [8, 40])
def test_complex_conjugate_pairs(n):
    from raft_b200 import solver
    rng = np.random.default_rng(100 + n)
    M = np.eye(n) + 0.1 * np.diag(rng.uniform(size=n))
    K = rng.normal(size=(n, n)) * 5.0 + np.eye(n) * 3.0               # nonsymmetric: complex-conjugate pairs
    w, v = np.linalg.eig(np.linalg.solve(M, K))
    assert np.iscomplexobj(w) and np.any(w.imag != 0)
    o = np.argsort(w)                                                # lexicographic: the pair's negative imaginary part first
    r = solver.solve_eigen(M, K, sort="ascending")
    assert r["lam"].dtype == np.complex128 and r["info"] & solver.EIG_COMPLEX
    np.testing.assert_allclose(r["lam"], w[o], rtol=0, atol=1e-12 * np.abs(w).max())
    assert np.array_equal(np.sign(r["lam"].imag), np.sign(w[o].imag))
    for j in range(n):                                               # vectors up to a unit phase, and the phase rule
        a, b = r["modes"][:, j], v[:, o[j]]
        ph = np.vdot(a, b) / abs(np.vdot(a, b))
        assert np.abs(a * ph - b).max() < 1e-9, j
        assert abs(np.linalg.norm(a) - 1) < 1e-14
        if w[o[j]].imag != 0:
            assert a[np.argmax(np.abs(a))].imag == 0.0


@gpu
@pytest.mark.parametrize("n", [6, 30, 200])
def test_batch_isolation_and_entry_points(n):
    import torch
    from raft_b200 import _lib, solver
    nS = 1000 if n < 100 else 40
    M, K = seeded(n, nS, seed=7 * n)
    one = solver.solve_eigen(M[17:18], K[17:18])
    full = solver.solve_eigen(M, K)
    assert np.array_equal(one["lam"][0], full["lam"][17]) and np.array_equal(one["modes"][0], full["modes"][17])
    # the device entry at several workspace sizes, bit-identical to the host entry
    dev = torch.device("cuda")
    Mt, Kt = torch.from_numpy(M).to(dev), torch.from_numpy(K).to(dev)
    need = solver.eigen_workspace_bytes(nS, n)
    slab = solver.eigen_workspace_bytes(1, n)
    for wsb in sorted({need, slab, 3 * slab}) if need else [0]:
        lam = torch.empty([nS, n], dtype=torch.complex128, device=dev)
        V = torch.empty([nS, n, n], dtype=torch.complex128, device=dev)
        info = torch.empty(nS, dtype=torch.int32, device=dev)
        ws = torch.empty(max(wsb, 1), dtype=torch.uint8, device=dev)
        e = solver._eigen_struct(nS, n, "dof", Mt.data_ptr(), Kt.data_ptr(), lam.data_ptr(), V.data_ptr(), info.data_ptr())
        _lib.check(_lib.lib.raftk_eigen_dev(C.byref(e), ws.data_ptr(), wsb, torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        lam_h = lam.cpu().numpy()
        assert np.array_equal(lam_h.real if full["lam"].dtype == np.float64 else lam_h, full["lam"]), wsb
        assert np.array_equal(V.cpu().numpy().real if full["modes"].dtype == np.float64 else V.cpu().numpy(), full["modes"]), wsb
        assert np.array_equal(info.cpu().numpy(), full["info"])
    if need:
        e = solver._eigen_struct(nS, n, "dof", Mt.data_ptr(), Kt.data_ptr(), lam.data_ptr(), V.data_ptr(), info.data_ptr())
        assert _lib.lib.raftk_eigen_dev(C.byref(e), ws.data_ptr(), slab - 8, None) == -1
        assert "less than one slab" in _lib.lib.raftk_last_error().decode()


@gpu
def test_flags_stay_in_their_row():
    from raft_b200 import solver
    n, nS = 12, 40
    M, K = seeded(n, nS, seed=3)
    M[5] = 5.0                                                        # exactly singular mass, diagonal above 1
    M[9, 2, 2] = 0.5                                                  # a diagonal below 1
    K[13] = np.eye(n) * 1e3                                           # an indefinite stiffness with diagonal above 1:
    K[13, 0, 1] = K[13, 1, 0] = 5e3                                   # one negative eigenvalue
    r = solver.solve_eigen(M, K, sort="dof")
    base = solver.solve_eigen(np.delete(M, [5, 9, 13], 0), np.delete(K, [5, 9, 13], 0), sort="dof")
    assert r["info"][5] & solver.EIG_SINGULAR and np.all(np.isnan(r["lam"][5]))
    assert r["info"][9] & solver.EIG_SMALL_DIAG
    assert r["info"][13] & solver.EIG_NONPOSITIVE
    rest = np.delete(np.arange(nS), [5, 9, 13])
    assert np.all(r["info"][rest] & ~solver.EIG_COMPLEX == 0) and np.array_equal(r["lam"][rest], base["lam"])
    assert np.array_equal(r["info"][rest], base["info"])
    with pytest.raises(np.linalg.LinAlgError):
        solver.eigen_fns_modes(M[5], K[5], "dof")
    with pytest.raises(RuntimeError, match="small or negative diagonals"):
        solver.eigen_fns_modes(M[9], K[9], "dof")
    with pytest.raises(RuntimeError, match="zero or negative system eigenvalues"):
        solver.eigen_fns_modes(M[13], K[13], "dof")


@gpu
def test_device_session_eigen_equals_solve_eigen():
    import torch
    from conftest import load_golden
    from raft_b200 import solver
    _, P = load_golden("cfg2_VolturnUS-S_nw64")
    Ps = []
    for s in range(5):
        Q = {k: (np.array(v) if isinstance(v, np.ndarray) else v) for k, v in P.items()}
        Q["M0"] = Q["M0"] * (1 + 0.05 * s)
        Q["C0"] = Q["C0"] * (1 + 0.03 * s)
        Ps.append(Q)
    cases = solver.CaseTable(dict(Hs=[6.0], Tp=[12.0], gamma=[0.0], beta_deg=[0.0], spec=np.zeros(1, dtype=np.int32)))
    sess = solver.DeviceSession(solver.DesignBatch(Ps), cases)
    A0 = np.diag([1e6, 1e6, 2e6, 1e9, 1e9, 1e8])
    yaw = np.linspace(1e7, 5e7, 5)
    r = sess.eigen(A0=A0, yawstiff=yaw)
    torch.cuda.synchronize()
    M = np.array([q["M0"] + A0 for q in Ps])
    K = np.array([q["C0"] for q in Ps])
    K[:, 5, 5] += yaw
    h = solver.solve_eigen(M, K)
    assert np.array_equal(r["lam"].cpu().numpy().real, h["lam"]) and np.array_equal(r["modes"].cpu().numpy().real, h["modes"])
    assert np.array_equal(r["info"].cpu().numpy(), h["info"])


@gpu
def test_general_batch_session_eigen_equals_solve_eigen():
    import torch
    from conftest import load_golden
    from raft_b200 import solver
    z, P = load_golden("flex_VolturnUS-S-flexible")
    designs = []
    for s in range(3):
        designs.append(dict(P=P, M=z["gen_M"] * (1 + 0.02 * s), B=z["gen_B"], Cm=z["gen_C"] * (1 + 0.01 * s)))
    cases = solver.CaseTable(dict(Hs=[6.0], Tp=[12.0], gamma=[0.0], beta_deg=[0.0], spec=np.zeros(1, dtype=np.int32)))
    sess = solver.GeneralBatchSession(designs, cases)
    A0 = np.diag([1e6, 1e6, 2e6, 1e9, 1e9, 1e8])
    r = sess.eigen(A0=A0, yawstiff=2e7)
    torch.cuda.synchronize()
    n = designs[0]["M"].shape[0]
    M = np.array([d["M"] for d in designs])
    M[:, :6, :6] += A0
    K = np.array([d["Cm"] for d in designs])
    K[:, 5, 5] += 2e7
    h = solver.solve_eigen(M, K, sort="ascending")
    lam = r["lam"].cpu().numpy()
    assert np.array_equal(lam.real if h["lam"].dtype == np.float64 else lam, h["lam"]) and lam.shape == (3, n)
    assert solver.last_dispatch()["kernel"] == "eig-cta-smem"


@gpu
@pytest.mark.parametrize("name", ["test_OC3spar", "test_VolturnUS-S"])
def test_fowt_solve_eigen_mirror(name):
    from raft_b200.fowt import FOWT
    z = fixture(name[5:])
    design = json.load(open(os.path.join(GOLDEN, "designs.json")))[name]
    mats = {k: z["fowt_" + k] for k in ("M_struc", "C_struc", "C_hydro", "C_moor", "C_elast", "A_BEM")}
    f = FOWT(design, np.array([0.05, 0.1]), depth=float(design["site"]["water_depth"]), matrices=mats)
    f.A_hydro_morison = z["fowt_A_hydro_morison"]
    assert f.yawstiff == z["fowt_yawstiff"]
    fns, modes = f.solveEigen()
    _check_mirror(fns, modes, z)
    with pytest.raises(NotImplementedError):
        f.solveEigen(outPath="modes.json")


def _check_mirror(fns, modes, z):
    """the fixture's fns, and its modes column by column, or as a subspace inside a degenerate pair"""
    np.testing.assert_allclose(fns, z["fns"], rtol=1e-9)
    for g in _clusters(np.asarray(z["fns"], dtype=complex), 1e-9 * np.abs(z["fns"]).max()):
        Qa, _ = np.linalg.qr(modes[:, g])
        Qb, _ = np.linalg.qr(z["modes"][:, g])
        assert np.linalg.svd(Qa.conj().T @ Qb, compute_uv=False).min() > 1 - 1e-9, g


@gpu
def test_model_solve_eigen_mirror_farm():
    from raft_b200.model import Model
    z = fixture("farm")
    design = json.load(open(os.path.join(GOLDEN, "designs.json")))["farm_VolturnUS-S_farm_nw48"]
    mats = [dict(M_struc=z["M_blocks"][i], C_struc=z["C_blocks"][i]) for i in range(len(z["M_blocks"]))]
    m = Model(design, matrices=mats, array_stiffness=z["C_array"])
    for f in m.fowtList:
        f.A_hydro_morison = np.zeros([6, 6])
    fns, modes = m.solveEigen()
    assert m.results["eigen"]["frequencies"] is fns and m.results["eigen"]["modes"] is modes
    _check_mirror(fns, modes, z)
    m.fowtList[0].C_struc = m.fowtList[0].C_struc.copy()
    m.fowtList[0].C_struc[2, 2] = -1e9                               # a negative diagonal: the reference's RuntimeError
    with pytest.raises(RuntimeError, match="Diagonal entry 2 of system stiffness matrix"):
        m.solveEigen()
