"""C-ABI checks that need no GPU: the library loads, exports every symbol include/raftk.h declares,
struct layouts agree with the header, and argument validation returns error codes (never throws)."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import ROOT, load_golden

HEADER = os.path.join(ROOT, "include", "raftk.h")


def header_functions():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(raftk_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_declared_symbols_and_version():
    """Every function include/raftk.h declares is exported and listed in _lib.SYMBOLS, and the library reports the header's
    RAFTK_VERSION (132 since raftk_last_dispatch was added)."""
    from raft_b200 import _lib
    declared = header_functions()
    assert len(declared) >= 15
    assert sorted(_lib.SYMBOLS) == declared
    for name in declared:
        assert hasattr(_lib.lib, name), name
    assert _lib.lib.raftk_version() == 132


def test_struct_layout_matches_header(tmp_path):
    """Compile a tiny C program against the header and compare sizeof/offsetof with the ctypes mirrors."""
    from raft_b200 import _lib
    prog = tmp_path / "layout.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "raftk.h"\nint main(){printf("%zu %zu %zu %zu %zu %zu %zu\\n",'
                    'sizeof(raftk_designs), offsetof(raftk_designs, X_BEM), sizeof(raftk_cases), offsetof(raftk_cases, zeta),'
                    'sizeof(raftk_solve_opts), sizeof(raftk_outputs), offsetof(raftk_designs, node_in_p1_w));'
                    'printf("%zu %zu %zu %zu %zu %zu\\n", sizeof(raftk_family_member), offsetof(raftk_family_member, Ca_End), sizeof(raftk_family),'
                    'offsetof(raftk_family, members), sizeof(raftk_family_tables), offsetof(raftk_family_tables, max_nodes));'
                    'printf("%zu %zu %zu %zu\\n", sizeof(raftk_dispatch), offsetof(raftk_dispatch, f0_global), offsetof(raftk_dispatch, chunks),'
                    'offsetof(raftk_dispatch, trains));return 0;}\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    want = [C.sizeof(_lib.RaftkDesigns), _lib.RaftkDesigns.X_BEM.offset, C.sizeof(_lib.RaftkCases), _lib.RaftkCases.zeta.offset,
            C.sizeof(_lib.RaftkSolveOpts), C.sizeof(_lib.RaftkOutputs), _lib.RaftkDesigns.node_in_p1_w.offset,
            C.sizeof(_lib.RaftkFamilyMember), _lib.RaftkFamilyMember.Ca_End.offset, C.sizeof(_lib.RaftkFamily), _lib.RaftkFamily.members.offset,
            C.sizeof(_lib.RaftkFamilyTables), _lib.RaftkFamilyTables.max_nodes.offset,
            C.sizeof(_lib.RaftkDispatch), _lib.RaftkDispatch.f0_global.offset, _lib.RaftkDispatch.chunks.offset, _lib.RaftkDispatch.trains.offset]
    assert got == want


def test_dispatch_record_names_match_header():
    """solver.last_dispatch() names the RAFTK_FAMILY_* / RAFTK_KERNEL_* values of include/raftk.h in order; a call that fails
    before launching anything leaves the record cleared."""
    from raft_b200 import _lib, solver
    src = open(HEADER).read()
    fam = dict((m[0], int(m[1])) for m in re.findall(r"RAFTK_FAMILY_([A-Z0-9_]+)\s*=\s*(\d+)", src))
    ker = dict((m[0], int(m[1])) for m in re.findall(r"RAFTK_KERNEL_([A-Z0-9_]+)\s*=\s*(\d+)", src))
    assert sorted(fam.values()) == list(range(len(solver.DISPATCH_FAMILIES)))
    assert sorted(ker.values()) == list(range(len(solver.DISPATCH_KERNELS)))
    for name, v in fam.items():
        assert solver.DISPATCH_FAMILIES[v] == name.lower().replace("_", "-"), name
    for name, v in ker.items():
        assert solver.DISPATCH_KERNELS[v] == name.lower().replace("_", "-"), name
    assert _lib.lib.raftk_system_solve_host(0, 1, 1, None, None, None) == -1
    rec = solver.last_dispatch()
    assert rec["family"] == "none" and rec["kernel"] == "none" and rec["chunks"] == 0 and not rec["direct_d2h"]
    assert _lib.lib.raftk_last_dispatch(None) == -1


def test_argument_validation_returns_codes():
    from raft_b200 import _lib
    lib = _lib.lib
    d, c, o, out = _lib.RaftkDesigns(), _lib.RaftkCases(), _lib.RaftkSolveOpts(), _lib.RaftkOutputs()
    assert lib.raftk_solve_dynamics_host(C.byref(d), C.byref(c), C.byref(o), C.byref(out)) == -1     # Xi/status missing
    buf = np.zeros(16)
    out.Xi, out.status = buf.ctypes.data, buf.ctypes.data
    assert lib.raftk_solve_dynamics_host(C.byref(d), C.byref(c), C.byref(o), C.byref(out)) == -1     # empty batch
    assert b"empty batch" in lib.raftk_last_error()
    assert lib.raftk_system_solve_host(0, 1, 1, None, None, None) == -1
    with pytest.raises(_lib.RaftkError):
        _lib.check(-1)
    with pytest.raises(ValueError):
        _lib.check(-4)
    assert lib.raftk_workspace_bytes(C.byref(d), 4) == 0


def test_design_batch_and_case_table():
    from raft_b200 import packer, solver
    _, P = load_golden("cfg2_VolturnUS-S_nw64")
    b = solver.DesignBatch([P, P, P])
    assert b.n_designs == 3 and b.n_nodes_total == 3 * 53 and b.max_nodes == 53 and b.max_members == 7
    assert b.arrays["member_offset"].tolist() == [0, 7, 14, 21]
    assert b.arrays["mem_node_start"][7] == 53 and b.arrays["mem_node_start"][-1] == 159
    np.testing.assert_allclose(b.arrays["mem_arm"][:7], P["mem_rA"] - P["prp"])
    s = b.struct(lambda n: b.arrays[n].ctypes.data)
    assert s.n_designs == 3 and s.nw == 64 and s.A_w is None and s.n_bem_head == 0
    cases = packer.pack_cases([dict(wave_spectrum="JONSWAP", wave_height=2, wave_period=9, wave_heading=10),
                               dict(wave_spectrum=["unit"], wave_height=[1], wave_period=[8], wave_heading=[-30], wave_gamma=[3.3])])
    ct = solver.CaseTable(cases)
    assert ct.n_cases == 2 and ct.arrays["spec"].tolist() == [0, 1] and ct.arrays["gamma"].tolist() == [0.0, 3.3]
    with pytest.raises(ValueError):
        packer.pack_cases([dict(wave_spectrum="bogus", wave_height=2, wave_period=9)])
    _, Pb = load_golden("cfg3_OC4semi-WAMIT_nw128")
    bb = solver.DesignBatch(Pb)
    assert bb.n_bem_head == 37 and bb.arrays["X_BEM"].shape == (1, 37, 6, 128) and bb.arrays["A_w"].shape == (1, 36, 128)
    with pytest.raises(ValueError):
        solver.DesignBatch([P, Pb])


def test_no_oracle_on_product_path():
    """The product package must not import, link or call anything under oracle/ (no CPU fallback)."""
    pkg = os.path.join(ROOT, "raft_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".h", ".cpp")):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"(import\s+oracle|from\s+oracle|raft_oracle|oracle\.|oracle/)", src), os.path.join(dirpath, f)
