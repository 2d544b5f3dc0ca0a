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


# (design, nw, designs per batch) -> (raftk_solve_workspace_bytes, raftk_workspace_bytes) for 1, 3, 64 and 200 cases.  The
# designs are regridded to nw bins up to 0.4 Hz (cfg3 without its BEM tables, which the sizes do not depend on).  The batches
# stay clear of 114-132 units: there k_rao_fused2's exchange rows depend on the device's SM count (132 without a device).
WORKSPACE_BYTES = {
    ("cfg2", 64, 1): [(8704, 115200), (25856, 237056), (547328, 3953664), (1710592, 12239872)],
    ("cfg2", 64, 3): [(25856, 344576), (77056, 708096), (1641984, 11795456), (5131264, 36514816)],
    ("cfg2", 151, 1): [(17152, 272384), (50944, 559872), (1081856, 9328384), (3380992, 28878848)],
    ("cfg2", 151, 3): [(50944, 813312), (152320, 1671168), (3245568, 27830016), (10142464, 86152448)],
    ("cfg2", 201, 1): [(83200, 362240), (234240, 744960), (4837888, 12417024), (10136832, 38441216)],
    ("cfg2", 201, 3): [(247808, 1082880), (700672, 2224384), (9744896, 37045248), (30409472, 114679808)],
    ("cfg2", 333, 1): [(34560, 600064), (103424, 1234176), (2200064, 20571648), (6875392, 63686144)],
    ("cfg2", 333, 3): [(103424, 1793536), (309504, 3684864), (6600192, 61373440), (20625664, 189991680)],
    ("cfg2", 501, 1): [(155136, 902144), (450048, 1856000), (9445888, 30949888), (24536832, 95815680)],
    ("cfg2", 501, 3): [(463616, 2697728), (1348352, 5543424), (23568896, 92336384), (73609472, 285842944)],
    ("cfg2", 601, 1): [(60416, 1082112), (180736, 2226688), (3846656, 37127424), (12020992, 114940416)],
    ("cfg2", 601, 3): [(180736, 3236352), (541184, 6650112), (11539968, 110766848), (36062464, 342897408)],
    ("cfg2", 1024, 1): [(280320, 1843200), (826368, 3792896), (17479168, 63258624), (49640704, 195837952)],
    ("cfg2", 1024, 3): [(839936, 5513216), (2477824, 11329536), (47668736, 188727296), (148921344, 584237056)],
    ("cfg1", 64, 1): [(7680, 59904), (22528, 126464), (478208, 2156544), (1494528, 6682624)],
    ("cfg1", 64, 3): [(22528, 178688), (67328, 376320), (1434624, 6404096), (4483328, 19843072)],
    ("cfg1", 151, 1): [(16128, 141824), (47616, 299008), (1012736, 5088256), (3164928, 15767040)],
    ("cfg1", 151, 3): [(47616, 422144), (142592, 888576), (3038208, 15109888), (9494528, 46817536)],
    ("cfg1", 201, 1): [(43776, 188672), (122880, 397568), (2537984, 6772992), (5414912, 20987904)],
    ("cfg1", 201, 3): [(129536, 561664), (367360, 1182208), (5204736, 20112896), (16243968, 62319872)],
    ("cfg1", 333, 1): [(33536, 312320), (100096, 658688), (2130944, 11220992), (6659328, 34770944)],
    ("cfg1", 333, 3): [(100096, 930304), (299776, 1958656), (6392832, 33321472), (19977728, 103246336)],
    ("cfg1", 501, 1): [(82176, 469504), (237824, 990464), (4995584, 16881920), (13094912, 52312832)],
    ("cfg1", 501, 3): [(244480, 1399296), (712448, 2946304), (12577536, 50132224), (39283968, 155334400)],
    ("cfg1", 601, 1): [(59392, 562944), (177408, 1188096), (3777536, 20251392), (11804928, 62754304)],
    ("cfg1", 601, 3): [(177408, 1678336), (531456, 3534336), (11332608, 60138496), (35414528, 186339072)],
    ("cfg1", 1024, 1): [(148736, 958464), (438528, 2023424), (9280000, 34504704), (26483456, 106921984)],
    ("cfg1", 1024, 3): [(445184, 2859008), (1314816, 6021120), (25430784, 102465536), (79450112, 317489152)],
    ("cfg3", 64, 1): [(7680, 59904), (22528, 126464), (478208, 2156544), (1494528, 6682624)],
    ("cfg3", 64, 3): [(22528, 178688), (67328, 376320), (1434624, 6404096), (4483328, 19843072)],
    ("cfg3", 151, 1): [(16128, 141824), (47616, 299008), (1012736, 5088256), (3164928, 15767040)],
    ("cfg3", 151, 3): [(47616, 422144), (142592, 888576), (3038208, 15109888), (9494528, 46817536)],
    ("cfg3", 201, 1): [(54272, 188672), (152576, 397568), (3156224, 6772992), (7345152, 20987904)],
    ("cfg3", 201, 3): [(160512, 561664), (456192, 1182208), (7059200, 20112896), (22034688, 62319872)],
    ("cfg3", 333, 1): [(33536, 312320), (100096, 658688), (2130944, 11220992), (6659328, 34770944)],
    ("cfg3", 333, 3): [(100096, 930304), (299776, 1958656), (6392832, 33321472), (19977728, 103246336)],
    ("cfg3", 501, 1): [(107008, 469504), (310784, 990464), (6535424, 16881920), (17905152, 52312832)],
    ("cfg3", 501, 3): [(318720, 1399296), (931072, 2946304), (17196800, 50132224), (53714688, 155334400)],
    ("cfg3", 601, 1): [(59392, 562944), (177408, 1188096), (3777536, 20251392), (11804928, 62754304)],
    ("cfg3", 601, 3): [(177408, 1678336), (531456, 3534336), (11332608, 60138496), (35414528, 186339072)],
    ("cfg3", 1024, 1): [(198656, 958464), (586752, 2023424), (12426496, 34504704), (36314624, 106921984)],
    ("cfg3", 1024, 3): [(594688, 2859008), (1759232, 6021120), (34870016, 102465536), (108943360, 317489152)],
}
SIZE_FIXTURES = dict(cfg2="cfg2_VolturnUS-S_nw64", cfg1="cfg1_OC3spar", cfg3="cfg3_OC4semi-WAMIT_nw128")


def test_workspace_size_queries(monkeypatch):
    """The workspace size queries answer without a device and give pinned byte counts: the solve's plan (k_rao_fused2,
    k_rao_fused<T> or the v1 tables) across both sides of every bin-range switch, one and three designs.  With RAFTK_FORCE_V1
    the solve asks for the v1 tables' workspace."""
    from raft_b200 import _lib, grid, solver
    lib = _lib.lib
    packed = {k: {n: v for n, v in load_golden(f)[1].items() if n not in ("A_w", "B_w", "X_BEM")} for k, f in SIZE_FIXTURES.items()}
    monkeypatch.delenv("RAFTK_FORCE_V1", raising=False)
    got, forced = {}, {}
    for (name, nw, nd) in WORKSPACE_BYTES:
        s = solver.DesignBatch([grid.regrid(packed[name], nw, 0.4)] * nd).struct(lambda n: None)
        got[name, nw, nd] = [(lib.raftk_solve_workspace_bytes(C.byref(s), nc), lib.raftk_workspace_bytes(C.byref(s), nc)) for nc in (1, 3, 64, 200)]
        monkeypatch.setenv("RAFTK_FORCE_V1", "1")
        forced[name, nw, nd] = [lib.raftk_solve_workspace_bytes(C.byref(s), nc) for nc in (1, 3, 64, 200)]
        monkeypatch.delenv("RAFTK_FORCE_V1")
    assert got == WORKSPACE_BYTES
    assert forced == {k: [t[1] for t in v] for k, v in WORKSPACE_BYTES.items()}


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
