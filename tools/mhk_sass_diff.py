"""Compare the rotor-free instantiations of the rigid solvers between two builds of libraftk.so (cuobjdump -sass dumps):
k_rao_fused2<GRID, OP> against k_rao_fused2<GRID, OP, false>, k_rao_fused<T> against k_rao_fused<T, false>, k_drag_solve with
itself.  Reports, per kernel, whether the instructions are identical, and otherwise how many lines differ only in an
immediate (the kernel-parameter offsets: raftk_designs.rot_* added 32 bytes to DesignsDev, so every later parameter moved).

    cuobjdump -sass parent/libraftk.so > a.sass; cuobjdump -sass raft_b200/csrc/libraftk.so > b.sass
    python tools/mhk_sass_diff.py a.sass b.sass
"""
import re
import sys


def funcs(path):
    out, cur = {}, None
    for line in open(path):
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            cur = m.group(1)
            out[cur] = []
        elif cur and re.search(r"/\*[0-9a-f]{4,}\*/", line):
            out[cur].append(re.sub(r"/\*[0-9a-f]{4,}\*/", "", line).split(";")[0].strip())
    return out


FP = "10DesignsDev8CasesDev11FusedParams"
PAIRS = [("_Z12k_rao_fused2ILb%dELb%dEEv%s" % (g, o, FP), "_Z12k_rao_fused2ILb%dELb%dELb0EEv%s" % (g, o, FP)) for g in (0, 1) for o in (0, 1)]
PAIRS += [("_Z11k_rao_fusedILi%dEEv%s" % (t, FP), "_Z11k_rao_fusedILi%dELb0EEv%s" % (t, FP)) for t in (128, 256)]
PAIRS += [("_Z12k_drag_solve10DesignsDev8CasesDev4Work11SolveParams",) * 2]


def main(a_path, b_path):
    a, b = funcs(a_path), funcs(b_path)
    mask = lambda s: re.sub(r"0x[0-9a-f]+", "#", s)          # noqa: E731
    for pa, pb in PAIRS:
        A, B = a[pa], b[pb]
        if len(A) != len(B):
            print("%-60s DIFFERENT length (%d vs %d)" % (pb, len(A), len(B)))
            continue
        other, shifts, n = 0, set(), 0
        for x, y in zip(A, B):
            if x == y:
                continue
            n += 1
            if mask(x) != mask(y):
                other += 1
                continue
            shifts |= {int(v, 16) - int(u, 16) for u, v in zip(re.findall(r"0x[0-9a-f]+", x), re.findall(r"0x[0-9a-f]+", y)) if u != v}
        print("%-60s %6d instructions, %4d lines differ, %d in opcode or registers, immediate shifts %s" % (pb, len(B), n, other, sorted(shifts)))


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
