#!/usr/bin/env python
"""Compare the SASS of two builds of the library, kernel by kernel (profiles/sm90a_farm_peer_sass.txt,
profiles/sm90a_farm_ragged_sass.txt, profiles/sm90a_farm_one_path_sass.txt).

The two inputs are `cuobjdump -sass` listings of raft_b200/csrc/raftk.cu compiled for sm_90a, one before and one after the
farm kernels gained a template flag (--flag PEER: the peer-store instantiations; --flag RAG: the ragged-batch ones).
Kernels are matched by demangled name and template arguments, not by parameter types (instantiations without the flag
spell their parameter struct through the FarmArg alias); a kernel that gained the flag as its last template argument is
matched through its flag = false instantiation.  --drop PEER compares across the removal of a template argument
instead: on the before side the farm kernels' PEER argument (the third) is dropped, and its true instantiations are listed
as found before only.  Instruction text is compared with addresses and encodings dropped.  Each matched farm kernel, and any kernel that differs, prints SAME or DIFF with its instruction counts; kernels
found on one side only are listed at the end.

Usage:  python tools/farm_sass_diff.py [--flag PEER|RAG | --drop PEER] BEFORE.sass AFTER.sass
"""
import argparse
import re
import subprocess

FLAG_KERNELS = {"PEER": ("k_farm_response", "k_farm_rows"), "RAG": ("k_farm_response", "k_farm_rows", "k_farm_response_global")}
PEER_KERNELS = FLAG_KERNELS["PEER"]
DROP_ARGS = {"PEER": (2, PEER_KERNELS)}        # position of the removed argument, kernels that had it
SHOWN = PEER_KERNELS + ("k_farm_response_global", "k_farm_channels", "k_farm_channels_ragged", "k_farm_publish")
# with --drop PEER: the publish kernel that was kept took the name of the one that was removed
DROP_RENAMES = {"PEER": {"k_farm_publish<>": "k_farm_publish<> (uniform)", "k_farm_publish_flat<>": "k_farm_publish<>"}}


def functions(path):
    """mangled name -> list of instruction strings of every function in a cuobjdump -sass listing."""
    out, cur = {}, None
    with open(path) as fh:
        for line in fh:
            m = re.match(r"\s*Function : (\S+)", line)
            if m:
                cur = m.group(1)
                out[cur] = []
                continue
            m = re.search(r"/\*[0-9a-f]{4,6}\*/\s+(.*?)\s*;", line)
            if cur and m:
                out[cur].append(m.group(1))
    return out


def demangle(names):
    res = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True)
    return dict(zip(names, res.stdout.splitlines()))


def key(demangled, after, flagged=PEER_KERNELS, drop=None):
    """Kernel name and template arguments; on the after side a trailing flag argument, or with `drop` (position, kernels)
    the dropped argument of the before side: (key, that argument is true)."""
    m = re.match(r"(?:void )?(\w+)(?:<(.*?)>)?\(", demangled)
    if not m:
        return demangled, False
    name, targs = m.group(1), [a.strip() for a in (m.group(2) or "").split(",") if a.strip()]
    peer = False
    if drop:
        if not after and name in drop[1]:
            peer = targs.pop(drop[0]) == "true"
    elif after and name in flagged:
        peer = targs.pop() == "true"
    return "%s<%s>" % (name, ", ".join(targs)), peer


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--flag", choices=sorted(FLAG_KERNELS), default="PEER")
    ap.add_argument("--drop", choices=sorted(DROP_ARGS))
    ap.add_argument("before")
    ap.add_argument("after")
    args = ap.parse_args()
    before, after = functions(args.before), functions(args.after)
    dm = demangle(sorted(set(before) | set(after)))
    drop = DROP_ARGS.get(args.drop)
    b_by_key, a_by_key, peer_only, dropped = {}, {}, [], []
    for n in before:
        k, peer = key(dm[n], False, drop=drop)
        if peer:
            dropped.append(k + " " + args.drop)
        else:
            b_by_key[DROP_RENAMES.get(args.drop, {}).get(k, k)] = n
    for n in after:
        k, peer = key(dm[n], True, FLAG_KERNELS[args.flag], drop)
        if peer:
            peer_only.append(k + " " + args.flag)
        else:
            a_by_key[k] = n
    same = diff = 0
    for k in sorted(set(b_by_key) & set(a_by_key)):
        b, a = before[b_by_key[k]], after[a_by_key[k]]
        ok = b == a
        same, diff = same + ok, diff + (not ok)
        if not ok or any(k.startswith(p + "<") for p in SHOWN):
            print("%-4s %6d %6d  %s" % ("SAME" if ok else "DIFF", len(b), len(a), k))
    print("matched kernels: %d identical, %d different" % (same, diff))
    print("only before: %s" % sorted((set(b_by_key) - set(a_by_key)) | set(dropped)))
    print("only after: %s" % sorted((set(a_by_key) - set(b_by_key)) | set(peer_only)))


if __name__ == "__main__":
    main()
