#!/bin/bash
# A/B of k_rao_fused2's exchange: a build of the parent commit (cluster exchange only) against this tree (grid exchange
# picked for cfg2), alternated three times on cfg2, dumps compared bit for bit, then the sweep shard alternated twice.
# usage: tools/fused2_xchg_ab.sh PARENT_LIB OUT_DIR   (the tree's own library is raft_b200/csrc/libraftk.so; the bench
# lines and output dumps go to OUT_DIR)
cd "$(dirname "$0")/.."
old=$(realpath "$1")
out=${2:?usage: tools/fused2_xchg_ab.sh PARENT_LIB OUT_DIR}
mkdir -p "$out"
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv,noheader
ms() { python -c "import json,sys; d=json.loads(open(sys.argv[1]).read().strip().splitlines()[-1]); print('ms_per_step %.4f  solves/s %.4g  sm_mhz %s' % (d['ms_per_step'], d['value'], d.get('clocks', {}).get('sm_mhz')))" $1; }
args="--steps 50 --warmup 5 --no-cpu-baseline --no-extras --no-parity --no-e2e"
for i in 1 2 3; do
  RAFTK_LIB=$old python bench.py $args --dump-outputs $out/old$i > $out/old$i.json 2>$out/old$i.err; echo "$i old (parent, cluster)  $(ms $out/old$i.json)"
  python bench.py $args --dump-outputs $out/new$i > $out/new$i.json 2>$out/new$i.err; echo "$i new (grid)              $(ms $out/new$i.json)"
done
RAFTK_FUSED2_XCHG=cluster python bench.py $args > $out/newc.json 2>$out/newc.err; echo "new, RAFTK_FUSED2_XCHG=cluster $(ms $out/newc.json)"
python - $out <<'EOF'
import glob, os, sys
import numpy as np
d = sys.argv[1]
for i in (1, 2, 3):
    for f in sorted(glob.glob(os.path.join(d, "old%d" % i, "*.npy"))):
        g = os.path.join(d, "new%d" % i, os.path.basename(f))
        print("dump %d %-14s bit-identical %s" % (i, os.path.basename(f), np.array_equal(np.load(f), np.load(g))))
EOF
sargs="--workload sweep --steps 20 --warmup 3 --no-cpu-baseline --no-extras --no-parity --no-e2e"
for i in 1 2; do
  RAFTK_LIB=$old python bench.py $sargs > $out/sold$i.json 2>$out/sold$i.err; echo "sweep $i old $(ms $out/sold$i.json)"
  python bench.py $sargs > $out/snew$i.json 2>$out/snew$i.err; echo "sweep $i new $(ms $out/snew$i.json)"
done
