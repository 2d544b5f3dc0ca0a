#!/usr/bin/env python
"""Generate tests/golden/farm24_VolturnUS-S_farm_nw48.npz: a 24-FOWT array (4 x 6 grid, 1600 m spacing, every fifth unit
turned by 180 deg) run by the UNMODIFIED reference with the recipe of make_golden.fixture_farm (seeded SPD array stiffness
through model.ms.getCoupledStiffnessA, moorMod 0), two cases, 48 bins.  Its 144-DOF system does not fit in one CTA's shared
memory, so it pins the global-memory farm kernel to the reference.  The design sections go into the .npz itself
(``design_json``) rather than designs.json.

Usage (build container, reference tree present):  python tests/golden/make_golden_farm24.py
"""
import json
import os
import sys
import tempfile

import numpy as np
import yaml

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg  # noqa: E402

NAME = "farm24_VolturnUS-S_farm_nw48"
ROWS, COLS, SPACING = 4, 6, 1600.0


def main():
    src = os.path.join(mg.REF, "designs", "VolturnUS-S_farm.yaml")
    with open(src) as f:
        design = yaml.load(f, Loader=yaml.FullLoader)
    ks = design["array"]["keys"]
    proto = list(design["array"]["data"][1])
    data = []
    for u in range(ROWS * COLS):
        row = list(proto)
        row[ks.index("x_location")] = SPACING * (u % COLS)
        row[ks.index("y_location")] = SPACING * (u // COLS)
        row[ks.index("heading_adjust")] = 180 if u % 5 == 0 else 0
        data.append(row)
    design["array"]["data"] = data
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "farm24.yaml")
        with open(path, "w") as f:
            yaml.dump(design, f)
        mg.fixture_farm(NAME, path, nw=48, max_freq=0.1024, cases=[(6.0, 12.0, 0.0), (3.5, 9.0, 40.0)])
    out = os.path.join(mg.OUT, NAME + ".npz")
    z = dict(np.load(out))
    z["design_json"] = np.array(json.dumps(mg.DESIGNS[NAME]))
    np.savez_compressed(out, **z)
    print("%s: %.0f KB" % (out, os.path.getsize(out) / 1024))


if __name__ == "__main__":
    main()
