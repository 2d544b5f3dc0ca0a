#!/usr/bin/env python
"""Generate tests/golden/eigen_<name>.npz: the natural frequencies and mode shapes of the UNMODIFIED reference's
FOWT.solveEigen / Model.solveEigen (raft_fowt.py:1646-1729, raft_model.py:436-547), run under oracle/ref_harness.py.

Each file stores what the reference itself computed: M_tot and C_tot (the arguments of its np.linalg.solve), the raw
eigenvals / eigenvectors of its np.linalg.eig, its output order (``order``: column k of ``modes`` is column order[k] of
``eigenvectors``), ``fns`` and ``modes``, ``sort`` (0 DOF claim, 1 ascending) and ``entry`` (FOWT or Model).  Single-FOWT
systems also store the live FOWT's matrices (``fowt_*``) so that packer.pack_eigen can be checked against M_tot / C_tot.

Cases (turbine and mooring stripped and rh.C_MOOR_DEFAULT on DOFs 0-5 as in make_golden.py, unless said otherwise):
  OC3spar (platform yaw_stiffness), VolturnUS-S, VolturnUS-S-pointInertia, OC4semi-WAMIT (nonzero A_BEM[:, :, 0]);
  the two-FOWT farm and the 24-FOWT farm with make_golden.fixture_farm's seeded SPD array stiffness on model.ms (DOF claim
  over 12 and 144 rows); VolturnUS-S-flexible (150 DOFs, ascending order) with make_golden.fixture_flexible's recipe.

Usage (build container, reference tree present):  python tests/golden/make_golden_eigen.py
"""
import contextlib
import copy
import io
import os
import sys

import numpy as np
import yaml

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg  # noqa: E402
import make_golden_farm24 as mf24  # noqa: E402

rh = mg.rh


@contextlib.contextmanager
def capture():
    """Record the arguments of np.linalg.solve and the results of np.linalg.eig while the reference runs."""
    rec = {}
    solve, eig = np.linalg.solve, np.linalg.eig

    def solve_(a, b):
        rec["M_tot"], rec["C_tot"] = np.array(a), np.array(b)
        return solve(a, b)

    def eig_(a):
        w, v = eig(a)
        rec["eigenvals"], rec["eigenvectors"] = np.array(w), np.array(v)
        return w, v
    np.linalg.solve, np.linalg.eig = solve_, eig_
    try:
        yield rec
    finally:
        np.linalg.solve, np.linalg.eig = solve, eig


def run(obj):
    with capture() as rec, contextlib.redirect_stdout(io.StringIO()):
        fns, modes = obj.solveEigen()
    V = rec["eigenvectors"]
    order = [next(k for k in range(V.shape[1]) if np.array_equal(modes[:, j], V[:, k])) for j in range(modes.shape[1])]
    rec.update(fns=np.array(fns), modes=np.array(modes), order=np.array(order, dtype=np.int32))
    return rec


def save(name, rec, sort, entry, fowt=None):
    out = dict(rec, sort=np.int32(sort), entry=np.array(entry))
    if fowt is not None:
        for k in ("M_struc", "A_hydro_morison", "A_BEM", "C_moor", "C_struc", "C_hydro", "C_elast"):
            a = np.asarray(getattr(fowt, k), dtype=float)
            out["fowt_" + k] = a[:, :, :1] if k == "A_BEM" else a
        out["fowt_yawstiff"] = np.float64(fowt.yawstiff)
    path = os.path.join(mg.OUT, "eigen_%s.npz" % name)
    np.savez_compressed(path, **out)
    lam = rec["eigenvals"]
    print("%-28s n=%3d  fns %.5g .. %.5g Hz  complex %s  %.0f KB" % (name, len(lam), np.min(rec["fns"].real), np.max(rec["fns"].real),
                                                                  bool(np.iscomplexobj(lam)), os.path.getsize(path) / 1024))


def rigid(name, path):
    model = rh.build_model(rh.load_design(path))
    f = model.fowtList[0]
    save(name, run(f), 0, "FOWT", f)


def farm(name, yaml_path, seed=5):
    """make_golden.fixture_farm's recipe: array rows with turbineID = mooringID = 0, array_mooring dropped, model.ms replaced
    by an object whose getCoupledStiffnessA returns the seeded SPD array stiffness, moorMod 0."""
    with open(yaml_path) as f:
        design = yaml.load(f, Loader=yaml.FullLoader)
    for k in ("turbine", "turbines", "mooring", "array_mooring"):
        design.pop(k, None)
    design["platform"]["potSecOrder"] = 0
    ks = design["array"]["keys"]
    for row in design["array"]["data"]:
        row[ks.index("turbineID")] = 0
        row[ks.index("mooringID")] = 0
    model = rh.build_model(design)
    n = model.nDOF
    rng = np.random.default_rng(seed)
    A = rng.normal(size=(n, n)) * 2e4
    C_arr = A @ A.T / n + np.diag([5e4] * n)

    class _MS:
        def getCoupledStiffnessA(self, lines_only=True):
            return C_arr
    model.ms, model.moorMod = _MS(), 0
    rec = run(model)
    rec["C_array"] = C_arr
    # each FOWT's diagonal blocks as Model.solveEigen sums them (raft_model.py:462-463), for a mirror Model built on them
    rec["M_blocks"] = np.array([fw.M_struc + fw.A_hydro_morison + fw.A_BEM[:, :, 0] for fw in model.fowtList])
    rec["C_blocks"] = np.array([fw.C_struc + fw.C_hydro + fw.C_moor + fw.C_elast for fw in model.fowtList])
    save(name, rec, 0, "Model")


def farm24():
    src = os.path.join(mg.REF, "designs", "VolturnUS-S_farm.yaml")
    with open(src) as f:
        design = yaml.load(f, Loader=yaml.FullLoader)
    ks = design["array"]["keys"]
    proto = list(design["array"]["data"][1])
    data = []
    for u in range(mf24.ROWS * mf24.COLS):
        row = list(proto)
        row[ks.index("x_location")] = mf24.SPACING * (u % mf24.COLS)
        row[ks.index("y_location")] = mf24.SPACING * (u // mf24.COLS)
        row[ks.index("heading_adjust")] = 180 if u % 5 == 0 else 0
        data.append(row)
    design["array"]["data"] = data
    import tempfile
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "farm24.yaml")
        with open(path, "w") as f:
            yaml.dump(design, f)
        farm("farm24", path)


def flexible(name, yaml_path):
    """make_golden.fixture_flexible's recipe: turbine kept (the tower is a flexible member), mooring stripped,
    rh.C_MOOR_DEFAULT on the rigid-body DOFs 0-5 of the 150-DOF system."""
    raft = rh.load_reference()
    design = rh.load_design(yaml_path, strip=False)
    design.pop("mooring", None)
    design["platform"]["potSecOrder"] = 0
    with contextlib.redirect_stdout(io.StringIO()):
        model = raft.Model(copy.deepcopy(design))
        fowt = model.fowtList[0]
        fowt.setPosition(np.zeros(fowt.nDOF))
        fowt.calcStatics()
        fowt.calcTurbineConstants(rh.make_case(), ptfm_pitch=0)
        fowt.calcHydroConstants()
    Cmoor = np.zeros([fowt.nDOF, fowt.nDOF])
    Cmoor[:6, :6] = rh.C_MOOR_DEFAULT
    fowt.C_moor = Cmoor
    save(name, run(fowt), 1, "FOWT", fowt)


def main():
    td = os.path.join(mg.REF, "tests", "test_data")
    rigid("OC3spar", os.path.join(td, "OC3spar.yaml"))
    rigid("VolturnUS-S", os.path.join(td, "VolturnUS-S.yaml"))
    rigid("VolturnUS-S-pointInertia", os.path.join(td, "VolturnUS-S-pointInertia.yaml"))
    rigid("OC4semi-WAMIT", os.path.join(mg.REF, "examples", "OC4semi-WAMIT_Coefs.yaml"))
    farm("farm", os.path.join(mg.REF, "designs", "VolturnUS-S_farm.yaml"))
    farm24()
    flexible("VolturnUS-S-flexible", os.path.join(td, "VolturnUS-S-flexible.yaml"))


if __name__ == "__main__":
    main()
