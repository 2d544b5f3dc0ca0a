#!/usr/bin/env python
"""Generate tests/golden/tmoor_<name>.npz: mooring line tension statistics from the UNMODIFIED reference's own output code,
Model.analyzeCases (raft_model.py:264-433) with FOWT.saveTurbineOutputs (raft_fowt.py:2355-2399, 2608), run under
oracle/ref_harness.py.

MoorPy is absent here, so the mooring systems are small stand-ins: ``fowt.ms`` / ``model.ms`` return an injected stiffness
and a seeded tension Jacobian from getCoupledStiffness(lines_only=True, tensions=True), seeded mean tensions from
getTensions(), and have ``lineList`` of the right length; ``lines2ss`` is the identity in raft.raft_fowt and raft.raft_model;
Model.solveStatics is a no-op and FOWT.calcStatics runs without the mooring system and then restores the injected C_moor,
so that analyzeCases runs its real solveDynamics, saveTurbineOutputs and array-level tension block (moorMod 0).

Each file stores the inputs (J, T0 per FOWT; J_arr, T0_arr, C_array for farms), the reference's Model.Xi per case
(``Xi_c<case>`` [nWaves+1, nDOF, nw]; for the flexible FOWT also Xi_PRP [nCases, nWaves+1, 6, nw], what J multiplies), w, and per case the
reference's Tmoor_avg/std/max/min/PSD per FOWT (``fowt<i>_*`` [nCases, ...]), wave_PSD and the array_mooring entries
(``arr_*``).

Cases: VolturnUS-S (rigid; one case with two wave trains), the two-FOWT farm with 5 array lines / 10 ends (like the
reference's farm golden), farm24 (144 DOFs), VolturnUS-S-flexible (150 DOFs).

Usage (build container, reference tree present):  python tests/golden/make_golden_tmoor.py
"""
import contextlib
import copy
import io
import os
import sys
import tempfile

import numpy as np
import yaml

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg  # noqa: E402
import make_golden_farm24 as mf24  # noqa: E402

rh = mg.rh
KEYS = ("Tmoor_avg", "Tmoor_std", "Tmoor_max", "Tmoor_min", "Tmoor_PSD")


class FakeMS:
    """Stands in for a MoorPy system after lines2ss: what saveTurbineOutputs / analyzeCases / solveDynamics ask of it."""

    def __init__(self, C, J, T0):
        self.C, self.J, self.T0 = C, J, T0
        self.lineList = [object() for _ in range(len(T0) // 2)]

    def getCoupledStiffness(self, lines_only=True, tensions=True):
        return self.C, self.J

    def getCoupledStiffnessA(self, lines_only=True):
        return self.C

    def getTensions(self):
        return self.T0


def seeded_tensions(rng, n_ends, n_dof):
    J = rng.normal(size=(n_ends, n_dof)) * 1e4
    J[:, 3:6] *= 1e2                                       # N/rad against N/m
    T0 = rng.uniform(1e6, 3e6, n_ends)
    return J, T0


def _without_ms(fn):
    """fn run with the mooring stand-in hidden (MoorPy equilibrium and stiffness are out of scope), the injected C_moor kept."""
    def wrapped(self, *a, **k):
        ms, C = self.ms, self.C_moor.copy()
        self.ms = None
        try:
            return fn(self, *a, **k)
        finally:
            self.ms = ms
            self.C_moor = C
    return wrapped


@contextlib.contextmanager
def patched(raft):
    """lines2ss -> identity, Model.solveStatics -> no-op, FOWT.setPosition / calcStatics without the mooring system."""
    fm, mm = raft.raft_fowt, raft.raft_model
    saved = (fm.lines2ss, mm.lines2ss, mm.Model.solveStatics, fm.FOWT.setPosition, fm.FOWT.calcStatics)
    fm.lines2ss = mm.lines2ss = lambda ms: ms
    mm.Model.solveStatics = lambda self, case, display=0: None
    fm.FOWT.setPosition, fm.FOWT.calcStatics = _without_ms(fm.FOWT.setPosition), _without_ms(fm.FOWT.calcStatics)
    try:
        yield
    finally:
        fm.lines2ss, mm.lines2ss, mm.Model.solveStatics, fm.FOWT.setPosition, fm.FOWT.calcStatics = saved


def set_cases(design, cases):
    keys = ["wind_speed", "wind_heading", "turbulence", "turbine_status", "yaw_misalign", "wave_spectrum", "wave_period",
            "wave_height", "wave_heading", "wave_gamma", "current_speed", "current_heading"]
    rows = []
    for c in cases:
        d = dict(rh.make_case(), **c)
        rows.append([d[k] for k in keys])
    design["cases"] = dict(keys=keys, data=rows)


def record_xi(model):
    """Model.Xi of every case, captured after each solveDynamics."""
    rec = []
    orig = model.solveDynamics

    def wrapped(case, **kw):
        r = orig(case, **kw)
        rec.append(np.array(model.Xi))
        return r
    model.solveDynamics = wrapped
    return rec


def run(model, out, n_fowt, nC, flexible=False):
    raft = rh.load_reference()
    rec = record_xi(model)
    prp = []
    if flexible:
        fowt = model.fowtList[0]
        orig_mm = np.matmul

        def cap(a, b, *x, **k):                                        # J_moor @ Xi_PRP[ih,:,iw] (raft_fowt.py:2367)
            if fowt.ms is not None and a is fowt.ms.J:
                prp.append(np.array(b))
            return orig_mm(a, b, *x, **k)
        np.matmul = cap
    try:
        with patched(raft), contextlib.redirect_stdout(io.StringIO()):
            model.analyzeCases()
    finally:
        if flexible:
            np.matmul = orig_mm
    cm = model.results["case_metrics"]
    for ic, x in enumerate(rec):
        out["Xi_c%d" % ic] = x
    out["w"] = np.array(model.w)
    if flexible:
        nH, nw = rec[0].shape[0], len(model.w)
        out["Xi_PRP"] = np.array(prp).reshape(nC, nH, nw, 6).transpose(0, 1, 3, 2)
    for i in range(n_fowt):
        for k in KEYS + ("wave_PSD",):
            if k in cm[0][i]:
                out["fowt%d_%s" % (i, k)] = np.array([cm[ic][i][k] for ic in range(nC)])
    if "array_mooring" in cm[0]:
        for k in KEYS:
            out["arr_" + k] = np.array([cm[ic]["array_mooring"][k] for ic in range(nC)])


def save(name, out):
    path = os.path.join(mg.OUT, "tmoor_%s.npz" % name)
    np.savez_compressed(path, **out)
    print("%-24s %s  %.0f KB" % (name, ", ".join("%s%s" % (k, list(v.shape)) for k, v in out.items() if "std" in k),
                                  os.path.getsize(path) / 1024))


def rigid(seed=21):
    td = os.path.join(mg.REF, "tests", "test_data")
    design = rh.load_design(os.path.join(td, "VolturnUS-S.yaml"))
    cases = [dict(wave_height=[6.0, 2.0], wave_period=[12.0, 7.0], wave_heading=[30.0, -60.0], wave_spectrum=["JONSWAP", "JONSWAP"],
                  wave_gamma=[0.0, 0.0]),
             dict(wave_height=3.5, wave_period=9.0, wave_heading=0.0)]
    set_cases(design, cases)
    model = rh.build_model(design)
    rng = np.random.default_rng(seed)
    J, T0 = seeded_tensions(rng, 6, 6)
    f = model.fowtList[0]
    f.ms, f.moorMod = FakeMS(f.C_moor.copy(), J, T0), 0
    out = dict(J0=J, T00=T0, n_fowt=np.int32(1))
    run(model, out, 1, len(cases))
    save("VolturnUS-S", out)


def farm(name, yaml_path, n_ends=10, seed=5, cases=None):
    with open(yaml_path) as fh:
        design = yaml.load(fh, Loader=yaml.FullLoader)
    for k in ("turbine", "turbines", "mooring", "array_mooring"):
        design.pop(k, None)
    design["platform"]["potSecOrder"] = 0
    ks = design["array"]["keys"]
    for row in design["array"]["data"]:
        row[ks.index("turbineID")] = 0
        row[ks.index("mooringID")] = 0
    design["settings"]["max_freq"], design["settings"]["min_freq"] = 0.1024, 0.1024 / 48
    cases = cases or [dict(wave_height=6.0, wave_period=12.0, wave_heading=0.0), dict(wave_height=3.5, wave_period=9.0, wave_heading=40.0)]
    set_cases(design, cases)
    model = rh.build_model(design)
    n = model.nDOF
    rng = np.random.default_rng(seed)
    A = rng.normal(size=(n, n)) * 2e4
    C_arr = A @ A.T / n + np.diag([5e4] * n)
    J, T0 = seeded_tensions(rng, n_ends, n)
    model.ms, model.moorMod = FakeMS(C_arr, J, T0), 0
    out = dict(C_array=C_arr, J_arr=J, T0_arr=T0, n_fowt=np.int32(model.nFOWT))
    run(model, out, model.nFOWT, len(cases))
    save(name, out)


def farm24():
    src = os.path.join(mg.REF, "designs", "VolturnUS-S_farm.yaml")
    with open(src) as fh:
        design = yaml.load(fh, Loader=yaml.FullLoader)
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
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "farm24.yaml")
        with open(path, "w") as fh:
            yaml.dump(design, fh)
        farm("farm24", path, n_ends=48, seed=6, cases=[dict(wave_height=6.0, wave_period=12.0, wave_heading=0.0)])


def flexible(seed=23):
    raft = rh.load_reference()
    td = os.path.join(mg.REF, "tests", "test_data")
    design = rh.load_design(os.path.join(td, "VolturnUS-S-flexible.yaml"), strip=False)
    design.pop("mooring", None)
    design["platform"]["potSecOrder"] = 0
    cases = [dict(wave_height=6.0, wave_period=12.0, wave_heading=30.0), dict(wave_height=2.0, wave_period=8.0, wave_heading=-60.0)]
    set_cases(design, cases)
    with contextlib.redirect_stdout(io.StringIO()):
        model = raft.Model(copy.deepcopy(design))
        fowt = model.fowtList[0]                                      # what solveStatics leaves for solveDynamics (A_aero ...)
        fowt.setPosition(np.zeros(fowt.nDOF))
        fowt.calcStatics()
        fowt.calcTurbineConstants(rh.make_case(), ptfm_pitch=0)
        fowt.calcHydroConstants()
    Cmoor = np.zeros([fowt.nDOF, fowt.nDOF])
    Cmoor[:6, :6] = rh.C_MOOR_DEFAULT
    fowt.C_moor = Cmoor
    rng = np.random.default_rng(seed)
    J, T0 = seeded_tensions(rng, 6, 6)
    fowt.ms, fowt.moorMod = FakeMS(rh.C_MOOR_DEFAULT.copy(), J, T0), 0
    out = dict(J0=J, T00=T0, n_fowt=np.int32(1))
    run(model, out, 1, len(cases), flexible=True)
    save("VolturnUS-S-flexible", out)


def main():
    only = sys.argv[1] if len(sys.argv) > 1 else None
    jobs = dict(rigid=rigid, farm=lambda: farm("farm", os.path.join(mg.REF, "designs", "VolturnUS-S_farm.yaml")), farm24=farm24,
                flexible=flexible)
    for k, fn in jobs.items():
        if only in (None, k):
            fn()


if __name__ == "__main__":
    main()
