import glob
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (select with -m gpu)")


def golden_names():
    names = sorted(os.path.splitext(os.path.basename(p))[0] for p in glob.glob(os.path.join(GOLDEN, "*.npz")))
    # design fixtures (not the raw WAMIT tables; the second-order fixture has its own tests)
    return [n for n in names if n.startswith(("test_", "cfg")) and n != QTF_GOLDEN]


QTF_GOLDEN = "cfg3q_OC4semi-QTF_nw96"       # potSecOrder 2: external .12d QTF (make_golden.fixture_qtf)


def load_golden(name):
    """-> (G, P): the raw npz dict and the packed design (keys without the P_ prefix)."""
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    G = {k: z[k] for k in z.files}
    P = {k[2:]: v for k, v in G.items() if k.startswith("P_")}
    return G, P


def relerr(a, b):
    """max |a-b| / max |b|  (array-level relative error)."""
    a, b = np.asarray(a), np.asarray(b)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


def response_err(Xi, ref, floor=1e-100):
    """Parity metric for responses [..,6,nw] (DESIGN.md section 6): per frequency, translations and rotations are each
    compared against the largest reference amplitude in their 3-DOF group at that frequency (every frequency is an
    independent linear solve; the three DOFs of a group share units).  Returns the max over everything of
    |Xi-ref| / group_max.  Bins whose group_max is below ``floor`` x the unit's peak amplitude are compared against that
    floor instead: there the wave spectrum itself is a SUBNORMAL double (JONSWAP's exp(-1.25 (Tp f)^-4) at the first
    non-zero bins, S ~ 1e-320 with a handful of significant bits), so the last-bit differences between two libm exp()
    implementations are O(1) relative there while the amplitudes are ~1e-160 of the response peak."""
    Xi, ref = np.asarray(Xi), np.asarray(ref)
    err = 0.0
    peak = np.abs(ref).max(axis=(-2, -1), keepdims=True) if ref.ndim >= 2 else np.abs(ref).max()
    for g in (slice(0, 3), slice(3, 6)):
        d = np.abs(Xi[..., g, :] - ref[..., g, :])
        scale = np.maximum(np.abs(ref[..., g, :]).max(axis=-2, keepdims=True), floor * peak)
        ok = scale > 0
        if np.any(ok):
            err = max(err, float((d / np.where(ok, scale, 1.0))[np.broadcast_to(ok, d.shape)].max()))
    return err


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as orc
    orc.build()
    return orc
