"""Second-order (difference-frequency) force from a QTF table: both kernels run_qtf can pick -- the tile kernel (k_qtf_tiles +
k_qtf_finish) and the diagonal kernel k_qtf_force<false> / <true> (one heading / heading interpolation) -- asserted through
solver.last_dispatch() and compared with oracle.hydro_force_2nd.  The diagonal kernel runs where the tile tables do not fit
in shared memory (nw > 3396 for the shipped 56-frequency table) or when RAFTK_QTF_DIAG=1."""
import numpy as np
import pytest

from conftest import QTF_GOLDEN, load_golden, relerr

pytestmark = pytest.mark.gpu
RTOL = 1e-10
D2R = 0.017453292519943295


def _sea_states(seed, n):
    rng = np.random.default_rng(seed)
    return dict(Hs=rng.uniform(1, 10, n), Tp=rng.uniform(5, 18, n), gamma=np.zeros(n), beta_deg=rng.uniform(-180, 180, n),
                spec=np.zeros(n, dtype=np.int32))


def _on_grid(P, nw):
    """The QTF design on an nw-bin grid up to 0.512 Hz (only the grid and the QTF fields matter to the force).  The grid
    reaches past the table's last frequency, and its difference frequencies past the table's span (2.75 rad/s)."""
    w = np.arange(1, nw + 1) * (2 * np.pi * 0.512 / nw)
    Q = dict(P, w=w, k=w ** 2 / 9.81, dw=w[1] - w[0])
    for key in ("A_w", "B_w", "X_BEM", "bem_headings"):
        Q.pop(key, None)
    return Q


def _four_headings(G, P):
    """The 4-heading table of test_gpu_parity.test_second_order_heading_interpolation_and_design_axis."""
    Pm = dict(P)
    Pm["qtf"] = np.stack([P["qtf"][:, :, 0, :] * s for s in G["mh_scale"]], axis=2)
    Pm["qtf_heads"] = G["mh_heads"]
    return Pm


def tile_limit(n_qtf_w):
    """Largest nw whose tile tables fit: run_qtf's nw*68 + (n_qtf_w - 1)*8 + 16 <= 226 KB (and nw <= 4096)."""
    return min(4096, (226 * 1024 - 16 - (n_qtf_w - 1) * 8) // 68)


def _force(monkeypatch, Ps, cs, diag):
    from raft_b200 import solver
    if diag:
        monkeypatch.setenv("RAFTK_QTF_DIAG", "1")
    else:
        monkeypatch.delenv("RAFTK_QTF_DIAG", raising=False)
    f = solver.second_order_force(solver.DesignBatch(Ps), solver.CaseTable(cs))
    return f, solver.last_dispatch()


def _vs_oracle(oracle, f, Ps, cs, cases, design=0):
    od = oracle.OracleDesign(Ps)
    err = 0.0
    for c in cases:
        S = oracle.jonswap(Ps["w"], cs["Hs"][c], cs["Tp"][c], 0.0)
        fm, fo = oracle.hydro_force_2nd(od, cs["beta_deg"][c] * D2R, S)
        assert relerr(f["F_2nd"][design, c], fo) < RTOL, c
        assert relerr(f["F_2nd_mean"][design, c], fm) < RTOL, c
        err = max(err, relerr(f["F_2nd"][design, c], fo))
    return err


def _beyond_span_zero(f, P, nw):
    w = _on_grid(P, nw)["w"]
    span = P["qtf_w"][-1] - P["qtf_w"][0]
    mu = np.arange(1, nw + 1) * (w[1] - w[0])              # bin m holds difference frequency (m+1) dw
    assert np.any(mu > span * (1 + 1e-12))
    assert np.all(f["F_2nd"][..., mu > span * (1 + 1e-12)] == 0.0)


@pytest.mark.parametrize("heads", [1, 4])
def test_diagonal_kernel_forced_vs_oracle_and_tiles(heads, monkeypatch, oracle):
    """RAFTK_QTF_DIAG=1 at nw = 2048: k_qtf_force<false> with one heading, <true> with the 4-heading table.  Equal to the
    oracle and, to 1e-13, to the tile kernel on the same inputs (its atomics change only the last bits)."""
    G, P = load_golden(QTF_GOLDEN)
    Ps = _on_grid(P if heads == 1 else _four_headings(G, P), 2048)
    cs = _sea_states(41, 4)
    fd, rec = _force(monkeypatch, Ps, cs, diag=True)
    assert rec["family"] == "qtf" and rec["kernel"] == ("qtf-diag" if heads == 1 else "qtf-diag-mix"), rec
    ft, rec_t = _force(monkeypatch, Ps, cs, diag=False)
    assert rec_t["kernel"] == "qtf-tiles", rec_t
    _vs_oracle(oracle, fd, Ps, cs, [0, 3])
    assert relerr(ft["F_2nd"], fd["F_2nd"]) < 1e-13 and relerr(ft["F_2nd_mean"], fd["F_2nd_mean"]) < 1e-13
    _beyond_span_zero(fd, P, 2048)
    _beyond_span_zero(ft, P, 2048)


def test_diagonal_kernel_two_design_batch(monkeypatch, oracle):
    """Two designs with different 4-heading tables in one batch (qtf_shared = 0) on the diagonal kernel: both against the oracle."""
    G, P = load_golden(QTF_GOLDEN)
    Pm = _on_grid(_four_headings(G, P), 1024)
    Pn = dict(Pm, qtf=Pm["qtf"][:, :, ::-1, :] * (0.5 - 0.25j))
    cs = _sea_states(42, 3)
    from raft_b200 import solver
    assert solver.DesignBatch([Pm, Pn]).qtf_shared == 0
    fd, rec = _force(monkeypatch, [Pm, Pn], cs, diag=True)
    assert rec["kernel"] == "qtf-diag-mix", rec
    for d, Pd in enumerate((Pm, Pn)):
        _vs_oracle(oracle, fd, Pd, cs, range(3), design=d)
    ft, _ = _force(monkeypatch, [Pm, Pn], cs, diag=False)
    assert relerr(ft["F_2nd"], fd["F_2nd"]) < 1e-13


def test_natural_fallback_at_the_tile_limit(monkeypatch, oracle):
    """The first nw past the tile kernel's shared-memory limit runs the diagonal kernel without any switch; the last nw below
    it still runs the tiles.  Both against the oracle (one case each: the oracle's cost grows as nw^2)."""
    G, P = load_golden(QTF_GOLDEN)
    lim = tile_limit(len(P["qtf_w"]))
    assert lim == 3396
    cs = _sea_states(43, 2)
    for nw, kernel in ((lim, "qtf-tiles"), (lim + 1, "qtf-diag")):
        Ps = _on_grid(P, nw)
        f, rec = _force(monkeypatch, Ps, cs, diag=False)
        assert rec["kernel"] == kernel, (nw, rec)
        _vs_oracle(oracle, f, Ps, cs, [nw % 2])
        _beyond_span_zero(f, P, nw)


@pytest.mark.parametrize("nw", [17, 31, 1001])
def test_tiles_at_odd_and_small_grids(nw, monkeypatch, oracle):
    """The tile kernel at odd nw and at nw < 32 (fewer bins than one warp), one and four headings, against the oracle and the
    diagonal kernel."""
    G, P = load_golden(QTF_GOLDEN)
    cs = _sea_states(44, 3)
    for Pq in (P, _four_headings(G, P)):
        Ps = _on_grid(Pq, nw)
        ft, rec = _force(monkeypatch, Ps, cs, diag=False)
        assert rec["kernel"] == "qtf-tiles", rec
        _vs_oracle(oracle, ft, Ps, cs, range(3))
        fd, _ = _force(monkeypatch, Ps, cs, diag=True)
        assert relerr(ft["F_2nd"], fd["F_2nd"]) < 1e-13 and relerr(ft["F_2nd_mean"], fd["F_2nd_mean"]) < 1e-13
