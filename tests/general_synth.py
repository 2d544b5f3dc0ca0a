"""Synthetic inputs for the generalised-DOF GPU path at the shapes its one flexible fixture (VolturnUS-S-flexible: n = 150,
nw = 40, fd support {0..5, 144..149}, nearly symmetric A_w / B_w, T0 = [I6 | 0]) never reaches.  Test infrastructure, seeded
and built in-test, in the style of the checker modules next to it:

* ``design``: ``test_dispatch_general.general_design`` (OC3spar regridded, seeded mode shapes, a modal stiffness that forces
  row swaps);
* ``fd_tables``: frequency-dependent added mass and damping on an arbitrary support, with a symmetric and an antisymmetric
  part (a transposed read changes the answer) and a per-entry variation over w; a seeded BEM table; a dense T0;
* ``qtf_table``: a Hermitian difference-frequency QTF whose frequency axis covers only part of the model grid;
* ``cases``: a train table (``packer.pack_case_trains``) mixing single- and multi-train cases, every secondary train with a
  heading of its own;
* ``CaptureZ``: an oracle proxy that keeps the last impedance the checkers solve with (conditioning checks).

The ``fd`` and ``qtf`` dicts have the layout of ``packer.pack_general_matrices`` / ``packer.pack_general_qtf``."""
import numpy as np

from test_dispatch_general import general_design

D2R = 0.017453292519943295


def design(n, nw, seed=0):
    """-> (P, M, B, C) of a synthetic n-DOF design on nw bins (``test_dispatch_general.general_design``)."""
    return general_design(n, nw, seed)


def support(n, extra=(0, 3, 7, 8, 15, 16)):
    """fd support ``(extra & [0, n)) | {n - 1}``: crosses the 8-column panels of the blocked LU and ends on the last DOF."""
    return np.array(sorted({i for i in extra if i < n} | {n - 1}), dtype=np.int32)


def _smooth(rng, shape, s, amp=0.5):
    """1 + amp cos(pi s + phase), a seeded phase per entry: every entry varies by >= amp / (1 + amp) of its peak over s in [0, 1]."""
    ph = rng.uniform(0.0, 2.0 * np.pi, shape)
    return 1.0 + amp * np.cos(np.pi * s + ph[..., None])


def _fd_matrix(rng, scale, s):
    """[nf, nf, nw]: (symmetric + antisymmetric) * a smooth per-entry function of w, entries scaled by sqrt(D_a D_b)."""
    nf = len(scale)
    S = rng.uniform(-0.1, 0.1, (nf, nf))
    S = 0.5 * (S + S.T)
    S[np.diag_indices(nf)] = rng.uniform(0.1, 0.3, nf)
    K = rng.uniform(0.08, 0.15, (nf, nf)) * rng.choice([-1.0, 1.0], (nf, nf))
    K = np.triu(K, 1)
    K = K - K.T
    base = (S + K) * np.sqrt(np.outer(scale, scale))
    return np.ascontiguousarray(base[:, :, None] * _smooth(rng, (nf, nf), s))


def fd_tables(P, M, B, idx, seed=0, bem=None, rotor=True, T0="dense", headings=None, heading_adjust=0.0, x_ref=0.0, y_ref=0.0):
    """The ``fd`` dict of a synthetic FOWT.

    ``rotor``: A_w, B_w [n_fd, n_fd, nw] on the support ``idx``, each a symmetric part (diagonal 0.1-0.3 of diag M, resp. of
    the damping scale below) plus an antisymmetric part of >= 20 % (Frobenius), times a per-entry smooth function of w that
    varies by >= 1/3 over the grid.  The damping scale is diag B, or 10 % of critical (0.1 sqrt(M C)) where B is zero.
    ``bem="table"``: X_BEM [nhead, 6, nw] (heading list ``headings``, default 0, 30, .., 330 deg), smooth in w, scaled per
    DOF like a unit-amplitude wave load on a spar (moments: forces at a 30 m lever arm, yaw 1 m), with ``heading_adjust``, ``x_ref``, ``y_ref``.  ``T0``: "dense" = [I6 | 0] plus a
    seeded dense perturbation of 5 % that also fills columns >= 6; "identity" = [I6 | 0]."""
    rng = np.random.default_rng(1000 + seed)
    n, w = M.shape[0], np.asarray(P["w"], dtype=float)
    nw = len(w)
    s = (w - w[0]) / max(w[-1] - w[0], 1e-300)
    idx = np.asarray(idx, dtype=np.int32)
    fd = dict(fd_idx=idx if rotor else np.zeros(0, dtype=np.int32))
    c6 = np.abs(np.diag(np.asarray(P["C0"], dtype=float).reshape(6, 6)))
    if rotor and len(idx):
        dM = np.diag(M)[idx]
        crit = 0.1 * np.sqrt(np.abs(dM) * np.where(idx < 6, c6[np.minimum(idx, 5)], np.abs(dM)))
        dB = np.where(np.diag(B)[idx] > 0, np.diag(B)[idx], crit)
        fd["A_w"] = _fd_matrix(rng, dM, s)
        fd["B_w"] = _fd_matrix(rng, dB, s)
    if bem == "table":
        hd = np.asarray(np.arange(0.0, 360.0, 30.0) if headings is None else headings, dtype=float)
        sc = 0.3 * np.maximum(c6, w[nw // 2] ** 2 * np.abs(np.diag(M)[:6]))
        sc[3:] = np.array([30.0, 30.0, 1.0]) * sc[:3].mean()     # roll, pitch: the forces at a 30 m lever arm; yaw: small
        X = np.zeros([len(hd), 6, nw], dtype=complex)
        for h in range(len(hd)):
            mag = _smooth(rng, (6,), s) * rng.uniform(0.5, 1.5, 6)[:, None]
            ph = rng.uniform(0, 2 * np.pi, 6)[:, None] + 1.5 * s[None, :] * rng.uniform(-1, 1, 6)[:, None]
            X[h] = sc[:, None] * mag * np.exp(1j * ph)
        T = np.zeros([6, n])
        T[:, :6] = np.eye(6)
        if T0 == "dense":                              # rotation rows in rad: 1 % of the translation rows' size off their block
            E = 0.05 * rng.uniform(-1.0, 1.0, (6, n))
            E[3:, :3] *= 0.01
            E[3:, 6:] *= 0.01
            T = T + E
        fd.update(X_BEM=X, bem_headings=hd, heading_adjust=float(heading_adjust), T0=np.ascontiguousarray(T))
    fd["x_ref"], fd["y_ref"] = float(x_ref), float(y_ref)
    return fd


def qtf_table(P, nq, heads, seed=0, scale=0.02):
    """The ``qtf`` dict of a synthetic FOWT: a Hermitian [nq, nq, nh, 6] table (Q[j, i] = conj Q[i, j], real diagonal) on
    ``nq`` frequencies from bin nw/6 to bin 2 nw/3 of the model grid, so bins at both ends lie outside it; headings ``heads``
    in deg (stored in rad).  The force entries are ``scale`` x the BEM table's per-DOF load scale per square metre, the moments
    those forces at a 30 m lever arm; smooth in both frequencies and different per heading."""
    rng = np.random.default_rng(2000 + seed)
    w = np.asarray(P["w"], dtype=float)
    nw = len(w)
    qw = np.linspace(w[nw // 6], w[(2 * nw) // 3], nq)
    s = (qw - qw[0]) / (qw[-1] - qw[0])
    M0, C0 = (np.asarray(P[k], dtype=float).reshape(6, 6) for k in ("M0", "C0"))
    sc = scale * 0.3 * np.maximum(np.abs(np.diag(C0)), w[nw // 2] ** 2 * np.abs(np.diag(M0)))
    sc[3:] = 30.0 * sc[:3].mean()                      # moments: the forces at a 30 m lever arm
    heads = np.asarray(heads, dtype=float)
    Q = np.zeros([nq, nq, len(heads), 6], dtype=complex)
    for h in range(len(heads)):
        for a in range(6):
            k1, k2, ph = rng.uniform(-2.0, 2.0), rng.uniform(-2.0, 2.0), rng.uniform(0, 2 * np.pi)
            G = (1.0 + 0.5 * np.cos(np.pi * s[:, None] + k1 * s[None, :])) * np.exp(1j * (ph + 3.0 * (k2 * s[:, None] - s[None, :])))
            Q[:, :, h, a] = sc[a] * 0.5 * (G + G.conj().T)
    return dict(qtf=np.ascontiguousarray(Q), qtf_w=qw, qtf_heads=heads * D2R)


def cases(ntrains, seed=0):
    """A train table mixing single- and multi-train cases: ``ntrains`` = trains per case, e.g. (1, 3, 1, 2).  Every secondary
    train has its own sea state and a heading 40-140 deg away from its primary's.
    -> (table of packer.pack_case_trains, owner [nT], first [nC], trains [per case: rows (Hs, Tp, heading deg)])."""
    from raft_b200 import packer
    rng = np.random.default_rng(3000 + seed)
    out, trains = [], []
    for nt in ntrains:
        b0 = rng.uniform(-90.0, 90.0)
        tr = np.stack([rng.uniform(2.0, 6.0, nt), rng.uniform(7.0, 14.0, nt),
                       b0 + np.concatenate([[0.0], rng.uniform(40.0, 140.0, nt - 1) * rng.choice([-1, 1], nt - 1)])], axis=1)
        trains.append(tr)
        out.append(dict(wave_spectrum=["JONSWAP"] * nt, wave_height=list(tr[:, 0]), wave_period=list(tr[:, 1]),
                        wave_heading=list(tr[:, 2]), wave_gamma=[0.0] * nt))
    table, owner, first = packer.pack_case_trains(out)
    return table, owner, first, trains


class CaptureZ:
    """The oracle module with ``system_response`` wrapped: keeps the impedance [nw, n, n] of the checker's last solve."""

    def __init__(self, orc):
        self._orc, self.Z = orc, None

    def __getattr__(self, name):
        return getattr(self._orc, name)

    def system_response(self, Z, F):
        self.Z = Z
        return self._orc.system_response(Z, F)


def max_cond(Z):
    """Largest 2-norm condition number over the bins of Z [nw, n, n]."""
    return float(np.linalg.cond(Z).max())


def row_errors(X, ref, floor=1e-6):
    """Per DOF row: max_w |X - ref| / max_w |ref| over the rows whose peak is >= ``floor`` x the whole response's peak,
    X and ref [n, nw] -> the largest such ratio."""
    X, ref = np.asarray(X), np.asarray(ref)
    pk = np.abs(ref).max(axis=-1)
    keep = pk >= floor * pk.max()
    return float((np.abs(X - ref).max(axis=-1)[keep] / pk[keep]).max())


def row(name, arg=None):
    """Inputs of one row of the GPU matrix (tests/test_general_edges.py), shared with the CPU sensitivity checks
    -> dict(P, M, B, Cm, fd, qtf, ct = cases(...) or an equivalent tuple, n_iter)."""
    from raft_b200 import packer
    qtf, n_iter = None, 10
    if name == "a":                                    # support across the panels and on the last DOF; trains, 129 bins
        P, M, B, Cm = design(arg, 129)
        fd, ct = fd_tables(P, M, B, support(arg), seed=arg, bem="table"), cases((1, 3, 2), seed=arg)
    elif name == "b":                                  # modal DOFs only, rotor tables without BEM, 257 bins
        P, M, B, Cm = design(64, 257)
        fd, ct = fd_tables(P, M, B, [6, 31, 32, 63], seed=2), cases((2, 1), seed=2)
    elif name == "c":                                  # BEM without rotor tables (n_fd = 0), arg = nw
        P, M, B, Cm = design(17, arg)
        fd, ct = fd_tables(P, M, B, support(17), seed=3, bem="table", rotor=False), cases((1, 1), seed=3)
    elif name == "d":                                  # every DOF on the support ("full", with BEM) or only the last
        P, M, B, Cm = design(17, 33)
        idx = np.arange(17) if arg == "full" else [16]
        fd, ct = fd_tables(P, M, B, idx, seed=4, bem="table" if arg == "full" else None), cases((1, 1), seed=4)
    elif name == "e":                                  # 256 DOFs: across the 128-thread stride ("stride") or every DOF
        P, M, B, Cm = design(256, 16)
        idx = [0, 1, 2, 3, 4, 5, 127, 128, 255] if arg == "stride" else np.arange(256)
        fd, ct, n_iter = fd_tables(P, M, B, idx, seed=5, bem="table"), cases((2,), seed=5), 4
    elif name == "f":                                  # second-order loads, arg = (n, nw)
        n, nw = arg
        P, M, B, Cm = design(n, nw)
        fd, ct = fd_tables(P, M, B, support(n), seed=6 + n, bem="table"), cases((1, 2), seed=6 + n)
        qtf = qtf_table(P, 20, [0.0, 90.0, 200.0], seed=n)
    elif name == "g":                                  # BEM heading tables, arg = headings; heading_adjust, x_ref, y_ref
        P, M, B, Cm = design(9, 129)
        fd = fd_tables(P, M, B, support(9), seed=7, bem="table", headings=arg, heading_adjust=12.5, x_ref=3.0, y_ref=-2.0)
        trains = [np.array([[3.0 + 0.5 * c, 8.0 + c, b]]) for c, b in enumerate([0.0, 20.0, 300.0, 355.0, -45.0])]
        table, owner, first = packer.pack_case_trains([dict(wave_spectrum="JONSWAP", wave_height=t[0, 0], wave_period=t[0, 1],
                                                            wave_heading=t[0, 2], wave_gamma=0.0) for t in trains])
        ct = (table, owner, first, trains)
    else:
        raise KeyError(name)
    return dict(P=P, M=M, B=B, Cm=Cm, fd=fd, qtf=qtf, ct=ct, n_iter=n_iter)


# every row of the GPU matrix, by (name, arg)
ROWS = ([("a", n) for n in (7, 9, 17)] + [("b", None)] + [("c", nw) for nw in (128, 129)] + [("d", "full"), ("d", "last")]
        + [("e", "stride"), ("e", "full")] + [("f", s) for s in ((6, 33), (9, 129), (17, 129), (64, 257))]
        + [("g", (40.0,)), ("g", (20.0, 95.0, 200.0, 290.0))])
