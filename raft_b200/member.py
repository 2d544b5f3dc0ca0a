"""Strip-theory member: discretisation, pose and per-node hydrodynamic coefficients (host pre-pass).

This is the node-table builder of SURVEY.md section 8(f) row 1 / section 8(a) row a12: it turns one entry of
``design['platform']['members']`` into the arrays the packer flattens for the kernels.  It restates, in
vectorised NumPy, the following parts of the reference (paths relative to /root/reference/raft/):

  * strip discretisation                       raft_member.py:190-271
  * heading copies / twist of vertical members raft_member.py:69-79, helpers.py:587-602
  * member frame q, p1, p2 (Z1Y2Z3 Euler)      raft_member.py:325-357, helpers.py:439-466
  * node positions                             raft_member.py:359-362
  * added-mass / inertia coefficients, a_i     raft_member.py:1295-1357, 1387-1448
  * MacCamy-Fuchs transverse coefficient       raft_member.py:1451-1486

Only what the response hot path needs is built: no shell mass, ballast, hydrostatics or FE stiffness
(statics are out of scope, DESIGN.md section 9).  Attribute names match the reference's ``Member`` so that
``raft_b200.packer`` treats both kinds of object alike.
"""
import numpy as np


def _tile(mi, key, n, default, index=None):
    """Scalar-or-list station property -> array of length n (semantics of helpers.getFromDict for 1-D shapes)."""
    if key not in mi:
        return np.full(n, float(default))
    v = mi[key]
    if np.isscalar(v):
        return np.full(n, float(v))
    a = np.array(v, dtype=float)
    if a.shape[0] != n and not (index is not None and a.ndim == 1):
        raise ValueError(f"Value for key '{key}' is not the expected size of {n} and is instead: {v}")
    if index is None:
        return a.astype(float)
    if a.ndim == 1:                       # a pair [c1, c2] given once for the whole member (n may equal 2: the
        if len(a) != n:                   # reference then reads it as per-station values; keep that quirk)
            raise ValueError(f"Value for key '{key}' is not the expected size of {n} and is instead: {v}")
        return np.full(n, a[index])
    return a[:, index].astype(float)


def rotation_matrix(x3, x2, x1):
    """Intrinsic z-y-x rotation (roll x3, pitch x2, yaw x1), helpers.py:439-466."""
    s1, c1, s2, c2, s3, c3 = np.sin(x1), np.cos(x1), np.sin(x2), np.cos(x2), np.sin(x3), np.cos(x3)
    return np.array([[c1 * c2, c1 * s2 * s3 - c3 * s1, s1 * s3 + c1 * c3 * s2],
                     [c2 * s1, c1 * c3 + s1 * s2 * s3, c3 * s1 * s2 - c1 * s3],
                     [-s2, c2 * s3, c2 * c3]])


def _heading(r, heading_deg):
    if heading_deg == 0.0:
        return r
    c, s = np.cos(np.deg2rad(heading_deg)), np.sin(np.deg2rad(heading_deg))
    return np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]]) @ r


class Member:
    """One rigid strip-theory member at a given heading (a design entry with ``heading: [..]`` yields several)."""

    def __init__(self, mi, nw=0, heading=0.0, part_of="platform"):
        self.name = str(mi["name"])
        self.type = str(mi.get("type", "rigid"))
        if self.type != "rigid":
            raise NotImplementedError("member %r: only rigid members are supported by the GPU path" % self.name)
        self.part_of = part_of
        rA0, rB0 = np.array(mi["rA"], dtype=float), np.array(mi["rB"], dtype=float)
        if rA0[2] == 0 or rB0[2] == 0:
            raise ValueError("RAFT Members cannot start or end on the waterplane")
        rAB0 = rB0 - rA0
        self.l = float(np.linalg.norm(rAB0))
        self.potMod = bool(mi.get("potMod", False))
        self.MCF = bool(mi.get("MCF", False))
        self.gamma = float(mi.get("gamma", 0.0))
        self.heading = float(heading)
        if heading != 0.0:
            rA0, rB0 = _heading(rA0, heading), _heading(rB0, heading)
            if rAB0[0] == 0.0 and rAB0[1] == 0:
                self.gamma += heading                     # a vertical member takes its heading as twist
        self.rA0, self.rB0 = rA0, rB0

        st = np.array(mi["stations"], dtype=float)
        n = len(st)
        if n < 2:
            raise ValueError("At least two stations entries must be provided")
        if np.any(np.diff(st) < 0):
            raise ValueError(f"Member {self.name}: the station list is not in ascending order.")
        self.stations = (st - st[0]) / (st[-1] - st[0]) * self.l
        shape = str(mi["shape"])[0].lower()
        if shape == "c":
            self.shape = "circular"
            d = _tile(mi, "d", n, None)
            self.gamma = 0.0
        elif shape == "r":
            self.shape = "rectangular"
            v = np.array(mi["d"], dtype=float)
            if v.shape == (n, 2):
                d = v
            elif v.ndim == 1 and len(v) == 2:
                d = np.tile(v, (n, 1))                    # one side-length pair for every station
            else:
                raise ValueError(f"Value for key 'd' is not a compatible size for target size of {[n, 2]} and is instead: {mi['d']}")
            self.MCF = False
        else:
            raise ValueError("The only allowable shape strings are circular and rectangular")
        self.d = d
        self.Cd_q = _tile(mi, "Cd_q", n, 0.0)
        self.Cd_p1 = _tile(mi, "Cd", n, 0.6, index=0)
        self.Cd_p2 = _tile(mi, "Cd", n, 0.6, index=1)
        self.Cd_End = _tile(mi, "CdEnd", n, 0.6)
        self.Ca_q = _tile(mi, "Ca_q", n, 0.0)
        self.Ca_p1 = _tile(mi, "Ca", n, 0.97, index=0)
        self.Ca_p2 = _tile(mi, "Ca", n, 0.97, index=1)
        self.Ca_End = _tile(mi, "CaEnd", n, 0.6)
        self._discretise(float(mi.get("dlsMax", 5.0)))
        self.nw = nw
        self.a_i = np.zeros(self.ns)
        self.Imat = np.zeros([self.ns, 3, 3])
        self.Amat = np.zeros([self.ns, 3, 3])
        self.Imat_MCF = np.zeros([self.ns, 3, 3, nw], dtype=complex)

    # raft_member.py:190-271 -------------------------------------------------------------------------
    def _discretise(self, dlsMax):
        d, s = self.d, self.stations
        half = lambda x: 0.5 * x
        ls, dls, ds, drs = [0.0], [0.0], [half(d[0])], [half(d[0])]
        for i in range(1, len(s)):
            lstrip = s[i] - s[i - 1]
            if lstrip > 0.0:
                ns = int(np.ceil(lstrip / dlsMax))
                dl = lstrip / ns
                m = 0.5 * (d[i] - d[i - 1]) / lstrip
                jj = 0.5 + np.arange(ns)
                ls += [s[i - 1] + dl * x for x in jj]
                dls += [dl] * ns
                ds += [d[i - 1] + dl * 2 * m * x for x in jj]
                drs += [dl * m] * ns
            elif lstrip == 0.0:
                ls.append(s[i - 1]); dls.append(0.0)
                ds.append(0.5 * (d[i - 1] + d[i])); drs.append(0.5 * (d[i] - d[i - 1]))
        ls.append(s[-1]); dls.append(0.0); ds.append(half(d[-1])); drs.append(-half(d[-1]))
        self.ns = len(ls)
        self.ls, self.dls = np.array(ls, dtype=float), np.array(dls, dtype=float)
        self.ds, self.drs = np.array(ds, dtype=float), np.array(drs, dtype=float)

    # raft_member.py:312-377 -------------------------------------------------------------------------
    def setPosition(self, r6=None):
        """Frame and node positions for a platform pose r6 = (x, y, z, roll, pitch, yaw)."""
        r6 = np.zeros(6) if r6 is None else np.asarray(r6, dtype=float)
        rAB = self.rB0 - self.rA0
        q = rAB / np.linalg.norm(rAB)
        beta = np.arctan2(q[1], q[0])
        phi = np.arctan2(np.sqrt(q[0] ** 2 + q[1] ** 2), q[2])
        s1, c1, s2, c2 = np.sin(beta), np.cos(beta), np.sin(phi), np.cos(phi)
        s3, c3 = np.sin(np.deg2rad(self.gamma)), np.cos(np.deg2rad(self.gamma))
        p1 = np.array([c1 * c2 * c3 - s1 * s3, c1 * s3 + c2 * c3 * s1, -c3 * s2])      # first column of Z1Y2Z3
        p2 = np.cross(q, p1)
        Rp = rotation_matrix(*r6[3:])
        self.rA = r6[:3] + Rp @ self.rA0                 # rigid link from the platform reference node
        self.q, self.p1, self.p2 = Rp @ q, Rp @ p1, Rp @ p2
        self.rB = self.rA + self.l * self.q
        self.r = self.rA[None, :] + (self.ls / self.l)[:, None] * (self.rB - self.rA)[None, :]
        return self

    # raft_member.py:1295-1357, 1387-1448 ---------------------------------------------------------------
    def calcHydroConstants(self, rho=1025.0, g=9.81, k_array=None):
        """Per-node added-mass / inertial-excitation coefficients in the member frame.

        Fills ``Imat``/``Amat`` [ns,3,3], ``a_i`` [ns] like the reference and additionally the scalar
        coefficients ``in_q, in_p1, in_p2, ad_q, ad_p1, ad_p2`` (Imat = in_q qq' + in_p1 p1p1' + in_p2 p2p2')."""
        ns = self.ns
        self.in_q, self.in_p1, self.in_p2 = np.zeros(ns), np.zeros(ns), np.zeros(ns)
        self.ad_q, self.ad_p1, self.ad_p2 = np.zeros(ns), np.zeros(ns), np.zeros(ns)
        self.a_i = np.zeros(ns)
        self.Imat[:] = 0; self.Amat[:] = 0
        sub = self.r[:, 2] < 0
        if self.potMod or not np.any(sub):
            return
        circ = self.shape == "circular"
        Ca_p1 = np.interp(self.ls, self.stations, self.Ca_p1)
        Ca_p2 = np.interp(self.ls, self.stations, self.Ca_p2)
        Ca_End = np.interp(self.ls, self.stations, self.Ca_End)
        if circ:
            v = 0.25 * np.pi * self.ds ** 2 * self.dls
            v_end = np.pi / 12.0 * np.abs((self.ds + self.drs) ** 3 - (self.ds - self.drs) ** 3)
            a_i = np.pi * self.ds * self.drs
        else:
            v = self.ds[:, 0] * self.ds[:, 1] * self.dls
            v_end = np.pi / 12.0 * (np.mean(self.ds + self.drs, axis=1) ** 3 - np.mean(self.ds - self.drs, axis=1) ** 3)
            a_i = ((self.ds[:, 0] + self.drs[:, 0]) * (self.ds[:, 1] + self.drs[:, 1])
                   - (self.ds[:, 0] - self.drs[:, 0]) * (self.ds[:, 1] - self.drs[:, 1]))
        # strips piercing the free surface: scale by the wetted fraction (uses r_z, not the axial coordinate: :1329)
        pierce = sub & (self.r[:, 2] + 0.5 * self.dls > 0)
        with np.errstate(divide="ignore", invalid="ignore"):
            v = np.where(pierce, v * (0.5 * self.dls - self.r[:, 2]) / self.dls, v)
        z = lambda x: np.where(sub, x, 0.0)
        self.ad_p1, self.ad_p2, self.ad_q = z(rho * v * Ca_p1), z(rho * v * Ca_p2), z(rho * v_end * Ca_End)
        self.in_p1, self.in_p2, self.in_q = z(rho * v * (1.0 + Ca_p1)), z(rho * v * (1.0 + Ca_p2)), z(rho * v_end * Ca_End)
        self.a_i = z(a_i)
        qq, p11, p22 = np.outer(self.q, self.q), np.outer(self.p1, self.p1), np.outer(self.p2, self.p2)
        self.Amat = (self.ad_p1[:, None, None] * p11 + self.ad_p2[:, None, None] * p22) + self.ad_q[:, None, None] * qq
        self.Imat = (self.in_p1[:, None, None] * p11 + self.in_p2[:, None, None] * p22) + self.in_q[:, None, None] * qq
        if self.MCF and k_array is not None:
            from scipy.special import hankel1
            k = np.asarray(k_array, dtype=float)
            self.Imat_MCF = np.zeros([ns, 3, 3, len(k)], dtype=complex)
            for il in np.where(sub)[0]:
                R = self.ds[il] / 2
                Hp1 = 0.5 * (hankel1(0, k * R) - hankel1(2, k * R))
                Cm = 4j / (np.pi * (k * R) ** 2 * Hp1)
                Tr = np.pi / 5 / R
                ramp = np.where(k < Tr, 0.5 * (1 - np.cos(np.pi * k / Tr)), 1.0)
                ramp = np.where(k <= 0, 0.0, ramp)
                Cm1 = Cm * ramp + (1.0 + Ca_p1[il]) * (1 - ramp)
                Cm2 = Cm * ramp + (1.0 + Ca_p2[il]) * (1 - ramp)
                sides = rho * v[il] * (Cm1[None, None, :] * p11[:, :, None] + Cm2[None, None, :] * p22[:, :, None])
                self.Imat_MCF[il] = sides + (self.in_q[il] * qq)[:, :, None]

    def added_mass_6dof(self, r_ref):
        """Member contribution to A_hydro_morison about ``r_ref`` (raft_member.py:1361 + raft_fowt.py:1625)."""
        A = np.zeros([6, 6])
        for il in np.where(self.r[:, 2] < 0)[0]:
            if not np.any(self.Amat[il]):
                continue
            r = self.r[il] - r_ref
            H = np.array([[0, r[2], -r[1]], [-r[2], 0, r[0]], [r[1], -r[0], 0]])
            m = self.Amat[il]
            A[:3, :3] += m
            mH = m @ H
            A[:3, 3:] += mH
            A[3:, :3] += mH.T
            A[3:, 3:] += H @ m @ H.T
        return A
