"""FOWT: host-side mirror of the reference's ``raft.FOWT`` for the response hot path.

Keeps the reference's method names, argument meaning and side-effect attributes for
``calcHydroConstants`` (raft_fowt.py:1589-1625), ``calcHydroExcitation`` (:1732-1888),
``calcHydroLinearization`` (:1891-1936) and ``calcDragExcitation`` (:1940-1957); the last three run on
the GPU through the C ABI (``raft_b200.solver``).  Everything the hot path does not compute -- structural
mass, hydrostatics, mooring, rotor aerodynamics, BEM coefficients -- is OUT OF SCOPE (DESIGN.md section 9) and is
injected as matrices (``matrices=dict(M_struc=..., C_hydro=..., C_moor=..., A_BEM=..., X_BEM=...)``).
Scope: one rigid 6-DOF body built from ``design['platform']['members']``.
"""
import copy

import numpy as np

from . import bem, grid, packer, solver
from .member import Member

_MATS6 = ("M_struc", "B_struc", "C_struc", "C_hydro", "C_moor", "C_elast")


class _RefNode:
    def __init__(self, r):
        self.r = np.array(r, dtype=float)


class FOWT:
    def __init__(self, design, w, mpb=None, depth=600, x_ref=0, y_ref=0, heading_adjust=0, matrices=None, k=None):
        self.design = design
        self.w = np.array(w, dtype=float)
        self.nw = len(self.w)
        self.dw = self.w[1] - self.w[0]
        self.depth = float(depth)
        self.k = grid.wave_number(self.w, self.depth) if k is None else np.array(k, dtype=float)
        self.x_ref, self.y_ref, self.heading_adjust = float(x_ref), float(y_ref), float(heading_adjust)
        site = design.get("site", {})
        self.rho_water = float(site.get("rho_water", 1025.0))
        self.g = float(site.get("g", 9.81))
        self.nDOF = self.nFullDOF = 6
        self.nrotors = 0
        self.body, self.ms, self.moorMod = mpb, None, 0
        plat = design["platform"]
        self.yawstiff = plat.get("yaw_stiffness", 0)                   # raft_fowt.py:377-380
        self.potModMaster = int(plat.get("potModMaster", 0))
        dlsMax = float(plat.get("dlsMax", 5.0))
        names = [m["name"] for m in plat["members"]]
        if len(names) != len(set(names)):
            raise Exception("Member names must be unique. Please check the input data.")
        self.memberList = []
        for mi in plat["members"]:
            mi = copy.deepcopy(mi)
            if self.potModMaster == 1:
                mi["potMod"] = False
            elif self.potModMaster in (2, 3):
                mi["potMod"] = True
            mi.setdefault("dlsMax", dlsMax)
            heads = mi.get("heading", 0.0)
            for h in (np.atleast_1d(heads) if not np.isscalar(heads) else [heads]):
                self.memberList.append(Member(mi, self.nw, heading=float(h) + self.heading_adjust, part_of="platform"))
        self.potMod = any(bool(m.potMod) for m in self.memberList)
        self.potFirstOrder = int(plat.get("potFirstOrder", 0))
        mats = dict(matrices or {})
        # second-order wave loads (raft_fowt.py:409-431): 0 none, 2 external QTF file <hydroPath>.12d (or an injected
        # table matrices['qtf'], ['qtf_w'], ['qtf_heads']); 1 (slender-body QTF) is outside the GPU path
        self.potSecOrder = int(plat.get("potSecOrder", 0) or 0)
        self.outFolderQTF = None
        if self.potSecOrder == 1:                                      # slender-body QTF on its own frequency grid (:411-426)
            if "min_freq2nd" not in plat or "max_freq2nd" not in plat:
                raise Exception("If potSecOrder==1, then both min_freq2nd and max_freq2nd must be specified in the platform input.")
            lo, hi = plat["min_freq2nd"], plat["max_freq2nd"]
            df = plat.get("df_freq2nd", lo)
            self.w1_2nd = np.arange(lo, hi + 0.5 * lo, df) * 2 * np.pi
            self.w2_2nd = self.w1_2nd.copy()
            self.k1_2nd = np.array([grid.wave_number(np.array([w_]), self.depth)[0] for w_ in self.w1_2nd])
            self.k2_2nd = self.k1_2nd.copy()
        if self.potSecOrder == 2:
            if "qtf" in mats:
                self.qtf = np.array(mats["qtf"], dtype=complex)
                self.w1_2nd = self.w2_2nd = np.array(mats["qtf_w"], dtype=float)
                self.heads_2nd = np.array(mats["qtf_heads"], dtype=float)
            else:
                if "hydroPath" not in plat:
                    raise Exception("If potSecOrder==2, then hydroPath must be specified in the platform input.")
                self.qtfPath = plat["hydroPath"] + ".12d"
                self.readQTF(self.qtfPath)
        for nm in _MATS6:
            setattr(self, nm, np.array(mats.get(nm, np.zeros([6, 6])), dtype=float))
        self.A_BEM = np.array(mats.get("A_BEM", np.zeros([6, 6, self.nw])), dtype=float)
        self.B_BEM = np.array(mats.get("B_BEM", np.zeros([6, 6, self.nw])), dtype=float)
        if "X_BEM" in mats:
            self.X_BEM = np.array(mats["X_BEM"], dtype=complex)
            self.BEM_headings = np.array(mats["BEM_headings"], dtype=float)
        self.B_gyro = np.zeros([6, 6, 0])
        # submerged rotors (MHK turbines), which this FOWT does not build: their inertial wave excitation as
        # packer.pack_rotor_excitation would pack it for the FOWT at x_ref = y_ref = 0 (dict(r3 [nR,3] hub positions relative
        # to the FOWT's reference point, G [nR,6,3]); pack_fowt adds (x_ref, y_ref)) and their reduced
        # added mass A_hydro_rotor [6,6], which calcHydroConstants adds to A_hydro_morison as the reference does
        # (raft_fowt.py:1616-1625)
        self.rotor_excitation = mats.get("rotor_excitation")
        self.A_hydro_rotor = np.array(mats.get("A_hydro_rotor", np.zeros([6, 6])), dtype=float)
        self.A_hydro_morison = np.zeros([6, 6])
        self.Xi = np.zeros([6, self.nw], dtype=complex)
        self.setPosition(np.array([self.x_ref, self.y_ref, 0, 0, 0, 0], dtype=float))

    # raft_fowt.py:754 ----------------------------------------------------------------------------------
    def setPosition(self, r6):
        self.r6 = np.array(r6, dtype=float)
        self.rigidBodyNode = _RefNode(self.r6)
        for mem in self.memberList:
            mem.setPosition(self.r6)

    def calcStatics(self):
        raise NotImplementedError("statics are outside the GPU hot path: inject M_struc, C_struc, C_hydro (DESIGN.md section 9)")

    # raft_fowt.py:1589-1625 -------------------------------------------------------------------------------
    def calcHydroConstants(self):
        A = np.zeros([6, 6])
        for mem in self.memberList:
            mem.calcHydroConstants(rho=self.rho_water, g=self.g, k_array=self.k if mem.MCF else None)
            A += mem.added_mass_6dof(self.r6[:3])
        self.A_hydro_morison = A + self.A_hydro_rotor
        self._batch = None
        return self.A_hydro_morison

    def pack(self):
        return packer.pack_fowt(self)

    def _get_batch(self):
        if getattr(self, "_batch", None) is None:
            self._batch = solver.DesignBatch(self.pack())
        return self._batch

    # raft_fowt.py:1646-1729 -------------------------------------------------------------------------------
    def solveEigen(self, display=0, outPath=None):
        """Natural frequencies [Hz] and mode shapes of the FOWT on the GPU -> (fns, modes), in the reference's order (the DOF
        claim for 6 DOFs, ascending otherwise) and with its exceptions.  Writing ``outPath`` and the ``display`` table are not
        provided."""
        if outPath is not None:
            raise NotImplementedError("solveEigen(outPath=...): writing the modes JSON is not provided")
        E = packer.pack_eigen(self)
        return solver.eigen_fns_modes(E["M"], E["C"], "dof" if self.nDOF == 6 else "ascending")

    # raft_fowt.py:1732-1888 -------------------------------------------------------------------------------
    def calcHydroExcitation(self, case, memberList=None):
        """Wave kinematics + linear excitation for ``case`` on the GPU; leaves nWaves, beta, zeta, F_BEM,
        F_hydro_iner like the reference (first wave train; multi-train cases loop over trains).  A submerged rotor's
        excitation goes to the last train only, as in the reference (raft_fowt.py:1861-1883): the trains form one group."""
        heads = np.atleast_1d(np.array(case.get("wave_heading", 0.0), dtype=float))
        self.nWaves = len(heads)
        trains = []
        for ih in range(self.nWaves):
            pick = lambda key, dflt: (case.get(key, dflt) if np.isscalar(case.get(key, dflt)) else case.get(key, dflt)[ih])
            trains.append(dict(wave_spectrum=pick("wave_spectrum", "JONSWAP"), wave_period=pick("wave_period", None),
                               wave_height=pick("wave_height", None), wave_heading=heads[ih], wave_gamma=pick("wave_gamma", 0.0)))
        table = packer.pack_cases(trains)                                  # ValueError on an unknown spectrum (:1774)
        if self.nWaves > 1:
            table["primary"] = np.zeros(self.nWaves, dtype=np.int32)
        self._cases = solver.CaseTable(table)
        self.beta = np.deg2rad(heads)
        out = solver.hydro_excitation(self._get_batch(), self._cases)
        self.zeta = out["zeta"]
        self.S = self.zeta ** 2 / (2 * self.dw)
        self.F_BEM = out["F_BEM"][0]
        self.F_hydro_iner = out["F_iner"][0]
        return self.F_hydro_iner

    # raft_fowt.py:2081-2128 -------------------------------------------------------------------------------
    def readQTF(self, flPath, ULEN=1):
        """Read a WAMIT .12d QTF file into self.qtf [nw1,nw2,nheads,6], self.w1_2nd, self.w2_2nd, self.heads_2nd."""
        self.qtf, self.w1_2nd, self.heads_2nd = bem.read_qtf(flPath, rho=self.rho_water, g=self.g, ULEN=ULEN)
        self.w2_2nd = self.w1_2nd.copy()
        self._batch = None

    # raft_fowt.py:1988-2078 -------------------------------------------------------------------------------
    def calcQTF_slenderBody(self, waveHeadInd, Xi0=None, verbose=False, iCase=None, iWT=None):
        """Slender-body difference-frequency QTF on the GPU for wave train ``waveHeadInd`` of the last
        calcHydroExcitation; ``Xi0`` [6,nw] motion RAOs on self.w (None: fixed body).  Leaves self.qtf
        [nw2,nw2,1,6] and self.heads_2nd = [beta] like the reference."""
        if self.potSecOrder != 1:
            raise RuntimeError("calcQTF_slenderBody needs potSecOrder 1 (min_freq2nd / max_freq2nd in the platform input)")
        if Xi0 is None:
            Xi0 = np.zeros([6, self.nw], dtype=complex)
        beta = float(self.beta[waveHeadInd])
        self.heads_2nd = [beta]
        Xi = np.array([np.interp(self.w1_2nd, self.w, np.asarray(Xi0)[a], left=0, right=0) for a in range(6)])   # :2021-2023
        q = solver.qtf_slender(self.pack(), [beta], Xi[None])
        self.qtf = np.ascontiguousarray(q[0][:, :, None, :])
        return self.qtf

    def _qtf_batch(self):
        """DesignBatch carrying self.qtf (read from a file, injected, or left by calcQTF_slenderBody)."""
        P = {k: v for k, v in self.pack().items() if not k.startswith(("qs_", "qtf"))}
        P.update(qtf=np.asarray(self.qtf, dtype=complex), qtf_w=np.asarray(self.w1_2nd, dtype=float),
                 qtf_heads=np.asarray(self.heads_2nd, dtype=float))
        return solver.DesignBatch(P)

    # raft_fowt.py:2158-2253 -------------------------------------------------------------------------------
    def calcHydroForce_2ndOrd(self, beta, S0, iCase=None, iWT=None, interpMode="qtf"):
        """Difference-frequency force amplitudes from the QTF table on the GPU: ``beta`` [rad], ``S0`` [nw] wave
        spectrum -> (f_mean [6], f [6,nw] real).  Only the reference's default ``interpMode='qtf'``."""
        if interpMode != "qtf":
            raise NotImplementedError("only interpMode='qtf' (the reference's default) is on the GPU path")
        S0 = np.asarray(S0, dtype=float)
        one = solver.CaseTable(dict(Hs=[0.0], Tp=[1.0], gamma=[0.0], beta_deg=[float(beta) * 57.29577951308232], spec=[0]),
                               zeta=np.sqrt(2.0 * S0 * self.dw)[None, :])
        out = solver.second_order_force(self._qtf_batch(), one)
        return out["F_2nd_mean"][0, 0], out["F_2nd"][0, 0]

    # raft_fowt.py:1891-1957 -------------------------------------------------------------------------------
    def calcHydroLinearization(self, Xi):
        """Linearised drag damping for response ``Xi`` [6,nw] (first wave train); also stores F_hydro_drag."""
        if not hasattr(self, "_cases"):
            raise RuntimeError("calcHydroExcitation must be called first (the reference needs mem.u as well)")
        one = solver.CaseTable({k: v[:1] for k, v in self._cases.arrays.items() if k != "primary"})
        out = solver.hydro_linearization(self._get_batch(), one, np.asarray(Xi, dtype=complex))
        self.B_hydro_drag = out["B_drag"][0, 0]
        self.F_hydro_drag = out["F_drag"][0, 0]
        self._Xi_lin = np.array(Xi, dtype=complex)
        return self.B_hydro_drag

    def calcDragExcitation(self, ih):
        """Drag excitation of wave train ``ih`` with the Bmat of the last calcHydroLinearization (:1940-1957)."""
        if not hasattr(self, "_Xi_lin"):
            raise RuntimeError("calcHydroLinearization must be called first")
        if ih == 0:
            return self.F_hydro_drag
        if ih < 0 or ih >= self._cases.n_cases:
            raise IndexError("wave train %d of %d" % (ih, self._cases.n_cases))
        # Bmat comes from train 0's linearisation about the Xi of the last calcHydroLinearization (raft_member.py:2128-2152):
        # one pass of the solver with train ih declared a secondary train of train 0 (cases.primary) and the loop started
        # at that Xi evaluates F = sum_nodes Bmat u[ih] with exactly those per-node coefficients.
        a = self._cases.arrays
        table = {k: a[k][[0, ih]] for k in ("Hs", "Tp", "gamma", "beta_deg", "spec")}
        table["primary"] = np.zeros(2, dtype=np.int32)
        Xi0 = np.broadcast_to(self._Xi_lin, (1, 2, 6, self.nw))
        out = solver.solve_dynamics(self._get_batch(), solver.CaseTable(table, Xi_init=Xi0), n_iter=0, want=("Xi", "status", "F_drag"))
        self.F_hydro_drag = out["F_drag"][0, 1]
        return self.F_hydro_drag
