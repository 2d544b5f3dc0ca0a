"""Model: host-side mirror of the reference's ``raft.Model`` for ``solveDynamics`` / ``analyzeCases``.

Reference: raft_model.py:30-176 (construction), :264-433 (analyzeCases), :966-1302 (solveDynamics).
The per-frequency work runs on the GPU through the C ABI; statics / mooring / aero are out of scope and are
injected per FOWT (see ``raft_b200.fowt``).  Farms: every FOWT is linearised independently on the GPU, then the
coupled 6N system (block-diagonal impedances + an injected array-mooring stiffness) is solved per frequency by
``raftk_system_solve`` (raft_model.py:1164-1216).
"""
import numpy as np

from . import grid, packer, solver
from .fowt import FOWT


class Model:
    def __init__(self, design, matrices=None, array_stiffness=None, channels=None, tension_jacobian=None, mean_tensions=None,
                 array_tension_jacobian=None, array_mean_tensions=None, rotors=None, turbine_constants=None, fatigue=None, stress=None):
        """``channels``: optional turbine output channels per FOWT (``packer.pack_turbine_channels`` dicts: nacelle
        accelerations, tower-base moment) -- the turbine itself is outside this path, its constants enter here.
        ``tension_jacobian`` [2L,6] / ``mean_tensions`` [2L] (one for every FOWT, or a list with None for a FOWT without its
        own lines) and ``array_tension_jacobian`` [2L,6N] / ``array_mean_tensions`` [2L]: the mooring line-end tensions of
        moorMod 0, standing in for fowt.ms / model.ms (MoorPy getCoupledStiffness(tensions=True)[1] and getTensions(), see
        ``packer.pack_mooring_tensions``) as ``array_stiffness`` stands in for getCoupledStiffnessA.
        ``rotors``: ``packer.pack_rotor_outputs`` of each FOWT for the cases ``analyzeCases`` will run (one dict for a single
        FOWT, a list with None for a FOWT without rotor outputs for an array): the rotors' control transfer functions, wind
        amplitudes, gains and operating points, standing in for Rotor.calcAero (CCBlade), as ``matrices`` stand in for the
        turbine's constants.
        ``turbine_constants``: per FOWT a list with one snapshot per case of the case table (a list of such lists for an
        array), each what the reference's calcTurbineConstants(case) leaves on the FOWT (a live FOWT or a dict with A_aero,
        B_aero, B_gyro; ``packer.pack_operating_points``).  Every case is then solved with its own aero-servo added mass and
        damping (raft_model.py:1005-1010, 1045-1046), on top of the case-independent ``matrices``; ``channels`` may then be
        a per-case list of ``pack_turbine_channels`` dicts per FOWT, taken after each case's calcTurbineConstants, so that
        Mbase's aero reaction and mean follow the case too.
        ``fatigue``: dict(m={channel name: Woehler exponent}, f_eq=1.0, method="dirlik", weights=None)
        (``solver.fatigue_options``), e.g. m={"Mbase": 4.0, "Tmoor": 3.0}: analyzeCases then adds, per case and FOWT,
        ``<name>_DEL`` of the named turbine channels ([nrot]) and ``Tmoor_DEL`` [2L] of the FOWT's lines,
        case_metrics[iCase]['array_mooring']['Tmoor_DEL'] of the array's, and with weights the lifetime DELs in
        results['fatigue'] (the same keys per FOWT, and 'array_mooring').  Without it the results are unchanged.
        ``stress``: dict(d=10.0, t=0.083, angles=None, m=None, f_eq=1.0, method="dirlik", weights=None, psd=False)
        (``solver.stress_options``): analyzeCases then adds, per case and FOWT with turbine channels, the tower-base axial
        stress around the circumference from each tower's Mbase (``solver.stress_ring``, helpers.getSigmaXPSD; a rigid tower
        has no side-side moment): ``sigmaX_avg/_std/_max/_min`` [nrot, nA], ``sigmaX_PSD`` [nrot, nA, nw] with psd,
        ``sigmaX_DEL`` [nrot, nA] with m, ``sigmaX_hot`` (``solver.stress_hot``), and with weights (and m)
        results['fatigue'][i]['sigmaX_DEL'] and ['sigmaX_hot'] of the lifetime.  Without it the results are unchanged."""
        s = design.setdefault("settings", {})
        min_freq, max_freq = float(s.get("min_freq", 0.01)), float(s.get("max_freq", 1.00))
        self.XiStart = float(s.get("XiStart", 0.1))
        self.nIter = int(s.get("nIter", 15))
        self.w = grid.make_w(min_freq, max_freq)
        self.nw = len(self.w)
        self.depth = float(design["site"]["water_depth"])
        self.k = grid.wave_number(self.w, self.depth)
        self.design = design
        self.fowtList, self.coords = [], []
        if "array" in design:
            keys, rows = design["array"]["keys"], design["array"]["data"]
            mats = matrices if isinstance(matrices, (list, tuple)) else [matrices] * len(rows)
            for i, row in enumerate(rows):
                info = dict(zip(keys, row))
                plats = design["platforms"] if "platforms" in design else [design["platform"]]     # raft_model.py:86-101
                d_i = dict(site=design["site"], platform=plats[int(info["platformID"]) - 1])
                self.fowtList.append(FOWT(d_i, self.w, depth=self.depth, x_ref=info["x_location"], y_ref=info["y_location"],
                                          heading_adjust=info.get("heading_adjust", 0), matrices=mats[i], k=self.k))
                self.coords.append([info["x_location"], info["y_location"]])
        else:
            self.fowtList.append(FOWT(design, self.w, depth=self.depth, matrices=matrices, k=self.k))
            self.coords.append([0.0, 0.0])
        self.nFOWT = len(self.fowtList)
        self.nDOF = 6 * self.nFOWT
        self.C_array = None if array_stiffness is None else np.array(array_stiffness, dtype=float)   # stands in for ms.getCoupledStiffnessA
        self.results = {}
        if self.nFOWT == 1 and isinstance(channels, (list, tuple)) and len(channels) > 1:
            channels = [channels]                                        # one FOWT's per-case list
        self.channels = list(channels) if isinstance(channels, (list, tuple)) else [channels] * self.nFOWT
        tc = turbine_constants
        if tc is not None and self.nFOWT == 1 and len(tc) and not isinstance(tc[0], (list, tuple)):
            tc = [tc]                                                    # one FOWT's per-case list
        if tc is not None and len(tc) != self.nFOWT:
            raise ValueError("turbine_constants: one per-case list per FOWT (%d), got %d" % (self.nFOWT, len(tc)))
        self.turbine_constants = None if tc is None else [list(t) for t in tc]
        per = lambda v: list(v) if isinstance(v, (list, tuple)) else [v] * self.nFOWT
        self.tensions = [None if J is None else packer.pack_mooring_tensions(dict(J=J, T0=T0))
                         for J, T0 in zip(per(tension_jacobian), per(mean_tensions))]
        self.array_tensions = (None if array_tension_jacobian is None else
                               packer.pack_mooring_tensions(dict(J=array_tension_jacobian, T0=array_mean_tensions)))
        self.rotors = per(rotors)
        for r in self.rotors:
            if r is not None and r["R"].shape[1] != 6:
                raise ValueError("rotors: the hub rows of a rigid FOWT must be [nrot, 6]")
        for t in self.tensions:
            if t is not None and t["J"].shape[1] != 6:
                raise ValueError("tension_jacobian must be [2L, 6]")
        if self.array_tensions is not None and self.array_tensions["J"].shape[1] != self.nDOF:
            raise ValueError("array_tension_jacobian must be [2L, %d]" % self.nDOF)
        self.fatigue = None if fatigue is None else solver.fatigue_options(fatigue)
        if self.fatigue is not None:
            known = {"Tmoor"} | {nm for ch in self.channels if ch is not None
                                 for nm, _ in (ch[0] if isinstance(ch, (list, tuple)) else ch)["names"]}
            missing = sorted(set(self.fatigue["m"]) - known)
            if missing:
                raise ValueError("fatigue=: no channel named %s" % missing)
        # FOWTs without turbine channels have no stress ring; when none has channels, stress= is refused like channels
        # without a tower-base moment
        have = [ch[0] if isinstance(ch, (list, tuple)) else ch for ch in self.channels if ch is not None]
        self.stress = solver.stress_options_for(stress, have or [dict(names=[])])
        for f in self.fowtList:
            f.calcHydroConstants()

    # raft_model.py:966-1302 -------------------------------------------------------------------------------
    def solveDynamics(self, case, tol=0.01, conv_plot=0, RAO_plot=0, display=0):
        """Response amplitudes for one load case -> self.Xi [nWaves+1, nDOF, nw] (last row zero, as :1195).  With
        ``turbine_constants`` the case's operating point is that of case ``case['iCase']`` of the table."""
        if self.turbine_constants is not None and "iCase" not in case:
            raise ValueError("solveDynamics: with turbine_constants the case must name its row of the case table (case['iCase'])")
        out = self._solve_batch([case], tol, icases=[int(case["iCase"])] if self.turbine_constants is not None else None)
        trains = out["Xi_trains"][0]                                      # [nWaves, nDOF, nw]
        Xi = np.zeros([len(trains) + 1, self.nDOF, self.nw], dtype=complex)
        Xi[:-1] = trains
        self.Xi = Xi
        for i, f in enumerate(self.fowtList):
            f.Xi = Xi[:, 6 * i:6 * i + 6, :]
            f.Xi_fullDOF = f.Xi
        self.results["response"] = {}
        return self.Xi

    # raft_model.py:264-433 (dynamics part) ---------------------------------------------------------------------
    def analyzeCases(self, display=0, meshDir=None, RAO_plot=False, cases=None, tol=0.01):
        """All load cases in ONE batched GPU call.  Positional arguments as the reference's
        ``analyzeCases(display=0, meshDir=..., RAO_plot=False)`` (raft_model.py:264; meshDir / RAO_plot concern the BEM mesh
        and plotting, outside this path and ignored); ``cases=``: list of case dicts (default: the design's table).
        Fills results['freq_rad'], results['Xi'] [nCases, nDOF, nw], results['status'] [nCases, nFOWT, 4], and per case and
        FOWT the saveTurbineOutputs statistics: PRP motions, turbine channels, wave_PSD and, with tension Jacobians, Tmoor_* of
        the FOWT's lines and case_metrics[iCase]['array_mooring'] of the array's (raft_fowt.py:2355-2399, raft_model.py:371-433;
        max / min = avg +- 3 std, Tmoor_PSD divided by w[0] as the reference does) and, with ``rotors``, the rotor entries
        omega / torque / bPitch / power and wind_PSD (raft_fowt.py:2610-2679; ``solver.rotor_metrics``)."""
        if cases is None:
            keys = self.design["cases"]["keys"]
            cases = [dict(zip(keys, row)) for row in self.design["cases"]["data"]]
        out = self._solve_batch(cases, tol)
        self.results["freq_rad"] = self.w
        self.results["Xi"] = out["Xi"]
        self.results["Xi_trains"] = out["Xi_trains"]
        self.results["status"] = out["status"]
        # response statistics per case and FOWT (raft_fowt.py:2299-2353; zero mean offsets: statics are out of scope).
        # getRMS / getPSD sum the squares over a case's wave trains (helpers.py:678-700), so the per-train device
        # reductions are combined here: std = sqrt(sum std_t^2), PSD = sum PSD_t (solver.combine_trains).
        nC = len(cases)
        owner = out["owner"]
        Xi_units = out["Xi_all"].reshape(len(owner), self.nFOWT, 6, self.nw)                  # [nTrains, nFOWT, 6, nw]
        sd_t, psd_t = solver.response_stats(Xi_units, self.w[1] - self.w[0])
        names = ("surge", "sway", "heave", "roll", "pitch", "yaw")
        ch_stats = [None if ch is None else self._channel_stats(ch, Xi_units[:, i], owner, nC) for i, ch in enumerate(self.channels)]
        # line-end tensions T = J Xi (moorMod 0): a FOWT's lines on its PRP motions through channel_stats (J constant over w),
        # the array's lines on the coupled response through farm_channel_stats; PSDs divided by w[0] (raft_fowt.py:2370, 2399)
        w0 = float(self.w[0])
        ten = [None if t is None else solver.channel_stats(np.repeat(t["J"][:, :, None], self.nw, axis=2) + 0j, Xi_units[:, i], w0)
               for i, t in enumerate(self.tensions)]
        arr = None if self.array_tensions is None else solver.farm_channel_stats(self.array_tensions["J"], out["Xi_all"], w0)
        dw = self.w[1] - self.w[0]
        rot = self._rotor_stats(cases, out, dw)
        fat = None if self.fatigue is None else self._fatigue(cases, out, Xi_units)
        sig = None if self.stress is None else self._stress(cases, out, Xi_units)
        self.results["case_metrics"] = {}
        for ic in range(nC):
            idx = np.nonzero(owner == ic)[0]
            sd, psd = solver.combine_trains(sd_t, psd_t, idx)
            self.results["case_metrics"][ic] = {}
            for i in range(self.nFOWT):
                m = {}
                for k_, nm in enumerate(names):
                    m[nm + "_avg"], m[nm + "_std"] = 0.0, sd[i, k_]
                    m[nm + "_max"], m[nm + "_min"] = 3 * sd[i, k_], -3 * sd[i, k_]
                    m[nm + "_PSD"] = psd[i, k_]
                    ra = np.zeros([len(idx) + 1, self.nw], dtype=complex)                     # all trains + the zero row (:1195)
                    ra[:-1] = Xi_units[idx, i, k_] * (57.29577951308232 if k_ >= 3 else 1.0)
                    m[nm + "_RA"] = ra
                if ch_stats[i] is not None:                                                   # raft_fowt.py:2401-2444, 2504-2538
                    ch = self.channels[i][ic] if isinstance(self.channels[i], (list, tuple)) else self.channels[i]
                    nrot = 1 + max(ir for _, ir in ch["names"])
                    sd_c, psd_c = solver.combine_trains(ch_stats[i][0], ch_stats[i][1], idx)
                    for k_, (nm, ir) in enumerate(ch["names"]):
                        solver.rotor_channel_entries(m, nm, ir, nrot, ch["avg"][k_], sd_c[k_], psd_c[k_])
                if ten[i] is not None:
                    m.update(solver.tension_metrics(self.tensions[i]["T0"], *solver.combine_trains(ten[i][0], ten[i][1], idx)))
                m["wave_PSD"] = (0.5 * np.abs(out["zeta"][idx]) ** 2 / dw).sum(axis=0)          # getPSD(zeta, dw) (:2608)
                if self.rotors[i] is not None:
                    k = rot[1][i]
                    m.update(solver.rotor_metrics(self.rotors[i], ic, rot[0][0][ic, k], rot[0][1][ic, k], dw))
                if fat is not None:
                    m.update(fat["case"][ic][i])
                if sig is not None and sig[i] is not None:
                    m.update(solver.stress_entries(sig[i], ic))
                self.results["case_metrics"][ic][i] = m
            if arr is not None:
                self.results["case_metrics"][ic]["array_mooring"] = solver.tension_metrics(self.array_tensions["T0"],
                                                                                           *solver.combine_trains(arr[0], arr[1], idx))
                if fat is not None and "array_mooring" in fat["case"][ic]:
                    self.results["case_metrics"][ic]["array_mooring"].update(fat["case"][ic]["array_mooring"])
        if fat is not None and fat["life"] is not None:
            self.results["fatigue"] = fat["life"]
        for i, r in enumerate(sig or []):
            if r is not None and "DEL_life" in r:
                self.results.setdefault("fatigue", {}).setdefault(i, {}).update(sigmaX_DEL=np.array(r["DEL_life"]),
                                                                                sigmaX_hot=solver.stress_hot(r))
        return self.results

    def _stress(self, cases, out, Xi_units):
        """The tower-base stress ring of every FOWT with turbine channels (``stress=``) on its trains Xi_units [nT, nFOWT, 6,
        nw]: each tower's Mbase coefficients (per case when ``channels`` is a per-case list) as the fore-aft moment.  -> per
        FOWT a solver.stress_ring result without the unit axis, or None."""
        o = self.stress
        owner = out["owner"]
        row0 = np.append(np.nonzero(np.diff(np.append(-1, owner)))[0], len(owner))
        first = row0[:-1]
        res = []
        for i, ch in enumerate(self.channels):
            if ch is None:
                res.append(None)
                continue
            per_case = isinstance(ch, (list, tuple))
            rows, _ = solver.stress_rows((ch[0] if per_case else ch)["names"])
            if per_case:
                fa = np.stack([np.asarray(ch[c]["coef"])[rows] for c in owner])[None]            # [1, nT, nrot, 6, nw]
                mean = np.stack([np.asarray(ch[owner[t]]["avg"])[rows] for t in first])[None, :, :, None]
                xi = Xi_units[None, :, i]
            else:
                fa, mean, xi = np.asarray(ch["coef"])[rows], np.asarray(ch["avg"])[rows][:, None], Xi_units[:, i]
            r = solver.stress_ring(xi, self.w, fa, None, o["angles"], o["d"], o["t"], m=o["m"], f_eq=o["f_eq"], method=o["method"],
                                   weights=o["weights"], case_row0=row0, psd=o["psd"], mean=mean, dw=self.w[1] - self.w[0])
            res.append({k: v[0] for k, v in r.items()} if per_case else r)
        return res

    def _fatigue(self, cases, out, Xi_units):
        """Fatigue DELs of every case (``fatigue=``) on the device: each FOWT's named turbine channels (their coefficients,
        per case when ``channels`` is a per-case list) and lines on its trains Xi_units [nT, nFOWT, 6, nw], the array's lines
        on the coupled response.  -> dict(case=[{FOWT i: entries, 'array_mooring': entries}], life={...} or None)."""
        o = self.fatigue
        nC, owner = len(cases), out["owner"]
        row0 = np.append(np.nonzero(np.diff(np.append(-1, owner)))[0], len(owner))
        kw = dict(case_row0=row0, f_eq=o["f_eq"], method=o["method"], weights=o["weights"], moments=False)
        case = [dict() for _ in range(nC)]
        life = {} if o["weights"] is not None else None

        def put(key, sel, r):
            for ic in range(nC):
                case[ic].setdefault(key, {}).update(solver.fatigue_entries(sel, r["DEL"][ic]))
            if life is not None:
                life.setdefault(key, {}).update(solver.fatigue_entries(sel, r["DEL_life"]))
        for i in range(self.nFOWT):
            ch = self.channels[i]
            if ch is not None:
                per_case = isinstance(ch, (list, tuple))
                sel = solver.fatigue_selection((ch[0] if per_case else ch)["names"], o["m"])
                if sel:
                    ks = [s_[1] for s_ in sel]
                    ms = [s_[3] for s_ in sel]
                    if per_case:
                        coef = np.stack([np.asarray(ch[c]["coef"])[ks] for c in owner])[None]      # [1, nT, nsel, 6, nw]
                        r = {k: v[0] for k, v in solver.fatigue(Xi_units[None, :, i], self.w, ms, coef=coef, **kw).items()}
                    else:
                        r = solver.fatigue(Xi_units[:, i], self.w, ms, coef=np.asarray(ch["coef"])[ks], **kw)
                    put(i, sel, r)
            if self.tensions[i] is not None and "Tmoor" in o["m"]:
                J = self.tensions[i]["J"]
                sel = [("Tmoor", k, k, float(o["m"]["Tmoor"])) for k in range(len(J))]
                put(i, sel, solver.fatigue(Xi_units[:, i], self.w, o["m"]["Tmoor"], R=J, **kw))
            for ic in range(nC):
                case[ic].setdefault(i, {})
        if self.array_tensions is not None and "Tmoor" in o["m"]:
            J = self.array_tensions["J"]
            sel = [("Tmoor", k, k, float(o["m"]["Tmoor"])) for k in range(len(J))]
            put("array_mooring", sel, solver.fatigue(out["Xi_all"], self.w, o["m"]["Tmoor"], R=J, **kw))
        return dict(case=case, life=life)

    def _channel_stats(self, ch, Xi, owner, nC):
        """Turbine channel statistics of one FOWT on its trains Xi [nT, 6, nw]: ``ch`` one pack_turbine_channels dict, or one
        per case (each train then takes its case's coefficients) -> (std [nT, nch], PSD [nT, nch, nw])."""
        dw = self.w[1] - self.w[0]
        if not isinstance(ch, (list, tuple)):
            return solver.channel_stats(ch["coef"], Xi, dw)[:2]
        if len(ch) != nC:
            raise ValueError("channels: a per-case list must hold one entry per case (%d), got %d" % (nC, len(ch)))
        sd, P, _ = solver.channel_stats(np.stack([ch[c]["coef"] for c in owner]), Xi[:, None], dw)
        return sd[:, 0], P[:, 0]

    def _ops(self, icases, owner, n_table=None):
        """The operating points of the trains (case ``icases[owner[t]]`` of the turbine constants) -> CaseTable ops, or None.
        ``n_table``: the case table's length, which every FOWT's list must have (analyzeCases)."""
        if self.turbine_constants is None:
            return None
        for i, tc in enumerate(self.turbine_constants):
            if n_table is not None and len(tc) != n_table:
                raise ValueError("turbine_constants: FOWT %d holds %d cases, the case table %d" % (i, len(tc), n_table))
            bad = [ic for ic in icases if not 0 <= ic < len(tc)]
            if bad:
                raise ValueError("turbine_constants: FOWT %d holds %d cases, case %d asked for" % (i, len(tc), bad[0]))
        P = packer.pack_operating_points([[tc[ic] for ic in icases] for tc in self.turbine_constants])
        return dict(op=P["op"][owner], A_w=P["A_w"], B_w=P["B_w"])

    def _rotor_stats(self, cases, out, dw):
        """Rotor statistics of every FOWT's rotors in one device call on the (coupled) response Xi_all [nTrains, 6N, nw]:
        FOWT i's hub rows read columns 6 i .. 6 i + 5.  -> ((std [nC, nrot, 3], PSD [nC, nrot, 3, nw]), per FOWT the slice of
        its rotors), or None without rotor inputs."""
        have = [i for i, r in enumerate(self.rotors) if r is not None]
        if not have:
            return None
        for i in have:
            if self.rotors[i]["C"].shape[0] != len(cases):
                raise ValueError("rotors: FOWT %d's are packed for %d cases, %d given" % (i, self.rotors[i]["C"].shape[0], len(cases)))
        cat = lambda k: np.concatenate([self.rotors[i][k] for i in have], axis=1 if k != "R" else 0)   # noqa: E731
        col0 = np.concatenate([np.full(len(self.rotors[i]["R"]), 6 * i) for i in have])
        first = np.nonzero(np.diff(np.append(-1, out["owner"])))[0]
        stats = solver.rotor_stats(cat("R"), cat("C"), cat("V_w"), cat("gains"), self.w, out["Xi_all"], dw,
                                   case_row0=np.append(first, len(out["owner"])), col0=col0)
        sl, k0 = [None] * self.nFOWT, 0
        for i in have:
            sl[i] = slice(k0, k0 + len(self.rotors[i]["R"]))
            k0 = sl[i].stop
        return stats, sl

    # raft_model.py:436-547 -------------------------------------------------------------------------------------
    def solveEigen(self, display=0, outPath=None):
        """Natural frequencies [Hz] and mode shapes of the floating system on the GPU -> (fns, modes), stored in
        results['eigen'].  The reference's assembly order: per FOWT M_struc + A_hydro_morison + A_BEM[:, :, 0] and
        C_struc + C_hydro + C_moor + C_elast on its diagonal block, yawstiff on its DOF 5, then the array mooring stiffness
        (``array_stiffness``, standing in for ms.getCoupledStiffnessA); its order of the modes (the DOF claim when every FOWT
        has 6 DOFs) and its exceptions.  Writing ``outPath`` and the ``display`` table are not provided."""
        if outPath is not None:
            raise NotImplementedError("solveEigen(outPath=...): writing the modes JSON is not provided")
        M_tot = np.zeros([self.nDOF, self.nDOF])
        C_tot = np.zeros([self.nDOF, self.nDOF])
        for i, fowt in enumerate(self.fowtList):
            i1, i2 = i * fowt.nDOF, (i + 1) * fowt.nDOF
            M_tot[i1:i2, i1:i2] += fowt.M_struc + fowt.A_hydro_morison + fowt.A_BEM[:, :, 0]
            C_tot[i1:i2, i1:i2] += fowt.C_struc + fowt.C_hydro + fowt.C_moor + fowt.C_elast
            C_tot[i1 + 5, i1 + 5] += fowt.yawstiff
        rigid = all(f.nDOF == 6 for f in self.fowtList)
        if self.C_array is not None:
            if not rigid:
                raise Exception('Currently, array-level mooring eigen analysis only supported for fully rigid FOWTs (6 DOFs).')
            C_tot += self.C_array
        fns, modes = solver.eigen_fns_modes(M_tot, C_tot, "dof" if rigid else "ascending")
        self.results['eigen'] = {'frequencies': fns, 'modes': modes}
        return fns, modes

    def _solve_batch(self, cases, tol, icases=None):
        table, owner, first = packer.pack_case_trains(cases)
        ops = self._ops(list(range(len(cases))) if icases is None else icases, owner, len(cases) if icases is None else None)
        ct = solver.CaseTable(table, ops=ops)
        nC = len(cases)
        packs = [f.pack() for f in self.fowtList]
        batch = solver.DesignBatch([{k: v for k, v in P.items() if not k.startswith("qs_")} for P in packs])
        want = ("Xi", "status", "B_drag", "F_drag", "F_iner", "F_BEM", "zeta")
        sec = [int(getattr(f, "potSecOrder", 0)) for f in self.fowtList]
        if any(s_ == 1 for s_ in sec):                                      # slender-body QTF inside the loop (raft_model.py:1106-1131)
            if not all(s_ == 1 for s_ in sec):
                raise NotImplementedError("mixing potSecOrder 1 with other settings in one array is not supported")
            o = solver.solve_dynamics_slender(packs, ct, n_iter=self.nIter, tol=tol, xi_start=self.XiStart, want=want)
            for i, f in enumerate(self.fowtList):
                f.qtf = np.ascontiguousarray(o["qtf"][i, -1][:, :, None, :])
                f.heads_2nd = [float(ct.arrays["beta_deg"][-1]) * 0.017453292519943295]
        else:
            if batch.n_qtf_w:                                               # potSecOrder 2 (raft_model.py:1035-1038)
                want += ("F_2nd", "F_2nd_mean")
            if self.nFOWT > 1 and self.C_array is not None:
                # coupled array: per-FOWT linearisation + block assembly + 6N x 6N solve in one device call (raft_model.py:1164-1216)
                o = solver.solve_dynamics_farm(batch, ct, C_arr=self.C_array, n_iter=self.nIter, tol=tol, xi_start=self.XiStart, want=want)
                if np.any(o["info"]):
                    raise np.linalg.LinAlgError("Singular matrix")          # np.linalg.inv at raft_model.py:1191
            else:
                o = solver.solve_dynamics(batch, ct, n_iter=self.nIter, tol=tol, xi_start=self.XiStart, want=want)
        if "primary" in table:                                              # secondary trains share their primary's B_drag
            o["B_drag"] = o["B_drag"][:, table["primary"]]
        st = o["status"][:, first]                                          # [nFOWT, nC, 4] (train 0 of every case)
        solver.raise_on_flags(st)                                           # raft_model.py:1089 (LinAlgError), :1098-1099 (NaN)
        w = self.w
        for i, f in enumerate(self.fowtList):
            P = f.pack()
            f.B_hydro_drag, f.F_hydro_drag = o["B_drag"][i, -1], o["F_drag"][i, -1]
            f.zeta, f.F_BEM, f.F_hydro_iner = o["zeta"][-1:], o["F_BEM"][i, -1:], o["F_iner"][i, -1:]
            last = np.nonzero(owner == nC - 1)[0]                           # the trains of the last case
            f.Fhydro_2nd = np.zeros([len(last), 6, self.nw], dtype=complex)
            f.Fhydro_2nd_mean = np.zeros([len(last), 6])
            if "F_2nd" in o:
                f.Fhydro_2nd[:] = o["F_2nd"][i, last]
                f.Fhydro_2nd_mean[:] = o["F_2nd_mean"][i, last]
            M = P["M0"][:, :, None] + self._tab(P, "A_w", ops, i, first[-1])
            B = (P["B0"] + f.B_hydro_drag)[:, :, None] + self._tab(P, "B_w", ops, i, first[-1])
            f.Z = -w ** 2 * M + 1j * w * B + P["C0"][:, :, None]             # raft_model.py:1086, 1155 (last case, its own aero)
        nT = ct.n_cases
        Xi_all = np.moveaxis(o["Xi"], 0, 1).reshape(nT, self.nDOF, self.nw)  # [nTrains, 6N, nw]
        if "Xi_sys" in o:
            Xi_all = o["Xi_sys"]                                            # coupled system response, computed on the device
        elif self.nFOWT > 1 and self.C_array is not None:
            # (slender-body QTF path) coupled system: Z_sys = blockdiag(Z_i) + C_array; F = Z_i Xi_i  (raft_model.py:1164-1216)
            Xi_all = self._couple(o, nT, ops)
        Xi_trains = [Xi_all[owner == ic] for ic in range(nC)]
        return dict(Xi=Xi_all[first], Xi_trains=Xi_trains, status=np.moveaxis(st, 0, 1), Xi_all=Xi_all, owner=owner, zeta=o["zeta"])

    @staticmethod
    def _tab(P, name, ops, i, t):
        """FOWT i's frequency-dependent A_w / B_w for train t: the design's plus the train's operating point (as the kernels
        sum them), 0.0 without either."""
        if ops is None:
            return P[name] if name in P else 0.0
        o = ops[name][i, ops["op"][t]]
        return P[name] + o if name in P else o

    def _couple(self, o, nC, ops=None):
        n, nw, w = self.nDOF, self.nw, self.w
        Xi = np.zeros([nC, n, nw], dtype=complex)
        packs = [f.pack() for f in self.fowtList]
        for c in range(nC):
            Z = np.zeros([nw, n, n], dtype=complex)
            F = np.zeros([nw, n], dtype=complex)
            for i, P in enumerate(packs):
                M = P["M0"][:, :, None] + Model._tab(P, "A_w", ops, i, c)
                B = (P["B0"] + o["B_drag"][i, c])[:, :, None] + Model._tab(P, "B_w", ops, i, c)
                Zi = np.moveaxis(-w ** 2 * M + 1j * w * B + P["C0"][:, :, None], 2, 0)     # [nw,6,6]
                Z[:, 6 * i:6 * i + 6, 6 * i:6 * i + 6] = Zi
                Fi = o["F_BEM"][i, c] + o["F_iner"][i, c] + o["F_drag"][i, c]
                if "F_2nd" in o:
                    Fi = Fi + o["F_2nd"][i, c]                              # raft_model.py:1212
                F[:, 6 * i:6 * i + 6] = np.moveaxis(Fi, 0, 1)
            Z += self.C_array[None, :, :]
            X, info = solver.system_solve(Z, F)
            if np.any(info):
                raise np.linalg.LinAlgError("singular system impedance matrix")
            Xi[c] = X.T
        return Xi
