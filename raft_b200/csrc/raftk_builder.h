// raftk_builder.h -- native (host C++) node-table builder for design families (included by raftk.cu only).
//
// Same formulas as raft_b200/batch_builder.py (which restates raft_member.py:190-271 strip discretisation, :325-362 frame and
// node positions, :1295-1357 / :1387-1448 per-node coefficients, :2061-2110 drag areas, raft_fowt.py:1625 A_hydro_morison),
// evaluated design by design in plain loops: a sweep shard of 1250 VolturnUS-S variants takes ~2 ms instead of ~80 ms of
// NumPy calls.  No CUDA in here: the tables are ordinary host arrays in the layout of raftk_designs.
#pragma once
#include <cmath>
#include <vector>

namespace rkb {

struct Node { double ls, cd_q, cd_p1, cd_p2, in_q, in_p1, in_p2, pa; };
struct MemberOut { double q[3], p1[3], p2[3], rA[3]; int circ; std::vector<Node> nodes; };

static inline double interp_station(double x, const double *xp, const double *fp, int n)
{
    // np.interp with the slope formula of batch_builder._interp_stations (repeated stations keep the left value)
    bool flat = true;
    for (int i = 1; i < n; i++) if (fp[i] != fp[0]) { flat = false; break; }
    if (flat) return fp[0];
    if (x <= xp[0]) return fp[0];
    if (x >= xp[n - 1]) return fp[n - 1];
    int cnt = 0;
    for (int i = 0; i < n; i++) cnt += (x >= xp[i]);
    int j = cnt - 1;
    if (j < 0) j = 0;
    if (j > n - 2) j = n - 2;
    const double x0 = xp[j], x1 = xp[j + 1], f0 = fp[j], f1 = fp[j + 1];
    if (x1 == x0) return f0;
    const double slope = (f1 - f0) / (x1 - x0);
    return slope * (x - x0) + f0;
}

static inline void matvec3(const double R[9], const double v[3], double o[3])
{
    // v @ R.T  (row vector times transpose) = R v, accumulated in NumPy's matmul order
    for (int a = 0; a < 3; a++) o[a] = v[0] * R[3 * a + 0] + v[1] * R[3 * a + 1] + v[2] * R[3 * a + 2];
}

// One member copy of one design.  Returns 0, or a negative code: -1 end point on the waterplane, -2 stations not ascending.
static int build_member(const raftk_family_member &M, int d, double rho, double g, const double Rp[9], const double r0[3],
                        MemberOut &out, double A[36], bool count_only = false)
{
    const int n = M.n_stations, nc = M.circular ? 1 : 2;
    const double PI = 3.141592653589793;
    double rA0[3], rB0[3];
    for (int a = 0; a < 3; a++) { rA0[a] = M.rA[3 * (size_t)d + a]; rB0[a] = M.rB[3 * (size_t)d + a]; }
    if (rA0[2] == 0.0 || rB0[2] == 0.0) return -1;
    double rAB0[3] = { rB0[0] - rA0[0], rB0[1] - rA0[1], rB0[2] - rA0[2] };
    const double L = std::sqrt(rAB0[0] * rAB0[0] + rAB0[1] * rAB0[1] + rAB0[2] * rAB0[2]);
    double gamma = M.gamma_deg;
    if (M.heading_deg != 0.0) {
        const double hr = M.heading_deg * (PI / 180.0);
        const double c = std::cos(hr), s = std::sin(hr);
        const bool vertical = rAB0[0] == 0.0 && rAB0[1] == 0.0;
        const double ax = c * rA0[0] + (-s) * rA0[1], ay = s * rA0[0] + c * rA0[1];
        const double bx = c * rB0[0] + (-s) * rB0[1], by = s * rB0[0] + c * rB0[1];
        rA0[0] = ax; rA0[1] = ay; rB0[0] = bx; rB0[1] = by;
        if (vertical) gamma += M.heading_deg;
    }
    if (M.circular) gamma = 0.0;
    const double *st = M.stations;
    for (int i = 1; i < n; i++) if (st[i] < st[i - 1]) return -2;
    static thread_local std::vector<double> s;               // scratch reused across calls: no allocation per member
    s.resize(n);
    for (int i = 0; i < n; i++) s[i] = ((st[i] - st[0]) / (st[n - 1] - st[0])) * L;
    const double *dd = M.d + (size_t)d * n * nc;           // [n][nc]

    // ---- strips (raft_member.py:190-271) ----
    struct Strip { double ls, dls, ds[2], drs[2]; };
    static thread_local std::vector<Strip> strips;
    strips.clear();
    {
        Strip t; t.ls = 0.0; t.dls = 0.0;
        for (int c = 0; c < nc; c++) { t.ds[c] = 0.5 * dd[c]; t.drs[c] = 0.5 * dd[c]; }
        strips.push_back(t);
    }
    for (int i = 1; i < n; i++) {
        const double lstrip = s[i] - s[i - 1];
        if (lstrip > 0.0) {
            const long ns = (long)std::ceil(lstrip / M.dls_max);
            const double dl = lstrip / (double)ns;
            double m[2];
            for (int c = 0; c < nc; c++) m[c] = 0.5 * (dd[i * nc + c] - dd[(i - 1) * nc + c]) / lstrip;
            for (long j = 0; j < ns; j++) {
                const double jj = 0.5 + (double)j;
                Strip t; t.ls = s[i - 1] + dl * jj; t.dls = dl;
                for (int c = 0; c < nc; c++) { t.ds[c] = dd[(i - 1) * nc + c] + ((dl * 2) * m[c]) * jj; t.drs[c] = dl * m[c]; }
                strips.push_back(t);
            }
        } else if (lstrip == 0.0) {
            Strip t; t.ls = s[i - 1]; t.dls = 0.0;
            for (int c = 0; c < nc; c++) { t.ds[c] = 0.5 * (dd[(i - 1) * nc + c] + dd[i * nc + c]); t.drs[c] = 0.5 * (dd[i * nc + c] - dd[(i - 1) * nc + c]); }
            strips.push_back(t);
        } else return -2;
    }
    {
        Strip t; t.ls = s[n - 1]; t.dls = 0.0;
        for (int c = 0; c < nc; c++) { t.ds[c] = 0.5 * dd[(n - 1) * nc + c]; t.drs[c] = -0.5 * dd[(n - 1) * nc + c]; }
        strips.push_back(t);
    }

    // ---- frame (raft_member.py:325-357) ----
    double rAB[3] = { rB0[0] - rA0[0], rB0[1] - rA0[1], rB0[2] - rA0[2] };
    const double nrm = std::sqrt(rAB[0] * rAB[0] + rAB[1] * rAB[1] + rAB[2] * rAB[2]);
    double q[3] = { rAB[0] / nrm, rAB[1] / nrm, rAB[2] / nrm };
    const double beta = std::atan2(q[1], q[0]);
    const double phi = std::atan2(std::sqrt(q[0] * q[0] + q[1] * q[1]), q[2]);
    const double s1 = std::sin(beta), c1 = std::cos(beta), s2 = std::sin(phi), c2 = std::cos(phi);
    const double gr = gamma * (PI / 180.0);
    const double s3 = std::sin(gr), c3 = std::cos(gr);
    double p1[3] = { c1 * c2 * c3 - s1 * s3, c1 * s3 + c2 * c3 * s1, -c3 * s2 };
    double p2[3] = { q[1] * p1[2] - q[2] * p1[1], q[2] * p1[0] - q[0] * p1[2], q[0] * p1[1] - q[1] * p1[0] };
    double t[3], rA[3], rB[3];
    matvec3(Rp, rA0, t);
    for (int a = 0; a < 3; a++) rA[a] = r0[a] + t[a];
    matvec3(Rp, q, t);  for (int a = 0; a < 3; a++) q[a] = t[a];
    matvec3(Rp, p1, t); for (int a = 0; a < 3; a++) p1[a] = t[a];
    matvec3(Rp, p2, t); for (int a = 0; a < 3; a++) p2[a] = t[a];
    for (int a = 0; a < 3; a++) rB[a] = rA[a] + L * q[a];
    for (int a = 0; a < 3; a++) { out.q[a] = q[a]; out.p1[a] = p1[a]; out.p2[a] = p2[a]; out.rA[a] = rA[a]; }
    out.circ = M.circular ? 1 : 0;
    out.nodes.clear();

    const double pref = 1.5957691216057308 * 0.5 * rho;       // sqrt(8/pi) rho / 2  (packer.SQRT_8_OVER_PI)
    for (const Strip &S : strips) {
        const double f = S.ls / L;
        double r[3];
        for (int a = 0; a < 3; a++) r[a] = rA[a] + f * (rB[a] - rA[a]);
        if (!(r[2] < 0.0)) continue;                                                       // submerged nodes only
        if (count_only) { Node N0 = {}; out.nodes.push_back(N0); continue; }                 // raftk_family_sizes: positions suffice
        const double dls = S.dls;
        double v, v_end, a_i, a_q, a_p1, a_p2, a_End;
        if (M.circular) {
            const double D = S.ds[0], DR = S.drs[0];
            v = 0.25 * PI * (D * D) * dls;
            const double u = D + DR, w_ = D - DR;
            v_end = PI / 12.0 * std::fabs(u * u * u - w_ * w_ * w_);
            a_i = PI * D * DR;
            a_q = PI * D * dls; a_p1 = D * dls; a_p2 = D * dls;
            a_End = std::fabs(PI * D * DR);
        } else {
            v = S.ds[0] * S.ds[1] * dls;
            const double mp = ((S.ds[0] + S.drs[0]) + (S.ds[1] + S.drs[1])) / 2.0, mm = ((S.ds[0] - S.drs[0]) + (S.ds[1] - S.drs[1])) / 2.0;
            v_end = PI / 12.0 * (mp * mp * mp - mm * mm * mm);
            a_i = (S.ds[0] + S.drs[0]) * (S.ds[1] + S.drs[1]) - (S.ds[0] - S.drs[0]) * (S.ds[1] - S.drs[1]);
            a_q = 2 * (S.ds[0] + S.ds[0]) * dls;                                           // sic, raft_member.py:2070
            a_p1 = S.ds[0] * dls; a_p2 = S.ds[1] * dls;
            a_End = std::fabs(a_i);
        }
        const double Cd_q = interp_station(S.ls, s.data(), M.Cd_q, n), Cd_p1 = interp_station(S.ls, s.data(), M.Cd_p1, n);
        const double Cd_p2 = interp_station(S.ls, s.data(), M.Cd_p2, n), Cd_End = interp_station(S.ls, s.data(), M.Cd_End, n);
        Node N;
        N.ls = S.ls;
        N.cd_q = pref * (a_q * Cd_q + a_End * Cd_End);
        N.cd_p1 = pref * a_p1 * Cd_p1;
        N.cd_p2 = pref * a_p2 * Cd_p2;
        if (M.pot_mod) { N.in_q = N.in_p1 = N.in_p2 = N.pa = 0.0; }
        else {
            const double Ca_p1 = interp_station(S.ls, s.data(), M.Ca_p1, n), Ca_p2 = interp_station(S.ls, s.data(), M.Ca_p2, n);
            const double Ca_End = interp_station(S.ls, s.data(), M.Ca_End, n);
            if (r[2] + 0.5 * dls > 0.0) v = v * (0.5 * dls - r[2]) / dls;                    // strip piercing the waterplane
            const double ad_p1 = rho * v * Ca_p1, ad_p2 = rho * v * Ca_p2, ad_q = rho * v_end * Ca_End;
            N.in_p1 = rho * v * (1.0 + Ca_p1); N.in_p2 = rho * v * (1.0 + Ca_p2); N.in_q = rho * v_end * Ca_End;
            N.pa = rho * g * a_i;
            // A_hydro_morison += translateMatrix3to6DOF(Amat, r - r_ref)  (raft_member.py:1361; helpers.py:537-560)
            double m[3][3], H[3][3] = { { 0, 0, 0 }, { 0, 0, 0 }, { 0, 0, 0 } };
            for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++)
                m[a][b] = (ad_p1 * (p1[a] * p1[b]) + ad_p2 * (p2[a] * p2[b])) + ad_q * (q[a] * q[b]);
            const double rr[3] = { r[0] - r0[0], r[1] - r0[1], r[2] - r0[2] };
            H[0][1] = rr[2]; H[0][2] = -rr[1]; H[1][0] = -rr[2]; H[1][2] = rr[0]; H[2][0] = rr[1]; H[2][1] = -rr[0];
            double mH[3][3], HmH[3][3];
            for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) { double x = 0; for (int l = 0; l < 3; l++) x += m[a][l] * H[l][b]; mH[a][b] = x; }
            for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) {                     // H m H^T
                double x = 0;
                for (int l = 0; l < 3; l++) { double y = 0; for (int k = 0; k < 3; k++) y += m[l][k] * H[b][k]; x += H[a][l] * y; }
                HmH[a][b] = x;
            }
            for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) {
                A[6 * a + b] += m[a][b];
                A[6 * a + 3 + b] += mH[a][b];
                A[6 * (3 + a) + b] += mH[b][a];
                A[6 * (3 + a) + 3 + b] += HmH[a][b];
            }
        }
        out.nodes.push_back(N);
    }
    return 0;
}

// step-class counts of one design by the fused kernels' rule (raftk_fused.cuh step_classes_warp): greedy in node order,
// a key joins the first class within the tolerance of its own key, else opens one (solver.DesignBatch._step_classes)
static void count_classes(const std::vector<MemberOut> &mem, int &nW, int &nH, int &nZ)
{
    std::vector<double> wk, hk, zk;
    for (const MemberOut &M : mem) {
        if (M.nodes.empty()) continue;
        const double z0 = M.rA[2] + M.nodes[0].ls * M.q[2];
        bool seen = false;
        for (double a : zk) if (std::fabs(a - z0) <= Z0_RTOL * std::fmax(1.0, std::fabs(z0))) { seen = true; break; }
        if (!seen) zk.push_back(z0);
        for (size_t j = 1; j < M.nodes.size(); j++) {
            const double step = M.nodes[j].ls - M.nodes[j - 1].ls;
            const double kx = M.q[0] * step, ky = M.q[1] * step, kz = M.q[2] * step;
            if (std::fabs(kx) > STEP_ZERO || std::fabs(ky) > STEP_ZERO) {
                const double tol = STEP_RTOL * (std::fabs(kx) + std::fabs(ky));
                bool s2 = false;
                for (size_t x = 0; x + 1 < wk.size(); x += 2) if (std::fabs(wk[x] - kx) <= tol && std::fabs(wk[x + 1] - ky) <= tol) { s2 = true; break; }
                if (!s2) { wk.push_back(kx); wk.push_back(ky); }
            }
            if (std::fabs(kz) > STEP_ZERO) {
                bool s3 = false;
                for (double a : hk) if (std::fabs(a - kz) <= STEP_RTOL * std::fabs(kz)) { s3 = true; break; }
                if (!s3) hk.push_back(kz);
            }
        }
    }
    nW = (int)(wk.size() / 2); nH = (int)hk.size(); nZ = (int)zk.size();
}

}  // namespace rkb
