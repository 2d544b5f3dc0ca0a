// raftk_slender.cuh -- slender-body difference-frequency QTF (potSecOrder 1): FOWT.calcQTF_slenderBody
// (raft_fowt.py:1988-2078), Member.calcQTF_slenderBody + correction_KAY (raft_member.py:1488-1792) and the second-order
// wave kinematics of helpers.py:239-373  (included by raftk.cu only).
//
// Two kernels per call.  k_slender_tables: per (case, node, frequency) first-order kinematics -- body displacement and
// transverse velocity, wave velocity and its gradient, relative axial velocity, pressure gradient --, per (case,
// member, frequency) the waterline quantities, and per (radius, frequency) the Hankel functions of the Kim & Yue
// correction; the reference recomputes all of these inside its frequency-pair loop.
// k_slender_pairs: one CTA per (frequency pair w2 >= w1, case); its threads split the strip nodes (and the members'
// waterline / Kim & Yue terms), evaluate Rainey's second-order terms and the second-order potential, and a fixed-order
// block reduction gives the six force components.  k_slender_fill adds the conjugate triangle.
//
// The reference's quirks are kept for parity (see oracle/raft_oracle.c): the amplitude factors of grad_u1, grad_pres1st
// and pot2ndOrd use cos/sin(deg2rad(beta)) of a heading already in radians; every use of the node velocity in the pair
// loop sees its transverse part only (in-place side effect of getWaveKin_axdivAcc) except nodeV_axial_rel.
#pragma once

#define SL_THREADS 64
#define SL_NODE_C 22          // complex numbers per (case, node, frequency): dr 3, vt 3, u 3, G 9, vax 1, gp 3
#define SL_MEM_C 10           // per (case, member, frequency): eta_r 1, ud_wl 3, a_wl 3, g_e1 3
#define SL_HANK 14            // Hankel orders -1 .. 12 per (radius, frequency) for the Kim & Yue correction
#define SL_DEG 0.017453292519943295

struct cx { double x, y; };
__host__ __device__ __forceinline__ cx mk(double a, double b = 0.0) { cx r; r.x = a; r.y = b; return r; }
__host__ __device__ __forceinline__ cx operator+(cx a, cx b) { return mk(a.x + b.x, a.y + b.y); }
__host__ __device__ __forceinline__ cx operator-(cx a, cx b) { return mk(a.x - b.x, a.y - b.y); }
__host__ __device__ __forceinline__ cx operator-(cx a) { return mk(-a.x, -a.y); }
__host__ __device__ __forceinline__ cx operator*(cx a, cx b) { return mk(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
__host__ __device__ __forceinline__ cx operator*(cx a, double s) { return mk(a.x * s, a.y * s); }
__host__ __device__ __forceinline__ cx operator*(double s, cx a) { return mk(a.x * s, a.y * s); }
__host__ __device__ __forceinline__ cx operator/(cx a, cx b) { const double d = b.x * b.x + b.y * b.y; return mk((a.x * b.x + a.y * b.y) / d, (a.y * b.x - a.x * b.y) / d); }
__host__ __device__ __forceinline__ cx operator/(cx a, double s) { return mk(a.x / s, a.y / s); }
__host__ __device__ __forceinline__ cx cj(cx a) { return mk(a.x, -a.y); }
__host__ __device__ __forceinline__ cx mulI(cx a) { return mk(-a.y, a.x); }       //  i a
__host__ __device__ __forceinline__ cx mulmI(cx a) { return mk(a.y, -a.x); }      // -i a
__host__ __device__ __forceinline__ cx cexpi(double t) { double s, c; sincos(t, &s, &c); return mk(c, s); }   // e^{i t}

struct c3 { cx v[3]; };
__host__ __device__ __forceinline__ c3 z3() { c3 r; r.v[0] = r.v[1] = r.v[2] = mk(0.0); return r; }
__host__ __device__ __forceinline__ c3 operator+(c3 a, c3 b) { c3 r; for (int i = 0; i < 3; i++) r.v[i] = a.v[i] + b.v[i]; return r; }
__host__ __device__ __forceinline__ c3 operator-(c3 a, c3 b) { c3 r; for (int i = 0; i < 3; i++) r.v[i] = a.v[i] - b.v[i]; return r; }
__host__ __device__ __forceinline__ c3 operator*(c3 a, cx s) { c3 r; for (int i = 0; i < 3; i++) r.v[i] = a.v[i] * s; return r; }
__host__ __device__ __forceinline__ c3 operator*(c3 a, double s) { c3 r; for (int i = 0; i < 3; i++) r.v[i] = a.v[i] * s; return r; }
__host__ __device__ __forceinline__ c3 cj(c3 a) { c3 r; for (int i = 0; i < 3; i++) r.v[i] = cj(a.v[i]); return r; }
__host__ __device__ __forceinline__ cx dotr(c3 a, const double *d) { return a.v[0] * d[0] + a.v[1] * d[1] + a.v[2] * d[2]; }
__host__ __device__ __forceinline__ cx dotc(c3 a, c3 b) { return a.v[0] * b.v[0] + a.v[1] * b.v[1] + a.v[2] * b.v[2]; }   // np.dot: no conjugation
__host__ __device__ __forceinline__ c3 vecr(const double *d, cx s) { c3 r; for (int i = 0; i < 3; i++) r.v[i] = s * d[i]; return r; }
struct m33 { cx a[3][3]; };
__host__ __device__ __forceinline__ c3 mul(const m33 &M, c3 x) { c3 r; for (int i = 0; i < 3; i++) r.v[i] = M.a[i][0] * x.v[0] + M.a[i][1] * x.v[1] + M.a[i][2] * x.v[2]; return r; }
__host__ __device__ __forceinline__ c3 mulc(const m33 &M, c3 x) { c3 r; for (int i = 0; i < 3; i++) r.v[i] = cj(M.a[i][0]) * x.v[0] + cj(M.a[i][1]) * x.v[1] + cj(M.a[i][2]) * x.v[2]; return r; }
// (a p1 p1' + b p2 p2') v   and   q q' v
__host__ __device__ __forceinline__ c3 projp(const double *p1, const double *p2, double a, double b, c3 v) { return vecr(p1, dotr(v, p1) * a) + vecr(p2, dotr(v, p2) * b); }
__host__ __device__ __forceinline__ c3 projq(const double *q, c3 v) { return vecr(q, dotr(v, q)); }
__host__ __device__ __forceinline__ void force6(c3 f, const double *r, cx (&F)[6])       // += translateForce3to6DOF(f, r)
{
    F[0] = F[0] + f.v[0]; F[1] = F[1] + f.v[1]; F[2] = F[2] + f.v[2];
    F[3] = F[3] + (f.v[2] * r[1] - f.v[1] * r[2]);
    F[4] = F[4] + (f.v[0] * r[2] - f.v[2] * r[0]);
    F[5] = F[5] + (f.v[1] * r[0] - f.v[0] * r[1]);
}

// helpers.py:239-278 getWaveKin_grad_u1
__host__ __device__ inline m33 sl_grad_u1(double w, double k, double beta, double h, const double *r)
{
    m33 G;
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) G.a[i][j] = mk(0.0);
    const double z = r[2];
    const double cosBeta = cos(beta * SL_DEG), sinBeta = sin(beta * SL_DEG);
    if (z <= 0 && k > 0) {
        double khz_xy, khz_z;
        if (k * h >= 10) { khz_xy = exp(k * z); khz_z = khz_xy; }
        else { khz_xy = cosh(k * (z + h)) / sinh(k * h); khz_z = sinh(k * (z + h)) / sinh(k * h); }
        const cx ph = cexpi(-(k * (cos(beta) * r[0] + sin(beta) * r[1])));
        cx aux = ph * (w * cosBeta);
        G.a[0][0] = mulmI(aux) * khz_xy * k * cosBeta;
        G.a[0][1] = mulmI(aux) * khz_xy * k * sinBeta;
        G.a[0][2] = aux * k * khz_z;
        aux = ph * (w * sinBeta);
        G.a[1][0] = G.a[0][1];
        G.a[1][1] = mulmI(aux) * khz_xy * k * sinBeta;
        G.a[1][2] = aux * k * khz_z;
        aux = mulI(ph * w);
        G.a[2][0] = G.a[0][2];
        G.a[2][1] = G.a[0][1];
        G.a[2][2] = aux * k * khz_xy;
    }
    return G;
}

// helpers.py:285-308 getWaveKin_grad_pres1st
__host__ __device__ inline c3 sl_grad_pres1st(double k, double beta, double h, const double *r, double rho, double g)
{
    c3 gr = z3();
    const double z = r[2];
    const double cosBeta = cos(beta * SL_DEG), sinBeta = sin(beta * SL_DEG);
    if (z <= 0 && k > 0) {
        double khz_xy, khz_z;
        if (k * h >= 10) { khz_xy = exp(k * z); khz_z = khz_xy; }
        else { khz_xy = cosh(k * (z + h)) / cosh(k * h); khz_z = sinh(k * (z + h)) / cosh(k * h); }
        const cx ph = cexpi(-(k * (cosBeta * r[0] + sinBeta * r[1])));
        gr.v[0] = (ph * (rho * g * khz_xy)) * mk(0.0, -k * cosBeta);
        gr.v[1] = (ph * (rho * g * khz_xy)) * mk(0.0, -k * sinBeta);
        gr.v[2] = ph * (rho * g * khz_z) * k;
    }
    return gr;
}

// helpers.py:188-236 getWaveKin at one frequency, unit amplitude
__host__ __device__ inline void sl_wave_kin(double beta, double w, double k, double h, const double *r, double rho, double g,
                                            c3 &u, c3 &ud, cx &pDyn)
{
    const cx zeta = cexpi(-(k * (cos(beta) * r[0] + sin(beta) * r[1])));
    const double z = r[2];
    u = z3(); ud = z3(); pDyn = mk(0.0);
    if (z <= 0) {
        double S_, C_, P_;
        if (k == 0.0) { S_ = 1.0; C_ = 99999.0; P_ = 99999.0; }
        else if (k * h > 89.4) { S_ = exp(k * z); C_ = exp(k * z); P_ = exp(k * z) + exp(-k * (z + 2.0 * h)); }
        else { S_ = sinh(k * (z + h)) / sinh(k * h); C_ = cosh(k * (z + h)) / sinh(k * h); P_ = cosh(k * (z + h)) / cosh(k * h); }
        u.v[0] = zeta * w * C_ * cos(beta);
        u.v[1] = zeta * w * C_ * sin(beta);
        u.v[2] = mulI(zeta * w) * S_;
        for (int c = 0; c < 3; c++) ud.v[c] = mulI(u.v[c] * w);
        pDyn = zeta * (rho * g) * P_;
    }
}

// helpers.py:149-184 getKinematics at one frequency: Xi6 = the 6 response amplitudes
__host__ __device__ inline void sl_kinematics(const double *r, const cx *Xi6, double w, c3 &dr, c3 &v, c3 &a)
{
    const cx th0 = Xi6[3], th1 = Xi6[4], th2 = Xi6[5];
    dr.v[0] = Xi6[0] + (th1 * r[2] - th2 * r[1]);
    dr.v[1] = Xi6[1] + (th2 * r[0] - th0 * r[2]);
    dr.v[2] = Xi6[2] + (th0 * r[1] - th1 * r[0]);
    for (int c = 0; c < 3; c++) { v.v[c] = mulI(dr.v[c] * w); a.v[c] = mulI(v.v[c] * w); }
}

// helpers.py:337-373 getWaveKin_pot2ndOrd (both wave components share the heading)
__host__ __device__ inline void sl_pot_2nd(double w1, double w2, double k1, double k2, double beta, double h, const double *r, double g,
                                           double rho, c3 &acc, cx &p)
{
    acc = z3(); p = mk(0.0);
    if (w1 == w2) return;
    const double b = beta * SL_DEG, cosB = cos(b), sinB = sin(b), z = r[2];
    if (z <= 0 && k1 > 0 && k2 > 0) {
        const double kx = k1 * cosB - k2 * cosB, ky = k1 * sinB - k2 * sinB;
        const double nk = sqrt(kx * kx + ky * ky);
        const double t1 = tanh(k1 * h), t2 = tanh(k2 * h);
        const double den12 = (w1 - w2) * (w1 - w2) / g - nk * tanh(nk * h), den21 = (w2 - w1) * (w2 - w1) / g - nk * tanh(nk * h);
        const cx g12 = mk(0.0, -g / (2 * w1)) * ((k1 * k1) * (1 - t1 * t1) - 2 * k1 * k2 * (1 + t1 * t2)) / den12;
        const cx g21 = mk(0.0, -g / (2 * w2)) * ((k2 * k2) * (1 - t2 * t2) - 2 * k2 * k1 * (1 + t2 * t1)) / den21;
        const cx aux = (g21 + cj(g12)) * 0.5;
        const double khz_xy = cosh(nk * (z + h)) / cosh(nk * h), khz_z = sinh(nk * (z + h)) / cosh(nk * h);
        const cx ph = cexpi(-(kx * r[0] + ky * r[1]));
        acc.v[0] = aux * khz_xy * ph; acc.v[1] = acc.v[0];
        acc.v[0] = acc.v[0] * ((w1 - w2) * kx);
        acc.v[1] = acc.v[1] * ((w1 - w2) * ky);
        acc.v[2] = mulI(aux * khz_z * ph) * ((w1 - w2) * nk);
        p = mulmI(aux * khz_xy * ph) * (rho * (w1 - w2));
    }
}

// Hankel function of the first kind H_n(x) = J_n + i Y_n, any integer order (H_{-n} = (-1)^n H_n)
__host__ __device__ inline cx sl_hankel1(int n, double x)
{
    const int m = n < 0 ? -n : n;
    cx hv = mk(jn(m, x), yn(m, x));
    return (n < 0 && (m & 1)) ? -hv : hv;
}
// raft_member.py:1700-1708 omega(k1R, k2R, n); h1 / h2: H_{-1..12}(k1 R), H_{-1..12}(k2 R) from the table (index order + 1)
__host__ __device__ inline cx sl_kay_omega(const cx *h1, const cx *h2, int n)
{
    const cx H_N_ii = (h1[n] - h1[n + 2]) * 0.5;
    const cx H_N_jj = cj(h2[n] - h2[n + 2]) * 0.5;
    const cx H_Nm1_ii = (h1[n + 1] - h1[n + 3]) * 0.5;
    const cx H_Nm1_jj = cj(h2[n + 1] - h2[n + 3]) * 0.5;
    return mk(1.0) / (H_Nm1_ii * H_N_jj) - mk(1.0) / (H_N_ii * H_Nm1_jj);
}

struct SlenderDev {
    int n_nodes, n_members, n_seg, nw;
    double depth, rho, g;
    const double *mem_q, *mem_p1, *mem_p2;
    const int *mem_mcf, *mem_wl;
    const double *mem_r_int, *mem_a_wl, *mem_rwl, *mem_R_wl;
    const int *mem_node_start;            // [Nm+1]
    const double *node_r, *node_v_side, *node_Ca_p1, *node_Ca_p2, *node_Ca_End, *node_v_end, *node_a_i;
    const int *seg_mem;
    const double *seg_z1, *seg_z2, *seg_R, *seg_rmid;
    const double *M_struc;
    const double *w, *k;                  // [nw] second-order grid (w1_2nd, k1_2nd)
};

// ------------------------------------------------------------------------------------------------
// tables: grid (n_nodes + n_members, n_cases), block SL_THREADS; thread loops over frequencies
// ------------------------------------------------------------------------------------------------
// One launch over units y = 0 .. gridDim.y-1 of a batch of designs: unit y is (design, case) = divmod(u0 + y, nC).  The
// design tables are concatenated (CSR: node / member / segment offsets [nD+1]; mem_node_start holds every design's own
// [n_members+1] starts, so design d's begin at mem_off[d] + d; seg_mem indexes the design's own members).  node_off NULL:
// one design, D as given.  Per unit the node and member tables are maxN / maxM rows apart; Th holds the Hankel rows of the
// designs from d0 on, each design's members then its segments.  Every design sees exactly the pointers, counts and loops
// of a single-design call, so a design's QTF has the same bits whichever batch, chunk or unit offset it is computed in.
struct SlenderLaunch {
    const int *node_off, *mem_off, *seg_off;
    int nC, u0, d0, maxN, maxM, maxS;
};

__device__ __forceinline__ SlenderDev sl_design(const SlenderDev &D, const SlenderLaunch &L, int d)
{
    if (!L.node_off) return D;
    SlenderDev V = D;
    const int n0 = L.node_off[d], m0 = L.mem_off[d], s0 = L.seg_off[d];
    V.n_nodes = L.node_off[d + 1] - n0; V.n_members = L.mem_off[d + 1] - m0; V.n_seg = L.seg_off[d + 1] - s0;
    V.mem_q += 3 * m0; V.mem_p1 += 3 * m0; V.mem_p2 += 3 * m0; V.mem_mcf += m0; V.mem_wl += m0;
    V.mem_r_int += 3 * m0; V.mem_a_wl += m0; V.mem_rwl += 3 * m0; V.mem_R_wl += m0;
    V.mem_node_start += m0 + d;
    V.node_r += 3 * n0; V.node_v_side += n0; V.node_Ca_p1 += n0; V.node_Ca_p2 += n0; V.node_Ca_End += n0; V.node_v_end += n0; V.node_a_i += n0;
    V.seg_mem += s0; V.seg_z1 += s0; V.seg_z2 += s0; V.seg_R += s0; V.seg_rmid += 3 * s0;
    V.M_struc += 36 * d;
    return V;
}

// first Hankel row of design d in Th
__device__ __forceinline__ size_t sl_th_row(const SlenderLaunch &L, int d)
{
    return L.node_off ? (size_t)(L.mem_off[d] - L.mem_off[L.d0]) + (L.seg_off[d] - L.seg_off[L.d0]) : 0;
}

__global__ void __launch_bounds__(SL_THREADS) k_slender_tables(SlenderDev D0, SlenderLaunch L, const double *beta_rad /*[nC]*/,
                                                               const cx *Xi /*[units][6][nw]*/, cx *Tn /*[units][maxN][nw][22]*/,
                                                               cx *Tm /*[units][maxM][nw][10]*/, cx *Th /*[rows][nw][14]*/)
{
    const int y = blockIdx.y, u = L.u0 + y, d = u / L.nC, c = u % L.nC, nw = D0.nw;
    const SlenderDev D = sl_design(D0, L, d);
    if ((int)blockIdx.x >= L.maxN + L.maxM) {
        // Hankel functions of the Kim & Yue correction: they depend on (radius, frequency) only, not on the pair or the case;
        // the design's first unit of the launch writes them
        if (y != 0 && c != 0) return;
        int x = blockIdx.x - L.maxN - L.maxM;
        if (x < L.maxM) { if (x >= D.n_members) return; }
        else { x -= L.maxM; if (x >= D.n_seg) return; x += D.n_members; }
        Th += sl_th_row(L, d) * nw * SL_HANK;
        const bool live = x < D.n_members ? (D.mem_mcf[x] != 0) : (D.mem_mcf[D.seg_mem[x - D.n_members]] != 0);
        const double R = x < D.n_members ? D.mem_R_wl[x] : D.seg_R[x - D.n_members];
        for (int t = threadIdx.x; t < nw * SL_HANK; t += SL_THREADS) {
            const int i = t / SL_HANK, n = t % SL_HANK - 1;
            Th[((size_t)x * nw + i) * SL_HANK + (n + 1)] = live ? sl_hankel1(n, D.k[i] * R) : mk(0.0);
        }
        return;
    }
    const double beta = beta_rad[c], h = D.depth;
    const cx *X = Xi + (size_t)y * 6 * nw;
    if ((int)blockIdx.x < L.maxN) {
        const int j = blockIdx.x;
        if (j >= D.n_nodes) return;
        int m = 0;
        while (D.mem_node_start[m + 1] <= j) m++;
        const double *r = D.node_r + 3 * j, *q = D.mem_q + 3 * m;
        for (int i = threadIdx.x; i < nw; i += SL_THREADS) {
            cx X6[6];
            for (int a = 0; a < 6; a++) X6[a] = X[(size_t)a * nw + i];
            c3 dr, v, acc, u, ud; cx pd;
            sl_kinematics(r, X6, D.w[i], dr, v, acc);
            sl_wave_kin(beta, D.w[i], D.k[i], h, r, D.rho, D.g, u, ud, pd);
            const m33 G = sl_grad_u1(D.w[i], D.k[i], beta, h, r);
            const cx vax = dotr(u - v, q);                      // nodeV_axial_rel, from the FULL node velocity (raft_member.py:1517)
            const c3 gp = sl_grad_pres1st(D.k[i], beta, h, r, D.rho, D.g);
            const c3 vt = v - projq(q, v);                      // transverse node velocity (side effect of getWaveKin_axdivAcc)
            cx *o = Tn + (((size_t)y * L.maxN + j) * nw + i) * SL_NODE_C;
            for (int a = 0; a < 3; a++) { o[a] = dr.v[a]; o[3 + a] = vt.v[a]; o[6 + a] = u.v[a]; o[19 + a] = gp.v[a]; }
            for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) o[9 + 3 * a + b] = G.a[a][b];
            o[18] = vax;
        }
    } else {
        const int m = blockIdx.x - L.maxN;
        if (m >= D.n_members) return;
        const double *p1 = D.mem_p1 + 3 * m, *p2 = D.mem_p2 + 3 * m, *r_int = D.mem_r_int + 3 * m;
        for (int i = threadIdx.x; i < nw; i += SL_THREADS) {
            cx X6[6];
            for (int a = 0; a < 6; a++) X6[a] = X[(size_t)a * nw + i];
            cx *o = Tm + (((size_t)y * L.maxM + m) * nw + i) * SL_MEM_C;
            for (int a = 0; a < SL_MEM_C; a++) o[a] = mk(0.0);
            if (D.mem_wl[m]) {                                     // raft_member.py:1524-1539
                c3 dr, v, acc, u, ud; cx eta;
                sl_kinematics(r_int, X6, D.w[i], dr, v, acc);
                sl_wave_kin(beta, D.w[i], D.k[i], h, r_int, 1.0, 1.0, u, ud, eta);
                o[0] = eta - dr.v[2];
                for (int a = 0; a < 3; a++) { o[1 + a] = ud.v[a]; o[4 + a] = acc.v[a]; }
            }
            const cx c1z = X6[3] * p1[1] - X6[4] * p1[0], c2z = X6[3] * p2[1] - X6[4] * p2[0];     // cross(theta, p)[2]
            for (int a = 0; a < 3; a++) o[7 + a] = (c1z * p1[a] + c2z * p2[a]) * (-D.g);
        }
    }
}

// one strip node's contribution to the pair (i1, i2): F += all force terms (raft_member.py:1556-1650)
__host__ __device__ inline void sl_node_terms(const SlenderDev &D, int m, int j, const cx *t1, const cx *t2, const m33 &O1, const m33 &O2,
                                              double w1, double w2, double k1, double k2, double beta, cx (&F)[6])
{
    const double *q = D.mem_q + 3 * m, *p1 = D.mem_p1 + 3 * m, *p2 = D.mem_p2 + 3 * m, *r = D.node_r + 3 * j;
    const double rho = D.rho, g = D.g, h = D.depth;
    const double Ca1 = D.node_Ca_p1[j], Ca2 = D.node_Ca_p2[j], CaE = D.node_Ca_End[j];
    const double v_i = D.node_v_side[j], v_e = D.node_v_end[j], a_i = D.node_a_i[j];
    c3 dr1, dr2, vt1, vt2, u1, u2, gp1, gp2;
    m33 G1, G2;
    for (int a = 0; a < 3; a++) {
        dr1.v[a] = t1[a]; vt1.v[a] = t1[3 + a]; u1.v[a] = t1[6 + a]; gp1.v[a] = t1[19 + a];
        dr2.v[a] = t2[a]; vt2.v[a] = t2[3 + a]; u2.v[a] = t2[6 + a]; gp2.v[a] = t2[19 + a];
    }
    for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) { G1.a[a][b] = t1[9 + 3 * a + b]; G2.a[a][b] = t2[9 + 3 * a + b]; }
    const cx vax1 = t1[18], vax2 = t2[18];

    c3 acc2; cx p2nd;
    sl_pot_2nd(w1, w2, k1, k2, beta, h, r, g, rho, acc2, p2nd);
    c3 f_2ndPot = projp(p1, p2, 1. + Ca1, 1. + Ca2, acc2) * (rho * v_i);
    const c3 conv_acc = (mul(G1, cj(u2)) + mulc(G2, u1)) * 0.25;
    c3 f_conv = projp(p1, p2, 1. + Ca1, 1. + Ca2, conv_acc) * (rho * v_i);
    // Rainey's axial-divergence acceleration (helpers.py:311-334)
    c3 f_axdv;
    {
        const c3 qv = vecr(q, mk(1.0));
        const cx dwdz1 = dotr(mul(G1, qv), q), dwdz2 = dotr(mul(G2, qv), q);
        const c3 a1 = vt1 - projq(q, vt1), a2 = vt2 - projq(q, vt2);
        const c3 b1 = u1 - projq(q, u1), b2 = u2 - projq(q, u2);
        c3 acc = cj(b2 - a2) * (dwdz1 * 0.25) + (b1 - a1) * (cj(dwdz2) * 0.25);
        acc = acc - projq(q, acc);
        f_axdv = projp(p1, p2, Ca1, Ca2, acc) * (rho * v_i);
    }
    m33 Gd1, Gd2;
    for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) { Gd1.a[a][b] = mulI(G1.a[a][b] * w1); Gd2.a[a][b] = mulI(G2.a[a][b] * w2); }
    const c3 acc_nabla = mul(Gd1, cj(dr2)) * 0.25 + mulc(Gd2, dr1) * 0.25;
    c3 f_nabla = projp(p1, p2, 1. + Ca1, 1. + Ca2, acc_nabla) * (rho * v_i);
    c3 f_rslb = projp(p1, p2, Ca1, Ca2, mul(O1, cj(vecr(q, vax2))) + mulc(O2, vecr(q, vax1))) * (-0.25 * 2);
    f_rslb = f_rslb * (rho * v_i);
    c3 u1a = u1 - vt1, u2a = u2 - vt2;
    m33 V1, V2;
    for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) { V1.a[a][b] = G1.a[a][b] + O1.a[a][b]; V2.a[a][b] = G2.a[a][b] + O2.a[a][b]; }
    c3 aux = (mul(V1, cj(projp(p1, p2, Ca1, Ca2, u2a))) + mulc(V2, projp(p1, p2, Ca1, Ca2, u1a))) * 0.25;
    aux = aux - projq(q, aux);
    f_rslb = f_rslb + aux * (rho * v_i);
    u1a = u1a - projq(q, u1a);
    u2a = u2a - projq(q, u2a);
    aux = (projp(p1, p2, Ca1, Ca2, mul(V1, cj(u2a))) + projp(p1, p2, Ca1, Ca2, mulc(V2, u1a))) * 0.25;
    f_rslb = f_rslb + aux * (-rho * v_i);
    // axial / end effects
    f_2ndPot = f_2ndPot + vecr(q, p2nd * a_i);
    f_2ndPot = f_2ndPot + projq(q, acc2) * (rho * v_e * CaE);
    f_conv = f_conv + projq(q, conv_acc) * (rho * v_e * CaE);
    f_nabla = f_nabla + projq(q, acc_nabla) * (rho * v_e * CaE);
    const cx p_nabla = dotc(gp1, cj(dr2)) * 0.25 + dotc(cj(gp2), dr1) * 0.25;
    f_nabla = f_nabla + vecr(q, p_nabla * a_i);
    const cx p_drop = dotc(projp(p1, p2, 1.0, 1.0, u1 - vt1), cj(projp(p1, p2, Ca1, Ca2, u2 - vt2))) * (-2 * 0.25 * 0.5 * rho);
    f_conv = f_conv + vecr(q, p_drop * a_i);
    u1a = projp(p1, p2, Ca1, Ca2, u1a);
    u2a = projp(p1, p2, Ca1, Ca2, u2a);
    f_conv = f_conv + (cj(u1a) * vax2 + u2a * cj(vax1)) * (0.25 * a_i * rho);
    force6(f_2ndPot, r, F); force6(f_conv, r, F); force6(f_axdv, r, F); force6(f_nabla, r, F); force6(f_rslb, r, F);
}

// member-level terms of the pair: relative-wave-elevation force at the waterline (raft_member.py:1655-1683) and the
// Kim & Yue correction (:1692-1792)
__host__ __device__ inline void sl_member_terms(const SlenderDev &D, int m, const cx *tm1, const cx *tm2, const cx *Th, int i1, int i2,
                                                double w1, double w2, double k1, double k2, double beta, cx (&F)[6])
{
    const double *p1 = D.mem_p1 + 3 * m, *p2 = D.mem_p2 + 3 * m;
    const double rho = D.rho, g = D.g, h = D.depth;
    if (D.mem_wl[m]) {
        const double a_i = D.mem_a_wl[m];
        const int jl = D.mem_node_start[m + 1] - 1;                // the loop variables keep the last submerged node's coefficients
        const bool any = D.mem_node_start[m + 1] > D.mem_node_start[m];
        const double Ca1 = any ? D.node_Ca_p1[jl] : 0.0, Ca2 = any ? D.node_Ca_p2[jl] : 0.0;
        c3 ud1, ud2, aw1, aw2, ge1, ge2;
        for (int a = 0; a < 3; a++) { ud1.v[a] = tm1[1 + a]; aw1.v[a] = tm1[4 + a]; ge1.v[a] = tm1[7 + a]; ud2.v[a] = tm2[1 + a]; aw2.v[a] = tm2[4 + a]; ge2.v[a] = tm2[7 + a]; }
        const cx er1 = tm1[0], er2 = tm2[0];
        c3 fe = (ud1 * cj(er2) + cj(ud2) * er1) * 0.25;
        fe = projp(p1, p2, 1. + Ca1, 1. + Ca2, fe) * (rho * a_i);
        const c3 ae = (aw1 * cj(er2) + cj(aw2) * er1) * 0.25;
        fe = fe - projp(p1, p2, Ca1, Ca2, ae) * (rho * a_i);
        fe = fe - (ge1 * cj(er2) + cj(ge2) * er1) * (0.25 * rho * a_i);
        force6(fe, D.mem_r_int + 3 * m, F);
    }
    if (D.mem_mcf[m]) {
        cx K[6];
        for (int a = 0; a < 6; a++) K[a] = mk(0.0);
        const double cosB = cos(beta), sinB = sin(beta);
        const double kx = k1 * cosB - k2 * cosB, ky = k1 * sinB - k2 * sinB;
        const double d1 = cosB * p1[0] + sinB * p1[1], d2 = cosB * p2[0] + sinB * p2[1];
        double pf[3] = { d1 * p1[0] + d2 * p2[0], d1 * p1[1] + d2 * p2[1], d1 * p1[2] + d2 * p2[2] };
        const double nrm = sqrt(pf[0] * pf[0] + pf[1] * pf[1] + pf[2] * pf[2]);
        for (int i = 0; i < 3; i++) pf[i] /= nrm;
        const double *rwl = D.mem_rwl + 3 * m;
        const cx ph = cexpi(-(kx * rwl[0] + ky * rwl[1]));
        {
            const double R = D.mem_R_wl[m], k1R = k1 * R, k2R = k2 * R;
            const cx *h1 = Th + ((size_t)m * D.nw + i1) * SL_HANK, *h2 = Th + ((size_t)m * D.nw + i2) * SL_HANK;
            cx Fwl = mk(0.0);
            for (int nn = 0; nn <= 10; nn++) Fwl = Fwl + mk(0.0, -rho * g * R * 2 / CUDART_PI / (k1R * k2R)) * sl_kay_omega(h1, h2, nn);
            force6(vecr(pf, ph * Fwl.x), rwl, K);
        }
        for (int s = 0; s < D.n_seg; s++) {
            if (D.seg_mem[s] != m) continue;
            const double z1 = D.seg_z1[s], z2 = D.seg_z2[s], R = D.seg_R[s], k1R = k1 * R, k2R = k2 * R;
            const double H = h / R, k1h = k1R * H, k2h = k2R * H;
            double Im, Ip;
            if (w1 == w2) {
                Im = 0.5 * (sinh((k1 + k2) * (z2 + h)) / (k1h + k2h) - (z2 + h) / h - sinh((k1 + k2) * (z1 + h)) / (k1h + k2h) + (z1 + h) / h);
                Ip = 0.5 * (sinh((k1 + k2) * (z2 + h)) / (k1h + k2h) + (z2 + h) / h - sinh((k1 + k2) * (z1 + h)) / (k1h + k2h) - (z1 + h) / h);
            } else {
                Im = 0.5 * (sinh((k1 + k2) * (z2 + h)) / (k1h + k2h) - sinh((k1 - k2) * (z2 + h)) / (k1h - k2h) - sinh((k1 + k2) * (z1 + h)) / (k1h + k2h) + sinh((k1 - k2) * (z1 + h)) / (k1h - k2h));
                Ip = 0.5 * (sinh((k1 + k2) * (z2 + h)) / (k1h + k2h) + sinh((k1 - k2) * (z2 + h)) / (k1h - k2h) - sinh((k1 + k2) * (z1 + h)) / (k1h + k2h) - sinh((k1 - k2) * (z1 + h)) / (k1h - k2h));
            }
            const double c1 = cosh(k1h), c2 = cosh(k2h);
            const cx *h1 = Th + ((size_t)(D.n_members + s) * D.nw + i1) * SL_HANK, *h2 = Th + ((size_t)(D.n_members + s) * D.nw + i2) * SL_HANK;
            cx dF = mk(0.0);
            for (int nn = 0; nn <= 10; nn++)
                dF = dF + mk(0.0, rho * g * R * 2 / CUDART_PI / (k1R * k2R)) * sl_kay_omega(h1, h2, nn)
                          * (k1h * k2h / sqrt(k1h * tanh(k1h)) / sqrt(k2h * tanh(k2h)) * (Im + Ip * nn * (nn + 1) / k1R / k2R) / c1 / c2);
            force6(vecr(pf, ph * dF.x), D.seg_rmid + 3 * s, K);
        }
        for (int a = 0; a < 6; a++) F[a] = F[a] + ((k1 < k2) ? cj(K[a]) : K[a]);
    }
}

// ------------------------------------------------------------------------------------------------
// pairs: grid (nw (nw + 1) / 2, units), block SL_THREADS.  qtf [units][nw][nw][6], upper triangle i2 >= i1.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SL_THREADS) k_slender_pairs(SlenderDev D0, SlenderLaunch L, const double *beta_rad, const cx *Xi, const cx *Tn,
                                                              const cx *Tm, const cx *Th, cx *qtf)
{
    __shared__ cx part[SL_THREADS][6];
    const int y = blockIdx.y, u = L.u0 + y, d = u / L.nC, c = u % L.nC, nw = D0.nw, tid = threadIdx.x;
    const SlenderDev D = sl_design(D0, L, d);
    Tn += (size_t)y * L.maxN * nw * SL_NODE_C;
    Tm += (size_t)y * L.maxM * nw * SL_MEM_C;
    Th += sl_th_row(L, d) * nw * SL_HANK;
    // pair index -> (i1, i2 >= i1), rows of decreasing length
    int i1 = 0, rem = blockIdx.x;
    while (rem >= nw - i1) { rem -= nw - i1; i1++; }
    const int i2 = i1 + rem;
    const double w1 = D.w[i1], w2 = D.w[i2], k1 = D.k[i1], k2 = D.k[i2], beta = beta_rad[c];
    const cx *X = Xi + (size_t)y * 6 * nw;
    cx F[6];
    for (int a = 0; a < 6; a++) F[a] = mk(0.0);
    if (!(w2 < w1)) {
        m33 O1, O2;                                               // OMEGA = -getH(1j w Xi[3:])
        {
            cx a1[3], a2[3];
            for (int a = 0; a < 3; a++) { a1[a] = mulI(X[(size_t)(3 + a) * nw + i1] * w1); a2[a] = mulI(X[(size_t)(3 + a) * nw + i2] * w2); }
            const cx z = mk(0.0);
            O1.a[0][0] = z; O1.a[0][1] = -a1[2]; O1.a[0][2] = a1[1]; O1.a[1][0] = a1[2]; O1.a[1][1] = z; O1.a[1][2] = -a1[0]; O1.a[2][0] = -a1[1]; O1.a[2][1] = a1[0]; O1.a[2][2] = z;
            O2.a[0][0] = z; O2.a[0][1] = -a2[2]; O2.a[0][2] = a2[1]; O2.a[1][0] = a2[2]; O2.a[1][1] = z; O2.a[1][2] = -a2[0]; O2.a[2][0] = -a2[1]; O2.a[2][1] = a2[0]; O2.a[2][2] = z;
        }
        for (int j = tid; j < D.n_nodes; j += SL_THREADS) {
            int m = 0;
            while (D.mem_node_start[m + 1] <= j) m++;
            const cx *t1 = Tn + ((size_t)j * nw + i1) * SL_NODE_C;
            const cx *t2 = Tn + ((size_t)j * nw + i2) * SL_NODE_C;
            sl_node_terms(D, m, j, t1, t2, O1, O2, w1, w2, k1, k2, beta, F);
        }
        for (int m = tid; m < D.n_members; m += SL_THREADS) {
            const cx *tm1 = Tm + ((size_t)m * nw + i1) * SL_MEM_C;
            const cx *tm2 = Tm + ((size_t)m * nw + i2) * SL_MEM_C;
            sl_member_terms(D, m, tm1, tm2, Th, i1, i2, w1, w2, k1, k2, beta, F);
        }
        if (tid == 0) {                                           // Pinkster IV: rotation of the first-order forces (raft_fowt.py:2044-2058)
            cx F1a[6], F1b[6];
            for (int a = 0; a < 6; a++) {
                cx s1 = mk(0.0), s2 = mk(0.0);
                for (int b = 0; b < 6; b++) {
                    s1 = s1 + X[(size_t)b * nw + i1] * (-w1 * w1) * D.M_struc[6 * a + b];
                    s2 = s2 + X[(size_t)b * nw + i2] * (-w2 * w2) * D.M_struc[6 * a + b];
                }
                F1a[a] = s1; F1b[a] = s2;
            }
            const cx x1[3] = { X[(size_t)3 * nw + i1], X[(size_t)4 * nw + i1], X[(size_t)5 * nw + i1] };
            const cx x2[3] = { cj(X[(size_t)3 * nw + i2]), cj(X[(size_t)4 * nw + i2]), cj(X[(size_t)5 * nw + i2]) };
            for (int half = 0; half < 2; half++) {
                const cx b0 = cj(F1b[3 * half]), b1 = cj(F1b[3 * half + 1]), b2 = cj(F1b[3 * half + 2]);
                const cx e0 = F1a[3 * half], e1 = F1a[3 * half + 1], e2 = F1a[3 * half + 2];
                F[3 * half + 0] = F[3 * half + 0] + ((x1[1] * b2 - x1[2] * b1) + (x2[1] * e2 - x2[2] * e1)) * 0.25;
                F[3 * half + 1] = F[3 * half + 1] + ((x1[2] * b0 - x1[0] * b2) + (x2[2] * e0 - x2[0] * e2)) * 0.25;
                F[3 * half + 2] = F[3 * half + 2] + ((x1[0] * b1 - x1[1] * b0) + (x2[0] * e1 - x2[1] * e0)) * 0.25;
            }
        }
    }
    for (int a = 0; a < 6; a++) part[tid][a] = F[a];
    __syncthreads();
    if (tid < 6) {                                                // fixed-order reduction over the CTA's threads
        cx s = mk(0.0);
        for (int t = 0; t < SL_THREADS; t++) s = s + part[t][tid];
        qtf[(((size_t)y * nw + i1) * nw + i2) * 6 + tid] = s;
    }
}

// Hermitian fill (raft_fowt.py:2068-2070): lower triangle = conj of the upper one.  grid (nw, units), block 64
__global__ void __launch_bounds__(64) k_slender_fill(int nw, cx *qtf)
{
    const int c = blockIdx.y, i2 = blockIdx.x;
    for (int t = threadIdx.x; t < i2 * 6; t += 64) {
        const int i1 = t / 6, a = t % 6;
        qtf[(((size_t)c * nw + i2) * nw + i1) * 6 + a] = cj(qtf[(((size_t)c * nw + i1) * nw + i2) * 6 + a]);
    }
}

// ------------------------------------------------------------------------------------------------
// The potSecOrder 1 flow on the device (raft_model.py:1106-1131): the glue between loop A, the QTF and loop B.
// ------------------------------------------------------------------------------------------------

// np.interp's complex path (real and imaginary parts separately) of helpers.getRAO's ratio, written with explicitly
// rounded operations so that no multiply-add is contracted: the bits are NumPy's.  getRAO divides a complex by a real
// zeta promoted to complex, i.e. NumPy's Smith division with a zero imaginary part.
__device__ __forceinline__ cx sl_rao(cx x, double z)
{
    if (!(fabs(z) > 1e-6)) return mk(0.0);
    const double rat = __ddiv_rn(0.0, z);
    const double scl = __ddiv_rn(1.0, __dadd_rn(z, __dmul_rn(0.0, rat)));
    return mk(__dmul_rn(__dadd_rn(x.x, __dmul_rn(x.y, rat)), scl), __dmul_rn(__dsub_rn(x.y, __dmul_rn(x.x, rat)), scl));
}

__device__ __forceinline__ double sl_lerp(double x, double x0, double x1, double y0, double y1, double inv_dx)
{
    const double slope = __dmul_rn(__dsub_rn(y1, y0), inv_dx);
    double r = __dadd_rn(__dmul_rn(slope, __dsub_rn(x, x0)), y0);
    if (isnan(r)) {                                   // NumPy tries the other end, then the flat segment
        r = __dadd_rn(__dmul_rn(slope, __dsub_rn(x, x1)), y1);
        if (isnan(r) && y0 == y1) r = y0;
    }
    return r;
}

// Motion RAOs of loop A on the second-order grid (raft_fowt.py:2021-2023, left = right = 0), zero for units whose loop A did
// not converge; units u < nC also write beta_rad[u] = beta_deg[u] * deg2rad.  grid (units), block 64.
__global__ void __launch_bounds__(64) k_slender_rao(int nC, int nw, int nw2, const double *w, const double *w2, const cx *Xi /*[units][6][nw]*/,
                                                    const double *zeta /*[nC][nw]*/, const int *status /*[units][4]*/,
                                                    const double *beta_deg, double *beta_rad, cx *rao /*[units][6][nw2]*/)
{
    const int u = blockIdx.x, c = u % nC;
    if (u < nC && threadIdx.x == 0) beta_rad[u] = __dmul_rn(beta_deg[u], 0.017453292519943295);
    const bool ok = status[(size_t)u * 4 + 1] == 1;
    const cx *X = Xi + (size_t)u * 6 * nw;
    const double *z = zeta + (size_t)c * nw;
    for (int t = threadIdx.x; t < 6 * nw2; t += 64) {
        const int a = t / nw2, i = t % nw2;
        const double x = w2[i];
        cx v = mk(0.0);
        if (ok && !(x > w[nw - 1]) && !(x < w[0])) {
            int j = 0, hi = nw - 1;                       // largest j with w[j] <= x
            if (x >= w[hi]) j = hi;
            else while (hi - j > 1) { const int mid = (j + hi) >> 1; if (w[mid] <= x) j = mid; else hi = mid; }
            const cx y0 = sl_rao(X[(size_t)a * nw + j], z[j]);
            if (j == nw - 1 || w[j] == x) v = y0;
            else {
                const cx y1 = sl_rao(X[(size_t)a * nw + j + 1], z[j + 1]);
                const double inv_dx = __ddiv_rn(1.0, __dsub_rn(w[j + 1], w[j]));
                v = mk(sl_lerp(x, w[j], w[j + 1], y0.x, y1.x, inv_dx), sl_lerp(x, w[j], w[j + 1], y0.y, y1.y, inv_dx));
            }
        }
        rao[((size_t)u * 6 + a) * nw2 + i] = v;
    }
}

// Loop B wrote every unit's outputs; where loop A did not converge they take loop A's values (kept in the workspace) and
// the second-order force and QTF are zero.  Where it did, passes add up and the flags are OR-ed.  Case rows of zeta are
// loop A's.  grid (units), block 256.
struct SlenderMerge {
    int nC, nw, nw2;
    const int *stA;
    const cx *XiA, *XlA, *FdA, *FiA, *FbA;
    const double *BdA, *zetaA;
    int *st;
    cx *Xi, *Xl, *Fd, *Fi, *Fb, *qtf;
    double *Bd, *zeta, *F2, *F2m;
};

__global__ void __launch_bounds__(256) k_slender_merge(SlenderMerge M)
{
    const int u = blockIdx.x, tid = threadIdx.x;
    const size_t n6 = (size_t)6 * M.nw, o6 = (size_t)u * n6;
    if (u < M.nC && M.zeta)
        for (int i = tid; i < M.nw; i += 256) M.zeta[(size_t)u * M.nw + i] = M.zetaA[(size_t)u * M.nw + i];
    const int *a = M.stA + (size_t)u * 4;
    int *s = M.st + (size_t)u * 4;
    if (a[1] == 1) {
        if (tid == 0) { s[0] = a[0] + s[0]; s[2] = a[2] | s[2]; }
        return;
    }
    if (tid < 4) s[tid] = a[tid];
    for (size_t t = tid; t < n6; t += 256) {
        M.Xi[o6 + t] = M.XiA[o6 + t];
        if (M.Xl) M.Xl[o6 + t] = M.XlA[o6 + t];
        if (M.Fd) M.Fd[o6 + t] = M.FdA[o6 + t];
        if (M.Fi) M.Fi[o6 + t] = M.FiA[o6 + t];
        if (M.Fb) M.Fb[o6 + t] = M.FbA[o6 + t];
        if (M.F2) M.F2[o6 + t] = 0.0;
    }
    if (M.Bd && tid < 36) M.Bd[(size_t)u * 36 + tid] = M.BdA[(size_t)u * 36 + tid];
    if (M.F2m && tid < 6) M.F2m[(size_t)u * 6 + tid] = 0.0;
    if (M.qtf) {
        const size_t nq = (size_t)M.nw2 * M.nw2 * 6;
        for (size_t t = tid; t < nq; t += 256) M.qtf[(size_t)u * nq + t] = mk(0.0);
    }
}
