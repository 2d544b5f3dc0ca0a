// A/B for the 6 x 6 complex impedance solve (north-star: "one warp owning one system in registers ... warp-shuffle elimination";
// product: one THREAD per system, whole augmented matrix in registers -- raftk_common.cuh:solve6).
//   variant T: thread per system, the product's solve6 (254 registers, 8 warps per SM)
//   variant W: 8 lanes per system (4 systems per warp): lane c holds column c of the augmented 6 x 7 system (12 registers of matrix),
//              pivot row and multipliers broadcast with __shfl_sync inside the 8-lane group, full occupancy
// Both read Z = C - w^2 M + i w B and F from global tables and write Xi; same pivot rule (|re| + |im|, first maximum).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o tools/micro/lu6_ab.bin tools/micro/lu6_ab.cu
#include <cstdio>
#include <cmath>
#include <type_traits>
#include <vector>
#include <cuda_runtime.h>
#include "../../raft_b200/csrc/raftk_common.cuh"

__global__ void __launch_bounds__(128, 2) k_thread(const double *M, const double *B, const double *C, const double *w, const double2 *F, double2 *X, int n)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double ar[6][6], ai[6][6], br[6], bi[6];
    const double ww = w[i], w2 = ww * ww;
#pragma unroll
    for (int a = 0; a < 6; a++)
#pragma unroll
        for (int b = 0; b < 6; b++) { ar[a][b] = fma(-w2, M[6 * a + b], C[6 * a + b]); ai[a][b] = ww * B[6 * a + b]; }
#pragma unroll
    for (int a = 0; a < 6; a++) { const double2 f = F[(size_t)a * n + i]; br[a] = f.x; bi[a] = f.y; }
    solve6(ar, ai, br, bi);
#pragma unroll
    for (int a = 0; a < 6; a++) X[(size_t)a * n + i] = make_double2(br[a], bi[a]);
}

// lane c (0..6) of an 8-lane group holds column c: cr[r], ci[r], r = 0..5 (c == 6: right-hand side)
__global__ void __launch_bounds__(256) k_warp(const double *M, const double *B, const double *C, const double *w, const double2 *F, double2 *X, int n)
{
    const int lane = threadIdx.x & 31, c = lane & 7, g = lane >> 3;
    const int sys = (blockIdx.x * blockDim.x + threadIdx.x) / 32 * 4 + g;
    const bool live = sys < n;
    const int i = live ? sys : 0;
    double cr[6], ci[6];
    const double ww = w[i], w2 = ww * ww;
    const int cc = c < 6 ? c : 0;
#pragma unroll
    for (int r = 0; r < 6; r++) {
        if (c < 6) { cr[r] = fma(-w2, M[6 * r + cc], C[6 * r + cc]); ci[r] = ww * B[6 * r + cc]; }
        else { const double2 f = F[(size_t)r * n + i]; cr[r] = f.x; ci[r] = f.y; }
    }
    const unsigned full = 0xffffffffu;
#pragma unroll
    for (int k = 0; k < 6; k++) {
        // owner of column k (lane k of the group) finds the pivot row and the multipliers
        int p = k; double best = fabs(cr[k]) + fabs(ci[k]);
#pragma unroll
        for (int r = k + 1; r < 6; r++) { const double t = fabs(cr[r]) + fabs(ci[r]); if (t > best) { best = t; p = r; } }
        p = __shfl_sync(full, p, k, 8);
        // row swap k <-> p in every column (register selects: p is dynamic)
        {
            double pr = cr[k], pi = ci[k];
#pragma unroll
            for (int r = k + 1; r < 6; r++) if (r == p) { const double tr = cr[r], ti = ci[r]; cr[r] = pr; ci[r] = pi; pr = tr; pi = ti; }
            cr[k] = pr; ci[k] = pi;
        }
        const double dr = __shfl_sync(full, cr[k], k, 8), di = __shfl_sync(full, ci[k], k, 8);
        const double inv = 1.0 / (dr * dr + di * di), rr = dr * inv, ri = -di * inv;
#pragma unroll
        for (int r = k + 1; r < 6; r++) {
            const double ar_ = __shfl_sync(full, cr[r], k, 8), ai_ = __shfl_sync(full, ci[r], k, 8);     // a_rk from the owner of column k
            const double lr = ar_ * rr - ai_ * ri, li = ar_ * ri + ai_ * rr;
            if (c > k) { cr[r] -= lr * cr[k] - li * ci[k]; ci[r] -= lr * ci[k] + li * cr[k]; }
        }
    }
    // back substitution on the right-hand-side lane (c == 6): needs U entries from the other lanes
    double xr[6], xi[6];
#pragma unroll
    for (int r = 5; r >= 0; r--) {
        double sr = __shfl_sync(full, cr[r], 6, 8), si = __shfl_sync(full, ci[r], 6, 8);
#pragma unroll
        for (int j = r + 1; j < 6; j++) {
            const double ur = __shfl_sync(full, cr[r], j, 8), ui = __shfl_sync(full, ci[r], j, 8);
            sr -= ur * xr[j] - ui * xi[j]; si -= ur * xi[j] + ui * xr[j];
        }
        const double dr = __shfl_sync(full, cr[r], r, 8), di = __shfl_sync(full, ci[r], r, 8);
        const double inv = 1.0 / (dr * dr + di * di);
        xr[r] = (sr * dr + si * di) * inv; xi[r] = (si * dr - sr * di) * inv;
    }
    if (live && c < 6) X[(size_t)c * n + i] = make_double2(xr[c < 6 ? c : 0], xi[c < 6 ? c : 0]);
}

int main()
{
    const int n = 1 << 20;
    std::vector<double> M(36), B(36), C(36), w(n);
    std::vector<double2> F((size_t)6 * n);
    srand(1);
    auto rnd = [] { return rand() / (double)RAND_MAX - 0.5; };
    for (int t = 0; t < 36; t++) { M[t] = rnd() + (t % 7 == 0 ? 4.0 : 0.0); B[t] = rnd() + (t % 7 == 0 ? 2.0 : 0.0); C[t] = rnd() + (t % 7 == 0 ? 8.0 : 0.0); }
    for (int i = 0; i < n; i++) w[i] = 0.05 + 3.0 * i / n;
    for (auto &f : F) f = make_double2(rnd(), rnd());
    double *dM, *dB, *dC, *dw; double2 *dF, *dX1, *dX2;
    cudaMalloc(&dM, 288); cudaMalloc(&dB, 288); cudaMalloc(&dC, 288); cudaMalloc(&dw, n * 8);
    cudaMalloc(&dF, (size_t)6 * n * 16); cudaMalloc(&dX1, (size_t)6 * n * 16); cudaMalloc(&dX2, (size_t)6 * n * 16);
    cudaMemcpy(dM, M.data(), 288, cudaMemcpyHostToDevice); cudaMemcpy(dB, B.data(), 288, cudaMemcpyHostToDevice); cudaMemcpy(dC, C.data(), 288, cudaMemcpyHostToDevice);
    cudaMemcpy(dw, w.data(), n * 8, cudaMemcpyHostToDevice); cudaMemcpy(dF, F.data(), (size_t)6 * n * 16, cudaMemcpyHostToDevice);
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    float msT = 0, msW = 0;
    for (int rep = 0; rep < 3; rep++) {
        cudaEventRecord(a); k_thread<<<(n + 127) / 128, 128>>>(dM, dB, dC, dw, dF, dX1, n); cudaEventRecord(b); cudaEventSynchronize(b); cudaEventElapsedTime(&msT, a, b);
        cudaEventRecord(a); k_warp<<<(n / 4 * 32 + 255) / 256, 256>>>(dM, dB, dC, dw, dF, dX2, n); cudaEventRecord(b); cudaEventSynchronize(b); cudaEventElapsedTime(&msW, a, b);
    }
    std::vector<double2> X1((size_t)6 * n), X2((size_t)6 * n);
    cudaMemcpy(X1.data(), dX1, (size_t)6 * n * 16, cudaMemcpyDeviceToHost); cudaMemcpy(X2.data(), dX2, (size_t)6 * n * 16, cudaMemcpyDeviceToHost);
    double err = 0, mx = 0;
    for (size_t t = 0; t < X1.size(); t++) { err = fmax(err, fmax(fabs(X1[t].x - X2[t].x), fabs(X1[t].y - X2[t].y))); mx = fmax(mx, fmax(fabs(X1[t].x), fabs(X1[t].y))); }
    printf("6x6 complex solve, %d systems: thread-per-system (solve6, registers) %.3f ms = %.3e systems/s ; 8-lanes-per-system warp-shuffle elimination %.3f ms = %.3e systems/s ; max |diff| / max |x| = %.2e (%s)\n",
           n, msT, n / (msT * 1e-3), msW, n / (msW * 1e-3), err / mx, cudaGetErrorString(cudaGetLastError()));
    return 0;
}
