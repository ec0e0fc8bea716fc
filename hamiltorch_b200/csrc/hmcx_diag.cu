// hmcx_diag.cu -- convergence diagnostics of a batched sample block: the two streaming passes behind split-R-hat,
// effective sample size and Monte-Carlo standard error (hamiltorch_b200/diagnostics.py runs the Geyer scan on their
// output; oracle/diagnostics_oracle.py is the fp64 definition they are tested against).
//
// The block is fp32 x[c, s, d] at x + c*chain_stride + s*draw_stride + d (unit stride along D, so a strided view such as
// res.samples[:, 1:] or a thinned block is read in place).  Half-chain 2c is draws [0, m) of chain c, half-chain 2c+1 is
// draws [n-m, n), m = n/2.  All accumulation is fp64; every reduction over half-chains runs in a fixed order (no atomics),
// so the same block gives the same bits on every call.
#include "hmcx_common.cuh"

namespace hmcx {
namespace {

constexpr int TB = HMCX_DIAG_LAG_BLOCK;   // lags per autocovariance pass
constexpr int DX = 8;                      // dimensions per CTA: a warp reads 8 consecutive floats (one 32-byte sector)
constexpr int JY = 32;                     // half-chain lanes per CTA
constexpr int SUB = 8;                     // draws loaded ahead per batch (loads in flight per thread)

__device__ __forceinline__ const float* half_chain(const float* x, long long cs, long long ds, int n, int m, int j, int d) {
    return x + (long long)(j >> 1) * cs + (long long)((j & 1) ? (n - m) : 0) * ds + d;
}

// mu[j, d] = mean of half-chain j in dimension d.  One thread per (half-chain, dimension); the draws are summed in order.
__global__ void __launch_bounds__(DX * JY) diag_means_kernel(const float* __restrict__ x, long long cs, long long ds,
                                                             int C, int n, int D, double* __restrict__ mu) {
    const int d = blockIdx.x * DX + threadIdx.x;
    const int j = blockIdx.y * JY + threadIdx.y;
    const int m = n / 2;
    if (d >= D || j >= 2 * C) return;
    const float* p = half_chain(x, cs, ds, n, m, j, d);
    double s = 0.0;
    int u = 0;
    for (; u + SUB <= m; u += SUB) {
        float v[SUB];
#pragma unroll
        for (int q = 0; q < SUB; ++q) v[q] = p[(long long)(u + q) * ds];
#pragma unroll
        for (int q = 0; q < SUB; ++q) s += (double)v[q];
    }
    for (; u < m; ++u) s += (double)p[(long long)u * ds];
    mu[(long long)j * D + d] = s / m;
}

// mu_sum[d] = sum_j mu[j, d], j ascending.
__global__ void diag_mu_sum_kernel(const double* __restrict__ mu, int K, int D, double* __restrict__ mu_sum) {
    const int d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= D) return;
    double s = 0.0;
    for (int j = 0; j < K; ++j) s += mu[(long long)j * D + d];
    mu_sum[d] = s;
}

// acov_out[k, d] = sum_j gamma_j(t0 + k), k < TB, with gamma_j(t) = (1/m) sum_{s < m-t} y_s y_{s+t}, y = x - mu_j.
// A CTA owns DX dimensions and all half-chains; thread (dx, ly) streams half-chains ly, ly + JY, ... .  For each it walks
// u = 0 .. m-1-t0: y_u goes into a TB-slot register ring and z = y_{u+t0} meets the TB trailing values, so lag t0 + k
// pairs y_{u-k} with y_{u+t0} (slots of negative u hold 0 and add nothing).  The u loop is unrolled by TB, so every ring
// index is a compile-time constant and the ring never moves.  Per-thread sums are then added over the JY lanes in lane
// order through shared memory.  With mu_bar, between_out[d] = sum_j (mu_j - mu_bar)^2 in the same order.
__global__ void __launch_bounds__(DX * JY, 1) diag_acov_kernel(const float* __restrict__ x, long long cs, long long ds,
                                                               int C, int n, int D, const double* __restrict__ mu,
                                                               const double* __restrict__ mu_bar, int t0,
                                                               double* __restrict__ acov_out,
                                                               double* __restrict__ between_out) {
    __shared__ double red[JY][SUB][DX];
    const int dx = threadIdx.x, ly = threadIdx.y;
    const int d = blockIdx.x * DX + dx;
    const int m = n / 2, K = 2 * C;
    const int U = m - t0;
    double acc[TB];
#pragma unroll
    for (int k = 0; k < TB; ++k) acc[k] = 0.0;
    double between = 0.0;
    if (d < D) {
        const double mb = mu_bar ? mu_bar[d] : 0.0;
        for (int j = ly; j < K; j += JY) {
            const float* p = half_chain(x, cs, ds, n, m, j, d);
            const double mj = mu[(long long)j * D + d];
            if (mu_bar) {
                const double e = mj - mb;
                between = fma(e, e, between);
            }
            double r[TB];
#pragma unroll
            for (int k = 0; k < TB; ++k) r[k] = 0.0;
            for (int u0 = 0; u0 < U; u0 += TB) {
#pragma unroll
                for (int sc = 0; sc < TB / SUB; ++sc) {
                    float fy[SUB], fz[SUB];
#pragma unroll
                    for (int q = 0; q < SUB; ++q) {
                        const int u = u0 + sc * SUB + q;
                        fz[q] = u < U ? p[(long long)(u + t0) * ds] : 0.f;
                        fy[q] = t0 == 0 ? fz[q] : (u < U ? p[(long long)u * ds] : 0.f);
                    }
#pragma unroll
                    for (int q = 0; q < SUB; ++q) {
                        const int slot = sc * SUB + q;
                        const bool ok = u0 + slot < U;
                        const double zv = ok ? (double)fz[q] - mj : 0.0;
                        r[slot] = ok ? (double)fy[q] - mj : 0.0;
#pragma unroll
                        for (int k = 0; k < TB; ++k) acc[k] = fma(r[(slot - k + TB) % TB], zv, acc[k]);
                    }
                }
            }
        }
    }
    const int tid = ly * DX + dx;
    const double inv_m = 1.0 / m;
#pragma unroll
    for (int tt = 0; tt < TB; tt += SUB) {
#pragma unroll
        for (int q = 0; q < SUB; ++q) red[ly][q][dx] = acc[tt + q];
        __syncthreads();
        if (tid < SUB * DX) {
            const int q = tid / DX, e = tid % DX, od = blockIdx.x * DX + e;
            double s = 0.0;
            for (int y = 0; y < JY; ++y) s += red[y][q][e];
            if (od < D) acov_out[(long long)(tt + q) * D + od] = s * inv_m;
        }
        __syncthreads();
    }
    if (mu_bar && between_out) {
        red[ly][0][dx] = between;
        __syncthreads();
        if (ly == 0 && d < D) {
            double s = 0.0;
            for (int y = 0; y < JY; ++y) s += red[y][0][dx];
            between_out[d] = s;
        }
    }
}

}  // namespace

int diag_means(const float* x, long long cs, long long ds, int C, int n, int D, double* mu, double* mu_sum,
               cudaStream_t st) {
    const int K = 2 * C;
    dim3 grid((D + DX - 1) / DX, (K + JY - 1) / JY);
    diag_means_kernel<<<grid, dim3(DX, JY), 0, st>>>(x, cs, ds, C, n, D, mu);
    diag_mu_sum_kernel<<<(D + 127) / 128, 128, 0, st>>>(mu, K, D, mu_sum);
    return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA;
}

int diag_acov(const float* x, long long cs, long long ds, int C, int n, int D, const double* mu, const double* mu_bar,
              int t0, double* acov_out, double* between_out, cudaStream_t st) {
    diag_acov_kernel<<<(D + DX - 1) / DX, dim3(DX, JY), 0, st>>>(x, cs, ds, C, n, D, mu, mu_bar, t0, acov_out,
                                                                  between_out);
    return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA;
}

}  // namespace hmcx
