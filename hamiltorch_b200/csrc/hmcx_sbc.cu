// hmcx_sbc.cu -- simulation-based calibration of Bayesian NNs (Talts et al. 2018; Modrák et al. 2023): prior draws,
// data simulated from the likelihood at a draw, and the rank of the true parameters among the posterior draws of a fit.
// hamiltorch_b200/sbc.py drives it; tests/sbc_oracle.py is the numpy definition.
//
// Every random value is keyed by the GLOBAL sim id m, never by the launch geometry, so a sim gets the same values
// whatever the number of sims of the call.  Two Philox streams of hmcx_common.cuh, chain word = m:
//   STREAM_SBC_PRIOR  counter (v, j lo, j hi | 6 << 24, m lo), key (seed lo, seed hi ^ m hi): row j of sim m, j = 0 the
//                     true parameters, j = 1 + r the start of chain r; elements 4v .. 4v + 3 by the canonical Box-Muller
//   STREAM_SBC_DATA   the same with j = 0: regression normals over the flattened (N O) outputs, one u01 word per output
//                     (binary), one u01 word x of vector = row (multi-class)
#include <algorithm>
#include <cmath>
#include "hmcx_common.cuh"

namespace hmcx {
namespace {

constexpr int PT = 256;                     // threads per CTA of the prior and data kernels
constexpr int RX = 32, RY = 8;              // rank kernel: 32 columns x 8 draw lanes per CTA

// The prior standard deviation of every parameter tensor, sqrt(prior_scale / tau_k), and where each tensor ends in the
// flat parameter vector (util.flatten order: W_0, b_0, W_1, b_1, ...).
struct PriorTable {
    int   end[2 * HMCX_MLP_MAX_LAYERS];
    float sd[2 * HMCX_MLP_MAX_LAYERS];
    int   num;
};

__global__ void __launch_bounds__(PT) sbc_prior_kernel(PriorTable tab, uint64_t seed, long long m0, int rows_per_sim,
                                                       int ld, long long total, float* __restrict__ out) {
    const int nv = ld >> 2;
    for (long long i = (long long)blockIdx.x * PT + threadIdx.x; i < total; i += (long long)gridDim.x * PT) {
        const long long row = i / nv;
        const int v = (int)(i - row * nv);
        const long long m = row / rows_per_sim;
        const int j = (int)(row - m * rows_per_sim);
        const uint4 r = philox_draw(seed, (uint64_t)(m0 + m), (uint64_t)j, (uint32_t)v, STREAM_SBC_PRIOR);
        float z[4];
        box_muller(r.x, r.y, z[0], z[1]);
        box_muller(r.z, r.w, z[2], z[3]);
        float o[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int d = 4 * v + e;
            int k = 0;
            while (k < tab.num && d >= tab.end[k]) ++k;
            o[e] = k < tab.num ? mul(z[e], tab.sd[k]) : 0.0f;
        }
        st4(out + row * ld + 4 * v, o);
    }
}

// Regression: y = f + z / sqrt(tau_out), one Philox block per 4 consecutive outputs of a sim.  Binary: y = 1 when the
// output's u01 word is below sigmoid(f) (fp64), else 0.  The element definitions are hmcx_common.cuh's sim_*.
__global__ void __launch_bounds__(PT) sbc_simulate_elem_kernel(const float* __restrict__ f, uint64_t seed, long long m0,
                                                               long long n_out, long long total, int binary,
                                                               float noise_sd, float* __restrict__ y) {
    const long long nvec = (n_out + 3) >> 2;
    for (long long i = (long long)blockIdx.x * PT + threadIdx.x; i < total; i += (long long)gridDim.x * PT) {
        const long long m = i / nvec;
        const long long v = i - m * nvec;
        const uint4 r = philox_draw(seed, (uint64_t)(m0 + m), 0, (uint32_t)v, STREAM_SBC_DATA);
        const uint32_t w[4] = {r.x, r.y, r.z, r.w};
        float z[4];
        if (!binary) {
            box_muller(r.x, r.y, z[0], z[1]);
            box_muller(r.z, r.w, z[2], z[3]);
        }
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const long long idx = 4 * v + e;
            if (idx >= n_out) break;
            const long long at = m * n_out + idx;
            const float fv = f[at];
            y[at] = binary ? sim_bernoulli(fv, w[e]) : sim_gaussian(fv, z[e], noise_sd);
        }
    }
}

// Multi-class: one label per row from Categorical(softmax f) (sim_categorical), u = u01(word x of vector = row).
__global__ void __launch_bounds__(PT) sbc_simulate_class_kernel(const float* __restrict__ f, uint64_t seed, long long m0,
                                                                int N, int O, long long total, float* __restrict__ y) {
    for (long long i = (long long)blockIdx.x * PT + threadIdx.x; i < total; i += (long long)gridDim.x * PT) {
        const long long m = i / N;
        const int row = (int)(i - m * N);
        const float* fr = f + i * O;
        const uint4 r = philox_draw(seed, (uint64_t)(m0 + m), 0, (uint32_t)row, STREAM_SBC_DATA);
        y[i] = (float)sim_categorical(fr, O, r.x);
    }
}

// ranks[m, d] = #{(r, s) : x[r K + m, s, d] < truth[m, d]}, r < R, 1 <= s < keep.  CTA (blockIdx.x, m): 32 columns, the
// 8 rows of threads stride over the R (keep - 1) draws so every warp reads 128 contiguous bytes of one draw; the
// per-lane counts are summed in a fixed order.  Each element of the block is read once.
__global__ void __launch_bounds__(RX * RY) sbc_rank_kernel(const float* __restrict__ x, long long cs, long long ds, int K,
                                                           int R, int keep, int D, const float* __restrict__ truth,
                                                           long long ts, int* __restrict__ ranks) {
    __shared__ int sh[RY][RX];
    const int d = blockIdx.x * RX + threadIdx.x, m = blockIdx.y;
    const int per = keep - 1, n = R * per;
    int cnt = 0;
    if (d < D) {
        const float thr = truth[(long long)m * ts + d];
        for (int t = threadIdx.y; t < n; t += RY) {
            const int r = t / per, s = 1 + (t - r * per);
            cnt += __ldcs(x + (long long)(r * K + m) * cs + (long long)s * ds + d) < thr ? 1 : 0;
        }
    }
    sh[threadIdx.y][threadIdx.x] = cnt;
    __syncthreads();
    if (threadIdx.y == 0 && d < D) {
        int s = 0;
#pragma unroll
        for (int i = 0; i < RY; ++i) s += sh[i][threadIdx.x];
        ranks[(long long)m * D + d] = s;
    }
}

int grid_of(long long total) { return (int)std::min<long long>((total + PT - 1) / PT, 65536LL); }

}  // namespace

int sbc_prior(const hmcx_target_t* target, uint64_t seed, long long m0, int M, int R, int ld, float* out,
              cudaStream_t st) {
    const hmcx_mlp_t& mlp = *target->mlp;
    PriorTable tab;
    tab.num = 2 * mlp.num_layers;
    int off = 0;
    for (int l = 0; l < mlp.num_layers; ++l) {
        off += mlp.widths[l] * mlp.widths[l + 1];
        tab.end[2 * l] = off;
        off += mlp.widths[l + 1];
        tab.end[2 * l + 1] = off;
    }
    // prior_two_var = 2 / tau_k (the reference's fp32 rounding of 2 scale^2), so prior_scale / tau_k = prior_scale two_var / 2
    for (int k = 0; k < tab.num; ++k)
        tab.sd[k] = (float)sqrt(0.5 * (double)mlp.prior_scale * (double)mlp.prior_two_var[k]);
    const long long total = (long long)M * (1 + R) * (ld / 4);
    sbc_prior_kernel<<<grid_of(total), PT, 0, st>>>(tab, seed, m0, 1 + R, ld, total, out);
    return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA;
}

int sbc_simulate(const hmcx_target_t* target, const float* f, uint64_t seed, long long m0, int M, float* y,
                 cudaStream_t st) {
    const hmcx_mlp_t& mlp = *target->mlp;
    const int N = mlp.num_rows, O = mlp.widths[mlp.num_layers];
    if (mlp.loss == HMCX_LOSS_MULTICLASS) {
        const long long total = (long long)M * N;
        sbc_simulate_class_kernel<<<grid_of(total), PT, 0, st>>>(f, seed, m0, N, O, total, y);
    } else {
        const long long n_out = (long long)N * O, total = (long long)M * ((n_out + 3) >> 2);
        const float noise_sd = (float)(1.0 / sqrt((double)mlp.tau_out));
        sbc_simulate_elem_kernel<<<grid_of(total), PT, 0, st>>>(f, seed, m0, n_out, total,
                                                                 mlp.loss == HMCX_LOSS_BINARY, noise_sd, y);
    }
    return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA;
}

int sbc_rank(const float* x, long long cs, long long ds, int C, int keep, int K, int D, const float* truth, long long ts,
             int* ranks, cudaStream_t st) {
    sbc_rank_kernel<<<dim3((D + RX - 1) / RX, K), dim3(RX, RY), 0, st>>>(x, cs, ds, K, C / K, keep, D, truth, ts, ranks);
    return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA;
}

}  // namespace hmcx
