// hmcx_temper.cu -- the swap round of replica exchange between the rungs of Bayesian-NN ladders (DESIGN.md 3.17).
//
// The C rows of q_cur are R = C / T ladders, ladder-major (row r*T + t = ladder r at beta_t).  Round k pairs the rungs
// (t, t + 1) with t = k (mod 2); the pairs of a round are disjoint, so one CTA per (ladder, pair) decides its pair and
// exchanges the two rows itself: no atomics, no ordering between CTAs, the same bytes on every call.
#include <float.h>
#include <math.h>
#include "hmcx_common.cuh"

namespace hmcx {

constexpr int SWAP_THREADS = 128;

struct SwapBetas { double v[HMCX_TEMPER_MAX_TEMPS]; };

__global__ void __launch_bounds__(SWAP_THREADS)
temper_swap_kernel(float* __restrict__ q, int ld, int T, const SwapBetas betas, const double* __restrict__ ll, int round,
                   int rng_mode, uint64_t seed, uint64_t ladder0, const double* __restrict__ log_uniforms,
                   int8_t* __restrict__ accepted) {
    __shared__ int s_acc;
    const int pairs = T - 1;
    const int r = blockIdx.x / pairs, t = blockIdx.x - r * pairs;
    const size_t o = (size_t)r * pairs + t;
    if ((t & 1) != (round & 1)) {                              // not paired in this round
        if (threadIdx.x == 0) accepted[o] = -1;
        return;
    }
    const size_t a = (size_t)r * T + t;                        // rows a (beta_t) and a + 1 (beta_{t+1})
    if (threadIdx.x == 0) {
        double logu;
        if (rng_mode == HMCX_RNG_INJECTED) {
            logu = log_uniforms[o];
        } else {
            const uint64_t ladder = ladder0 + (uint64_t)r;
            logu = log((double)u01(philox_draw(seed, ladder, (uint64_t)round, (uint32_t)t, STREAM_SWAP).x));
        }
        const double x = (betas.v[t] - betas.v[t + 1]) * (ll[a + 1] - ll[a]);
        const int acc = logu < x ? 1 : 0;                      // NaN log-likelihoods never swap
        accepted[o] = (int8_t)acc;
        s_acc = acc;
    }
    __syncthreads();
    if (!s_acc) return;
    float4* x0 = reinterpret_cast<float4*>(q + a * ld);
    float4* x1 = reinterpret_cast<float4*>(q + (a + 1) * ld);
    for (int v = threadIdx.x; v < (ld >> 2); v += SWAP_THREADS) {
        const float4 u = x0[v], w = x1[v];
        x0[v] = w;
        x1[v] = u;
    }
}

int temper_swap(float* q_cur, int C, int ld, int T, const double* betas, const double* ll, int round,
                const hmcx_rng_t* rng, const double* log_uniforms, int8_t* accepted, cudaStream_t st) {
    if (!q_cur || !betas || !ll || !accepted || !rng || C < 1 || T < 2 || T > HMCX_TEMPER_MAX_TEMPS || C % T != 0 ||
        ld < 4 || (ld & 3) || (reinterpret_cast<size_t>(q_cur) & 15) || round < 0)
        return HMCX_ERR_INVALID_ARG;
    SwapBetas b = {};
    for (int t = 0; t < T; ++t) {
        if (!(betas[t] >= 0.0) || !(betas[t] <= DBL_MAX) || (t == 0 && betas[0] != 1.0) || (t > 0 && !(betas[t] < betas[t - 1])))
            return HMCX_ERR_INVALID_ARG;
        b.v[t] = betas[t];
    }
    if (rng->mode == HMCX_RNG_INJECTED) {
        if (!log_uniforms) return HMCX_ERR_INVALID_ARG;
    } else if (rng->mode == HMCX_RNG_PHILOX) {
        if (rng->chain_offset % (uint64_t)T != 0) return HMCX_ERR_INVALID_ARG;
    } else {
        return HMCX_ERR_INVALID_ARG;
    }
    const int R = C / T;
    temper_swap_kernel<<<R * (T - 1), SWAP_THREADS, 0, st>>>(q_cur, ld, T, b, ll, round, rng->mode, rng->seed,
                                                             rng->chain_offset / (uint64_t)T, log_uniforms, accepted);
    return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA;
}

}  // namespace hmcx
