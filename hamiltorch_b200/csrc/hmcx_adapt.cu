// hmcx_adapt.cu -- the pooled diagonal mass estimate of a warm-up window (Stan's windowed adaptation, pooled over every
// chain of the batch) and the restart of the step-size dual averaging that follows a mass update (include/hmcx.h,
// hmcx_adapt_diag_mass).
//
// Input: per-chain compensated running sums of the window's draws, [C, ld] each (hi + lo), as the sink forms of
// hmc_run_kernel / mlp_run_kernel leave them with hmcx_sink_t.moments_all.  One thread per dimension walks the chains in
// index order: the per-chain variances and their sum are fp64, every operation is an explicit IEEE round-to-nearest
// intrinsic and there are no atomics, so the estimate has one definition, bit for bit (tests/adapt_oracle.py restates it
// in numpy).  The same pass zeroes the sums for the next window.
#include "hmcx_common.cuh"

namespace hmcx {
namespace {

constexpr int ADAPT_THREADS = 128;

__global__ void __launch_bounds__(ADAPT_THREADS)
adapt_diag_mass_kernel(float* __restrict__ sum, float* __restrict__ sumsq, float* __restrict__ sum_lo,
                       float* __restrict__ sumsq_lo, int C, int ld, int D, int n, const float* __restrict__ eps,
                       int C_chains, float* __restrict__ inv_mass, float* __restrict__ mass_factor,
                       double* __restrict__ mu_chain, double* __restrict__ h_bar, double* __restrict__ eps_bar) {
    const int i = blockIdx.x * ADAPT_THREADS + threadIdx.x;
    if (i < C_chains) {
        // the restarted dual averaging (Stan: x_bar = 0, s_bar = 0, mu = log(10 eps)); 10 * eps rounds in fp32 as
        // engine.nuts_mu's FloatTensor product does, the log is the correctly rounded fp32 one
        const float e10 = __fmul_rn(10.0f, eps[i]);
        mu_chain[i] = (double)__double2float_rn(log((double)e10));
        h_bar[i] = 0.0;
        eps_bar[i] = 1.0;
    }
    if (i >= ld) return;
    float im = 0.0f, mf = 0.0f;
    if (i < D) {
        const double dn = (double)n, dn1 = (double)(n - 1);
        double w = 0.0;
#pragma unroll 4
        for (int c = 0; c < C; ++c) {
            const size_t o = (size_t)c * ld + i;
            const double s1 = __dadd_rn((double)sum[o], (double)sum_lo[o]);
            const double s2 = __dadd_rn((double)sumsq[o], (double)sumsq_lo[o]);
            const double m = __ddiv_rn(s1, dn);
            w = __dadd_rn(w, __ddiv_rn(__dsub_rn(s2, __dmul_rn(s1, m)), dn1));
        }
        w = __ddiv_rn(w, (double)C);
        const double N = __dmul_rn((double)C, dn);
        const double var = __dadd_rn(__dmul_rn(__ddiv_rn(N, __dadd_rn(N, 5.0)), w),
                                     __dmul_rn(1e-3, __ddiv_rn(5.0, __dadd_rn(N, 5.0))));
        im = __double2float_rn(var);
        mf = __fsqrt_rn(__fdiv_rn(1.0f, im));                 // engine.NativeMass: (1 / inv_mass) ** 0.5
    }
    inv_mass[i] = im;
    mass_factor[i] = mf;
    for (int c = 0; c < C; ++c) {                             // the next window starts from zero
        const size_t o = (size_t)c * ld + i;
        sum[o] = 0.0f; sumsq[o] = 0.0f; sum_lo[o] = 0.0f; sumsq_lo[o] = 0.0f;
    }
}

}  // namespace

int adapt_diag_mass(float* sum, float* sumsq, float* sum_lo, float* sumsq_lo, int C, int ld, int D, int n, const float* eps,
                    int C_chains, float* inv_mass, float* mass_factor, double* mu_chain, double* h_bar, double* eps_bar,
                    cudaStream_t st) {
    const int threads = ld > C_chains ? ld : C_chains;
    const int blocks = (threads + ADAPT_THREADS - 1) / ADAPT_THREADS;
    adapt_diag_mass_kernel<<<blocks, ADAPT_THREADS, 0, st>>>(sum, sumsq, sum_lo, sumsq_lo, C, ld, D, n, eps, C_chains,
                                                              inv_mass, mass_factor, mu_chain, h_bar, eps_bar);
    return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA;
}

}  // namespace hmcx
