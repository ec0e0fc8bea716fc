// hmcx_ppc.cu -- posterior predictive checks of Bayesian NNs (Gelman, Meng & Stern 1996; BDA3 ch. 6; Gabry et al. 2019):
// one replicated data set y_rep ~ p(y | theta_g) per posterior draw g, its test statistics and the realised deviances of
// y_rep and of the observed y under theta_g.  hamiltorch_b200/ppc.py drives it; tests/ppc_oracle.py is the numpy
// definition.  LOO-PIT, the other half of ppc.py, runs on the PSIS pass of hmcx_loo.cu.
//
// A call handles a slab of k draws whose network outputs f [k, N, O] come from hmcx_mlp_pointwise_out; draw j of the slab
// is the pooled draw g = draws[j] (g = c n + s).  One CTA per draw:
//   1. y_rep is simulated from the draw's outputs with the element definitions of hmcx_sbc_simulate (hmcx_common.cuh's
//      sim_*) on Philox stream STREAM_PPC, chain word g, so a draw's replicate depends on (seed, g) only: regression
//      normals and binary uniforms one block per 4 consecutive outputs e = i O + o, multi-class one block per row.  It is
//      written to y_rep, and the two deviances accumulate on the way;
//   2. after a barrier the statistics are read back from the CTA's own y_rep rows.
// Every sum is thread-strided in fp64, then a fixed xor tree and the warp partials in warp order; there are no atomics,
// so a draw's results are the same bytes whatever the slab size and on every call.
#include <cfloat>
#include "hmcx_common.cuh"

namespace hmcx {
namespace {

constexpr int PT = 256;                     // threads per draw
constexpr int PW = PT / 32;

// Fixed-order CTA reduction of one double per thread; every thread gets the result.
template <class Op>
__device__ __forceinline__ double cta_reduce(double v, double* sh, Op op) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    double s = sh[0];
#pragma unroll
    for (int w = 1; w < PW; ++w) s = op(s, sh[w]);
    __syncthreads();
    return s;
}
struct Sum { __device__ double operator()(double a, double b) const { return a + b; } };
struct Min { __device__ double operator()(double a, double b) const { return fmin(a, b); } };
struct Max { __device__ double operator()(double a, double b) const { return fmax(a, b); } };

// -BCEWithLogits(f, y) in torch's stable form, fp64
__device__ __forceinline__ double bce(double f, double y) { return fmax(f, 0.0) - f * y + log1p(exp(-fabs(f))); }

// -log p(label | f) of one row: log-softmax of the logits, or f[label] itself for a LogSoftmax output
__device__ __forceinline__ double class_nll(const float* fr, int O, int label, bool logsoftmax) {
    if (logsoftmax) return -(double)fr[label];
    double mx = (double)fr[0];
    for (int c = 1; c < O; ++c) mx = fmax(mx, (double)fr[c]);
    double tot = 0.0;
    for (int c = 0; c < O; ++c) tot += exp((double)fr[c] - mx);
    return -(((double)fr[label] - mx) - log(tot));
}

// stats[j, :K]: regression mean, sd (ddof 1), min, max of every output column (column-major in o), binary the mean of
// every column, multi-class the frequency of every class; then the deviance -2 sum_i ll_i(y_rep | theta).  dev_obs[j] =
// -2 sum_i ll_i(y | theta).  A draw with a non-finite output: NaN statistics and deviances, nonfinite[j] = 1.
__global__ void __launch_bounds__(PT) ppc_kernel(const float* __restrict__ f, int N, int O, int loss, float tau_target,
                                                 const float* __restrict__ y, const long long* __restrict__ draws,
                                                 uint64_t seed, const float* __restrict__ tau, float* yrep,
                                                 double* __restrict__ stats, double* __restrict__ dev_obs,
                                                 int* __restrict__ nonfinite) {
    __shared__ double sh[PW];
    const int j = blockIdx.x, tid = threadIdx.x;
    const long long g = draws[j];
    const bool classes = loss == HMCX_LOSS_MULTICLASS || loss == HMCX_LOSS_MULTICLASS_LOGSOFTMAX;
    const int yc = classes ? 1 : O, K = (loss == HMCX_LOSS_REGRESSION ? 4 * O : O) + 1;
    const float* fj = f + (long long)j * N * O;
    float* yj = yrep + (long long)j * N * yc;
    double* out = stats + (long long)j * K;
    const float tj = tau ? tau[j] : tau_target;
    double drep = 0.0, dobs = 0.0, bad = 0.0;
    // 1. simulate, accumulating the deviance terms (regression: squared errors; classification: -ll)
    if (!classes) {
        const bool binary = loss == HMCX_LOSS_BINARY;
        const float sd = noise_sd(tj);
        const long long n_out = (long long)N * O, nvec = (n_out + 3) >> 2;
        for (long long v = tid; v < nvec; v += PT) {
            const uint4 r = philox_draw(seed, (uint64_t)g, 0, (uint32_t)v, STREAM_PPC);
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
                const float fv = fj[idx];
                if (!finite_f(fv)) bad += 1.0;
                const float yr = binary ? sim_bernoulli(fv, w[e]) : sim_gaussian(fv, z[e], sd);
                yj[idx] = yr;
                const double fd = (double)fv, yo = (double)y[idx];
                if (binary) {
                    drep += bce(fd, (double)yr);
                    dobs += bce(fd, yo);
                } else {
                    drep += (fd - (double)yr) * (fd - (double)yr);
                    dobs += (fd - yo) * (fd - yo);
                }
            }
        }
    } else {
        const bool ls = loss == HMCX_LOSS_MULTICLASS_LOGSOFTMAX;
        for (int i = tid; i < N; i += PT) {
            const float* fr = fj + (long long)i * O;
            for (int c = 0; c < O; ++c) if (!finite_f(fr[c])) bad += 1.0;
            const uint4 r = philox_draw(seed, (uint64_t)g, 0, (uint32_t)i, STREAM_PPC);
            const int label = sim_categorical(fr, O, r.x);
            yj[i] = (float)label;
            drep += class_nll(fr, O, label, ls);
            dobs += class_nll(fr, O, (int)y[i], ls);
        }
    }
    bad = cta_reduce(bad, sh, Sum());
    drep = cta_reduce(drep, sh, Sum());
    dobs = cta_reduce(dobs, sh, Sum());
    if (bad > 0.0) {                                            // CTA-uniform
        if (tid == 0) {
            const double nan = __longlong_as_double(0x7ff8000000000000LL);
            for (int q = 0; q < K; ++q) out[q] = nan;
            dev_obs[j] = nan;
            nonfinite[j] = 1;
        }
        return;
    }
    // the deviances: regression -2 sum_i (sum_o -tau/2 sq + O/2 log(tau / 2 pi)) = tau sum sq - N O log(tau / 2 pi)
    double d_rep, d_obs;
    if (loss == HMCX_LOSS_REGRESSION) {
        const double td = (double)tj, lc = (double)N * O * log(td / (2.0 * 3.14159265358979323846));
        d_rep = td * drep - lc;
        d_obs = td * dobs - lc;
    } else {
        d_rep = 2.0 * drep;
        d_obs = 2.0 * dobs;
    }
    __syncthreads();                                            // y_rep rows of every thread are visible to the CTA
    // 2. statistics of y_rep
    if (classes) {
        for (int c = 0; c < O; ++c) {
            double cnt = 0.0;
            for (int i = tid; i < N; i += PT) cnt += yj[i] == (float)c ? 1.0 : 0.0;
            cnt = cta_reduce(cnt, sh, Sum());
            if (tid == 0) out[c] = cnt / N;
        }
    } else {
        for (int o = 0; o < O; ++o) {
            double s = 0.0, lo = DBL_MAX, hi = -DBL_MAX;
            for (int i = tid; i < N; i += PT) {
                const double v = (double)yj[(long long)i * O + o];
                s += v;
                lo = fmin(lo, v);
                hi = fmax(hi, v);
            }
            const double mean = cta_reduce(s, sh, Sum()) / N;
            if (loss == HMCX_LOSS_BINARY) {
                if (tid == 0) out[o] = mean;
                continue;
            }
            lo = cta_reduce(lo, sh, Min());
            hi = cta_reduce(hi, sh, Max());
            double ss = 0.0;
            for (int i = tid; i < N; i += PT) {
                const double d = (double)yj[(long long)i * O + o] - mean;
                ss += d * d;
            }
            ss = cta_reduce(ss, sh, Sum());
            if (tid == 0) {
                out[4 * o] = mean;
                out[4 * o + 1] = sqrt(ss / (N - 1));
                out[4 * o + 2] = lo;
                out[4 * o + 3] = hi;
            }
        }
    }
    if (tid == 0) {
        out[K - 1] = d_rep;
        dev_obs[j] = d_obs;
        nonfinite[j] = 0;
    }
}

}  // namespace

int ppc_pass(const hmcx_target_t* target, const float* f, int k, const long long* draws, uint64_t seed,
             const float* tau, float* yrep, double* stats, double* dev_obs, int* nonfinite, cudaStream_t st) {
    const hmcx_mlp_t& m = *target->mlp;
    ppc_kernel<<<k, PT, 0, st>>>(f, m.num_rows, m.widths[m.num_layers], m.loss, m.tau_out, (const float*)m.y, draws,
                                 seed, tau, yrep, stats, dev_obs, nonfinite);
    return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA;
}

}  // namespace hmcx
