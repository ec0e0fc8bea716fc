// hmcx_psens.cu -- power-scaling prior and likelihood sensitivity (Kallioinen, Paananen, Buerkner & Vehtari 2023).
// hamiltorch_b200/sensitivity.py drives it; tests/psens_oracle.py is the numpy definition.
//
// Four passes, all on the caller's stream, with no floating-point atomics: every output is a function of its inputs
// alone, not of the slab size or the launch geometry.
//   * hmcx_mlp_log_prior: one CTA per draw sums the Normal prior terms of a subset of the parameter tensors in fp64,
//     tensor by tensor in parameter order, each a thread-strided sum of squares and the fixed tree of cta_sum.
//   * hmcx_psens_ll_totals: one warp per draw adds a slab of its pointwise log-likelihoods to its running total in
//     128-row groups, in row order.  A group's sum is a fixed lane order and xor tree, so with slab boundaries on
//     multiples of 128 rows the total is the same bits whatever the slab size.
//   * hmcx_psens_weights: the K negated log-ratio columns -r (the role of -ll in hmcx_loo.cu) go through rank_sort with
//     one segment per weight set, then one CTA per set runs psis_smooth (hmcx_psis.cuh) and scatters the normalised
//     weights back to flat-draw order through the sort's flat indices.
//   * hmcx_psens_pass: rank_sort of a slab of columns, then one CTA per column sweeps its sorted draws twice.  The
//     forward sweep forms the prefix sums P, Q of every weight set in ascending x order and the cjs+ sums, plus the
//     weighted means; the reverse sweep does the same in ascending -x order (the cjs- sums) plus the weighted variances.
//     A sweep goes in tiles of LT * PE sorted positions: each thread scans PE consecutive positions, a fixed-order CTA
//     scan of the thread totals places them, and a carry takes the tile total to the next tile.
#include "hmcx_psis.cuh"

namespace hmcx {

size_t rank_sort_workspace_bytes(int C, int n, int k);
int rank_sort(const float* x, long long cs, long long ds, int C, int n, int d0, int k, int* nonfinite, void* ws,
              const uint32_t** sorted_keys, const int** sorted_idx, cudaStream_t st);
int loo_tail_cap(int S, double r_eff);

namespace {

constexpr int MAX_TENSORS = 2 * HMCX_MLP_MAX_LAYERS;
constexpr int NSET = HMCX_PSENS_SETS;       // weight sets: (prior, lo), (prior, hi), (lik, lo), (lik, hi)
constexpr int PE = 8;                       // sorted positions per thread per tile of a sweep
constexpr double LOG_2PI = 1.8378770664093454836;

struct PriorArgs {
    int T;
    int off[MAX_TENSORS + 1];
    double tau[MAX_TENSORS];                // 0: the tensor is left out
};

// out[g] = sum over the tensors t with tau_t > 0 of -tau_t/2 sum_i w_i^2 + n_t/2 (log tau_t - log 2 pi), g = c n + s.
__global__ void __launch_bounds__(LT) mlp_log_prior_kernel(const float* __restrict__ x, long long cs, long long ds,
                                                           int n, PriorArgs a, double* __restrict__ out) {
    __shared__ double sh[LW];
    const int g = blockIdx.x, c = g / n, s = g - c * n;
    const float* xp = x + (long long)c * cs + (long long)s * ds;
    double lp = 0.0;
    for (int t = 0; t < a.T; ++t) {
        if (!(a.tau[t] > 0.0)) continue;
        double ss = 0.0;
        for (int i = a.off[t] + (int)threadIdx.x; i < a.off[t + 1]; i += LT) {
            const double v = (double)xp[i];
            ss += v * v;
        }
        ss = cta_sum(ss, sh);
        lp += -0.5 * a.tau[t] * ss + 0.5 * (double)(a.off[t + 1] - a.off[t]) * (log(a.tau[t]) - LOG_2PI);
    }
    if (threadIdx.x == 0) out[g] = lp;
}

// totals[g] += the slab's rows [0, k) of draw g, coefficient coef[r0 + i] (1 when coef is NULL), in 128-row groups.
__global__ void __launch_bounds__(256) psens_ll_kernel(const float* __restrict__ ll, long long cs, long long ds, int n,
                                                       int S, int k, int r0, const double* __restrict__ coef,
                                                       double* __restrict__ totals) {
    const int g = (int)blockIdx.x * 8 + ((int)threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (g >= S) return;
    const int c = g / n, s = g - c * n;
    const float* lp = ll + (long long)c * cs + (long long)s * ds;
    double t = totals[g];
    for (int b = 0; b < k; b += 128) {
        double v = 0.0;
#pragma unroll
        for (int m = 0; m < 4; ++m) {
            const int i = b + lane + 32 * m;
            if (i < k) v += coef ? (double)lp[i] * coef[r0 + i] : (double)lp[i];
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        t += v;
    }
    if (lane == 0) totals[g] = t;
}

// One weight set per CTA: w[j * S + g_p] = exp(lw(p) - lse_w) over the sorted positions p of set j; pareto_k[j],
// tail[j] = M'.  A set with a non-finite log-ratio: NaN weights and k-hat, tail 0.
__global__ void __launch_bounds__(LT) psens_weights_kernel(const uint32_t* __restrict__ keys,
                                                           const int* __restrict__ idx, int S, int M,
                                                           const int* __restrict__ nonfinite, double* __restrict__ w,
                                                           double* __restrict__ pareto_k, int* __restrict__ tail) {
    extern __shared__ double sL[];
    __shared__ double sh[LW];
    const int j = blockIdx.x, tid = threadIdx.x;
    const uint32_t* kp = keys + (long long)j * S;
    const int* ip = idx + (long long)j * S;
    double* wj = w + (long long)j * S;
    if (nonfinite[j]) {
        for (int p = tid; p < S; p += LT) write_nan(wj + p);
        if (tid == 0) {
            write_nan(pareto_k + j);
            tail[j] = 0;
        }
        return;
    }
    const Psis ps = psis_smooth(kp, S, M, sL, sh);
    for (int p = tid; p < S; p += LT) wj[ip[p]] = exp(ps.lw(p) - ps.lse_w);
    if (tid == 0) {
        pareto_k[j] = ps.khat;
        tail[j] = ps.Mt;
    }
}

__device__ __forceinline__ double value_of_key(uint32_t k) { return ll_of_key(k); }

// Exclusive prefix of one double per thread in thread order (warp shuffle scan, then the warp totals in warp order);
// *total is the CTA total, the same bits in every thread.
__device__ __forceinline__ double cta_exscan(double v, double* sh, double* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const double u = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += u;
    }
    double ex = __shfl_up_sync(0xffffffffu, inc, 1);
    if (lane == 0) ex = 0.0;
    if (lane == 31) sh[warp] = inc;
    __syncthreads();
    double before = 0.0, tot = 0.0;
#pragma unroll
    for (int w = 0; w < LW; ++w) {
        if (w == warp) before = tot;
        tot += sh[w];
    }
    __syncthreads();
    *total = tot;
    return before + ex;
}

// P log2(2P / (P + Q)) + Q log2(2Q / (P + Q)), 0 log 0 = 0 (P > 0 always).
__device__ __forceinline__ double cjs_term(double P, double Q) {
    const double m = P + Q;
    double t = P * log2(2.0 * P / m);
    if (Q > 0.0) t += Q * log2(2.0 * Q / m);
    return t;
}

// One sweep over a column's S sorted draws.  REV = false: the sequence y_r = x_(r) (ascending x); REV = true: y_r =
// -x_(S-1-r) (ascending -x).  Per weight set k: num / den of the cjs formula with P_r = (r + 1) / S and Q_r the prefix
// sum of q_k in y order, widths y_(r+1) - y_(r) (the last one y_(S-1) - y_(S-2)).  mom[k] gets sum q_k x (forward) or
// sum q_k (x - mean[k + 1])^2 (reverse), mom[NSET] sum x or sum (x - mean[0])^2.  Results are CTA totals.
template <bool REV>
__device__ __forceinline__ void sweep(const uint32_t* __restrict__ kp, const int* __restrict__ ip, int S,
                                      const double* __restrict__ w, const double* mean, double* sh, double cjs[NSET],
                                      double mom[NSET + 1]) {
    const int tid = threadIdx.x;
    auto yv = [&](int r) { return REV ? -value_of_key(kp[S - 1 - r]) : value_of_key(kp[r]); };
    double num[NSET], den[NSET], acc[NSET + 1], carry[NSET];
#pragma unroll
    for (int k = 0; k < NSET; ++k) num[k] = den[k] = acc[k] = carry[k] = 0.0;
    acc[NSET] = 0.0;
    const double Sd = (double)S;
    for (int t0 = 0; t0 < S; t0 += LT * PE) {
        const int r0 = t0 + tid * PE;
        double y[PE], dl[PE];
        int gi[PE];
#pragma unroll
        for (int e = 0; e < PE; ++e) {
            const int r = r0 + e;
            y[e] = 0.0;
            dl[e] = 0.0;
            gi[e] = 0;
            if (r < S) {
                y[e] = yv(r);
                gi[e] = ip[REV ? S - 1 - r : r];
                const int rn = r < S - 1 ? r + 1 : S - 1;
                dl[e] = yv(rn) - yv(rn - 1);
                const double x = REV ? -y[e] : y[e];
                if (REV) {
                    const double d = x - mean[0];
                    acc[NSET] += d * d;
                } else {
                    acc[NSET] += x;
                }
            }
        }
#pragma unroll
        for (int k = 0; k < NSET; ++k) {
            double q[PE], a[PE], s = 0.0;
#pragma unroll
            for (int e = 0; e < PE; ++e) {
                q[e] = r0 + e < S ? w[(long long)k * S + gi[e]] : 0.0;
                s += q[e];
                a[e] = s;
            }
            double tot;
            const double start = carry[k] + cta_exscan(s, sh, &tot);
#pragma unroll
            for (int e = 0; e < PE; ++e) {
                const int r = r0 + e;
                if (r < S) {
                    const double P = (double)(r + 1) / Sd, Q = start + a[e];
                    num[k] += dl[e] * cjs_term(P, Q);
                    den[k] += dl[e] * (P + Q);
                    const double x = REV ? -y[e] : y[e];
                    if (REV) {
                        const double d = x - mean[k + 1];
                        acc[k] += q[e] * (d * d);
                    } else {
                        acc[k] += q[e] * x;
                    }
                }
            }
            carry[k] += tot;
        }
    }
#pragma unroll
    for (int k = 0; k < NSET; ++k) {
        const double nk = cta_sum(num[k], sh), dk = cta_sum(den[k], sh);
        cjs[k] = dk > 0.0 ? sqrt(fmax(nk, 0.0) / dk) : 0.0;
        mom[k] = cta_sum(acc[k], sh);
    }
    mom[NSET] = cta_sum(acc[NSET], sh);
}

// One column per CTA (blockIdx.x = d - d0): out[row * D + d], rows 0..3 cjs = max(cjs+, cjs-) of the weight sets, 4 the
// mean, 5..8 the weighted means, 9 the sd, 10..13 the weighted sds.  A flagged column: NaN in every row.
__global__ void __launch_bounds__(LT) psens_col_kernel(const uint32_t* __restrict__ keys, const int* __restrict__ idx,
                                                       int S, int D, int d0, const double* __restrict__ w,
                                                       const int* __restrict__ nonfinite, double* __restrict__ out) {
    __shared__ double sh[LW];
    const int j = blockIdx.x, d = d0 + j;
    if (nonfinite[d]) {
        if (threadIdx.x < HMCX_PSENS_ROWS) write_nan(out + (long long)threadIdx.x * D + d);
        return;
    }
    const uint32_t* kp = keys + (long long)j * S;
    const int* ip = idx + (long long)j * S;
    double cp[NSET], cm[NSET], m1[NSET + 1], m2[NSET + 1], mean[NSET + 1];
    sweep<false>(kp, ip, S, w, nullptr, sh, cp, m1);
    mean[0] = m1[NSET] / (double)S;
#pragma unroll
    for (int k = 0; k < NSET; ++k) mean[k + 1] = m1[k];
    sweep<true>(kp, ip, S, w, mean, sh, cm, m2);
    if (threadIdx.x == 0) {
#pragma unroll
        for (int k = 0; k < NSET; ++k) {
            out[(long long)k * D + d] = fmax(cp[k], cm[k]);
            out[(long long)(NSET + 1 + k) * D + d] = mean[k + 1];
            out[(long long)(2 * NSET + 2 + k) * D + d] = sqrt(m2[k]);
        }
        out[(long long)NSET * D + d] = mean[0];
        out[(long long)(2 * NSET + 1) * D + d] = sqrt(m2[NSET] / (double)S);
    }
}

}  // namespace

int mlp_log_prior(const float* x, long long cs, long long ds, int C, int n, int T, const int* sizes, const double* tau,
                  double* out, cudaStream_t st) {
    PriorArgs a;
    a.T = T;
    a.off[0] = 0;
    for (int t = 0; t < T; ++t) {
        a.off[t + 1] = a.off[t] + sizes[t];
        a.tau[t] = tau[t];
    }
    mlp_log_prior_kernel<<<C * n, LT, 0, st>>>(x, cs, ds, n, a, out);
    return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA;
}

int psens_ll_totals(const float* ll, long long cs, long long ds, int C, int n, int r0, int k, const double* coef,
                    double* totals, cudaStream_t st) {
    const int S = C * n;
    psens_ll_kernel<<<(S + 7) / 8, 256, 0, st>>>(ll, cs, ds, n, S, k, r0, coef, totals);
    return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA;
}

size_t psens_workspace_bytes(int C, int n, int k) { return rank_sort_workspace_bytes(C, n, k); }

int psens_weights(const float* nr, long long cs, long long ds, int C, int n, int K, double r_eff, double* w,
                  double* pareto_k, int* tail, int* nonfinite, void* ws, cudaStream_t st) {
    const int S = C * n;
    const uint32_t* keys = nullptr;
    const int* idx = nullptr;
    int rc = rank_sort(nr, cs, ds, C, n, 0, K, nonfinite, ws, &keys, &idx, st);
    if (rc != HMCX_OK) return rc;
    const int M = loo_tail_cap(S, r_eff);
    const size_t smem = (size_t)(30 + (int)floor(sqrt((double)M))) * sizeof(double);
    if (cudaFuncSetAttribute(psens_weights_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) !=
        cudaSuccess)
        return HMCX_ERR_CUDA;
    psens_weights_kernel<<<K, LT, smem, st>>>(keys, idx, S, M, nonfinite, w, pareto_k, tail);
    return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA;
}

int psens_pass(const float* x, long long cs, long long ds, int C, int n, int D, int d0, int k, const double* w,
               double* out, int* nonfinite, void* ws, cudaStream_t st) {
    const int S = C * n;
    const uint32_t* keys = nullptr;
    const int* idx = nullptr;
    int rc = rank_sort(x, cs, ds, C, n, d0, k, nonfinite, ws, &keys, &idx, st);
    if (rc != HMCX_OK) return rc;
    psens_col_kernel<<<k, LT, 0, st>>>(keys, idx, S, D, d0, w, nonfinite, out);
    return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA;
}

}  // namespace hmcx
