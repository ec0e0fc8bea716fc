// hmcx_psis.cuh -- the Pareto smoothing of one sorted column of draws (psis_smooth) and the fixed-order CTA reductions
// (cta_sum / cta_max) shared by the PSIS kernels: hmcx_loo.cu (PSIS-LOO, LOO-PIT, per-chain PSIS-LOO) and hmcx_psens.cu
// (the power-scaling importance weights).  The input is a column of rank_sort keys (hmcx_rank.cu): ascending ll, i.e.
// descending log-ratio r = -ll.
#pragma once
#include <cfloat>
#include "hmcx_common.cuh"

namespace hmcx {
namespace {

constexpr int LT = 256;                     // threads per column
constexpr int LW = LT / 32;

__device__ __forceinline__ double ll_of_key(uint32_t k) {
    return (double)__uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// Fixed-order CTA sum / max of one double per thread; every thread gets the result.  The xor tree leaves the same bits
// in every lane (each level adds the same two operands), the warp partials are summed in warp order.
__device__ __forceinline__ double cta_sum(double v, double* sh) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    double s = sh[0];
#pragma unroll
    for (int w = 1; w < LW; ++w) s += sh[w];
    __syncthreads();
    return s;
}

__device__ __forceinline__ double cta_max(double v, double* sh) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    double s = sh[0];
#pragma unroll
    for (int w = 1; w < LW; ++w) s = fmax(s, sh[w]);
    __syncthreads();
    return s;
}

// The Pareto smoothing of one column's S sorted draws (steps 3-6 of hmcx_loo.cu): the tail cut, the generalised-Pareto
// fit and the normalised log-weights lw(p) - lse_w of sorted position p.  Called by every thread of the CTA; sL holds
// 30 + floor(sqrt(M)) doubles, sh one per warp.
struct Psis {
    const uint32_t* kp;
    double rmax, ec, khat, sigma, lse_w;
    int Mt;
    bool smooth;
    __device__ __forceinline__ double llv(int p) const { return ll_of_key(kp[p]); }
    __device__ __forceinline__ double rr(int p) const { return -llv(p) - rmax; }   // shifted log-ratio, rr(0) = 0
    // 6. log-ratios: the tail (ascending z = Mt - p) replaced by the GPD quantiles, then capped at 0 (the largest raw one)
    __device__ __forceinline__ double lw(int p) const {
        double v;
        if (smooth && p < Mt) {
            const double pz = (Mt - p - 0.5) / Mt;
            const double q = khat == 0.0 ? -sigma * log1p(-pz) : sigma * expm1(-khat * log1p(-pz)) / khat;
            v = log(q + ec);
        } else {
            v = rr(p);
        }
        return v > 0.0 ? 0.0 : v;
    }
};

__device__ __forceinline__ Psis psis_smooth(const uint32_t* kp, int S, int M, double* sL, double* sh) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    Psis w;
    w.kp = kp;
    w.rmax = -w.llv(0);
    // 3-4. cutoff = the (M+1)-th largest r, floored; the tail is {r > cutoff} = sorted positions [0, Mt)
    const double c = fmax(w.rr(M), log(DBL_MIN));
    int lo = 0, hi = M;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (w.rr(mid) > c) lo = mid + 1; else hi = mid;
    }
    const int Mt = lo;
    w.Mt = Mt;
    const double ec = exp(c);
    w.ec = ec;
    auto xt = [&](int t) { return exp(w.rr(Mt - t)) - ec; };   // ascending exceedances, t = 1..Mt
    // 5. generalised-Pareto fit (Zhang & Stephens 2009, with the weakly informative prior of Vehtari et al.)
    double khat = __longlong_as_double(0x7ff0000000000000LL), sigma = 0.0;
    if (Mt > 4) {
        const int m = 30 + (int)floor(sqrt((double)Mt));
        const double x_max = xt(Mt), x_q = xt((int)floor(Mt / 4.0 + 0.5));
        auto b_of = [&](int jj) { return 1.0 / x_max + (1.0 - sqrt(m / (jj - 0.5))) / (3.0 * x_q); };
        for (int jj = 1 + warp; jj <= m; jj += LW) {            // a warp per j: lane-strided sum, xor tree
            const double b = b_of(jj);
            double s = 0.0;
            for (int t = 1 + lane; t <= Mt; t += 32) s += log1p(-b * xt(t));
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            const double k = s / Mt;
            if (lane == 0) sL[jj - 1] = Mt * (log(-b / k) - k - 1.0);
        }
        __syncthreads();
        double wsum = 0.0, wbsum = 0.0;
        for (int jj = 1 + tid; jj <= m; jj += LT) {
            const double Lj = sL[jj - 1];
            double d = 0.0;
            for (int l = 0; l < m; ++l) d += exp(sL[l] - Lj);
            const double wj = 1.0 / d;
            if (wj >= 10.0 * DBL_EPSILON) { wsum += wj; wbsum += wj * b_of(jj); }
        }
        const double bbar = cta_sum(wbsum, sh) / cta_sum(wsum, sh);
        double s = 0.0;
        for (int t = 1 + tid; t <= Mt; t += LT) s += log1p(-bbar * xt(t));
        const double xi = cta_sum(s, sh) / Mt;
        sigma = -xi / bbar;
        khat = (Mt * xi + 5.0) / (Mt + 10.0);
    }
    w.khat = khat;
    w.sigma = sigma;
    w.smooth = Mt > 4 && isfinite(khat);
    // normalisation: lse_w = logsumexp over the draws of the capped log-ratios
    double mx = -DBL_MAX;
    for (int p = tid; p < S; p += LT) mx = fmax(mx, w.lw(p));
    mx = cta_max(mx, sh);
    double s = 0.0;
    for (int p = tid; p < S; p += LT) s += exp(w.lw(p) - mx);
    w.lse_w = mx + log(cta_sum(s, sh));
    return w;
}

__device__ __forceinline__ void write_nan(double* p) { *p = __longlong_as_double(0x7ff8000000000000LL); }

}  // namespace
}  // namespace hmcx
