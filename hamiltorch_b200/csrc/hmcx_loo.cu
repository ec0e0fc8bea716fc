// hmcx_loo.cu -- Pareto-smoothed importance-sampling leave-one-out (PSIS-LOO, Vehtari, Gelman & Gabry 2017; Vehtari,
// Simpson, Gelman, Yao & Gabry 2024) and WAIC per data point, from a pointwise log-likelihood block.
// hamiltorch_b200/loo.py drives it; tests/loo_oracle.py is the numpy definition.
//
// The block is fp32 ll[c, s, i] at ll + c*chain_stride + s*draw_stride + i: C chains of n draws, S = C*n pooled draws per
// data point i.  A call handles a slab of k points [i0, i0 + k):
//   1-2. the key build and segmented radix sort of hmcx_rank.cu (rank_sort), segments = points: every point's S draws in
//        ascending ll order, i.e. descending r = -ll;
//   3.   one CTA per point, in fp64: the tail cut, the Zhang & Stephens (2009) generalised-Pareto fit, the smoothed
//        log-ratios and the LOO / WAIC terms.  Every draw-sum is a thread-strided loop over the sorted draws followed by a
//        fixed shuffle tree and a fixed in-order sum over warps; there are no atomics, so the outputs depend on the block
//        alone (not on k or the launch geometry) and the same block gives the same bits.
// The smoothed tail needs no draw index: each term of every sum is a function of the sorted position only.  LOO-PIT
// (hmcx_loo_pit_pass, hamiltorch_b200/ppc.py) runs the same sort and the same smoothing (psis_smooth), then reads each
// sorted draw's network outputs and noise precision through the flat index c*n + s the sort carries alongside the key.
// Per-chain PSIS-LOO (hmcx_loo_chain_pass, loo.psis_loo_chains) runs PSIS over each chain's n draws alone: one CTA per
// (point, chain) sorts the chain's keys in shared memory and calls the same psis_smooth and sums.  psis_smooth and the
// CTA reductions live in hmcx_psis.cuh, shared with the power-scaling weights of hmcx_psens.cu.
#include "hmcx_psis.cuh"

namespace hmcx {

size_t rank_sort_workspace_bytes(int C, int n, int k);
int rank_sort(const float* x, long long cs, long long ds, int C, int n, int d0, int k, int* nonfinite, void* ws,
              const uint32_t** sorted_keys, const int** sorted_idx, cudaStream_t st);

namespace {

// One point per CTA.  keys: the slab's sorted keys, S per point.  M = ceil(min(0.2 S, 3 sqrt(S / r_eff))) (host).
// out[row * N + i], rows: 0 elpd_loo, 1 p_loo, 2 pareto_k, 3 lppd, 4 p_waic, 5 elpd_waic; tail[i] = M'.
// Dynamic shared memory: 30 + floor(sqrt(M)) doubles (the L_j of the fit).
__global__ void __launch_bounds__(LT) loo_point_kernel(const uint32_t* __restrict__ keys, int S, int M, int N, int i0,
                                                       const int* __restrict__ nonfinite, double* __restrict__ out,
                                                       int* __restrict__ tail) {
    extern __shared__ double sL[];
    __shared__ double sh[LW];
    const int j = blockIdx.x, i = i0 + j, tid = threadIdx.x;
    const uint32_t* kp = keys + (long long)j * S;
    if (nonfinite[i]) {
        if (tid == 0) {
            for (int r = 0; r < 6; ++r) write_nan(out + (long long)r * N + i);
            tail[i] = 0;
        }
        return;
    }
    const Psis w = psis_smooth(kp, S, M, sL, sh);
    const double lse_w = w.lse_w;
    // 7. elpd_loo = logsumexp(lw + ll), lw normalised
    double mx = -DBL_MAX;
    for (int p = tid; p < S; p += LT) mx = fmax(mx, (w.lw(p) - lse_w) + w.llv(p));
    mx = cta_max(mx, sh);
    double s = 0.0;
    for (int p = tid; p < S; p += LT) s += exp(((w.lw(p) - lse_w) + w.llv(p)) - mx);
    const double elpd = mx + log(cta_sum(s, sh));
    // lppd = logsumexp(ll) - log S (the largest ll is the last sorted draw); p_waic = var(ll), ddof 1
    const double llmax = w.llv(S - 1);
    double se = 0.0, sm = 0.0;
    for (int p = tid; p < S; p += LT) { const double v = w.llv(p); se += exp(v - llmax); sm += v; }
    const double lppd = (llmax + log(cta_sum(se, sh))) - log((double)S);
    const double mean = cta_sum(sm, sh) / S;
    double sv = 0.0;
    for (int p = tid; p < S; p += LT) { const double d = w.llv(p) - mean; sv += d * d; }
    const double pw = cta_sum(sv, sh) / (S - 1);
    if (tid == 0) {
        out[i] = elpd;
        out[(long long)N + i] = lppd - elpd;
        out[2LL * N + i] = w.khat;
        out[3LL * N + i] = lppd;
        out[4LL * N + i] = pw;
        out[5LL * N + i] = lppd - pw;
        tail[i] = w.Mt;
    }
}

// LOO-PIT, one point per CTA: pit[i, o] = sum_p w~_p Phi((y_io - f_{g_p, i, o}) sqrt(tau_{g_p})) over the sorted positions p
// of the point's draws, w~_p = exp(lw(p) - lse_w) the normalised PSIS weights of psis_smooth and g_p = c n + s the flat
// index the sort carried.  Phi(x) = erfc(-x / sqrt 2) / 2 in fp64; each output's sum is thread-strided over p, then the
// fixed tree of cta_sum.  pareto_k[i] = k-hat.  A point with a non-finite draw: NaN pit and k-hat.
__global__ void __launch_bounds__(LT) loo_pit_kernel(const uint32_t* __restrict__ keys, const int* __restrict__ idx,
                                                     int S, int M, int n, int O, int i0, const float* __restrict__ f,
                                                     long long fcs, long long fds, const float* __restrict__ y,
                                                     const float* __restrict__ tau, long long tcs, long long tds,
                                                     const int* __restrict__ nonfinite, double* __restrict__ pit,
                                                     double* __restrict__ pareto_k) {
    extern __shared__ double sL[];
    __shared__ double sh[LW];
    const int j = blockIdx.x, i = i0 + j, tid = threadIdx.x;
    const uint32_t* kp = keys + (long long)j * S;
    const int* ip = idx + (long long)j * S;
    if (nonfinite[i]) {
        if (tid == 0) {
            for (int o = 0; o < O; ++o) write_nan(pit + (long long)i * O + o);
            write_nan(pareto_k + i);
        }
        return;
    }
    const Psis w = psis_smooth(kp, S, M, sL, sh);
    for (int o = 0; o < O; ++o) {
        const double yo = (double)y[(long long)i * O + o];
        double s = 0.0;
        for (int p = tid; p < S; p += LT) {
            const int g = ip[p], c = g / n, t = g - c * n;
            const double fv = (double)f[(long long)c * fcs + (long long)t * fds + (long long)i * O + o];
            const double sq = sqrt((double)tau[(long long)c * tcs + (long long)t * tds]);
            s += exp(w.lw(p) - w.lse_w) * (0.5 * erfc(-((yo - fv) * sq) * 0.70710678118654752440));
        }
        s = cta_sum(s, sh);
        if (tid == 0) pit[(long long)i * O + o] = s;
    }
    if (tid == 0) pareto_k[i] = w.khat;
}

// The order-preserving key of rank_sort (hmcx_rank.cu): -0.0 canonicalised to +0.0, ascending keys = ascending values.
__device__ __forceinline__ uint32_t chain_key(float v) {
    if (v == 0.f) v = 0.f;
    const uint32_t u = __float_as_uint(v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// Per-chain PSIS-LOO, one CTA per (point, chain) of the slab: blockIdx.x = i - i0, blockIdx.y = c.  The chain's n keys
// are sorted in shared memory by an LSD radix sort (four 8-bit passes; each pass a digit histogram, an exclusive scan
// over the 256 digits and a stable scatter in rounds of LT keys, ordered by warp then lane), then psis_smooth and the
// elpd_loo / lppd loops of loo_point_kernel run on them unchanged.  A sorted key sequence does not depend on how it was
// sorted, so column c holds the bits hmcx_loo_pass writes for the one-chain block ll[c:c+1].
// out[r * C * N + c * N + i], rows: 0 elpd_loo, 1 lppd, 2 pareto_k; tail[c * N + i] = M', nonfinite[c * N + i].
// Dynamic shared memory: nL = 30 + floor(sqrt(M)) doubles (the L_j of the fit), then 2 n uint32 keys (ping-pong).
__global__ void __launch_bounds__(LT) loo_chain_kernel(const float* __restrict__ ll, long long cs, long long ds, int C,
                                                       int n, int N, int i0, int M, int nL, double* __restrict__ out,
                                                       int* __restrict__ tail, int* __restrict__ nonfinite) {
    extern __shared__ double sL[];
    __shared__ double sh[LW];
    __shared__ uint32_t base[256];
    __shared__ uint32_t wc[LW][256];
    __shared__ uint32_t wsum[LW];
    __shared__ int bad;
    const int i = i0 + (int)blockIdx.x, c = (int)blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const long long o = (long long)c * N + i, CN = (long long)C * N;
    uint32_t* src = reinterpret_cast<uint32_t*>(sL + nL);
    uint32_t* dst = src + n;
    if (tid == 0) bad = 0;
    __syncthreads();
    const float* lp = ll + (long long)c * cs + i;
    for (int s = tid; s < n; s += LT) {
        const float v = lp[(long long)s * ds];
        if (!finite_f(v)) bad = 1;
        src[s] = chain_key(v);
    }
    __syncthreads();
    if (bad) {
        if (tid == 0) {
            for (int r = 0; r < 3; ++r) write_nan(out + r * CN + o);
            tail[o] = 0;
            nonfinite[o] = 1;
        }
        return;
    }
    const uint32_t lt_mask = (1u << lane) - 1u;
    for (int shift = 0; shift < 32; shift += 8) {
        base[tid] = 0;
        __syncthreads();
        for (int s = tid; s < n; s += LT) atomicAdd(&base[(src[s] >> shift) & 255u], 1u);
        __syncthreads();
        // exclusive scan over the digits: thread tid owns digit tid
        const uint32_t h = base[tid];
        uint32_t incl = h;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t u = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += u;
        }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        uint32_t run = incl - h;
        for (int w = 0; w < warp; ++w) run += wsum[w];
        base[tid] = run;
        __syncthreads();
        for (int r0 = 0; r0 < n; r0 += LT) {
            const int s = r0 + tid;
            const bool valid = s < n;
            const uint32_t key = valid ? src[s] : 0u;
            const uint32_t dg = valid ? (key >> shift) & 255u : 256u;
#pragma unroll
            for (int w = 0; w < LW; ++w) wc[w][tid] = 0;
            __syncthreads();
            const uint32_t peers = __match_any_sync(0xffffffffu, dg);
            if (valid && lane == __ffs(peers) - 1) wc[warp][dg] = __popc(peers);
            __syncthreads();
            uint32_t b = base[tid];
#pragma unroll
            for (int w = 0; w < LW; ++w) {
                const uint32_t cnt = wc[w][tid];
                wc[w][tid] = b;
                b += cnt;
            }
            base[tid] = b;
            __syncthreads();
            if (valid) dst[wc[warp][dg] + __popc(peers & lt_mask)] = key;
            __syncthreads();
        }
        uint32_t* t = src; src = dst; dst = t;
    }
    // four passes: the sorted keys are back in the first buffer (src)
    const int S = n;
    const Psis w = psis_smooth(src, S, M, sL, sh);
    const double lse_w = w.lse_w;
    double mx = -DBL_MAX;
    for (int p = tid; p < S; p += LT) mx = fmax(mx, (w.lw(p) - lse_w) + w.llv(p));
    mx = cta_max(mx, sh);
    double s = 0.0;
    for (int p = tid; p < S; p += LT) s += exp(((w.lw(p) - lse_w) + w.llv(p)) - mx);
    const double elpd = mx + log(cta_sum(s, sh));
    const double llmax = w.llv(S - 1);
    double se = 0.0;
    for (int p = tid; p < S; p += LT) se += exp(w.llv(p) - llmax);
    const double lppd = (llmax + log(cta_sum(se, sh))) - log((double)S);
    if (tid == 0) {
        out[o] = elpd;
        out[CN + o] = lppd;
        out[2 * CN + o] = w.khat;
        tail[o] = w.Mt;
        nonfinite[o] = 0;
    }
}

}  // namespace

int loo_tail_cap(int S, double r_eff) {
    return (int)ceil(fmin(0.2 * S, 3.0 * sqrt(S / r_eff)));
}

size_t loo_workspace_bytes(int C, int n, int k) { return rank_sort_workspace_bytes(C, n, k); }

// dynamic shared memory of the PSIS kernels: the 30 + floor(sqrt(M')) <= 30 + floor(sqrt(M)) L_j of the fit
static size_t fit_smem(int M) { return (size_t)(30 + (int)floor(sqrt((double)M))) * sizeof(double); }

int loo_pass(const float* ll, long long cs, long long ds, int C, int n, int N, int i0, int k, double r_eff, double* out,
             int* tail, int* nonfinite, void* ws, cudaStream_t st) {
    const int S = C * n;
    const uint32_t* keys = nullptr;
    const int* idx = nullptr;
    int rc = rank_sort(ll, cs, ds, C, n, i0, k, nonfinite, ws, &keys, &idx, st);
    if (rc != HMCX_OK) return rc;
    const int M = loo_tail_cap(S, r_eff);
    const size_t smem = fit_smem(M);
    if (cudaFuncSetAttribute(loo_point_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
        return HMCX_ERR_CUDA;
    loo_point_kernel<<<k, LT, smem, st>>>(keys, S, M, N, i0, nonfinite, out, tail);
    return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA;
}

int loo_pit_pass(const float* ll, long long cs, long long ds, const float* f, long long fcs, long long fds, int C, int n,
                 int O, int i0, int k, double r_eff, const float* y, const float* tau, long long tcs, long long tds,
                 double* pit, double* pareto_k, int* nonfinite, void* ws, cudaStream_t st) {
    const int S = C * n;
    const uint32_t* keys = nullptr;
    const int* idx = nullptr;
    int rc = rank_sort(ll, cs, ds, C, n, i0, k, nonfinite, ws, &keys, &idx, st);
    if (rc != HMCX_OK) return rc;
    const int M = loo_tail_cap(S, r_eff);
    const size_t smem = fit_smem(M);
    if (cudaFuncSetAttribute(loo_pit_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
        return HMCX_ERR_CUDA;
    loo_pit_kernel<<<k, LT, smem, st>>>(keys, idx, S, M, n, O, i0, f, fcs, fds, y, tau, tcs, tds, nonfinite, pit,
                                        pareto_k);
    return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA;
}

// Per-chain PSIS-LOO of the points [i0, i0 + k): one launch, no workspace (every chain's keys live in shared memory).
int loo_chain_pass(const float* ll, long long cs, long long ds, int C, int n, int N, int i0, int k, double r_eff,
                   double* out, int* tail, int* nonfinite, cudaStream_t st) {
    const int M = loo_tail_cap(n, r_eff);
    const int nL = 30 + (int)floor(sqrt((double)M));
    const size_t smem = (size_t)nL * sizeof(double) + 2 * (size_t)n * sizeof(uint32_t);
    if (cudaFuncSetAttribute(loo_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
        return HMCX_ERR_CUDA;
    loo_chain_kernel<<<dim3((unsigned)k, (unsigned)C), LT, smem, st>>>(ll, cs, ds, C, n, N, i0, M, nL, out, tail,
                                                                      nonfinite);
    return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA;
}

}  // namespace hmcx
