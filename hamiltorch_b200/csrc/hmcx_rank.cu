// hmcx_rank.cu -- the rank pass behind rank-normalised split-R-hat, bulk-ESS and tail-ESS (Vehtari et al. 2021), and
// the indicator pass behind tail-ESS.  hamiltorch_b200/diagnostics.py::rank_summary feeds the z and indicator blocks
// these write through the split-R-hat / ESS passes of hmcx_diag.cu; tests/rank_oracle.py is the numpy definition.
//
// The block is fp32 x[c, s, d] at x + c*chain_stride + s*draw_stride + d, C chains of n draws, L = C*n draws per
// dimension, flat draw index f = c*n + s.  The split set drops the middle draw s == m of an odd n (m = n/2); it holds
// Ns = 2*C*m draws.  One call of the rank pass handles a slab of k dimensions [d0, d0 + k):
//   1. key build: the slab's rows are read coalesced through a shared-memory transpose and written dimension-major as
//      an order-preserving uint32 key (-0.0 canonicalised to +0.0, so the two tie) with its flat index;
//   2. segmented LSD radix sort, segments = dimensions: four 8-bit passes, each a per-(dimension, tile) digit
//      histogram, a per-dimension exclusive scan and a stable in-tile scatter (warp match + per-warp digit offsets);
//   3. the kept-prefix P[i] = number of split-set draws among the first i sorted draws (a tile scan);
//   4. the quantiles of the full set, read off the sorted keys with numpy's 'linear' arithmetic, and the first sorted
//      position u0 whose value is >= the median;
//   5. the rank / z pass: every sorted draw finds its tie run by a galloping search from its own position (O(1) for a
//      draw without ties), the bulk rank is the mean split-set position over the run, z = Phi^-1((r - 3/8)/(Ns + 1/4))
//      in fp64, stored as fp32 at the draw's (c, s).  Folded ranks need no second sort: the draws at [u0, L) ascending
//      and those at [0, u0) descending are two sequences already sorted by |x - median|, so a draw's folded rank is
//      read off its own sequence's tie run plus a galloping search into the other one, started from where the
//      previous draw of the same lane landed (each warp walks a short contiguous stretch, a merge in all but name).
// Integer atomics count digits in shared memory and OR the non-finite flags; there are no floating-point atomics, and
// every output is a function of the block alone (not of k or of the launch geometry).
#include "hmcx_common.cuh"

namespace hmcx {
namespace {

constexpr int RT = 256;                    // threads of the sort / scan CTAs
constexpr int RI = 8;                      // draws per thread per tile
constexpr int TILE = RT * RI;              // draws per (dimension, tile)
constexpr int SCAN_T = 1024;               // threads of the per-dimension scan
constexpr int FOLD_E = 16;                 // sorted draws per thread in the rank / z pass

__device__ __forceinline__ uint32_t to_key(float v) {
    if (v == 0.f) v = 0.f;                                     // -0.0 -> +0.0
    const uint32_t u = __float_as_uint(v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float from_key(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// 1. keys[j*L + f] = to_key(x[f, d0 + j]), idx[j*L + f] = f; nonfinite[d0 + j] |= 1 for a non-finite draw.  A CTA
// transposes a 32-draw x 32-dimension tile through shared memory.
__global__ void __launch_bounds__(32 * 8) rank_keys_kernel(const float* __restrict__ x, long long cs, long long ds,
                                                          int n, int L, int d0, int k, uint32_t* __restrict__ keys,
                                                          int* __restrict__ idx, int* __restrict__ nonfinite) {
    __shared__ uint32_t tile[32][33];
    __shared__ int bad[32];
    const int tx = threadIdx.x, ty = threadIdx.y;
    const int f0 = blockIdx.x * 32, j0 = blockIdx.y * 32;
    if (ty == 0) bad[tx] = 0;
    __syncthreads();
    for (int r = ty; r < 32; r += 8) {
        const int f = f0 + r, j = j0 + tx;
        if (f < L && j < k) {
            const int c = f / n, s = f - c * n;
            const float v = x[(long long)c * cs + (long long)s * ds + d0 + j];
            if (!finite_f(v)) bad[tx] = 1;
            tile[r][tx] = to_key(v);
        }
    }
    __syncthreads();
    if (ty == 0 && bad[tx] && j0 + tx < k) atomicOr(&nonfinite[d0 + j0 + tx], 1);
    for (int r = ty; r < 32; r += 8) {
        const int j = j0 + r, f = f0 + tx;
        if (j < k && f < L) {
            keys[(long long)j * L + f] = tile[tx][r];
            idx[(long long)j * L + f] = f;
        }
    }
}

// 2a. cnt[j][digit][t] = number of draws of tile t of segment j with that digit.
__global__ void __launch_bounds__(RT) radix_hist_kernel(const uint32_t* __restrict__ keys, int L, int nt, int shift,
                                                        uint32_t* __restrict__ cnt) {
    __shared__ uint32_t h[256];
    const int t = blockIdx.x, j = blockIdx.y;
    h[threadIdx.x] = 0;
    __syncthreads();
    const uint32_t* kp = keys + (long long)j * L;
#pragma unroll
    for (int q = 0; q < RI; ++q) {
        const int i = t * TILE + q * RT + threadIdx.x;
        if (i < L) atomicAdd(&h[(kp[i] >> shift) & 255u], 1u);
    }
    __syncthreads();
    cnt[((long long)j * 256 + threadIdx.x) * nt + t] = h[threadIdx.x];
}

// In-place exclusive scan of len uint32 per segment (segment = blockIdx.x); each thread owns a contiguous stretch.
__global__ void __launch_bounds__(SCAN_T) seg_scan_kernel(uint32_t* __restrict__ a, int len) {
    __shared__ uint32_t warp_sum[SCAN_T / 32];
    uint32_t* p = a + (long long)blockIdx.x * len;
    const int per = (len + SCAN_T - 1) / SCAN_T;
    const int b = threadIdx.x * per, e = min(b + per, len);
    uint32_t s = 0;
    for (int i = b; i < e; ++i) s += p[i];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    uint32_t incl = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    if (lane == 31) warp_sum[w] = incl;
    __syncthreads();
    if (w == 0) {
        uint32_t v = warp_sum[lane], iv = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t u = __shfl_up_sync(0xffffffffu, iv, o);
            if (lane >= o) iv += u;
        }
        warp_sum[lane] = iv - v;
    }
    __syncthreads();
    uint32_t run = warp_sum[w] + incl - s;
    for (int i = b; i < e; ++i) {
        const uint32_t v = p[i];
        p[i] = run;
        run += v;
    }
}

// 2c. Stable scatter of one tile by the digit at `shift`: rounds of RT draws in order; inside a round, draws are
// ordered by warp, then by lane (peers of a digit from __match_any_sync, offsets across warps from a shared table).
__global__ void __launch_bounds__(RT) radix_scatter_kernel(const uint32_t* __restrict__ kin, const int* __restrict__ iin,
                                                           uint32_t* __restrict__ kout, int* __restrict__ iout, int L,
                                                           int nt, int shift, const uint32_t* __restrict__ cnt) {
    __shared__ uint32_t base[256];
    __shared__ uint32_t wc[RT / 32][256];
    const int t = blockIdx.x, j = blockIdx.y;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const long long off = (long long)j * L;
    base[threadIdx.x] = cnt[((long long)j * 256 + threadIdx.x) * nt + t];
    uint32_t key[RI];
    int id[RI];
#pragma unroll
    for (int q = 0; q < RI; ++q) {
        const int i = t * TILE + q * RT + threadIdx.x;
        key[q] = i < L ? kin[off + i] : 0u;
        id[q] = i < L ? iin[off + i] : 0;
    }
    const uint32_t lt_mask = (1u << lane) - 1u;
#pragma unroll
    for (int q = 0; q < RI; ++q) {
        const bool valid = t * TILE + q * RT + threadIdx.x < L;
        const uint32_t dg = valid ? (key[q] >> shift) & 255u : 256u;
#pragma unroll
        for (int ww = 0; ww < RT / 32; ++ww) wc[ww][threadIdx.x] = 0;
        __syncthreads();
        const uint32_t peers = __match_any_sync(0xffffffffu, dg);
        if (valid && lane == __ffs(peers) - 1) wc[w][dg] = __popc(peers);
        __syncthreads();
        uint32_t run = base[threadIdx.x];
#pragma unroll
        for (int ww = 0; ww < RT / 32; ++ww) {
            const uint32_t c = wc[ww][threadIdx.x];
            wc[ww][threadIdx.x] = run;
            run += c;
        }
        base[threadIdx.x] = run;
        __syncthreads();
        if (valid) {
            const uint32_t pos = wc[w][dg] + __popc(peers & lt_mask);
            kout[off + pos] = key[q];
            iout[off + pos] = id[q];
        }
        __syncthreads();
    }
}

__device__ __forceinline__ bool kept(int f, int n, int m) {
    const int s = f % n;
    return s < m || s >= n - m;
}

// 3a. cnt[j][t] = split-set draws in sorted tile t of segment j.
__global__ void __launch_bounds__(RT) kept_count_kernel(const int* __restrict__ idx, int L, int n, int nt,
                                                        uint32_t* __restrict__ cnt) {
    __shared__ uint32_t ws[RT / 32];
    const int t = blockIdx.x, j = blockIdx.y;
    uint32_t c = 0;
#pragma unroll
    for (int q = 0; q < RI; ++q) {
        const int i = t * TILE + threadIdx.x * RI + q;
        if (i < L) c += kept(idx[(long long)j * L + i], n, n / 2);
    }
    for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t s = 0;
        for (int w = 0; w < RT / 32; ++w) s += ws[w];
        cnt[(long long)j * nt + t] = s;
    }
}

// 3b. P[j*(L+1) + i] = split-set draws among sorted positions < i of segment j; P[.. + L] = Ns.
__global__ void __launch_bounds__(RT) kept_prefix_kernel(const int* __restrict__ idx, int L, int n, int nt,
                                                         const uint32_t* __restrict__ cnt, int* __restrict__ P) {
    __shared__ uint32_t ws[RT / 32];
    const int t = blockIdx.x, j = blockIdx.y;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int fl[RI];
    uint32_t s = 0;
#pragma unroll
    for (int q = 0; q < RI; ++q) {
        const int i = t * TILE + threadIdx.x * RI + q;
        fl[q] = i < L ? kept(idx[(long long)j * L + i], n, n / 2) : 0;
        s += fl[q];
    }
    uint32_t incl = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    if (lane == 31) ws[w] = incl;
    __syncthreads();
    uint32_t run = cnt[(long long)j * nt + t] + incl - s;
    for (int ww = 0; ww < w; ++ww) run += ws[ww];
    int* pj = P + (long long)j * (L + 1);
#pragma unroll
    for (int q = 0; q < RI; ++q) {
        const int i = t * TILE + threadIdx.x * RI + q;
        if (i < L) pj[i] = (int)run;
        run += fl[q];
    }
    if (t == nt - 1 && threadIdx.x == RT - 1) pj[L] = (int)run;
}

// numpy 2.3 np.quantile(method='linear') on L sorted values, 0 < q < 1: virtual index vi = (L-1)*q (so 0 <= vi < L-1
// and both neighbours exist), gamma = vi - floor(vi), and _lerp's two branches (b - (b-a)*(1-g) when g >= 0.5).
__device__ double quantile_linear(const uint32_t* __restrict__ k, int L, double q) {
    const double vi = (double)(L - 1) * q;
    const int lo = (int)floor(vi);
    const double a = from_key(k[lo]), b = from_key(k[lo + 1]);
    const double gamma = vi - (double)lo;
    const double diff = b - a;
    return gamma >= 0.5 ? b - diff * (1.0 - gamma) : a + diff * gamma;
}

// 4. q[0*D + d] = q05, q[1*D + d] = median, q[2*D + d] = q95 (NaN for a flagged dimension); u0[j] = first sorted
// position with value >= median.  One thread per dimension.
__global__ void rank_quantiles_kernel(const uint32_t* __restrict__ keys, int L, int D, int d0, int k,
                                      const int* __restrict__ nonfinite, double* __restrict__ q, int* __restrict__ u0) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= k) return;
    const uint32_t* kp = keys + (long long)j * L;
    const int d = d0 + j;
    double med;
    if (L & 1) {
        med = from_key(kp[L / 2]);
    } else {
        med = ((double)from_key(kp[L / 2 - 1]) + (double)from_key(kp[L / 2])) / 2.0;
    }
    const double q05 = quantile_linear(kp, L, 0.05), q95 = quantile_linear(kp, L, 0.95);
    int lo = 0, hi = L;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if ((double)from_key(kp[mid]) < med) lo = mid + 1; else hi = mid;
    }
    u0[j] = lo;
    const bool bad = nonfinite[d] != 0;
    const double nan = __longlong_as_double(0x7ff8000000000000LL);
    q[d] = bad ? nan : q05;
    q[D + d] = bad ? nan : med;
    q[2 * D + d] = bad ? nan : q95;
}

// First b in [0, N] with !pred(b), for pred monotone (true on a prefix), searched outward from the hint h: a
// doubling stride brackets the answer, then a bisection.  Costs O(log |answer - h|) calls of pred.  The bracket is
// 64-bit: near HMCX_RANK_MAX_DRAWS a doubling stride can pass INT_MAX before the bracket is clamped to [0, N].
template <class Pred>
__device__ __forceinline__ int gallop(Pred pred, int N, int h) {
    h = min(max(h, 0), N);
    long long lo, hi;
    if (h < N && pred(h)) {
        lo = h + 1;
        long long step = 1;
        while (lo + step - 1 < N && pred((int)(lo + step - 1))) { lo += step; step <<= 1; }
        hi = min(lo + step - 1, (long long)N);
    } else {
        hi = h;
        long long step = 1;
        while (hi - step >= 0 && !pred((int)(hi - step))) { hi -= step; step <<= 1; }
        lo = max(hi - step + 1, 0LL);
    }
    while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        if (pred((int)mid)) lo = mid + 1; else hi = mid;
    }
    return (int)lo;
}

__device__ __forceinline__ float z_of(double twice_rank, double ns) {
    return (float)normcdfinv((0.5 * twice_rank - 0.375) / (ns + 0.25));
}

// 5. bulk and folded z; grid (ceil(L / (FOLD_E * RT)), k).  A warp owns 32 * FOLD_E consecutive sorted draws and lane l
// takes draws l, l + 32, ..., so the loads of the sorted keys, indices and kept prefix are coalesced; each lane's search
// into the other sequence starts from where its previous draw (32 positions back) landed.
__global__ void __launch_bounds__(RT) rank_z_kernel(const uint32_t* __restrict__ keys, const int* __restrict__ idx,
                                                    const int* __restrict__ P, const int* __restrict__ u0s,
                                                    const double* __restrict__ q, int C, int n, int D, int d0,
                                                    float* __restrict__ bz, long long bcs, long long bds,
                                                    float* __restrict__ fz, long long fcs, long long fds) {
    const int j = blockIdx.y;
    const int L = C * n, m = n / 2;
    const uint32_t* kp = keys + (long long)j * L;
    const int* pj = P + (long long)j * (L + 1);
    const int u0 = u0s[j];
    const double med = q[D + d0 + j];
    const double ns = (double)(2 * C * m);
    const int nu = L - u0, nl = u0;                           // sizes of the upper and lower sequences
    auto fold_up = [&](int a) { return fabs((double)from_key(kp[u0 + a]) - med); };      // ascending in a
    auto fold_lo = [&](int b) { return fabs((double)from_key(kp[u0 - 1 - b]) - med); };  // ascending in b
    int hint_other = 0;
    const int i0 = (blockIdx.x * RT + (threadIdx.x & ~31)) * FOLD_E + (threadIdx.x & 31);
    for (int i = i0; i < min(i0 + 32 * FOLD_E, L); i += 32) {
        const int f = idx[(long long)j * L + i];
        const int c = f / n, s = f - c * n;
        float zb = 0.f, zf = 0.f;
        if (s < m || s >= n - m) {
            const uint32_t key = kp[i];
            const int r0 = gallop([&](int b) { return kp[b] < key; }, L, i);
            const int r1 = gallop([&](int b) { return kp[b] <= key; }, L, i + 1);
            zb = z_of(2.0 * pj[r0] + (double)(pj[r1] - pj[r0]) + 1.0, ns);
            const double fv = fabs((double)from_key(key) - med);
            int less, leq;
            if (i >= u0) {                                     // own sequence: upper; other: lower
                const int a = i - u0;
                const int o0 = gallop([&](int t) { return fold_up(t) < fv; }, nu, a);
                const int o1 = gallop([&](int t) { return fold_up(t) <= fv; }, nu, a + 1);
                const int x0 = gallop([&](int t) { return fold_lo(t) < fv; }, nl, hint_other);
                const int x1 = gallop([&](int t) { return fold_lo(t) <= fv; }, nl, x0);
                hint_other = x0;
                less = (pj[u0 + o0] - pj[u0]) + (pj[u0] - pj[u0 - x0]);
                leq = (pj[u0 + o1] - pj[u0]) + (pj[u0] - pj[u0 - x1]);
            } else {                                           // own: lower; other: upper
                const int b = u0 - 1 - i;
                const int o0 = gallop([&](int t) { return fold_lo(t) < fv; }, nl, b);
                const int o1 = gallop([&](int t) { return fold_lo(t) <= fv; }, nl, b + 1);
                const int x0 = gallop([&](int t) { return fold_up(t) < fv; }, nu, hint_other);
                const int x1 = gallop([&](int t) { return fold_up(t) <= fv; }, nu, x0);
                hint_other = x0;
                less = (pj[u0] - pj[u0 - o0]) + (pj[u0 + x0] - pj[u0]);
                leq = (pj[u0] - pj[u0 - o1]) + (pj[u0 + x1] - pj[u0]);
            }
            zf = z_of(2.0 * less + (double)(leq - less) + 1.0, ns);
        }
        bz[(long long)c * bcs + (long long)s * bds + d0 + j] = zb;
        fz[(long long)c * fcs + (long long)s * fds + d0 + j] = zf;
    }
}

// out[c, s, d] = x[c, s, d] <= thr[d] (fp64 comparison) as 0 / 1.
__global__ void rank_indicator_kernel(const float* __restrict__ x, long long cs, long long ds, int n, int D,
                                      long long total, const double* __restrict__ thr, float* __restrict__ out,
                                      long long ocs, long long ods) {
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total;
         e += (long long)gridDim.x * blockDim.x) {
        const int d = (int)(e % D);
        const long long f = e / D;
        const int c = (int)(f / n), s = (int)(f - (long long)c * n);
        const float v = x[(long long)c * cs + (long long)s * ds + d];
        out[(long long)c * ocs + (long long)s * ods + d] = (double)v <= thr[d] ? 1.f : 0.f;
    }
}

struct RankWs {
    uint32_t *ka, *kb, *cnt;
    int *ia, *ib, *P, *u0;
};

// Byte sizes of the workspace pieces for a slab of k dimensions of L draws, each rounded up to 256 bytes: keys and
// indices twice (the sort ping-pongs), the kept prefix, the digit counts, u0.
void ws_sizes(int L, int k, size_t sz[7]) {
    const size_t nt = (size_t)(L + TILE - 1) / TILE, e = (size_t)L * k * 4;
    const size_t raw[7] = {e, e, e, e, (size_t)(L + 1) * k * 4, (size_t)k * 256 * nt * 4, (size_t)k * 4};
    for (int i = 0; i < 7; ++i) sz[i] = (raw[i] + 255) / 256 * 256;
}

RankWs carve(void* base, int L, int k) {
    size_t sz[7];
    ws_sizes(L, k, sz);
    char* p[7];
    p[0] = (char*)base;
    for (int i = 1; i < 7; ++i) p[i] = p[i - 1] + sz[i - 1];
    return RankWs{(uint32_t*)p[0], (uint32_t*)p[1], (uint32_t*)p[5], (int*)p[2], (int*)p[3], (int*)p[4], (int*)p[6]};
}

// Stages 1-2 on a slab of k segments: nonfinite[d0, d0 + k) cleared then flagged, the keys built into (ka, ia) and
// sorted by four LSD passes that ping-pong through (kb, ib); the sorted keys and flat indices end back in (ka, ia).
int sort_slab(const float* x, long long cs, long long ds, int n, int L, int d0, int k, int* nonfinite, uint32_t* ka,
              uint32_t* kb, int* ia, int* ib, uint32_t* cnt, cudaStream_t st) {
    const int nt = (L + TILE - 1) / TILE;
    if (cudaMemsetAsync(nonfinite + d0, 0, (size_t)k * sizeof(int), st) != cudaSuccess) return HMCX_ERR_CUDA;
    rank_keys_kernel<<<dim3((L + 31) / 32, (k + 31) / 32), dim3(32, 8), 0, st>>>(x, cs, ds, n, L, d0, k, ka, ia,
                                                                                 nonfinite);
    uint32_t *ki = ka, *ko = kb;
    int *ii = ia, *io = ib;
    for (int shift = 0; shift < 32; shift += 8) {
        radix_hist_kernel<<<dim3(nt, k), RT, 0, st>>>(ki, L, nt, shift, cnt);
        seg_scan_kernel<<<k, SCAN_T, 0, st>>>(cnt, 256 * nt);
        radix_scatter_kernel<<<dim3(nt, k), RT, 0, st>>>(ki, ii, ko, io, L, nt, shift, cnt);
        uint32_t* tk = ki; ki = ko; ko = tk;
        int* ti = ii; ii = io; io = ti;
    }
    return HMCX_OK;
}

}  // namespace

size_t rank_workspace_bytes(int C, int n, int k) {
    size_t sz[7], b = 0;
    ws_sizes(C * n, k, sz);
    for (int i = 0; i < 7; ++i) b += sz[i];
    return b;
}

// The sort alone (stages 1-2) for the PSIS passes of hmcx_loo.cu: keys and indices twice plus the digit counts -- the
// pieces 0-3 and 5 of ws_sizes, carved in that order.  Hands back the sorted keys and their flat draw indices c*n + s.
size_t rank_sort_workspace_bytes(int C, int n, int k) {
    size_t sz[7];
    ws_sizes(C * n, k, sz);
    return sz[0] + sz[1] + sz[2] + sz[3] + sz[5];
}

int rank_sort(const float* x, long long cs, long long ds, int C, int n, int d0, int k, int* nonfinite, void* ws,
              const uint32_t** sorted_keys, const int** sorted_idx, cudaStream_t st) {
    const int L = C * n;
    size_t sz[7];
    ws_sizes(L, k, sz);
    char* p = (char*)ws;
    uint32_t* ka = (uint32_t*)p;
    uint32_t* kb = (uint32_t*)(p += sz[0]);
    int* ia = (int*)(p += sz[1]);
    int* ib = (int*)(p += sz[2]);
    uint32_t* cnt = (uint32_t*)(p += sz[3]);
    *sorted_keys = ka;
    *sorted_idx = ia;
    const int rc = sort_slab(x, cs, ds, n, L, d0, k, nonfinite, ka, kb, ia, ib, cnt, st);
    if (rc != HMCX_OK) return rc;
    return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA;
}

int rank_pass(const float* x, long long cs, long long ds, int C, int n, int D, int d0, int k, float* bz, long long bcs,
              long long bds, float* fz, long long fcs, long long fds, double* q, int* nonfinite, void* ws,
              cudaStream_t st) {
    const int L = C * n, nt = (L + TILE - 1) / TILE;
    const RankWs w = carve(ws, L, k);
    const int rc = sort_slab(x, cs, ds, n, L, d0, k, nonfinite, w.ka, w.kb, w.ia, w.ib, w.cnt, st);
    if (rc != HMCX_OK) return rc;
    uint32_t* ki = w.ka;
    int* ii = w.ia;
    // four passes: the sorted keys and indices are back in (ka, ia)
    kept_count_kernel<<<dim3(nt, k), RT, 0, st>>>(ii, L, n, nt, w.cnt);
    seg_scan_kernel<<<k, SCAN_T, 0, st>>>(w.cnt, nt);
    kept_prefix_kernel<<<dim3(nt, k), RT, 0, st>>>(ii, L, n, nt, w.cnt, w.P);
    rank_quantiles_kernel<<<(k + 127) / 128, 128, 0, st>>>(ki, L, D, d0, k, nonfinite, q, w.u0);
    const int per_cta = FOLD_E * RT;
    rank_z_kernel<<<dim3((L + per_cta - 1) / per_cta, k), RT, 0, st>>>(ki, ii, w.P, w.u0, q, C, n, D, d0, bz, bcs, bds,
                                                                      fz, fcs, fds);
    return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA;
}

int rank_indicator(const float* x, long long cs, long long ds, int C, int n, int D, const double* thr, float* out,
                   long long ocs, long long ods, cudaStream_t st) {
    const long long total = (long long)C * n * D;
    const long long blocks = min((total + 255) / 256, 8192LL);
    rank_indicator_kernel<<<(int)blocks, 256, 0, st>>>(x, cs, ds, n, D, total, thr, out, ocs, ods);
    return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA;
}

}  // namespace hmcx
