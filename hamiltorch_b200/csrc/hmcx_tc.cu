// hmcx_tc.cu -- Hopper tensor-core (wgmma) building block for the dense contractions of the path:
//     D[M x N] = A[M x K] . B[N x K]^T        (A, B, D row-major fp32; fp32-accurate via 3xTF32 split operands)
// This is the GEMM behind full-covariance Gaussian targets / full mass matrices at large D
// (grad log p = -(q - mu) P for ALL chains at once is exactly this contraction with M = chains, N = K = D,
// samplers.py:294, :812 and targets.GaussianFull) -- SURVEY.md section 8f item 2.
//
// sm_90a mechanics (one CTA per 128 x BN output tile):
//   * operands sit in shared memory in the canonical K-major / no-swizzle layout (8-row x 16-byte core matrices), each
//     fp32 split into tf32 hi + tf32 lo;
//   * one warpgroup issues wgmma.mma_async m64nBNk8 tf32 for the two 64-row halves of the tile, three per k-step:
//     hi*hi + hi*lo + lo*hi, accumulating in fp32 REGISTERS (hmcx_wgmma.cuh);
//   * the epilogues need one thread per chain row, so the accumulator tile is handed over through shared memory.
#include <cstdlib>
#include "hmcx_common.cuh"
#include "hmcx_wgmma.cuh"

namespace hmcx {

// hmcx_flow.cu: the persistent small-D form of the flows below
bool flow_small_ok(int D, int ld);
int flow_small_hmc_run(const hmcx_target_t*, const hmcx_mass_t*, const hmcx_rng_t*, const hmcx_nuts_t*, const float*, float*,
                       float*, int, int, int, int, int, int, int, float*, uint8_t*, uint8_t*, float*, int32_t*, cudaStream_t);
int flow_small_rmhmc_run(const hmcx_target_t*, const hmcx_rmhmc_t*, const hmcx_const_metric_t*, const hmcx_rng_t*, const float*,
                         float*, const float*, int, int, int, int, int, int, int, float*, uint8_t*, uint8_t*, float*, int32_t*,
                         float, float, cudaStream_t);

constexpr int TC_M = 128, TC_N = 128, TC_KC = 32;        // CTA tile and K chunk (fp32 elements)
constexpr int TC_THREADS = 128;                           // one warpgroup: the MMAs and the epilogue rows
constexpr int DENSE_THREADS = TC_THREADS + 32;            // + one warp whose lane 0 is the TMA producer

// Stage a [128 rows x KC] fp32 slab (row stride `ld`) into the canonical layout, split into tf32 hi and lo copies.
// Core matrix (rg = row/8, kc = k/4) lives at ((kc * 16 + rg) * 128) bytes: SBO = 128 B, LBO = 16*128 = 2048 B.
__device__ __forceinline__ void stage_operand(const float* __restrict__ g, int ld, float* s_hi, float* s_lo) {
    // 128 rows x 8 float4 per row = 1024 float4; 128 threads -> 8 each.  Thread t handles row r = t, all 8 chunks:
    // consecutive threads touch consecutive rows => conflict-free 16-byte shared stores (row stride 16 B in a core).
    const int r = threadIdx.x;
    const float4* src = reinterpret_cast<const float4*>(g + (size_t)r * ld);
#pragma unroll
    for (int kc = 0; kc < TC_KC / 4; ++kc) {
        const float4 v = __ldg(src + kc);
        float4 h, l;
        h.x = to_tf32(v.x); h.y = to_tf32(v.y); h.z = to_tf32(v.z); h.w = to_tf32(v.w);
        l.x = to_tf32(v.x - h.x); l.y = to_tf32(v.y - h.y); l.z = to_tf32(v.z - h.z); l.w = to_tf32(v.w - h.w);
        const int off = ((kc * 16 + (r >> 3)) * 128 + (r & 7) * 16) >> 2;     // in floats
        *reinterpret_cast<float4*>(s_hi + off) = h;
        *reinterpret_cast<float4*>(s_lo + off) = l;
    }
}

// The three 3xTF32 products of one k-step for both 64-row halves of a 128-row A block: acc[h] += A[64h..] . B^T.
// sa / sb: shared addresses of the hi blocks at this k-step, lo blocks `a_lo` / `b_lo` bytes further.
template <int BN>
__device__ __forceinline__ void mma_kstep_3xtf32(float (&acc)[2][BN / 2], uint32_t sa, uint32_t a_lo, uint32_t sb,
                                                 uint32_t b_lo) {
    constexpr uint32_t A_LBO = (TC_M / 8) * 128, B_LBO = (BN / 8) * 128;
    const uint64_t bh = make_kmajor_desc(sb, B_LBO, 128), bl = make_kmajor_desc(sb + b_lo, B_LBO, 128);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const uint64_t ah = make_kmajor_desc(sa + h * 1024u, A_LBO, 128), al = make_kmajor_desc(sa + a_lo + h * 1024u, A_LBO, 128);
        wgmma_tf32_ss<BN>(acc[h], ah, bh);
        wgmma_tf32_ss<BN>(acc[h], ah, bl);
        wgmma_tf32_ss<BN>(acc[h], al, bh);
    }
}

__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_nt_tf32x3_kernel(const float* __restrict__ A, const float* __restrict__ B, float* __restrict__ D, int M, int N,
                      int K) {
    extern __shared__ __align__(1024) float smem[];
    float* a_hi = smem;                          // each 128 x 32 fp32 = 16 KB
    float* a_lo = a_hi + TC_M * TC_KC;
    float* b_hi = a_lo + TC_M * TC_KC;
    float* b_lo = b_hi + TC_N * TC_KC;

    const int tile_n = blockIdx.x, tile_m = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float* Ag = A + (size_t)tile_m * TC_M * K;
    const float* Bg = B + (size_t)tile_n * TC_N * K;
    float acc[2][TC_N / 2];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < TC_N / 2; ++i) acc[h][i] = 0.0f;
    for (int k0 = 0; k0 < K; k0 += TC_KC) {
        stage_operand(Ag + k0, K, a_hi, a_lo);
        stage_operand(Bg + k0, K, b_hi, b_lo);
        fence_async_smem();                                                    // generic-proxy writes -> wgmma operands
        __syncthreads();
        wgmma_fence();
#pragma unroll
        for (int s = 0; s < TC_KC / 8; ++s) {                                  // wgmma K = 8 tf32 = two core matrices
            const uint32_t koff = (uint32_t)s * 2u * 2048u;
            mma_kstep_3xtf32<TC_N>(acc, smem_u32(a_hi) + koff, (uint32_t)(TC_M * TC_KC * 4), smem_u32(b_hi) + koff,
                                   (uint32_t)(TC_N * TC_KC * 4));
        }
        wgmma_commit();
        wgmma_wait<0>();                                                       // MMAs done: smem may be overwritten
        __syncthreads();
    }
    // ---- epilogue: straight from the accumulator fragments (hmcx_wgmma.cuh) to global memory ----
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int i = 0; i < TC_N / 2; i += 2) {
            const int row = tile_m * TC_M + 64 * h + 16 * warp + (lane >> 2) + 8 * ((i >> 1) & 1);
            const int col = tile_n * TC_N + 8 * (i >> 2) + 2 * (lane & 3);
            if (row < M) *reinterpret_cast<float2*>(D + (size_t)row * N + col) = make_float2(acc[h][i], acc[h][i + 1]);
        }
    }
}


// =========================================================================================================
// Dense-target plain HMC / HMC_NUTS: full-covariance Gaussian at large D, all chains per step on the tensor cores
//   grad log p (samplers.py:297 via autograd of targets.GaussianFull) for ALL chains = -(Q - mu) P : one tensor-core GEMM
//   per leapfrog step with the kick (:281/:298/:302) and the drift (:284/:296) fused into its epilogue.
// Step-synchronous: a trajectory is L+1 launches of dense_step_kernel (each needs every column of the new Q, a
// grid-wide dependency), bracketed by dense_gibbs_kernel and dense_mh_kernel; launched back-to-back on one stream
// from hmcx_hmc_run, no host synchronisation.  State lives in the caller-provided workspace.
// =========================================================================================================
struct DenseArgs {
    int C, Cp, D, Dp, NT, BN;     // NT = Dp / BN column tiles
    const float* prec;        // [Dp, Dp] zero-padded precision
    const float* mean;        // [Dp]
    float log_norm;
    int mk;
    const float* im;          // [Dp] inverse mass (diag) or null
    const float* sd;          // [Dp] sqrt(mass) or null
    int tk;                   // target kind (full-mass path: GAUSS_ISO / GAUSS_DIAG / GAUSS_FULL)
    const float* ivar;        // [Dp] GAUSS_DIAG inverse variances
};

enum { DENSE_FIRST = 0, DENSE_MIDDLE = 1, DENSE_LAST = 2, DENSE_EVAL = 3 };

// ---- packed operand layout ---------------------------------------------------------------------------------------
// Operands are kept in global memory ALREADY in the canonical wgmma layout and ALREADY split into tf32 hi / lo, one
// contiguous block per (row tile, 32-wide K chunk, hi|lo): a block of R rows is R*32 floats, element (r, k) at
//     ((k/4) * (R/8) + r/8) * 32 + (r%8) * 4 + (k%4)            [8-row x 16-byte core matrices, K-major, no swizzle]
// so that the GEMM main loop is nothing but 1-D bulk TMA copies (cp.async.bulk -> UBLKCP) into the stage buffers.
__device__ __forceinline__ size_t pack_block_base(int tile, int kchunk, int hl, int kchunks, int R) {
    return ((size_t)(tile * kchunks + kchunk) * 2 + hl) * (size_t)(R * TC_KC);
}
__device__ __forceinline__ int pack_elem_off(int r, int k, int R) {     // k in [0,32), multiple of 4 for float4 access
    return ((k >> 2) * (R >> 3) + (r >> 3)) * 32 + (r & 7) * 4 + (k & 3);
}
__device__ __forceinline__ void split_store4(float* pack_hi, float* pack_lo, int off, const float v[4]) {
    float4 h, l;
    h.x = to_tf32(v[0]); h.y = to_tf32(v[1]); h.z = to_tf32(v[2]); h.w = to_tf32(v[3]);
    l.x = to_tf32(v[0] - h.x); l.y = to_tf32(v[1] - h.y); l.z = to_tf32(v[2] - h.z); l.w = to_tf32(v[3] - h.w);
    *reinterpret_cast<float4*>(pack_hi + off) = h;
    *reinterpret_cast<float4*>(pack_lo + off) = l;
}

// pack a zero-padded row-major [rows x Dp] matrix (minus `mean` if given) into blocks of R rows
__global__ void dense_pack_kernel(const float* __restrict__ src, const float* __restrict__ mean, int rows, int Dp, int R,
                                  float* __restrict__ dst) {
    const int kchunks = Dp / TC_KC, vec_per_row = Dp / 4;
    const size_t n = (size_t)rows * vec_per_row;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int row = (int)(i / vec_per_row), k = 4 * (int)(i % vec_per_row);
        float v[4];
        ld4(src + (size_t)row * Dp + k, v);
        if (mean) {
#pragma unroll
            for (int t = 0; t < 4; ++t) v[t] = sub(v[t], mean[k + t]);
        }
        const int tile = row / R, kc = k / TC_KC;
        const int off = pack_elem_off(row % R, k % TC_KC, R);
        split_store4(dst + pack_block_base(tile, kc, 0, kchunks, R), dst + pack_block_base(tile, kc, 1, kchunks, R), off, v);
    }
}

__host__ __device__ constexpr int dense_stages(int BN) { return BN == 128 ? 3 : 4; }
__host__ __device__ constexpr int dense_stage_floats(int BN) { return 2 * TC_M * TC_KC + 2 * BN * TC_KC; }

// Programmatic dependent launch: the step-synchronous dense paths are chains of short GEMM launches on one stream.  Each
// kernel lets its successor start launching at once (griddepcontrol.launch_dependents) and itself waits for its
// predecessor's completion + memory flush (griddepcontrol.wait) only after its prologue (mbarrier init),
// so launch latency and prologue overlap the previous kernel's main loop and epilogue.  All global reads and writes of a
// kernel come after its wait.  HMCX_PDL=0 in the environment falls back to plain stream order.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

static bool pdl_enabled() {
    static const bool on = [] { const char* e = getenv("HMCX_PDL"); return !(e && e[0] == '0'); }();
    return on;
}
template <typename... KArgs, typename... Args>
static void launch_pdl(void (*kernel)(KArgs...), dim3 grid, int threads, size_t smem, cudaStream_t st, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = dim3(threads); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = pdl_enabled() ? 1 : 0;
    cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

// Prologue shared by the dense kernels: the mbarrier ring.
template <int ST>
__device__ __forceinline__ void dense_prologue(uint64_t* s_full, uint64_t* s_empty) {
    if (threadIdx.x == 0) {
        for (int s = 0; s < ST; ++s) { mbar_init(smem_u32(&s_full[s]), 1); mbar_init(smem_u32(&s_empty[s]), 1); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
}

// The warp-specialised main loop shared by the dense kernels: thread TC_THREADS (lane 0 of the last warp) = TMA producer
// (1-D bulk copies of the packed hi|lo operand blocks into an ST-stage ring), threads [0, TC_THREADS) = the MMA warpgroup
// (three tf32 wgmmas per 8-wide k-step and 64-row half: hi*hi + hi*lo + lo*hi, fp32 accumulators in registers).  One
// wgmma group stays in flight: a stage is released when the group that read it has completed.  On return the ring is
// idle and `acc` holds the 128 x BN tile in the fragment layout of hmcx_wgmma.cuh (MMA threads only).
template <int BN, int ST>
__device__ __forceinline__ void dense_mainloop(float* smem, uint64_t* s_full, uint64_t* s_empty, float (&acc)[2][BN / 2],
                                               const float* __restrict__ QpIn, const float* __restrict__ Ppack,
                                               int tile_m, int tile_n, int kchunks) {
    constexpr int A_BLK = TC_M * TC_KC, B_BLK = BN * TC_KC;
    constexpr uint32_t STAGE_BYTES = (uint32_t)dense_stage_floats(BN) * 4u;
    if (threadIdx.x == TC_THREADS) {
        // ===== TMA producer: bulk copies per stage (A hi, A lo, B hi, B lo are adjacent pairs in global memory) =====
        for (int i = 0; i < kchunks; ++i) {
            const int s = i % ST;
            mbar_wait(smem_u32(&s_empty[s]), ((i / ST) & 1) ^ 1);
            const uint32_t full = smem_u32(&s_full[s]);
            mbar_expect_tx(full, STAGE_BYTES);
            float* st = smem + (size_t)s * dense_stage_floats(BN);
            bulk_g2s(smem_u32(st), QpIn + pack_block_base(tile_m, i, 0, kchunks, TC_M), 2 * A_BLK * 4, full);
            bulk_g2s(smem_u32(st + 2 * A_BLK), Ppack + pack_block_base(tile_n, i, 0, kchunks, BN), 2 * B_BLK * 4, full);
        }
    } else if (threadIdx.x < TC_THREADS) {
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int j = 0; j < BN / 2; ++j) acc[h][j] = 0.0f;
        for (int i = 0; i < kchunks; ++i) {
            const int s = i % ST;
            mbar_wait(smem_u32(&s_full[s]), (i / ST) & 1);
            const uint32_t sa = smem_u32(smem + (size_t)s * dense_stage_floats(BN));
            const uint32_t sb = sa + 2 * A_BLK * 4;
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < TC_KC / 8; ++k)
                mma_kstep_3xtf32<BN>(acc, sa + k * 2 * (TC_M / 8) * 128, A_BLK * 4, sb + k * 2 * (BN / 8) * 128, B_BLK * 4);
            wgmma_commit();
            wgmma_wait<1>();                                   // the previous chunk's group has read its stage
            if (i > 0 && threadIdx.x == 0) mbar_arrive(smem_u32(&s_empty[(i - 1) % ST]));
        }
        wgmma_wait<0>();
    }
    __syncwarp();
    __syncthreads();
}

// The accumulator tile -> shared memory (row pitch BN + 4 floats), so that the epilogue can give each thread one row.
template <int BN>
__device__ __forceinline__ void dense_stage_acc(const float (&acc)[2][BN / 2], float* stg) {
    if (threadIdx.x < TC_THREADS) {
        const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int i = 0; i < BN / 2; i += 2) {
                const int r = 64 * h + 16 * warp + (lane >> 2) + 8 * ((i >> 1) & 1), c = 8 * (i >> 2) + 2 * (lane & 3);
                *reinterpret_cast<float2*>(stg + r * (BN + 4) + c) = make_float2(acc[h][i], acc[h][i + 1]);
            }
    }
    __syncthreads();
}
__device__ __forceinline__ void stage_ld32(const float* src, uint32_t (&v)[32]) {
#pragma unroll
    for (int j = 0; j < 32; j += 4) {
        const float4 t = *reinterpret_cast<const float4*>(src + j);
        v[j] = __float_as_uint(t.x); v[j + 1] = __float_as_uint(t.y); v[j + 2] = __float_as_uint(t.z); v[j + 3] = __float_as_uint(t.w);
    }
}

// One leapfrog step for all chains:  acc = (Q - mu) P  on the tensor cores, then kick / drift in the epilogue.
//   grid (Dp/BN, Cp/128), 160 threads: warps 0-3 = MMA warpgroup + epilogue (one chain row each), thread 128 = TMA producer.
template <int BN>
__global__ void __launch_bounds__(DENSE_THREADS, 1)
dense_step_kernel(const DenseArgs a, const float* __restrict__ Qin, const float* __restrict__ QpIn,
                  const float* __restrict__ Ppack, float* __restrict__ Qout, float* __restrict__ QpOut,
                  float* __restrict__ P, const float* __restrict__ eps, int mode, float* __restrict__ upart) {
    constexpr int ST = dense_stages(BN);
    extern __shared__ __align__(1024) float smem[];
    __shared__ __align__(8) uint64_t s_full[ST], s_empty[ST];
    pdl_launch_dependents();
    const int tile_n = blockIdx.x, tile_m = blockIdx.y;
    const int Dp = a.Dp, kchunks = Dp / TC_KC;

    dense_prologue<ST>(s_full, s_empty);

    pdl_wait();               // the barrier set-up overlapped the previous launch's tail; its writes are visible now
    float acc[2][BN / 2];
    dense_mainloop<BN, ST>(smem, s_full, s_empty, acc, QpIn, Ppack, tile_m, tile_n, kchunks);
    dense_stage_acc<BN>(acc, smem);
    // ===== epilogue: acc = ((Q-mu) P)[row, cols]; g = -acc; kick, optional drift (+ packed copy for the next GEMM) =====
    const int row = tile_m * TC_M + threadIdx.x;
    const bool live = threadIdx.x < TC_THREADS && row < a.C;
    const float* srow = smem + (size_t)threadIdx.x * (BN + 4);
    const float e = live ? eps[row] : 0.0f, half = mul(0.5f, e);
    const float ck = (mode == DENSE_FIRST) ? half : e;
    const bool drift = (mode == DENSE_FIRST || mode == DENSE_MIDDLE);
    float udot = 0.0f;
    const size_t base = (size_t)row * Dp + (size_t)tile_n * BN;
#pragma unroll 1
    for (int c0 = 0; c0 < BN; c0 += 32) {
        if (live) {
            uint32_t v[32];
            stage_ld32(srow + c0, v);
            const int colbase = tile_n * BN + c0;                           // a 32-aligned column block = one K chunk
            float* qp_hi = QpOut + pack_block_base(tile_m, colbase / TC_KC, 0, kchunks, TC_M);
            float* qp_lo = QpOut + pack_block_base(tile_m, colbase / TC_KC, 1, kchunks, TC_M);
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
                const int col = colbase + j;
                const float4 q4 = *reinterpret_cast<const float4*>(Qin + base + c0 + j);
                const float4 m4 = *reinterpret_cast<const float4*>(a.mean + col);
                const float acc[4] = {__uint_as_float(v[j]), __uint_as_float(v[j + 1]), __uint_as_float(v[j + 2]),
                                      __uint_as_float(v[j + 3])};
                const float qv[4] = {q4.x, q4.y, q4.z, q4.w}, mv[4] = {m4.x, m4.y, m4.z, m4.w};
                float pn[4], yn[4], qn[4];
                float4 p4 = make_float4(0.f, 0.f, 0.f, 0.f);
                if (mode != DENSE_EVAL) p4 = *reinterpret_cast<const float4*>(P + base + c0 + j);
                const float pv[4] = {p4.x, p4.y, p4.z, p4.w};
#pragma unroll
                for (int t = 0; t < 4; ++t) {
                    udot = add(udot, mul(sub(qv[t], mv[t]), acc[t]));
                    const float g = -acc[t];
                    pn[t] = add(pv[t], mul(ck, g));                                             // :281 / :298
                    if (mode == DENSE_LAST) pn[t] = sub(pn[t], mul(half, g));                   // :302
                    const float cd = (a.mk == HMCX_MASS_DIAG) ? mul(e, a.im[col + t]) : e;
                    qn[t] = add(qv[t], mul(cd, pn[t]));                                         // :284 / :296
                    yn[t] = sub(qn[t], mv[t]);
                }
                if (mode != DENSE_EVAL) *reinterpret_cast<float4*>(P + base + c0 + j) = make_float4(pn[0], pn[1], pn[2], pn[3]);
                if (drift) {
                    *reinterpret_cast<float4*>(Qout + base + c0 + j) = make_float4(qn[0], qn[1], qn[2], qn[3]);
                    split_store4(qp_hi, qp_lo, pack_elem_off(row % TC_M, j, TC_M), yn);       // next step's A operand
                }
            }
        }
    }
    if (live && upart) upart[(size_t)row * a.NT + tile_n] = udot;
}


// =========================================================================================================
// Generic "linear flow" kernel on the tensor cores:  acc[row, col] = sum_k A[row, k] * B[col, k]   (all chains at once,
// A = a packed state operand, B = a packed D x D matrix), with a fused update epilogue
//     X[row, col]  <-  X + k1 * s*acc  [ - k2 * s*acc ]      (or X <- acc),     k = eps[row] or 0.5*eps[row]
//     Xpack        <-  split_tf32(X_new - shift[col])          the NEXT GEMM's A operand, already packed
//     part[row, tile_n] = sum_col (Y[row, col] - yshift[col]) * acc[row, col]       quadratic forms y.(B y)
// It is the building block of everything on the path that is a (chains x D) . (D x D) contraction and not the
// diagonal-mass dense step above:
//   * full (2-D) inv_mass at D > 16 (samplers.py:294 drift q += eps*(M^-1 p), :812 kinetic 0.5 p.(M^-1 p), gibbs
//     :199 p = chol(M) z) for GaussianIso / GaussianDiag / GaussianFull targets;
//   * the constant-metric RMHMC flows dH/dp = G~^-1 p and dH/dtheta = P (theta - mu) (samplers.py:389-462).
// =========================================================================================================
enum { LIN_K_E = 1, LIN_K_HALF = 2 };
struct LinEpi {
    float* X;              // [Cp, Dp] updated in place (null: no update)
    float* Xpack;          // packed copy of X_new - shift (null: none)
    const float* shift;    // [Dp] or null
    const float* Y;        // [Cp, Dp] dot partner (null: no dot)
    const float* yshift;   // [Dp] or null
    float* part;           // [Cp, NT]
    const float* eps;      // [C]
    int assign;            // X <- s*acc
    int k1, k2;            // LIN_K_* (k2 = 0: no second term)
    int k2add;             // second term is added instead of subtracted
    float sign;            // s = +1 / -1
};

template <int BN>
__global__ void __launch_bounds__(DENSE_THREADS, 1)
dense_lin_kernel(int C, int Dp, int NT, const float* __restrict__ Apack, const float* __restrict__ Bpack, const LinEpi ep) {
    constexpr int ST = dense_stages(BN);
    extern __shared__ __align__(1024) float smem[];
    __shared__ __align__(8) uint64_t s_full[ST], s_empty[ST];
    pdl_launch_dependents();
    const int tile_n = blockIdx.x, tile_m = blockIdx.y;
    const int kchunks = Dp / TC_KC;

    dense_prologue<ST>(s_full, s_empty);

    pdl_wait();
    float acc[2][BN / 2];
    dense_mainloop<BN, ST>(smem, s_full, s_empty, acc, Apack, Bpack, tile_m, tile_n, kchunks);
    dense_stage_acc<BN>(acc, smem);

    const int row = tile_m * TC_M + threadIdx.x;
    const bool live = threadIdx.x < TC_THREADS && row < C;
    const float* srow = smem + (size_t)threadIdx.x * (BN + 4);
    const float e = (live && ep.eps) ? ep.eps[row] : 0.0f, half = mul(0.5f, e);
    const float k1 = (ep.k1 == LIN_K_HALF) ? half : e, k2 = (ep.k2 == LIN_K_HALF) ? half : e;
    const bool neg = ep.sign < 0.0f;
    float dot = 0.0f;
    const size_t base = (size_t)row * Dp + (size_t)tile_n * BN;
#pragma unroll 1
    for (int c0 = 0; c0 < BN; c0 += 32) {
        if (live) {
            uint32_t v[32];
            stage_ld32(srow + c0, v);
            const int colbase = tile_n * BN + c0;                           // a 32-aligned column block = one K chunk
            float* xp_hi = ep.Xpack ? ep.Xpack + pack_block_base(tile_m, colbase / TC_KC, 0, kchunks, TC_M) : nullptr;
            float* xp_lo = ep.Xpack ? ep.Xpack + pack_block_base(tile_m, colbase / TC_KC, 1, kchunks, TC_M) : nullptr;
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
                const int col = colbase + j;
                const float acc[4] = {__uint_as_float(v[j]), __uint_as_float(v[j + 1]), __uint_as_float(v[j + 2]),
                                      __uint_as_float(v[j + 3])};
                if (ep.Y) {
                    float yv[4];
                    ld4(ep.Y + base + c0 + j, yv);
#pragma unroll
                    for (int t = 0; t < 4; ++t) {
                        const float y = ep.yshift ? sub(yv[t], ep.yshift[col + t]) : yv[t];
                        dot = add(dot, mul(y, acc[t]));
                    }
                }
                if (ep.X) {
                    float xv[4] = {0.f, 0.f, 0.f, 0.f}, xn[4], yn[4];
                    if (!ep.assign) ld4(ep.X + base + c0 + j, xv);
#pragma unroll
                    for (int t = 0; t < 4; ++t) {
                        const float g = neg ? -acc[t] : acc[t];
                        xn[t] = ep.assign ? g : add(xv[t], mul(k1, g));
                        if (ep.k2) xn[t] = ep.k2add ? add(xn[t], mul(k2, g)) : sub(xn[t], mul(k2, g));
                        yn[t] = ep.shift ? sub(xn[t], ep.shift[col + t]) : xn[t];
                    }
                    st4(ep.X + base + c0 + j, xn);
                    if (ep.Xpack) split_store4(xp_hi, xp_lo, pack_elem_off(row % TC_M, j, TC_M), yn);
                }
            }
        }
    }
    if (live && ep.part) ep.part[(size_t)row * NT + tile_n] = dot;
}

static bool lin_launch(int BN, dim3 grid, cudaStream_t st, int C, int Dp, int NT, const float* Apack, const float* Bpack,
                       const LinEpi& ep) {
    const size_t sm = (size_t)dense_stages(BN) * dense_stage_floats(BN) * sizeof(float);
    if (BN == 128) launch_pdl(dense_lin_kernel<128>, grid, DENSE_THREADS, sm, st, C, Dp, NT, Apack, Bpack, ep);
    else if (BN == 64) launch_pdl(dense_lin_kernel<64>, grid, DENSE_THREADS, sm, st, C, Dp, NT, Apack, Bpack, ep);
    else launch_pdl(dense_lin_kernel<32>, grid, DENSE_THREADS, sm, st, C, Dp, NT, Apack, Bpack, ep);
    return true;
}
static bool lin_configure() {
    bool ok = true;
    ok = ok && cudaFuncSetAttribute(dense_lin_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)((size_t)dense_stages(128) * dense_stage_floats(128) * 4)) == cudaSuccess;
    ok = ok && cudaFuncSetAttribute(dense_lin_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)((size_t)dense_stages(64) * dense_stage_floats(64) * 4)) == cudaSuccess;
    ok = ok && cudaFuncSetAttribute(dense_lin_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)((size_t)dense_stages(32) * dense_stage_floats(32) * 4)) == cudaSuccess;
    if (!ok) cudaGetLastError();
    return ok;
}

// zero-padded copies into the workspace
__global__ void dense_pad_matrix_kernel(const float* __restrict__ src, int D, float* __restrict__ dst, int Dp) {
    const size_t n = (size_t)Dp * Dp;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int r = (int)(i / Dp), c = (int)(i % Dp);
        dst[i] = (r < D && c < D) ? src[(size_t)r * D + c] : 0.0f;
    }
}
__global__ void dense_pad_vector_kernel(const float* __restrict__ src, int D, float* __restrict__ dst, int Dp) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < Dp; i += gridDim.x * blockDim.x)
        dst[i] = (src && i < D) ? src[i] : 0.0f;
}
// rows of a caller (C, ld) array -> padded (Cp, Dp) work array
__global__ void dense_load_rows_kernel(const float* __restrict__ src, int C, int ld, int D, float* __restrict__ dst,
                                       int Cp, int Dp) {
    const int r = blockIdx.x;
    for (int j = threadIdx.x; j < Dp; j += blockDim.x) dst[(size_t)r * Dp + j] = (r < C && j < D) ? src[(size_t)r * ld + j] : 0.0f;
}

struct DenseRun {
    DenseArgs a;
    int ld, rng_mode;
    uint64_t seed, chain_offset;
    const float* normals;
    const float* logu;
    int nuts;
    double delta, mu;
    const double* table;
    double* h_bar;
    double* eps_bar;
    const float* eps_schedule;
    float* eps_trace;
    const float* q_init;
    float* q_cur;
    float* eps;
    int S, burn, it0;
    float* samples;
    uint8_t* accept;
    uint8_t* diverged;
    float* ham;
    int32_t* num_rejected;
    // workspace
    float* kin0;
    float* U_cur;
    float* U_init;
    // full (2-D) inv_mass: gibbs packs z (p = chol(M) z is a GEMM), kinetic energies arrive as per-tile partials
    float* zpack;
    const float* kpart0;
    const float* kpartL;
    // constant-metric RMHMC: H = -log p + 0.5*D*log(2 pi) + 0.5*log det G + 0.5 p.(G^-1 p)   (samplers.py:731)
    int rm;
    float ham_c1, ham_c2;
};

// gibbs (:969) for iteration n: p = z * sqrt(mass) -> P rows, q_cur -> Q work rows, kinetic of p
__global__ void __launch_bounds__(256)
dense_gibbs_kernel(const DenseRun r, int n, float* __restrict__ Q, float* __restrict__ P, float* __restrict__ Qpack) {
    __shared__ float sred[32];
    const DenseArgs& a = r.a;
    const int c = blockIdx.x, Dp = a.Dp, D = a.D;
    const uint64_t chain_id = r.chain_offset + (uint64_t)c;
    if (r.eps_schedule && threadIdx.x == 0) r.eps[c] = r.eps_schedule[(size_t)n * a.C + c];
    float kin[1] = {0.0f};
    for (int v = threadIdx.x; 4 * v < Dp; v += blockDim.x) {
        float z[4] = {0.f, 0.f, 0.f, 0.f}, qv[4] = {0.f, 0.f, 0.f, 0.f};
        if (4 * v < r.ld) {
            if (r.rng_mode == HMCX_RNG_INJECTED) ld4_stream(r.normals + ((size_t)(n - r.it0) * a.C + c) * r.ld + 4 * v, z);
            else philox_normal4(r.seed, chain_id, (uint64_t)n, (uint32_t)v, z);
            ld4(r.q_cur + (size_t)c * r.ld + 4 * v, qv);
        }
        float pv[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int i = 4 * v + j;
            if (i >= D) { z[j] = 0.0f; qv[j] = 0.0f; }
            pv[j] = (a.mk == HMCX_MASS_DIAG) ? mul(z[j], a.sd[i]) : z[j];
            kin[0] = add(kin[0], (a.mk == HMCX_MASS_DIAG) ? mul(pv[j], mul(a.im[i], pv[j])) : mul(pv[j], pv[j]));
        }
        const int kchunks = Dp / TC_KC, kc = (4 * v) / TC_KC;
        if (a.mk == HMCX_MASS_FULL)                                              // :199: p = scale_tril . z, a GEMM
            split_store4(r.zpack + pack_block_base(c / TC_M, kc, 0, kchunks, TC_M),
                         r.zpack + pack_block_base(c / TC_M, kc, 1, kchunks, TC_M), pack_elem_off(c % TC_M, (4 * v) % TC_KC, TC_M), z);
        else
            st4(P + (size_t)c * Dp + 4 * v, pv);
        st4(Q + (size_t)c * Dp + 4 * v, qv);
        float y[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) y[j] = sub(qv[j], a.mean[4 * v + j]);
        split_store4(Qpack + pack_block_base(c / TC_M, kc, 0, kchunks, TC_M),
                     Qpack + pack_block_base(c / TC_M, kc, 1, kchunks, TC_M), pack_elem_off(c % TC_M, (4 * v) % TC_KC, TC_M), y);
    }
    block_sum<1>(kin, sred);
    if (threadIdx.x == 0 && r.kin0) r.kin0[c] = kin[0];
}

// log p from the per-tile partials of y.(P y)   (targets.GaussianFull: -0.5*dot(y, P y) + log_norm)
__device__ __forceinline__ float dense_log_prob(const DenseArgs& a, const float* upart, int c) {
    float s = 0.0f;
    for (int t = 0; t < a.NT; ++t) s = add(s, upart[(size_t)c * a.NT + t]);
    return add(mul(-0.5f, s), a.log_norm);
}

__global__ void dense_store_u_kernel(const DenseArgs a, const float* __restrict__ upart, float* __restrict__ U) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c < a.C) U[c] = dense_log_prob(a, upart, c);
}

// MH + bookkeeping + dual averaging for iteration n (samplers.py:995-1067), one CTA per chain
__global__ void __launch_bounds__(256)
dense_mh_kernel(const DenseRun r, int n, const float* __restrict__ Qprop, const float* __restrict__ P,
                const float* __restrict__ upart) {
    __shared__ float sred[32];
    __shared__ int s_flag[2];
    const DenseArgs& a = r.a;
    const int c = blockIdx.x, Dp = a.Dp, D = a.D, tid = threadIdx.x;
    const uint64_t chain_id = r.chain_offset + (uint64_t)c;
    float kin[1] = {0.0f};
    if (a.mk != HMCX_MASS_FULL) {
        for (int i = tid; i < D; i += blockDim.x) {
            const float p = P[(size_t)c * Dp + i];
            kin[0] = add(kin[0], (a.mk == HMCX_MASS_DIAG) ? mul(p, mul(a.im[i], p)) : mul(p, p));
        }
        block_sum<1>(kin, sred);
    }
    if (tid == 0) {
        float kin_old = 0.0f;
        if (a.mk == HMCX_MASS_FULL) {                                        // p.(M^-1 p): per-tile partials, fixed order
            for (int t = 0; t < a.NT; ++t) {
                kin_old = add(kin_old, r.kpart0[(size_t)c * a.NT + t]);
                kin[0] = add(kin[0], r.kpartL[(size_t)c * a.NT + t]);
            }
        } else {
            kin_old = r.kin0[c];
        }
        const float lp_cur = r.U_cur[c], lp_new = dense_log_prob(a, upart, c);
        float h_old, h_new;
        if (r.rm) {
            h_old = add(add(add(-lp_cur, r.ham_c1), r.ham_c2), mul(0.5f, kin_old));
            h_new = add(add(add(-lp_new, r.ham_c1), r.ham_c2), mul(0.5f, kin[0]));
        } else {
            h_old = add(-lp_cur, mul(0.5f, kin_old));
            h_new = add(-lp_new, mul(0.5f, kin[0]));
        }
        const bool bad = !finite_f(lp_cur) || !finite_f(lp_new) || (r.rm && (!finite_f(h_old) || !finite_f(h_new)));
        const float x = add(-h_new, h_old);
        const float rho = (x < 0.0f) ? x : 0.0f;
        const float logu = (r.rng_mode == HMCX_RNG_INJECTED) ? r.logu[(size_t)(n - r.it0) * a.C + c]
                                                             : philox_log_uniform(r.seed, chain_id, (uint64_t)n);
        const bool acc = !bad && (rho >= logu);
        const bool quirk = !acc && (n == r.burn + 1);
        if (acc) r.U_cur[c] = lp_new;
        else if (quirk) r.U_cur[c] = r.U_init[c];
        if (!acc && r.num_rejected) r.num_rejected[c] += 1;
        const size_t o = (size_t)c * r.S + n;
        if (r.accept) r.accept[o] = acc ? 1 : 0;
        if (r.diverged) r.diverged[o] = bad ? 1 : 0;
        if (r.ham) { r.ham[2 * o] = h_old; r.ham[2 * o + 1] = h_new; }
        float e = r.eps[c];
        if (r.nuts && n <= r.burn) {                                         // :1030-1035, :1060-1067
            double h_bar = r.h_bar[c], eps_bar = r.eps_bar[c];
            if (n < r.burn || bad) {
                const double* T = r.table + 5 * (size_t)n;
                const double alpha = bad ? 0.0 : (double)expf(rho);
                h_bar = __dadd_rn(__dmul_rn(T[0], h_bar), __dmul_rn(T[1], r.delta - alpha));
                const double x_new = r.mu - __dmul_rn(T[2], h_bar);
                e = expf((float)x_new);
                const float xb = add((float)__dmul_rn(T[3], x_new), mul((float)T[4], logf((float)eps_bar)));
                eps_bar = (double)expf(xb);
            }
            if (n == r.burn) e = (float)eps_bar;
            r.h_bar[c] = h_bar; r.eps_bar[c] = eps_bar;
            r.eps[c] = e;
        }
        if (r.eps_trace) r.eps_trace[o] = e;
        s_flag[0] = acc ? 1 : 0;
        s_flag[1] = quirk ? 1 : 0;
    }
    __syncthreads();
    const bool acc = s_flag[0] != 0, quirk = s_flag[1] != 0;
    float* qc = r.q_cur + (size_t)c * r.ld;
    float* dst = (n > r.burn && r.samples) ? r.samples + ((size_t)c * (r.S - r.burn) + (n - r.burn)) * r.ld : nullptr;
    for (int i = tid; i < r.ld; i += blockDim.x) {
        float v;
        if (acc) v = i < D ? Qprop[(size_t)c * Dp + i] : 0.0f;
        else if (quirk) v = r.q_init[(size_t)c * r.ld + i];
        else v = qc[i];
        if (acc || quirk) qc[i] = v;
        if (dst) dst[i] = v;
    }
}

size_t dense_workspace_floats(int C, int D, int full_mass) {
    const size_t Cp = (size_t)(C + 127) / 128 * 128, Dp = (size_t)(D + 127) / 128 * 128;
    if (full_mass)
        return 8 * Cp * Dp        // Q, P, Qpack, Ppack, Zpack (hi+lo each)
               + 7 * Dp * Dp      // padding scratch + packed precision, inv_mass, chol(mass)
               + 2 * Dp + 3 * Cp * (Dp / 32) + 2 * Cp + 64;
    return 7 * Cp * Dp            // Q[2], Qpack[2] (hi+lo each), P
           + 3 * Dp * Dp          // padded precision + its packed hi/lo
           + 3 * Dp + Cp * (Dp / 32) + 3 * Cp + 64;
}

// Element-wise targets under a full mass matrix: the kick has no contraction.  One CTA per chain: g = grad log p(q)
// in the reference's op order, p <- p + k1*g [- k2*g], packed copy of p for the drift GEMM, and the U-terms sum
// (slot 0 of the chain's partials; the other slots are zeroed so dense_log_prob's fixed-order sum is unchanged).
__global__ void __launch_bounds__(256)
dense_kick_elem_kernel(const DenseArgs a, const float* __restrict__ Q, float* __restrict__ P, float* __restrict__ Ppack,
                       const float* __restrict__ eps, int k1m, int k2m, float* __restrict__ upart, int k2add = 0) {
    __shared__ float sred[32];
    const int c = blockIdx.x, Dp = a.Dp, D = a.D;
    const float e = eps[c], half = mul(0.5f, e);
    const float k1 = (k1m == LIN_K_HALF) ? half : e, k2 = (k2m == LIN_K_HALF) ? half : e;
    const int kchunks = Dp / TC_KC;
    float us[1] = {0.0f};
    for (int v = threadIdx.x; 4 * v < Dp; v += blockDim.x) {
        float qv[4], pv[4];
        ld4(Q + (size_t)c * Dp + 4 * v, qv);
        if (k1m) ld4(P + (size_t)c * Dp + 4 * v, pv);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int i = 4 * v + j;
            float g = 0.0f, u = 0.0f;
            if (i < D) {
                if (a.tk == HMCX_TARGET_GAUSS_ISO) { g = -qv[j]; u = mul(qv[j], qv[j]); }
                else { const float y = sub(qv[j], a.mean[i]); g = -mul(a.ivar[i], y); u = mul(mul(y, y), a.ivar[i]); }
            }
            us[0] = add(us[0], u);
            if (k1m) {
                pv[j] = add(pv[j], mul(k1, g));                               // :281 / :298
                if (k2m) pv[j] = k2add ? add(pv[j], mul(k2, g)) : sub(pv[j], mul(k2, g));   // :302 | a second, separate kick
            }
        }
        if (k1m) {
            st4(P + (size_t)c * Dp + 4 * v, pv);
            const int kc = (4 * v) / TC_KC;
            split_store4(Ppack + pack_block_base(c / TC_M, kc, 0, kchunks, TC_M),
                         Ppack + pack_block_base(c / TC_M, kc, 1, kchunks, TC_M), pack_elem_off(c % TC_M, (4 * v) % TC_KC, TC_M), pv);
        }
    }
    block_sum<1>(us, sred);
    if (upart) for (int t = threadIdx.x; t < a.NT; t += blockDim.x) upart[(size_t)c * a.NT + t] = (t == 0) ? us[0] : 0.0f;
}

// sample() loop with a full (2-D) inv_mass at D > 16 (samplers.py:199, :294, :812): every drift, the momentum
// refresh and both kinetic energies are (chains x D) . (D x D) GEMMs on the tensor cores (dense_lin_kernel); a GaussianFull
// target adds the gradient GEMM, GaussianIso / GaussianDiag kick element-wise.  2L+4 (L+3) GEMMs per iteration.
// Column-tile width of the dense GEMMs over `mt` 128-row tiles and Dp (a multiple of 32) columns: the widest of 128/64/32
// that divides Dp and still gives the GPU ~100 CTAs (each CTA re-streams its 128 chain rows).  HMCX_DENSE_BN (tests only)
// forces the width so that every instantiation is reachable at small batches; it is read on every call, and a value that
// is not 32/64/128 dividing Dp gives 0 (the run returns HMCX_ERR_INVALID_ARG rather than run a width nobody asked for).
static int dense_tile_width(int Dp, int mt) {
    if (const char* e = getenv("HMCX_DENSE_BN")) {
        char* end = nullptr;
        const long bn = strtol(e, &end, 10);
        return (end != e && *end == '\0' && (bn == 32 || bn == 64 || bn == 128) && Dp % bn == 0) ? (int)bn : 0;
    }
    int bn = (Dp % 128 == 0) ? 128 : (Dp % 64 == 0) ? 64 : 32;
    while (bn > 32 && mt * (Dp / bn) < 96) bn >>= 1;
    return bn;
}

// K / N padding to multiples of 32 (one K chunk); false: HMCX_DENSE_BN forces a width that does not fit
static bool dense_geometry(DenseArgs& a) {
    a.Dp = (a.D + 31) / 32 * 32;
    a.BN = dense_tile_width(a.Dp, a.Cp / 128);
    if (!a.BN) return false;
    a.NT = a.Dp / a.BN;
    return true;
}

static inline float mul_host(float x, float y) { volatile float r = x * y; return r; }

static int dense_fullmass_hmc_run(const hmcx_target_t* target, const hmcx_mass_t* mass, const hmcx_rng_t* rng,
                                  const hmcx_nuts_t* nuts, const float* q_init, float* q_cur, float* eps, int C, int ld,
                                  int L, int S, int burn, int it0, int it1, float* samples, uint8_t* accept,
                                  uint8_t* diverged, float* ham, int32_t* num_rejected, float* ws, cudaStream_t st) {
    const int D = target->dim, tk = target->kind;
    if (!mass->inv_mass || !mass->mass_factor) return HMCX_ERR_INVALID_ARG;
    if (tk == HMCX_TARGET_GAUSS_DIAG && !target->inv_var) return HMCX_ERR_INVALID_ARG;
    DenseRun r = {};
    DenseArgs& a = r.a;
    a.C = C; a.D = D; a.Cp = (C + 127) / 128 * 128;
    a.log_norm = target->log_norm; a.mk = HMCX_MASS_FULL; a.tk = tk;
    if (!dense_geometry(a)) return HMCX_ERR_INVALID_ARG;
    const size_t CD = (size_t)a.Cp * a.Dp, DD = (size_t)a.Dp * a.Dp;
    float* Q = ws;
    float* P = ws + CD;
    float* Qpack = ws + 2 * CD;
    float* Ppack = ws + 4 * CD;
    float* Zpack = ws + 6 * CD;
    float* scratch = ws + 8 * CD;
    float* precpack = scratch + DD;
    float* impack = precpack + 2 * DD;
    float* trilpack = impack + 2 * DD;
    float* mean = trilpack + 2 * DD;
    float* ivar = mean + a.Dp;
    float* upart = ivar + a.Dp;
    float* kpart0 = upart + (size_t)a.Cp * (a.Dp / 32);
    float* kpartL = kpart0 + (size_t)a.Cp * (a.Dp / 32);
    r.U_cur = kpartL + (size_t)a.Cp * (a.Dp / 32);
    r.U_init = r.U_cur + a.Cp;
    r.kin0 = nullptr; r.zpack = Zpack; r.kpart0 = kpart0; r.kpartL = kpartL;
    a.mean = mean; a.ivar = ivar; a.prec = nullptr; a.im = nullptr; a.sd = nullptr;
    r.ld = ld; r.rng_mode = rng->mode; r.seed = rng->seed; r.chain_offset = rng->chain_offset;
    r.normals = rng->normals; r.logu = rng->log_uniforms;
    r.nuts = (nuts && nuts->enabled) ? 1 : 0;
    if (r.nuts) {
        if (!nuts->table || !nuts->h_bar || !nuts->eps_bar || burn < 1) return HMCX_ERR_INVALID_ARG;
        r.delta = nuts->desired_accept_rate; r.mu = nuts->mu; r.table = nuts->table;
        r.h_bar = nuts->h_bar; r.eps_bar = nuts->eps_bar;
        r.eps_schedule = nuts->eps_schedule; r.eps_trace = nuts->eps_trace;
    }
    r.q_init = q_init; r.q_cur = q_cur; r.eps = eps; r.S = S; r.burn = burn; r.it0 = it0;
    r.samples = samples; r.accept = accept; r.diverged = diverged; r.ham = ham; r.num_rejected = num_rejected;
    if (!lin_configure()) return HMCX_ERR_CUDA;

    const bool gemm_target = tk == HMCX_TARGET_GAUSS_FULL;
    auto pack_matrix = [&](const float* src, float* dst) {
        dense_pad_matrix_kernel<<<296, 256, 0, st>>>(src, D, scratch, a.Dp);
        dense_pack_kernel<<<296, 256, 0, st>>>(scratch, nullptr, a.Dp, a.Dp, a.BN, dst);
    };
    if (gemm_target) pack_matrix(target->prec, precpack);
    pack_matrix(mass->inv_mass, impack);
    pack_matrix(mass->mass_factor, trilpack);
    dense_pad_vector_kernel<<<8, 256, 0, st>>>(tk == HMCX_TARGET_GAUSS_ISO ? nullptr : target->mean, D, mean, a.Dp);
    dense_pad_vector_kernel<<<8, 256, 0, st>>>(tk == HMCX_TARGET_GAUSS_DIAG ? target->inv_var : nullptr, D, ivar, a.Dp);
    cudaMemsetAsync(ws, 0, 8 * CD * sizeof(float), st);

    const dim3 ggrid(a.NT, a.Cp / 128);
    // kick: p <- p + k1*g [- k2*g], g = grad log p(q); also leaves the U-terms partials of q in `upart`.  k1 = 0: U only.
    auto kick = [&](int k1, int k2) {
        if (gemm_target) {
            LinEpi ep = {};
            ep.X = k1 ? P : nullptr; ep.Xpack = k1 ? Ppack : nullptr; ep.Y = Q; ep.yshift = mean; ep.part = upart;
            ep.eps = eps; ep.k1 = k1; ep.k2 = k2; ep.sign = -1.0f;
            lin_launch(a.BN, ggrid, st, C, a.Dp, a.NT, Qpack, precpack, ep);
        } else {
            dense_kick_elem_kernel<<<C, 256, 0, st>>>(a, Q, P, Ppack, eps, k1, k2, upart);
        }
    };
    auto kinetic = [&](float* kpart) {                                       // :812  p.(M^-1 p)
        LinEpi ep = {};
        ep.Y = P; ep.part = kpart;
        lin_launch(a.BN, ggrid, st, C, a.Dp, a.NT, Ppack, impack, ep);
    };
    auto load_q = [&](const float* src) {
        dense_load_rows_kernel<<<a.Cp, 256, 0, st>>>(src, C, ld, D, Q, a.Cp, a.Dp);
        if (gemm_target) dense_pack_kernel<<<296, 256, 0, st>>>(Q, mean, a.Cp, a.Dp, TC_M, Qpack);
    };
    load_q(q_init);
    kick(0, 0);
    dense_store_u_kernel<<<(C + 127) / 128, 128, 0, st>>>(a, upart, r.U_init);
    load_q(q_cur);
    kick(0, 0);
    dense_store_u_kernel<<<(C + 127) / 128, 128, 0, st>>>(a, upart, r.U_cur);
    if (it0 == 0 && samples) {                                                      // slot 0 = params_init (:959)
        cudaMemcpy2DAsync(samples, (size_t)(S - burn) * ld * sizeof(float), q_init, (size_t)ld * sizeof(float),
                          (size_t)ld * sizeof(float), (size_t)C, cudaMemcpyDeviceToDevice, st);
    }
    for (int n = it0; n < it1; ++n) {
        dense_gibbs_kernel<<<C, 256, 0, st>>>(r, n, Q, P, Qpack);            // q_cur -> Q (+ packed), z -> Zpack
        {
            LinEpi ep = {};                                                  // :199  p = chol(M) z
            ep.X = P; ep.Xpack = Ppack; ep.assign = 1; ep.sign = 1.0f;
            lin_launch(a.BN, ggrid, st, C, a.Dp, a.NT, Zpack, trilpack, ep);
        }
        kinetic(kpart0);
        kick(LIN_K_HALF, 0);                                                 // :281
        for (int l = 1; l <= L; ++l) {
            LinEpi ep = {};                                                  // :294  q <- q + eps*(M^-1 p)
            ep.X = Q; ep.Xpack = gemm_target ? Qpack : nullptr; ep.shift = mean; ep.eps = eps; ep.k1 = LIN_K_E;
            ep.sign = 1.0f;
            lin_launch(a.BN, ggrid, st, C, a.Dp, a.NT, Ppack, impack, ep);
            kick(LIN_K_E, l == L ? LIN_K_HALF : 0);                          // :298 (:302)
        }
        kinetic(kpartL);
        dense_mh_kernel<<<C, 256, 0, st>>>(r, n, Q, P, upart);
    }
    return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA;
}

int dense_hmc_run(const hmcx_target_t* target, const hmcx_mass_t* mass, const hmcx_rng_t* rng, const hmcx_nuts_t* nuts,
                  const float* q_init, float* q_cur, float* eps, int C, int ld, int L, int S, int burn, int it0,
                  int it1, float* samples, uint8_t* accept, uint8_t* diverged, float* ham, int32_t* num_rejected,
                  float* ws, cudaStream_t st) {
    if (!target) return HMCX_ERR_INVALID_ARG;
    const bool full_mass = mass && mass->kind == HMCX_MASS_FULL;
    if (target->kind == HMCX_TARGET_GAUSS_FULL ? !target->prec
                                               : !(full_mass && (target->kind == HMCX_TARGET_GAUSS_ISO ||
                                                                 target->kind == HMCX_TARGET_GAUSS_DIAG)))
        return HMCX_ERR_INVALID_ARG;
    const int D = target->dim;
    if (!rng || !q_init || !q_cur || !eps || !ws || C < 1 || ld < D || (ld & 3) || L < 1 || S < 1 || burn < 0 ||
        burn >= S || it0 < 0 || it1 > S || it0 > it1)
        return HMCX_ERR_INVALID_ARG;
    const int mk = mass ? mass->kind : HMCX_MASS_NONE;
    if (mk == HMCX_MASS_DIAG && (!mass->inv_mass || !mass->mass_factor)) return HMCX_ERR_INVALID_ARG;
    if (rng->mode == HMCX_RNG_INJECTED) {
        if (!rng->normals || !rng->log_uniforms) return HMCX_ERR_INVALID_ARG;
    } else if (rng->mode != HMCX_RNG_PHILOX) {
        return HMCX_ERR_INVALID_ARG;
    }
    if (flow_small_ok(D, ld))                    // D <= 128: the whole run in one persistent launch (hmcx_flow.cu)
        return flow_small_hmc_run(target, mass, rng, nuts, q_init, q_cur, eps, C, ld, L, S, burn, it0, it1, samples, accept,
                                  diverged, ham, num_rejected, st);
    if (mk == HMCX_MASS_FULL)
        return dense_fullmass_hmc_run(target, mass, rng, nuts, q_init, q_cur, eps, C, ld, L, S, burn, it0, it1, samples,
                                      accept, diverged, ham, num_rejected, ws, st);
    DenseRun r = {};
    DenseArgs& a = r.a;
    a.C = C; a.D = D; a.Cp = (C + 127) / 128 * 128; a.Dp = (D + 127) / 128 * 128;
    a.log_norm = target->log_norm; a.mk = mk; a.tk = target->kind;
    const int mt = a.Cp / 128;
    a.BN = dense_tile_width(a.Dp, mt);
    if (!a.BN) return HMCX_ERR_INVALID_ARG;
    a.NT = a.Dp / a.BN;
    // carve the workspace
    const size_t CD = (size_t)a.Cp * a.Dp, DD = (size_t)a.Dp * a.Dp;
    float* Qbuf[2] = {ws, ws + CD};
    float* Qp[2] = {ws + 2 * CD, ws + 4 * CD};
    float* P = ws + 6 * CD;
    float* prec = ws + 7 * CD;
    float* ppack = prec + DD;
    float* mean = ppack + 2 * DD;
    float* im = mean + a.Dp;
    float* sd = im + a.Dp;
    float* upart = sd + a.Dp;
    r.kin0 = upart + (size_t)a.Cp * (a.Dp / 32);
    r.U_cur = r.kin0 + a.Cp;
    r.U_init = r.U_cur + a.Cp;
    a.prec = prec; a.mean = mean; a.im = (mk == HMCX_MASS_DIAG) ? im : nullptr; a.sd = (mk == HMCX_MASS_DIAG) ? sd : nullptr;
    r.ld = ld; r.rng_mode = rng->mode; r.seed = rng->seed; r.chain_offset = rng->chain_offset;
    r.normals = rng->normals; r.logu = rng->log_uniforms;
    r.nuts = (nuts && nuts->enabled) ? 1 : 0;
    if (r.nuts) {
        if (!nuts->table || !nuts->h_bar || !nuts->eps_bar || burn < 1) return HMCX_ERR_INVALID_ARG;
        r.delta = nuts->desired_accept_rate; r.mu = nuts->mu; r.table = nuts->table;
        r.h_bar = nuts->h_bar; r.eps_bar = nuts->eps_bar;
        r.eps_schedule = nuts->eps_schedule; r.eps_trace = nuts->eps_trace;
    }
    r.q_init = q_init; r.q_cur = q_cur; r.eps = eps; r.S = S; r.burn = burn; r.it0 = it0;
    r.samples = samples; r.accept = accept; r.diverged = diverged; r.ham = ham; r.num_rejected = num_rejected;

    const dim3 ggrid(a.NT, mt);
    auto step = [&](const float* qin, const float* qpin, float* qout, float* qpout, int mode) -> bool {
        const size_t sm = (size_t)dense_stages(a.BN) * dense_stage_floats(a.BN) * sizeof(float);
        if (a.BN == 128) launch_pdl(dense_step_kernel<128>, ggrid, DENSE_THREADS, sm, st, a, qin, qpin, ppack, qout, qpout, P, eps, mode, upart);
        else if (a.BN == 64) launch_pdl(dense_step_kernel<64>, ggrid, DENSE_THREADS, sm, st, a, qin, qpin, ppack, qout, qpout, P, eps, mode, upart);
        else launch_pdl(dense_step_kernel<32>, ggrid, DENSE_THREADS, sm, st, a, qin, qpin, ppack, qout, qpout, P, eps, mode, upart);
        return true;
    };
    {
        bool ok = true;
        ok = ok && cudaFuncSetAttribute(dense_step_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)((size_t)dense_stages(128) * dense_stage_floats(128) * 4)) == cudaSuccess;
        ok = ok && cudaFuncSetAttribute(dense_step_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)((size_t)dense_stages(64) * dense_stage_floats(64) * 4)) == cudaSuccess;
        ok = ok && cudaFuncSetAttribute(dense_step_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)((size_t)dense_stages(32) * dense_stage_floats(32) * 4)) == cudaSuccess;
        if (!ok) { cudaGetLastError(); return HMCX_ERR_CUDA; }
    }
    dense_pad_matrix_kernel<<<296, 256, 0, st>>>(target->prec, D, prec, a.Dp);
    dense_pack_kernel<<<296, 256, 0, st>>>(prec, nullptr, a.Dp, a.Dp, a.BN, ppack);
    dense_pad_vector_kernel<<<8, 256, 0, st>>>(target->mean, D, mean, a.Dp);
    if (mk == HMCX_MASS_DIAG) {
        dense_pad_vector_kernel<<<8, 256, 0, st>>>(mass->inv_mass, D, im, a.Dp);
        dense_pad_vector_kernel<<<8, 256, 0, st>>>(mass->mass_factor, D, sd, a.Dp);
    }
    cudaMemsetAsync(ws, 0, 7 * CD * sizeof(float), st);                              // Q, Qpack, P (incl. pad rows)
    // log p of params_init (needed again by the :1018 quirk) and of the current state
    dense_load_rows_kernel<<<a.Cp, 256, 0, st>>>(q_init, C, ld, D, Qbuf[0], a.Cp, a.Dp);
    dense_pack_kernel<<<296, 256, 0, st>>>(Qbuf[0], mean, a.Cp, a.Dp, TC_M, Qp[0]);
    step(Qbuf[0], Qp[0], Qbuf[1], Qp[1], DENSE_EVAL);
    dense_store_u_kernel<<<(C + 127) / 128, 128, 0, st>>>(a, upart, r.U_init);
    dense_load_rows_kernel<<<a.Cp, 256, 0, st>>>(q_cur, C, ld, D, Qbuf[0], a.Cp, a.Dp);
    dense_pack_kernel<<<296, 256, 0, st>>>(Qbuf[0], mean, a.Cp, a.Dp, TC_M, Qp[0]);
    step(Qbuf[0], Qp[0], Qbuf[1], Qp[1], DENSE_EVAL);
    dense_store_u_kernel<<<(C + 127) / 128, 128, 0, st>>>(a, upart, r.U_cur);
    if (it0 == 0 && samples) {                                                      // slot 0 = params_init (:959)
        cudaMemcpy2DAsync(samples, (size_t)(S - burn) * ld * sizeof(float), q_init, (size_t)ld * sizeof(float),
                          (size_t)ld * sizeof(float), (size_t)C, cudaMemcpyDeviceToDevice, st);
    }
    for (int n = it0; n < it1; ++n) {
        dense_gibbs_kernel<<<C, 256, 0, st>>>(r, n, Qbuf[0], P, Qp[0]);
        for (int l = 0; l <= L; ++l) {
            const int mode = (l == 0) ? DENSE_FIRST : (l == L ? DENSE_LAST : DENSE_MIDDLE);
            step(Qbuf[l & 1], Qp[l & 1], Qbuf[(l + 1) & 1], Qp[(l + 1) & 1], mode);
        }
        dense_mh_kernel<<<C, 256, 0, st>>>(r, n, Qbuf[L & 1], P, upart);
    }
    return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA;
}

// ---------------------------------------------------------------------------------------------------------
// sampler=RMHMC on Gaussian targets without jitter: the metric G = -Hessian (HESSIAN) or its softabs map is the SAME
// matrix at every point, so dH/dtheta = -grad log p(theta) and dH/dp = G^-1 p (samplers.py:389-462 through autograd of
// :677-736), and every flow of the explicit integrator (A-B-C-B-A on the augmented state, :427-458) and of the
// implicit one (:363-386; its fixed points converge in two sweeps) is a (chains x D).(D x D) GEMM on the tensor cores with the
// metric solve G^-1 p as one of them.  The host supplies G^-1, chol(G) (gibbs :183-184) and log det G, all computed
// with the reference's torch ops.
// ---------------------------------------------------------------------------------------------------------
// H_C flow (:435-450): the SEQUENTIAL rotation of (theta, p, theta~, p~) with c = cos(2 w eps), s = sin(2 w eps)
__global__ void __launch_bounds__(256)
dense_rm_bind_kernel(const DenseArgs a, float cw, float sw, float* __restrict__ Q, float* __restrict__ P,
                     float* __restrict__ Qc, float* __restrict__ Pc, float* __restrict__ Qpack, float* __restrict__ Ppack,
                     float* __restrict__ Qcpack, float* __restrict__ Pcpack) {
    const int c = blockIdx.x, Dp = a.Dp, kchunks = Dp / TC_KC;
    for (int v = threadIdx.x; 4 * v < Dp; v += blockDim.x) {
        const size_t o = (size_t)c * Dp + 4 * v;
        float q[4], p[4], qt[4], pt[4], yq[4], yqt[4];
        ld4(Q + o, q); ld4(P + o, p); ld4(Qc + o, qt); ld4(Pc + o, pt);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float qn = mul(0.5f, add(add(add(q[j], qt[j]), mul(cw, sub(q[j], qt[j]))), mul(sw, sub(p[j], pt[j]))));
            const float pn = mul(0.5f, add(sub(add(p[j], pt[j]), mul(sw, sub(qn, qt[j]))), mul(cw, sub(p[j], pt[j]))));
            const float qtn = mul(0.5f, sub(sub(add(qn, qt[j]), mul(cw, sub(qn, qt[j]))), mul(sw, sub(pn, pt[j]))));
            const float ptn = mul(0.5f, sub(add(add(pn, pt[j]), mul(sw, sub(qn, qtn))), mul(cw, sub(pn, pt[j]))));
            q[j] = qn; p[j] = pn; qt[j] = qtn; pt[j] = ptn;
            yq[j] = sub(qn, a.mean[4 * v + j]); yqt[j] = sub(qtn, a.mean[4 * v + j]);
        }
        st4(Q + o, q); st4(P + o, p); st4(Qc + o, qt); st4(Pc + o, pt);
        const int kc = (4 * v) / TC_KC, off = pack_elem_off(c % TC_M, (4 * v) % TC_KC, TC_M);
        const size_t bh = pack_block_base(c / TC_M, kc, 0, kchunks, TC_M), bl = pack_block_base(c / TC_M, kc, 1, kchunks, TC_M);
        split_store4(Ppack + bh, Ppack + bl, off, p);
        split_store4(Pcpack + bh, Pcpack + bl, off, pt);
        if (Qpack) { split_store4(Qpack + bh, Qpack + bl, off, yq); split_store4(Qcpack + bh, Qcpack + bl, off, yqt); }
    }
}

size_t dense_rmhmc_workspace_floats(int C, int D) {
    const size_t Cp = (size_t)(C + 127) / 128 * 128, Dp = (size_t)(D + 31) / 32 * 32;
    return 14 * Cp * Dp + 7 * Dp * Dp + 2 * Dp + 3 * Cp * (Dp / 32) + 2 * Cp + 64;
}

int dense_rmhmc_run(const hmcx_target_t* target, const hmcx_rmhmc_t* cfg, const hmcx_const_metric_t* gm,
                    const hmcx_rng_t* rng, const float* q_init, float* q_cur, const float* eps, int C, int ld, int L,
                    int S, int burn, int it0, int it1, float* samples, uint8_t* accept, uint8_t* diverged, float* ham,
                    int32_t* num_rejected, float* ws, cudaStream_t st) {
    if (!target || !cfg || !gm || !rng || !q_init || !q_cur || !eps || !ws) return HMCX_ERR_INVALID_ARG;
    const int D = target->dim, tk = target->kind;
    if (tk != HMCX_TARGET_GAUSS_ISO && tk != HMCX_TARGET_GAUSS_DIAG && tk != HMCX_TARGET_GAUSS_FULL) return HMCX_ERR_UNSUPPORTED;
    if (cfg->jitter >= 0.0f) return HMCX_ERR_UNSUPPORTED;                  // jitter makes the metric a per-call random matrix
    if (cfg->integrator != 1 && cfg->integrator != 2) return HMCX_ERR_INVALID_ARG;
    if (!gm->metric_inv || !gm->metric_chol || (tk == HMCX_TARGET_GAUSS_FULL && !target->prec) ||
        (tk == HMCX_TARGET_GAUSS_DIAG && !target->inv_var))
        return HMCX_ERR_INVALID_ARG;
    if (C < 1 || D < 1 || ld < D || (ld & 3) || L < 1 || S < 1 || burn < 0 || burn >= S || it0 < 0 || it1 > S || it0 > it1)
        return HMCX_ERR_INVALID_ARG;
    if (rng->mode == HMCX_RNG_INJECTED) {
        if (!rng->normals || !rng->log_uniforms) return HMCX_ERR_INVALID_ARG;
    } else if (rng->mode != HMCX_RNG_PHILOX) {
        return HMCX_ERR_INVALID_ARG;
    }
    if (flow_small_ok(D, ld))                    // D <= 128: the whole run in one persistent launch (hmcx_flow.cu)
        return flow_small_rmhmc_run(target, cfg, gm, rng, q_init, q_cur, eps, C, ld, L, S, burn, it0, it1, samples, accept,
                                    diverged, ham, num_rejected, mul_host(0.5f, cfg->pi_term), mul_host(0.5f, gm->log_det), st);
    DenseRun r = {};
    DenseArgs& a = r.a;
    a.C = C; a.D = D; a.Cp = (C + 127) / 128 * 128;
    a.log_norm = target->log_norm; a.mk = HMCX_MASS_FULL; a.tk = tk;
    if (!dense_geometry(a)) return HMCX_ERR_INVALID_ARG;
    const size_t CD = (size_t)a.Cp * a.Dp, DD = (size_t)a.Dp * a.Dp;
    float* Q = ws;           float* P = ws + CD;          float* Qc = ws + 2 * CD;      float* Pc = ws + 3 * CD;
    float* Qpack = ws + 4 * CD;  float* Ppack = ws + 6 * CD;  float* Qcpack = ws + 8 * CD;  float* Pcpack = ws + 10 * CD;
    float* Zpack = ws + 12 * CD;
    float* scratch = ws + 14 * CD;
    float* precpack = scratch + DD;
    float* ginvpack = precpack + 2 * DD;
    float* cholpack = ginvpack + 2 * DD;
    float* mean = cholpack + 2 * DD;
    float* ivar = mean + a.Dp;
    float* upart = ivar + a.Dp;
    float* kpart0 = upart + (size_t)a.Cp * (a.Dp / 32);
    float* kpartL = kpart0 + (size_t)a.Cp * (a.Dp / 32);
    r.U_cur = kpartL + (size_t)a.Cp * (a.Dp / 32);
    r.U_init = r.U_cur + a.Cp;
    r.zpack = Zpack; r.kpart0 = kpart0; r.kpartL = kpartL;
    a.mean = mean; a.ivar = ivar;
    r.ld = ld; r.rng_mode = rng->mode; r.seed = rng->seed; r.chain_offset = rng->chain_offset;
    r.normals = rng->normals; r.logu = rng->log_uniforms;
    r.q_init = q_init; r.q_cur = q_cur; r.eps = const_cast<float*>(eps); r.S = S; r.burn = burn; r.it0 = it0;
    r.samples = samples; r.accept = accept; r.diverged = diverged; r.ham = ham; r.num_rejected = num_rejected;
    r.rm = 1; r.ham_c1 = mul_host(0.5f, cfg->pi_term); r.ham_c2 = mul_host(0.5f, gm->log_det);
    if (!lin_configure()) return HMCX_ERR_CUDA;

    const bool gemm_target = tk == HMCX_TARGET_GAUSS_FULL;
    auto pack_matrix = [&](const float* src, float* dst) {
        dense_pad_matrix_kernel<<<296, 256, 0, st>>>(src, D, scratch, a.Dp);
        dense_pack_kernel<<<296, 256, 0, st>>>(scratch, nullptr, a.Dp, a.Dp, a.BN, dst);
    };
    if (gemm_target) pack_matrix(target->prec, precpack);
    pack_matrix(gm->metric_inv, ginvpack);
    pack_matrix(gm->metric_chol, cholpack);
    dense_pad_vector_kernel<<<8, 256, 0, st>>>(tk == HMCX_TARGET_GAUSS_ISO ? nullptr : target->mean, D, mean, a.Dp);
    dense_pad_vector_kernel<<<8, 256, 0, st>>>(tk == HMCX_TARGET_GAUSS_DIAG ? target->inv_var : nullptr, D, ivar, a.Dp);
    cudaMemsetAsync(ws, 0, 14 * CD * sizeof(float), st);

    const dim3 ggrid(a.NT, a.Cp / 128);
    // p_ <- p_ - k*dH/dtheta(q_) = p_ + k*grad log p(q_)  (k = 0: U-terms of q_ only)
    // `twice`: the same kick applied two times (two separately rounded updates, one contraction) -- the last A flow of an
    // explicit step and the first A flow of the next act on the same (theta, p~)
    auto kick = [&](float* q_, float* qpack_, float* p_, float* ppack_, int k1, float* part, bool twice = false) {
        if (gemm_target) {
            LinEpi ep = {};
            ep.X = k1 ? p_ : nullptr; ep.Xpack = k1 ? ppack_ : nullptr; ep.Y = part ? q_ : nullptr; ep.yshift = mean;
            ep.part = part; ep.eps = eps; ep.k1 = k1; ep.sign = -1.0f;
            if (twice) { ep.k2 = k1; ep.k2add = 1; }
            lin_launch(a.BN, ggrid, st, C, a.Dp, a.NT, qpack_, precpack, ep);
        } else {
            dense_kick_elem_kernel<<<C, 256, 0, st>>>(a, q_, p_, ppack_, eps, k1, twice ? k1 : 0, part, twice ? 1 : 0);
        }
    };
    // q_ <- q_ + k*G^-1 p_  [+ k*G^-1 p_]
    auto drift = [&](float* q_, float* qpack_, float* ppack_, bool twice) {
        LinEpi ep = {};
        ep.X = q_; ep.Xpack = gemm_target ? qpack_ : nullptr; ep.shift = mean; ep.eps = eps; ep.k1 = LIN_K_HALF;
        ep.k2 = twice ? LIN_K_HALF : 0; ep.k2add = 1; ep.sign = 1.0f;
        lin_launch(a.BN, ggrid, st, C, a.Dp, a.NT, ppack_, ginvpack, ep);
    };
    auto kinetic = [&](float* kpart) {                                       // p.(G^-1 p)  (:729-730)
        LinEpi ep = {};
        ep.Y = P; ep.part = kpart;
        lin_launch(a.BN, ggrid, st, C, a.Dp, a.NT, Ppack, ginvpack, ep);
    };
    auto load_q = [&](const float* src) {
        dense_load_rows_kernel<<<a.Cp, 256, 0, st>>>(src, C, ld, D, Q, a.Cp, a.Dp);
        if (gemm_target) dense_pack_kernel<<<296, 256, 0, st>>>(Q, mean, a.Cp, a.Dp, TC_M, Qpack);
    };
    load_q(q_init);
    kick(Q, Qpack, P, Ppack, 0, upart);
    dense_store_u_kernel<<<(C + 127) / 128, 128, 0, st>>>(a, upart, r.U_init);
    load_q(q_cur);
    kick(Q, Qpack, P, Ppack, 0, upart);
    dense_store_u_kernel<<<(C + 127) / 128, 128, 0, st>>>(a, upart, r.U_cur);
    if (it0 == 0 && samples) {                                                      // slot 0 = params_init (:959)
        cudaMemcpy2DAsync(samples, (size_t)(S - burn) * ld * sizeof(float), q_init, (size_t)ld * sizeof(float),
                          (size_t)ld * sizeof(float), (size_t)C, cudaMemcpyDeviceToDevice, st);
    }
    const bool explicit_int = cfg->integrator == 1;
    for (int n = it0; n < it1; ++n) {
        dense_gibbs_kernel<<<C, 256, 0, st>>>(r, n, Q, P, Qpack);
        {
            LinEpi ep = {};                                                  // :183-184  p = chol(G) z
            ep.X = P; ep.Xpack = Ppack; ep.assign = 1; ep.sign = 1.0f;
            lin_launch(a.BN, ggrid, st, C, a.Dp, a.NT, Zpack, cholpack, ep);
        }
        kinetic(kpart0);
        if (explicit_int) {
            cudaMemcpyAsync(Qc, Q, 2 * CD * sizeof(float), cudaMemcpyDeviceToDevice, st);          // theta~, p~ (:425-426)
            cudaMemcpyAsync(Qcpack, Qpack, 4 * CD * sizeof(float), cudaMemcpyDeviceToDevice, st);
            // The last A flow of step l (:457-458) and the first A flow of step l+1 (:429-430) act on the same (theta, p~):
            // one contraction each for dH/dtheta and G^-1 p~, applied twice in the epilogue (6L+2 GEMMs per trajectory
            // instead of 8L; the same bits -- the second application re-reads the identical accumulator)
            kick(Q, Qpack, P, Ppack, LIN_K_HALF, nullptr);                                          // A (:429-430)
            drift(Qc, Qcpack, Pcpack, false);
            for (int l = 0; l < L; ++l) {
                const bool last = l == L - 1;
                drift(Q, Qpack, Ppack, false);                                                      // B (:432-433)
                kick(Qc, Qcpack, Pc, Pcpack, LIN_K_HALF, nullptr);
                dense_rm_bind_kernel<<<C, 256, 0, st>>>(a, cfg->cos_2we, cfg->sin_2we, Q, P, Qc, Pc,  // C (:435-450)
                                                      gemm_target ? Qpack : nullptr, Ppack, Qcpack, Pcpack);
                drift(Q, Qpack, Ppack, false);                                                      // B (:454-455)
                kick(Qc, Qcpack, Pc, Pcpack, LIN_K_HALF, nullptr);
                kick(Q, Qpack, P, Ppack, LIN_K_HALF, last ? upart : nullptr, !last);                // A (:457-458) [+ :429-430]
                drift(Qc, Qcpack, Pcpack, !last);
            }
        } else {
            for (int l = 0; l < L; ++l) {
                kick(Q, Qpack, P, Ppack, LIN_K_HALF, nullptr);                                      // :363
                drift(Q, Qpack, Ppack, true);                                                       // :364
                kick(Q, Qpack, P, Ppack, LIN_K_HALF, upart);                                        // :368-383
            }
        }
        kinetic(kpartL);
        dense_mh_kernel<<<C, 256, 0, st>>>(r, n, Q, P, upart);
    }
    return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA;
}


// wgmma takes tf32 operands from shared memory in K-major form only: an operand that an epilogue produces "row per
// thread" is written transposed into its packed K-major block.

int gemm_nt_tf32x3(const float* A, const float* B, float* D, int M, int N, int K, cudaStream_t st) {
    if (!A || !B || !D || M < 1 || N < 1 || K < 1) return HMCX_ERR_INVALID_ARG;
    if ((M % TC_M) || (N % TC_N) || (K % TC_KC)) return HMCX_ERR_UNSUPPORTED;
    const size_t smem = (size_t)(2 * TC_M + 2 * TC_N) * TC_KC * sizeof(float);          // 64 KB
    if (cudaFuncSetAttribute(gemm_nt_tf32x3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
        cudaGetLastError();
        return HMCX_ERR_CUDA;
    }
    dim3 grid(N / TC_N, M / TC_M);
    gemm_nt_tf32x3_kernel<<<grid, TC_THREADS, smem, st>>>(A, B, D, M, N, K);
    return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA;
}

}  // namespace hmcx
