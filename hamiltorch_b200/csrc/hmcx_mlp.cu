// hmcx_mlp.cu -- Bayesian dense-stack (MLP) HMC on sm_90a (H100): the BNN rows of the hot path.
//
//   define_model_log_prob / define_split_model_log_prob   samplers.py:1093-1258  -> mlp_log_prob(), mlp_grad_split()
//   leapfrog SPLITTING / SPLITTING_RAND / SPLITTING_KMID  samplers.py:465-603    -> trajectory in mlp_run_kernel
//   sample() loop around them (sample_model / sample_split_model, :1261-1466)    -> mlp_run_kernel (persistent)
//   predict_model                                          samplers.py:1468-1562  -> mlp_predict_kernel
//   collect_gradients (autograd) is replaced by a hand-written backward pass      -> mlp_grad_split()
//
// Design of the fp32 SIMT form (the tensor-core first layer is further below, DESIGN.md 3.4):
// one CTA of 256 threads owns one chain for the whole run.  The chain's flat parameter vector q, its momentum p and
// the split gradient g live in SHARED MEMORY in the reference's flat layout (util.py:121-136), so every weight is
// read from smem by the GEMM loops and the leapfrog kick/drift are conflict-free element-wise passes.  A gradient
// evaluation streams the split's data rows through in tiles of 32 rows: forward (Linear+activation per layer,
// register micro-tiles 4x4 with interleaved columns and a per-lane k-rotation that makes the strided weight reads
// bank-conflict-free), loss gradient, backward (dW += dZ^T A, db, dA = dZ W) accumulating straight into g.
// Multiply-adds inside the GEMM loops use FMA: these sums have no bit-parity counterpart in the reference (its
// sgemm order is unknowable); everything element-wise (kicks, drifts, prior, Hamiltonian assembly, MH) keeps the
// reference's separately-rounded fp32 operation order.
#include "hmcx_common.cuh"
#include "hmcx_wgmma.cuh"
#include <cooperative_groups.h>
#include <cfloat>

namespace cg = cooperative_groups;

namespace hmcx {

constexpr int MLP_THREADS = 512;
constexpr int MLP_T_MAX = 64;             // data rows per tile: 64 when the tile buffers fit next to q,p,g, else 32 / 16
// (rows of a 4x4 micro-tile are rg, rg+T/4, rg+2T/4, rg+3T/4)

struct MlpDev {
    int L, D, Dp, N, M, has_data, loss;
    int n[HMCX_MLP_MAX_LAYERS + 1], act[HMCX_MLP_MAX_LAYERS];
    int woff[HMCX_MLP_MAX_LAYERS], boff[HMCX_MLP_MAX_LAYERS];
    int aoff[HMCX_MLP_MAX_LAYERS + 1];    // smem offsets (floats, relative to the tile area) of A[l] (T x n[l])
    int dzoff[2];                         // two delta buffers (T x maxw)
    int tile_floats;
    int tile_base;                        // float offset of the tile area in dynamic shared memory (after the state vectors)
    int T;                                // rows per tile (multiple of 4)
    int tc;                               // 1: the first layer's GEMMs run on the tensor cores (layout below), 0: SIMT tiles
    int tc_f0, tc_f1, tc_b, tc_part;      // tile-area offsets (floats): two forward X operand buffers, the backward one, partials
    int tc_yraw;                          // cp.async landing buffer of the tile's targets
    const float* xp;                      // packed X operands (hmcx_mlp_pack_x): per tile [fwd hi|lo (128 n0) | bwd hi|lo (128 n0)]
    int tb[HMCX_MLP_MAX_SPLITS + 1];      // first packed tile of split s (tiles of a split start at its first row)
    int flat_base;                        // first packed tile of the all-rows tiling (rows 0, 64, ...)
    float tau_out, prior_scale, c_ll;     // c_ll = fp32(-0.5*tau_out) (regression, :1184) or fp32(-tau_out) (:1172-1180)
    float two_var[2 * HMCX_MLP_MAX_LAYERS], log_scale[2 * HMCX_MLP_MAX_LAYERS], gcoef[2 * HMCX_MLP_MAX_LAYERS];
    const float* x;
    const float* y;
    int sb[HMCX_MLP_MAX_SPLITS + 1];
};

__device__ __forceinline__ float act_fwd(float z, int a) {
    if (a == HMCX_ACT_RELU) return z > 0.0f ? z : 0.0f;
    if (a == HMCX_ACT_TANH) return tanhf(z);
    if (a == HMCX_ACT_SIGMOID) return 1.0f / (1.0f + expf(-z));
    return z;
}
// derivative expressed through the activation's OUTPUT (what the backward pass has at hand)
__device__ __forceinline__ float act_bwd(float aout, int a) {
    if (a == HMCX_ACT_RELU) return aout > 0.0f ? 1.0f : 0.0f;
    if (a == HMCX_ACT_TANH) return 1.0f - aout * aout;
    if (a == HMCX_ACT_SIGMOID) return aout * (1.0f - aout);
    return 1.0f;
}

// ---- tile primitives (all 256 threads; callers place the __syncthreads) ---------------------------------------
__device__ __forceinline__ void mlp_load_x(const MlpDev& m, float* A0, int r0, int cnt) {
    const int n0 = m.n[0];
    for (int i = threadIdx.x; i < m.T * n0; i += MLP_THREADS)
        A0[i] = (i < cnt * n0) ? __ldg(m.x + (size_t)r0 * n0 + i) : 0.0f;
}

// ---- "thin" layers (few outputs, e.g. the scalar regression head): split the reduction over a lane group ---------
// S = lanes per output (power of two, S | 32); each group's lanes stride the reduction index, then shuffle-reduce.
__device__ __forceinline__ int thin_group(int outputs) {
    int s = 32;
    while (s > 1 && outputs * s > MLP_THREADS) s >>= 1;
    return s;
}
__device__ __forceinline__ float group_sum(float v, int S) {
    for (int o = S >> 1; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ void mlp_linear_fwd_thin(const float* Ain, const float* W, const float* b, float* Aout,
                                                    int n_in, int n_out, int act, int T) {
    const int outputs = T * n_out, S = thin_group(outputs);
    for (int base = 0; base < outputs; base += MLP_THREADS / S) {
        const int o = base + threadIdx.x / S, s = threadIdx.x % S;
        const bool live = o < outputs;
        const int r = live ? o / n_out : 0, j = live ? o % n_out : 0;
        float acc = 0.0f;
        for (int k = s; k < n_in; k += S) acc = fmaf(Ain[r * n_in + k], W[j * n_in + k], acc);
        acc = group_sum(acc, S);
        if (live && s == 0) Aout[r * n_out + j] = act_fwd(acc + b[j], act);
    }
}

// Aout[T x n_out] = act(Ain[T x n_in] . W^T + b),  W row-major (n_out, n_in) in shared memory.
// 4x4 register micro-tiles (rows rg+8i, columns cg+ncg*jj); the reduction index is rotated per lane so that the
// strided weight reads are bank-conflict-free; with n_in % 4 == 0 and 16-byte aligned rows the loads are float4.
__device__ __forceinline__ void mlp_linear_fwd(const float* Ain, const float* W, const float* b, float* Aout,
                                               int n_in, int n_out, int act, int T) {
    const int ncg = (n_out + 3) >> 2, RG = T >> 2;
    if (RG * ncg * 4 <= MLP_THREADS) { mlp_linear_fwd_thin(Ain, W, b, Aout, n_in, n_out, act, T); return; }
    const bool vec = ((n_in & 3) == 0) && ((((size_t)W) & 15) == 0) && ((((size_t)Ain) & 15) == 0);
    for (int tile = threadIdx.x; tile < RG * ncg; tile += MLP_THREADS) {
        const int cg = tile % ncg, rg = tile / ncg;
        int jc[4];
        float acc[4][4];
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
            const int j = cg + jj * ncg;
            jc[jj] = j < n_out ? j : n_out - 1;
            const float bj = b[jc[jj]];
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[i][jj] = bj;
        }
        if (vec) {
            const int n4 = n_in >> 2, rot = cg % n4;          // rotation in units of float4
            const float4* ap[4];
            const float4* wp[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                ap[i] = reinterpret_cast<const float4*>(Ain) + (rg + i * RG) * n4;
                wp[i] = reinterpret_cast<const float4*>(W) + jc[i] * n4;
            }
            auto body = [&](int kk) {
                float4 a[4], w[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) { a[i] = ap[i][kk]; w[i] = wp[i][kk]; }
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int jj = 0; jj < 4; ++jj) acc[i][jj] = fmaf(a[i].x, w[jj].x, acc[i][jj]);
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int jj = 0; jj < 4; ++jj) acc[i][jj] = fmaf(a[i].y, w[jj].y, acc[i][jj]);
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int jj = 0; jj < 4; ++jj) acc[i][jj] = fmaf(a[i].z, w[jj].z, acc[i][jj]);
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int jj = 0; jj < 4; ++jj) acc[i][jj] = fmaf(a[i].w, w[jj].w, acc[i][jj]);
            };
            int kk = rot;                                     // uniform trip count: no divergence across lanes
#pragma unroll 2
            for (int k = 0; k < n4; ++k) {
                body(kk);
                kk = (kk + 1 == n4) ? 0 : kk + 1;
            }
        } else {
            int kk = cg % n_in;                               // per-lane rotation of the reduction index
            for (int k = 0; k < n_in; ++k) {
                float a[4], w[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) a[i] = Ain[(rg + i * RG) * n_in + kk];
#pragma unroll
                for (int jj = 0; jj < 4; ++jj) w[jj] = W[jc[jj] * n_in + kk];
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int jj = 0; jj < 4; ++jj) acc[i][jj] = fmaf(a[i], w[jj], acc[i][jj]);
                if (++kk == n_in) kk = 0;
            }
        }
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
            const int j = cg + jj * ncg;
            if (j < n_out) {
#pragma unroll
                for (int i = 0; i < 4; ++i) Aout[(rg + i * RG) * n_out + j] = act_fwd(acc[i][jj], act);
            }
        }
    }
}

// gW[n_out x n_in] += dz^T[n_out x T] . Ain[T x n_in];   gb[n_out] += column sums of dz
__device__ __forceinline__ void mlp_weight_grad(const float* Ain, const float* dz, float* gW, float* gb, int n_in,
                                                int n_out, int T) {
    const int njg = (n_out + 3) >> 2;
    if (n_out * n_in * 2 <= MLP_THREADS * 4 && n_out * n_in <= MLP_THREADS) {
        // thin: one output (j,k) per lane group, the T rows split over the group's lanes
        const int outputs = n_out * n_in, S = thin_group(outputs);
        for (int base = 0; base < outputs; base += MLP_THREADS / S) {
            const int o = base + threadIdx.x / S, s = threadIdx.x % S;
            const bool live = o < outputs;
            const int j = live ? o / n_in : 0, k = live ? o % n_in : 0;
            float acc = 0.0f;
            for (int r = s; r < T; r += S) acc = fmaf(dz[r * n_out + j], Ain[r * n_in + k], acc);
            acc = group_sum(acc, S);
            if (live && s == 0) gW[j * n_in + k] += acc;
        }
    } else if (((n_in & 3) == 0) && ((((size_t)gW) & 15) == 0) && ((((size_t)Ain) & 15) == 0)) {
        // 4 (rows of gW: j = jg + jj*njg) x 4 (contiguous k) micro-tiles, float4 activations and float4 RMW of gW
        const int nk4 = n_in >> 2;
        const float4* A4 = reinterpret_cast<const float4*>(Ain);
        for (int tile = threadIdx.x; tile < njg * nk4; tile += MLP_THREADS) {
            const int k4 = tile % nk4, jg = tile / nk4;
            int jc[4];
#pragma unroll
            for (int t = 0; t < 4; ++t) { const int j = jg + t * njg; jc[t] = j < n_out ? j : n_out - 1; }
            float4 acc[4];
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) acc[jj] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
            for (int r = 0; r < T; ++r) {
                const float4 a = A4[r * nk4 + k4];
#pragma unroll
                for (int jj = 0; jj < 4; ++jj) {
                    const float d = dz[r * n_out + jc[jj]];
                    acc[jj].x = fmaf(d, a.x, acc[jj].x); acc[jj].y = fmaf(d, a.y, acc[jj].y);
                    acc[jj].z = fmaf(d, a.z, acc[jj].z); acc[jj].w = fmaf(d, a.w, acc[jj].w);
                }
            }
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
                const int j = jg + jj * njg;
                if (j >= n_out) continue;
                float4* dst = reinterpret_cast<float4*>(gW + j * n_in) + k4;
                float4 v = *dst;
                v.x += acc[jj].x; v.y += acc[jj].y; v.z += acc[jj].z; v.w += acc[jj].w;
                *dst = v;
            }
        }
    } else {
        const int nkg = (n_in + 3) >> 2;
        for (int tile = threadIdx.x; tile < njg * nkg; tile += MLP_THREADS) {
            const int kg = tile % nkg, jg = tile / nkg;
            int jc[4], kc[4];
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                const int j = jg + t * njg, k = kg + t * nkg;
                jc[t] = j < n_out ? j : n_out - 1;
                kc[t] = k < n_in ? k : n_in - 1;
            }
            float acc[4][4];
#pragma unroll
            for (int jj = 0; jj < 4; ++jj)
#pragma unroll
                for (int t = 0; t < 4; ++t) acc[jj][t] = 0.0f;
            for (int r = 0; r < T; ++r) {
                float d[4], a[4];
#pragma unroll
                for (int t = 0; t < 4; ++t) { d[t] = dz[r * n_out + jc[t]]; a[t] = Ain[r * n_in + kc[t]]; }
#pragma unroll
                for (int jj = 0; jj < 4; ++jj)
#pragma unroll
                    for (int t = 0; t < 4; ++t) acc[jj][t] = fmaf(d[jj], a[t], acc[jj][t]);
            }
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
                const int j = jg + jj * njg;
                if (j >= n_out) continue;
#pragma unroll
                for (int t = 0; t < 4; ++t) {
                    const int k = kg + t * nkg;
                    if (k < n_in) gW[j * n_in + k] += acc[jj][t];
                }
            }
        }
    }
    for (int j = threadIdx.x; j < n_out; j += MLP_THREADS) {
        float s = 0.0f;
        for (int r = 0; r < T; ++r) s += dz[r * n_out + j];
        gb[j] += s;
    }
}

// dz_prev[T x n_in] = (dz[T x n_out] . W[n_out x n_in]) * act'(A[T x n_in])
__device__ __forceinline__ void mlp_input_grad(const float* dz, const float* W, const float* A, float* dz_prev,
                                               int n_in, int n_out, int act_prev, int T) {
    const int nkg = (n_in + 3) >> 2, MLP_RG = T >> 2;
    for (int tile = threadIdx.x; tile < MLP_RG * nkg; tile += MLP_THREADS) {
        const int kg = tile % nkg, rg = tile / nkg;
        int kc[4];
#pragma unroll
        for (int t = 0; t < 4; ++t) { const int k = kg + t * nkg; kc[t] = k < n_in ? k : n_in - 1; }
        float acc[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int t = 0; t < 4; ++t) acc[i][t] = 0.0f;
        for (int j = 0; j < n_out; ++j) {
            float d[4], w[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) d[i] = dz[(rg + i * MLP_RG) * n_out + j];
#pragma unroll
            for (int t = 0; t < 4; ++t) w[t] = W[j * n_in + kc[t]];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int t = 0; t < 4; ++t) acc[i][t] = fmaf(d[i], w[t], acc[i][t]);
        }
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const int k = kg + t * nkg;
            if (k >= n_in) continue;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int o = (rg + i * MLP_RG) * n_in + k;
                dz_prev[o] = acc[i][t] * act_bwd(A[o], act_prev);
            }
        }
    }
}

// forward pass of one tile; returns nothing, leaves A[0..L] in the tile area
__device__ __forceinline__ void mlp_forward_tile(const MlpDev& m, const float* q, float* tile, int r0, int cnt) {
    mlp_load_x(m, tile + m.aoff[0], r0, cnt);
    __syncthreads();
    for (int l = 0; l < m.L; ++l) {
        mlp_linear_fwd(tile + m.aoff[l], q + m.woff[l], q + m.boff[l], tile + m.aoff[l + 1], m.n[l], m.n[l + 1],
                       m.act[l], m.T);
        __syncthreads();
    }
}

// Loss stage of a forwarded tile: returns the thread's partial of the loss sum (ll = c_ll * sum, or c_ll * sum / rows
// for the mean-reduced nll_loss) and, when dz != nullptr, writes dz_L = d ll / d out.  `rows` = data rows of the closure
// being evaluated (the split), only used by the mean reduction.  With log_softmax_out the tile's outputs are replaced
// by their log-softmax (what predict_model returns for such a model).
__device__ __forceinline__ float mlp_loss_tile(const MlpDev& m, float* out, float* dz, int r0, int cnt, int rows,
                                               bool log_softmax_out = false, const float* ytile = nullptr) {
    const int nL = m.n[m.L];
    float sum = 0.0f;
    if (m.loss == HMCX_LOSS_REGRESSION || m.loss == HMCX_LOSS_BINARY) {
        const float c2 = mul(m.c_ll, 2.0f);                               // regression, autograd: ds * (2*diff)
        for (int i = threadIdx.x; i < m.T * nL; i += MLP_THREADS) {
            float d = 0.0f, gz = 0.0f;
            if (i < cnt * nL) {
                const float yv = ytile ? ytile[i] : __ldg(m.y + (size_t)r0 * nL + i), z = out[i];
                if (m.loss == HMCX_LOSS_REGRESSION) {
                    d = sub(z, yv);
                    sum = add(sum, mul(d, d));
                    gz = mul(c2, d);
                } else {                                                  // BCE with logits, sum reduction
                    sum += (1.0f - yv) * z + fmaxf(-z, 0.0f) + log1pf(expf(-fabsf(z)));
                    gz = m.c_ll * (1.0f / (1.0f + expf(-z)) - yv);
                }
            }
            if (dz) dz[i] = gz;
        }
        return sum;
    }
    // multi-class: one thread per data row
    const float cg = (m.loss == HMCX_LOSS_MULTICLASS_LOGSOFTMAX) ? m.c_ll / (float)rows : m.c_ll;
    for (int r = threadIdx.x; r < m.T; r += MLP_THREADS) {
        float* z = out + r * nL;
        if (r < cnt) {
            float mx = z[0];
            for (int k = 1; k < nL; ++k) mx = fmaxf(mx, z[k]);
            float se = 0.0f;
            for (int k = 0; k < nL; ++k) se += expf(z[k] - mx);
            const float lse = mx + logf(se);
            int label = (int)(ytile ? ytile[r] : __ldg(m.y + r0 + r));
            label = label < 0 ? 0 : (label >= nL ? nL - 1 : label);
            sum += lse - z[label];
            for (int k = 0; k < nL; ++k) {
                if (dz) dz[r * nL + k] = cg * (expf(z[k] - lse) - (k == label ? 1.0f : 0.0f));
                if (log_softmax_out) z[k] = z[k] - lse;
            }
        } else if (dz) {
            for (int k = 0; k < nL; ++k) dz[r * nL + k] = 0.0f;
        }
    }
    return sum;
}

// ll of one closure from its reduced loss sum
__device__ __forceinline__ float mlp_ll_from_sum(const MlpDev& m, float sum, int rows) {
    if (m.loss == HMCX_LOSS_MULTICLASS_LOGSOFTMAX) return mul(m.c_ll, __fdiv_rn(sum, (float)rows));
    return mul(m.c_ll, sum);
}

// ---- thread-block clusters: a chain may be owned by CS cooperating CTAs (CS SMs) --------------------------------
// Every CTA of the cluster keeps the full q, p, g in its own shared memory and does the (cheap) element-wise work
// redundantly and identically; the expensive part -- the data rows of a gradient / log-prob evaluation -- is divided
// by tile index (tile i -> rank i % CS), and the partial results are combined through DISTRIBUTED SHARED MEMORY in
// the fixed order rank 0, 1, ... so that all CTAs hold bit-identical sums.  CS is a function of the data layout only
// (never of the number of chains), so results do not depend on how chains are sharded over GPUs.
struct ClusterCtx { int rank, size; };

template <int CS>
__device__ __forceinline__ void cluster_sum_vector(float* v, int n) {
    if (CS == 1) return;
    cg::cluster_group cluster = cg::this_cluster();
    cluster.sync();                                            // every partial is complete
    constexpr int MAXPT = 36;                                  // n <= 512*36 (the three state vectors must fit smem anyway)
    float acc[MAXPT];
#pragma unroll
    for (int t = 0; t < MAXPT; ++t) {
        const int i = threadIdx.x + t * MLP_THREADS;
        float sum = 0.0f;
        if (i < n) {
#pragma unroll
            for (int r = 0; r < CS; ++r) {
                const float x = cluster.map_shared_rank(v, r)[i];
                sum = (r == 0) ? x : add(sum, x);
            }
        }
        acc[t] = sum;
    }
    cluster.sync();                                            // everybody has read everybody's partial
#pragma unroll
    for (int t = 0; t < MAXPT; ++t) {
        const int i = threadIdx.x + t * MLP_THREADS;
        if (i < n) v[i] = acc[t];
    }
    __syncthreads();
}

// scalar version: `slot` is a shared-memory word of this CTA; returns sum over ranks in rank order
template <int CS>
__device__ __forceinline__ float cluster_sum_scalar(float x, float* slot) {
    if (CS == 1) return x;
    cg::cluster_group cluster = cg::this_cluster();
    if (threadIdx.x == 0) *slot = x;
    cluster.sync();
    float sum = 0.0f;
#pragma unroll
    for (int r = 0; r < CS; ++r) {
        const float y = *cluster.map_shared_rank(slot, r);
        sum = (r == 0) ? y : add(sum, y);
    }
    cluster.sync();                                            // slot may be rewritten after this
    return sum;
}


// =========================================================================================================
// First-layer GEMMs on the Hopper tensor cores (wgmma, fp32 accumulators in registers), for one-hidden-layer stacks
//   n0 -> 128 -> nL   (n0 in {16,32,48,64}, nL <= 4; BASELINE config 4 is 64-128-1)
// where  H = X W1^T  (forward) and  dW1 = dH^T X  (backward) carry ~all of the flops.  Per 64-row tile of the split the
// CTA's four warpgroups split the work 2 x 2: warpgroup wg takes hidden units [64 (wg & 1), +64) and tile rows
// [32 (wg >> 1), +32):
//   forward, TRANSPOSED:  H^T[64 units x 32 rows] = W1[64 x n0] . X_rows^T  -- A = W1 as register fragments read from the
//       chain's q in shared memory, B = the X tile (bulk TMA copy of a pre-packed operand); 3xTF32 split operands
//       (hi*hi + hi*lo + lo*hi) keep fp32-level accuracy;
//   epilogue 1: bias + activation on the accumulator fragments (two units x 8 rows per thread), the thin output layer
//       as shuffle sums over the units -> z2 in shared memory -> the usual loss stage;
//   epilogue 2: dH^T = (W2^T dz2) * act'(H) in the same registers; db1 and dW2 are thread-local sums;
//   backward:  dW1[64 units x n0] += dH^T[64 x 32 rows] . X_rows  with dH^T's fragments used AS the A operand
//       (registers, no shared-memory round trip); the accumulators stay in registers across all tiles of the split and
//       the two row halves are added once per evaluation.
// The contraction index of each GEMM is stored in a permuted order in the packed X operands (tc_kpos_fwd / tc_row_bwd)
// so that every A fragment is a plain float4 of W1 (forward) or a set of accumulator registers (backward).  Everything
// around (prior, schedules, kicks, drifts, Hamiltonians, MH, clusters) is the code of the SIMT path.
// =========================================================================================================
constexpr int TC_TR = 64;                 // data rows per tile (MMA N forward, MMA K backward)
constexpr int TC_H = 128;                 // hidden units
constexpr int TC_NLMAX = 4;               // outputs handled by the register head

static_assert(TC_TR / 4 == MLP_THREADS / 32 && TC_TR == 64, "the thread maps assume 16 warps and 64-row tiles");

struct TcCtx { uint32_t barF[2], barB, parF[2], parB; int pre_id; };   // pre_id: tile whose operands an earlier evaluation already prefetched (-1: none)

#ifdef HMCX_TC_PROF
__device__ long long g_tc_prof[512];
__device__ int g_tc_prof_n;
#define TC_MARK(id) do { if (threadIdx.x == 0 && blockIdx.x == 0) { int k_ = g_tc_prof_n; if (k_ < 510) { g_tc_prof[k_] = ((long long)(id) << 48) | (clock64() & 0xFFFFFFFFFFFFll); g_tc_prof_n = k_ + 1; } } } while (0)
#else
#define TC_MARK(id) do {} while (0)
#endif

__device__ __forceinline__ void tc_init(TcCtx& tc, uint64_t* bars) {
    if (threadIdx.x == 0) {
        for (int b = 0; b < 3; ++b) mbar_init(smem_u32(&bars[b]), 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    tc.barF[0] = smem_u32(&bars[0]); tc.barF[1] = smem_u32(&bars[1]); tc.barB = smem_u32(&bars[2]);
    tc.parF[0] = tc.parF[1] = tc.parB = 0;
    tc.pre_id = -1;
}

// round-to-nearest (ties away) tf32 in an fp32 container == cvt.rna.tf32.f32 for finite inputs, as two full-rate
// integer instructions instead of a conversion-pipe instruction (the epilogues split ~50 values per thread per tile)
__device__ __forceinline__ float tf32_rn(float x) {
    return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u);
}
__device__ __forceinline__ void tc_split(const float (&v)[4], uint32_t (&hi)[4], uint32_t (&lo)[4]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float h = tf32_rn(v[i]);
        hi[i] = __float_as_uint(h);
        lo[i] = __float_as_uint(tf32_rn(v[i] - h));
    }
}

// X never changes during a run, so its tf32 hi / lo split and both operand layouts are built ONCE (hmcx_mlp_pack_x ->
// mlp_pack_x_kernel) and a tile's operands arrive ready-made by one bulk TMA copy each:
//   forward B operand  [64 rows hi | 64 rows lo (N = 128)] x [n0 (K)], K-major core matrices (8 rows x 16 B);
//   backward B operand [n0 hi | n0 lo (N = 2 n0)] x [64 rows (K)], K-major (4 K positions of one input column per 16 B).
// K orders: forward position 16 t + 8 e + c + 4 h holds input feature 16 t + 4 c + 2 e + h (wgmma k-step 2 t + e, A
// fragment column c + 4 h), so thread column c finds the A fragments of k-steps 2t and 2t+1 in ONE float4 of its W1 row;
// backward position 8 s + c + 4 h holds tile row 8 s + 2 c + h, the row of forward accumulator register 4 s + h of
// thread column c.  Rows past the end of a ragged last tile are zero in the packed copy.
__device__ __forceinline__ int tc_pack_off_fwd(int r, int c) { return (c * (2 * TC_TR >> 3) + (r >> 3)) * 32 + (r & 7) * 4; }
__device__ __forceinline__ int tc_pack_off_bwd(int a, int n, int n0) { return (a * (2 * n0 >> 3) + (n >> 3)) * 32 + (n & 7) * 4; }
__device__ __forceinline__ int tc_kpos_fwd(int k) { return (k & ~15) + 8 * ((k >> 1) & 1) + ((k >> 2) & 3) + 4 * (k & 1); }
__device__ __forceinline__ int tc_row_bwd(int p) { return (p & ~7) + 2 * (p & 3) + ((p >> 2) & 1); }

__global__ void __launch_bounds__(256) mlp_pack_x_kernel(const MlpDev m, float* __restrict__ out) {
    const int n0 = m.n[0], tile_id = blockIdx.x;
    int r0, r_end;
    if (tile_id >= m.flat_base && m.flat_base >= m.tb[m.M]) {        // the all-rows tiling (only packed when it differs)
        r0 = TC_TR * (tile_id - m.flat_base); r_end = m.N;
    } else {
        int sp = 0;
        while (sp + 1 < m.M && tile_id >= m.tb[sp + 1]) ++sp;
        r0 = m.sb[sp] + TC_TR * (tile_id - m.tb[sp]); r_end = m.sb[sp + 1];
    }
    const int cnt = min(TC_TR, r_end - r0);
    float* fwd = out + (size_t)tile_id * (2 * 2 * TC_TR * n0);
    float* bwd = fwd + 2 * TC_TR * n0;
    for (int i = threadIdx.x; i < TC_TR * n0; i += blockDim.x) {
        const int r = i / n0, k = i - r * n0, p = tc_kpos_fwd(k);
        const float v = r < cnt ? m.x[(size_t)(r0 + r) * n0 + k] : 0.0f, h = tf32_rn(v);
        const int off = tc_pack_off_fwd(r, p >> 2) + (p & 3);
        fwd[off] = h;
        fwd[off + (TC_TR >> 3) * 32] = tf32_rn(v - h);
    }
    for (int i = threadIdx.x; i < TC_TR * n0; i += blockDim.x) {
        const int p = i / n0, n = i - p * n0, r = tc_row_bwd(p);
        const float v = r < cnt ? m.x[(size_t)(r0 + r) * n0 + n] : 0.0f, h = tf32_rn(v);
        const int off = tc_pack_off_bwd(p >> 2, n, n0) + (p & 3);
        bwd[off] = h;
        bwd[off + (n0 >> 3) * 32] = tf32_rn(v - h);
    }
}

// one bulk TMA copy per operand (thread 0; completion on the buffer's mbarrier)
__device__ __forceinline__ void tc_prefetch_fwd(const MlpDev& m, float* tile, const TcCtx& tc, int tile_id, int buf) {
    if (threadIdx.x == 0) {
        const uint32_t bytes = (uint32_t)(2 * TC_TR * m.n[0]) * 4u;
        mbar_expect_tx(tc.barF[buf], bytes);
        bulk_g2s(smem_u32(tile + (buf ? m.tc_f1 : m.tc_f0)), m.xp + (size_t)tile_id * (4 * TC_TR * m.n[0]), bytes, tc.barF[buf]);
    }
}
__device__ __forceinline__ void tc_prefetch_bwd(const MlpDev& m, float* tile, const TcCtx& tc, int tile_id) {
    if (threadIdx.x == 0) {
        const uint32_t bytes = (uint32_t)(2 * TC_TR * m.n[0]) * 4u;
        mbar_expect_tx(tc.barB, bytes);
        bulk_g2s(smem_u32(tile + m.tc_b), m.xp + (size_t)tile_id * (4 * TC_TR * m.n[0]) + 2 * TC_TR * m.n[0], bytes, tc.barB);
    }
}
// the tile's targets: 4-byte cp.async by warp 1 (waited for by the same warp at the top of tc_forward_tile)
__device__ __forceinline__ void tc_prefetch_y(const MlpDev& m, float* tile, int r0, int cnt) {
    if (threadIdx.x >= 32 && threadIdx.x < 64) {
        const int ycols = (m.loss == HMCX_LOSS_REGRESSION || m.loss == HMCX_LOSS_BINARY) ? m.n[2] : 1;
        const uint32_t yraw = smem_u32(tile + m.tc_yraw);
        for (int t = threadIdx.x - 32; t < cnt * ycols; t += 32)
            asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" :: "r"(yraw + 4u * (uint32_t)t), "l"(m.y + (size_t)r0 * ycols + t) : "memory");
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
}

// per-thread constants / accumulators of the register epilogues.  Accumulator register i = 4 j + 2 uu + b of a thread
// holds hidden unit u[uu] and tile row rbase + 8 j + b (hmcx_wgmma.cuh fragment layout, offset by the warpgroup's block)
struct TcEpi {
    int u[2], rbase, rh, grp;             // rh: the warpgroup's row half; grp: its 16-unit group (0..7)
    float b1u[2], w2[2][TC_NLMAX];
    float db1[2], dw2[2][TC_NLMAX], db2;
};
__device__ __forceinline__ void tc_epi_begin(const MlpDev& m, const float* q, TcEpi& e) {
    const int wg = threadIdx.x >> 7, wl = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
    e.u[0] = 64 * (wg & 1) + 16 * wl + (lane >> 2);
    e.u[1] = e.u[0] + 8;
    e.rh = wg >> 1;
    e.rbase = 32 * e.rh + 2 * (lane & 3);
    e.grp = 4 * (wg & 1) + wl;
#pragma unroll
    for (int uu = 0; uu < 2; ++uu) {
        e.b1u[uu] = q[m.boff[0] + e.u[uu]];
        e.db1[uu] = 0.0f;
#pragma unroll
        for (int j = 0; j < TC_NLMAX; ++j) {
            e.w2[uu][j] = j < m.n[2] ? q[m.woff[1] + j * TC_H + e.u[uu]] : 0.0f;
            e.dw2[uu][j] = 0.0f;
        }
    }
    e.db2 = 0.0f;
}

// bias + activation / activation derivative over a thread's 16 values, the activation kind resolved once
template <int A>
__device__ __forceinline__ void tc_act16_t(const float (&v)[16], const float (&b)[2], float (&act)[16]) {
#pragma unroll
    for (int i = 0; i < 16; ++i) act[i] = act_fwd(v[i] + b[(i >> 1) & 1], A);
}
__device__ __forceinline__ void tc_act16(const float (&v)[16], const float (&b)[2], float (&act)[16], int a) {
    if (a == HMCX_ACT_RELU) tc_act16_t<HMCX_ACT_RELU>(v, b, act);
    else if (a == HMCX_ACT_TANH) tc_act16_t<HMCX_ACT_TANH>(v, b, act);
    else if (a == HMCX_ACT_SIGMOID) tc_act16_t<HMCX_ACT_SIGMOID>(v, b, act);
    else tc_act16_t<HMCX_ACT_NONE>(v, b, act);
}
template <int A>
__device__ __forceinline__ void tc_dact16_t(const float (&act)[16], float (&d)[16]) {
#pragma unroll
    for (int i = 0; i < 16; ++i) d[i] = act_bwd(act[i], A);
}
__device__ __forceinline__ void tc_dact16(const float (&act)[16], float (&d)[16], int a) {
    if (a == HMCX_ACT_RELU) tc_dact16_t<HMCX_ACT_RELU>(act, d);
    else if (a == HMCX_ACT_TANH) tc_dact16_t<HMCX_ACT_TANH>(act, d);
    else if (a == HMCX_ACT_SIGMOID) tc_dact16_t<HMCX_ACT_SIGMOID>(act, d);
    else tc_dact16_t<HMCX_ACT_NONE>(act, d);
}

// H^T block of this warpgroup = W1 . X^T: per 16 input features one float4 of each of the thread's two W1 rows gives the
// A fragments of two k-steps; three wgmmas per k-step (W1_hi X_hi, W1_hi X_lo, W1_lo X_hi).  wgmma reads its register A
// operands asynchronously, so each group is waited for before the next 16 features overwrite those registers.
__device__ __forceinline__ void tc_mma_fwd(const MlpDev& m, const float* q, const TcEpi& e, uint32_t xop, float (&h)[16]) {
    constexpr uint32_t B_LBO = (2 * TC_TR / 8) * 128;
    const int n0 = m.n[0], c = threadIdx.x & 3;
    const float* w0 = q + m.woff[0] + e.u[0] * n0 + 4 * c;
    const float* w1 = q + m.woff[0] + e.u[1] * n0 + 4 * c;
    xop += 512u * (uint32_t)e.rh;                         // this warpgroup's 32 rows = 4 of the operand's 8-row groups
#pragma unroll
    for (int i = 0; i < 16; ++i) h[i] = 0.0f;
    for (int t = 0; t < (n0 >> 4); ++t) {
        const float4 x0 = *reinterpret_cast<const float4*>(w0 + 16 * t), x1 = *reinterpret_cast<const float4*>(w1 + 16 * t);
        uint32_t ah0[4], al0[4], ah1[4], al1[4];
        tc_split({x0.x, x1.x, x0.y, x1.y}, ah0, al0);
        tc_split({x0.z, x1.z, x0.w, x1.w}, ah1, al1);
        const uint32_t b0 = xop + (uint32_t)(2 * t) * 2u * B_LBO, b1 = b0 + 2u * B_LBO;
        wgmma_fence();
        wgmma_tf32_rs<32>(h, ah0, make_kmajor_desc(b0, B_LBO, 128));
        wgmma_tf32_rs<32>(h, ah0, make_kmajor_desc(b0 + 1024u, B_LBO, 128));
        wgmma_tf32_rs<32>(h, al0, make_kmajor_desc(b0, B_LBO, 128));
        wgmma_tf32_rs<32>(h, ah1, make_kmajor_desc(b1, B_LBO, 128));
        wgmma_tf32_rs<32>(h, ah1, make_kmajor_desc(b1 + 1024u, B_LBO, 128));
        wgmma_tf32_rs<32>(h, al1, make_kmajor_desc(b1, B_LBO, 128));
        wgmma_commit();
        wgmma_wait<0>();
    }
}

// dW1 block (+)= dH^T . X over this warpgroup's 32 rows: the A fragment of k-step j is accumulator registers
// 4j, 4j+2, 4j+1, 4j+3 (tc_row_bwd); N = n0
template <int N0>
__device__ __forceinline__ void tc_mma_bwd_n(float (&dw)[32], const uint32_t (&hi)[16], const uint32_t (&lo)[16], uint32_t xb,
                                             int rh) {
    constexpr uint32_t B_LBO = (uint32_t)(2 * N0 / 8) * 128, LO = (uint32_t)(N0 / 8) * 128;
    float (&d)[N0 / 2] = *reinterpret_cast<float (*)[N0 / 2]>(&dw[0]);
    uint32_t ah[4][4], al[4][4];                 // every A fragment is written before the fence that precedes the wgmmas
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        ah[j][0] = hi[4 * j]; ah[j][1] = hi[4 * j + 2]; ah[j][2] = hi[4 * j + 1]; ah[j][3] = hi[4 * j + 3];
        al[j][0] = lo[4 * j]; al[j][1] = lo[4 * j + 2]; al[j][2] = lo[4 * j + 1]; al[j][3] = lo[4 * j + 3];
    }
    wgmma_fence();
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const uint32_t b = xb + (uint32_t)(4 * rh + j) * 2u * B_LBO;
        wgmma_tf32_rs<N0>(d, ah[j], make_kmajor_desc(b, B_LBO, 128));
        wgmma_tf32_rs<N0>(d, ah[j], make_kmajor_desc(b + LO, B_LBO, 128));
        wgmma_tf32_rs<N0>(d, al[j], make_kmajor_desc(b, B_LBO, 128));
    }
    wgmma_commit();
    wgmma_wait<0>();
}
__device__ __forceinline__ void tc_mma_bwd(int n0, float (&dw)[32], const uint32_t (&hi)[16], const uint32_t (&lo)[16],
                                           uint32_t xb, int rh) {
    if (n0 == 16) tc_mma_bwd_n<16>(dw, hi, lo, xb, rh);
    else if (n0 == 32) tc_mma_bwd_n<32>(dw, hi, lo, xb, rh);
    else if (n0 == 48) tc_mma_bwd_n<48>(dw, hi, lo, xb, rh);
    else tc_mma_bwd_n<64>(dw, hi, lo, xb, rh);
}

// forward of one (prefetched) tile up to the network outputs: out[r * nL + j] (the loss stage's layout); the hidden
// activations of this thread's (2 units, 8 rows) block stay in `act`.  Ends with every thread past a __syncthreads.
__device__ __forceinline__ void tc_forward_tile(const MlpDev& m, const float* q, float* tile, TcCtx& tc, const TcEpi& e,
                                                float (&act)[16], int buf) {
    const int nL = m.n[2], lane = threadIdx.x & 31;
    if (threadIdx.x >= 32 && threadIdx.x < 64) asm volatile("cp.async.wait_group 0;" ::: "memory");    // the targets
    mbar_wait(tc.barF[buf], tc.parF[buf]);                        // this tile's forward operand has landed
    tc.parF[buf] ^= 1;
    TC_MARK(3);
    float h[16];
    tc_mma_fwd(m, q, e, smem_u32(tile + (buf ? m.tc_f1 : m.tc_f0)), h);
    TC_MARK(5);
    tc_act16(h, e.b1u, act, m.act[0]);
    float* part = tile + m.tc_part;
#pragma unroll
    for (int j = 0; j < TC_NLMAX; ++j) {
        if (j < nL) {
            float t[8];                                           // rows rbase + 8 (k >> 1) + (k & 1), summed over 2 units
#pragma unroll
            for (int k = 0; k < 8; ++k) t[k] = e.w2[0][j] * act[4 * (k >> 1) + (k & 1)] + e.w2[1][j] * act[4 * (k >> 1) + 2 + (k & 1)];
#pragma unroll
            for (int k = 0; k < 8; ++k) {                         // ... and over the 8 lanes of the same column
                t[k] += __shfl_xor_sync(0xffffffffu, t[k], 4);
                t[k] += __shfl_xor_sync(0xffffffffu, t[k], 8);
                t[k] += __shfl_xor_sync(0xffffffffu, t[k], 16);
            }
            if (lane < 4) {
#pragma unroll
                for (int k = 0; k < 8; ++k) part[(e.grp * TC_TR + e.rbase + 8 * (k >> 1) + (k & 1)) * TC_NLMAX + j] = t[k];
            }
        }
    }
    __syncthreads();
    TC_MARK(6);
    float* out = tile + m.aoff[2];
    for (int i = threadIdx.x; i < TC_TR * nL; i += MLP_THREADS) {
        const int r = i / nL, j = i - r * nL;
        float s = part[r * TC_NLMAX + j];
        for (int g = 1; g < 8; ++g) s += part[(g * TC_TR + r) * TC_NLMAX + j];
        out[i] = s + q[m.boff[1] + j];
    }
    __syncthreads();
    TC_MARK(7);
}

// g += d ll_split / dq over this rank's 64-row tiles of [r_begin, r_end)
__device__ __forceinline__ void tc_backprop_rows(const MlpDev& m, const float* q, float* g, float* tile, TcCtx& tc,
                                                 int r_begin, int r_end, int tile0, ClusterCtx cc, int next_s = -2) {
    const int nL = m.n[2], n0 = m.n[0], lane = threadIdx.x & 31;
    TcEpi e;
    tc_epi_begin(m, q, e);
    float* out = tile + m.aoff[2];
    float* dz = tile + m.dzoff[0];
    const float* ytile = tile + m.tc_yraw;
    const int stride = TC_TR * cc.size;
    float dw[32];                                                 // this warpgroup's dW1 block (first n0 / 2 registers)
#pragma unroll
    for (int i = 0; i < 32; ++i) dw[i] = 0.0f;
    int done = 0;
    int r0 = r_begin + TC_TR * cc.rank;                           // this rank's tiles: rank, rank + size, ...
    int id = tile0 + cc.rank;                                     // ... and their packed operands
    if (r0 < r_end && tc.pre_id != id) {                          // (else: the previous evaluation already fetched them)
        tc_prefetch_fwd(m, tile, tc, id, 0);
        tc_prefetch_bwd(m, tile, tc, id);
        tc_prefetch_y(m, tile, r0, min(TC_TR, r_end - r0));
    }
    tc.pre_id = -1;
    for (; r0 < r_end; r0 += stride, id += cc.size) {
        const int cnt = min(TC_TR, r_end - r0), buf = done & 1;
        const bool has_next = r0 + stride < r_end;
        if (has_next) tc_prefetch_fwd(m, tile, tc, id + cc.size, buf ^ 1);   // last read by the forward MMA of tile t-1: complete
        float act[16];
        tc_forward_tile(m, q, tile, tc, e, act, buf);
        mlp_loss_tile(m, out, dz, r0, cnt, r_end - r_begin, false, ytile);
        __syncthreads();
        TC_MARK(8);
        if (has_next) tc_prefetch_y(m, tile, r0 + stride, min(TC_TR, r_end - r0 - stride));   // the target buffer is free
        if (threadIdx.x < TC_TR * nL) e.db2 += dz[threadIdx.x];   // element (r, j) of every tile; reduced over r at the end
        float dact[16];
        tc_dact16(act, dact, m.act[0]);
        uint32_t hi[16], lo[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const int r = e.rbase + 8 * (i >> 2) + (i & 1), uu = (i >> 1) & 1;
            float da = 0.0f;
#pragma unroll
            for (int j = 0; j < TC_NLMAX; ++j) {
                if (j < nL) {
                    const float d = dz[r * nL + j];
                    da = fmaf(d, e.w2[uu][j], da);
                    e.dw2[uu][j] = fmaf(d, act[i], e.dw2[uu][j]);
                }
            }
            const float dh = da * dact[i];
            e.db1[uu] += dh;
            const float h = tf32_rn(dh);
            hi[i] = __float_as_uint(h);
            lo[i] = __float_as_uint(tf32_rn(dh - h));
        }
        TC_MARK(10);
        mbar_wait(tc.barB, tc.parB);                              // the backward operand has landed (long ago)
        tc.parB ^= 1;
        tc_mma_bwd(n0, dw, hi, lo, smem_u32(tile + m.tc_b), e.rh);
        ++done;
        TC_MARK(11);
        __syncthreads();                                          // every warpgroup is done with the backward operand
        if (has_next) tc_prefetch_bwd(m, tile, tc, id + cc.size);
        TC_MARK(12);
    }
    if (done == 0) return;                                        // (uniform over the CTA)
    // The first tile of the NEXT evaluation (the schedule knows its split): its operands do not depend on q, so they are
    // requested now and land while this evaluation finishes (dW1 read-out, reductions, cluster sum, kick, drift).
    int nid = -1;
    if (next_s > -2) {
        const int nb = next_s < 0 ? 0 : m.sb[next_s], ne = next_s < 0 ? m.N : m.sb[next_s + 1];
        const int nr0 = nb + TC_TR * cc.rank;
        if (nr0 < ne) {
            nid = (next_s < 0 ? m.flat_base : m.tb[next_s]) + cc.rank;
            tc_prefetch_fwd(m, tile, tc, nid, 0);                 // every forward MMA of this evaluation has completed
            tc_prefetch_y(m, tile, nr0, min(TC_TR, ne - nr0));    // the last loss stage is over
        }
    }
    // ---- dW1: the two row halves' blocks -> padded staging (first half stores, second half adds) -> g
    float* stg = tile + m.tc_f1;                 // forward buffer 1 | backward buffer (adjacent, both idle now)
    const int pitch = n0 + 4;
    for (int half = 0; half < 2; ++half) {
        if (e.rh == half) {
#pragma unroll
            for (int i = 0; i < 32; i += 2) {
                if (i < n0 / 2) {
                    float2* s2 = reinterpret_cast<float2*>(stg + e.u[(i >> 1) & 1] * pitch + 8 * (i >> 2) + 2 * (lane & 3));
                    float2 v = make_float2(dw[i], dw[i + 1]);
                    if (half) { const float2 o = *s2; v.x = o.x + v.x; v.y = o.y + v.y; }
                    *s2 = v;
                }
            }
        }
        __syncthreads();
    }
    float* gW = g + m.woff[0];
    for (int i4 = threadIdx.x; i4 < TC_H * n0 / 4; i4 += MLP_THREADS) {
        const int u = (4 * i4) / n0, k = 4 * i4 - u * n0;
        const float4 d = *reinterpret_cast<const float4*>(stg + u * pitch + k);
        float4 a = *reinterpret_cast<float4*>(gW + 4 * i4);
        a.x += d.x; a.y += d.y; a.z += d.z; a.w += d.w;
        *reinterpret_cast<float4*>(gW + 4 * i4) = a;
    }
    // ---- db1, dW2: summed over the 4 lanes that share a unit, then two per-unit partials (one per row half) in a fixed
    // order; db2
    float* red = tile + m.tc_part;
#pragma unroll
    for (int uu = 0; uu < 2; ++uu) {
        float v = e.db1[uu];
        v += __shfl_xor_sync(0xffffffffu, v, 1);
        v += __shfl_xor_sync(0xffffffffu, v, 2);
        if ((lane & 3) == 0) red[(e.rh * TC_H + e.u[uu]) * (1 + TC_NLMAX)] = v;
#pragma unroll
        for (int j = 0; j < TC_NLMAX; ++j) {
            float w = e.dw2[uu][j];
            w += __shfl_xor_sync(0xffffffffu, w, 1);
            w += __shfl_xor_sync(0xffffffffu, w, 2);
            if ((lane & 3) == 0) red[(e.rh * TC_H + e.u[uu]) * (1 + TC_NLMAX) + 1 + j] = w;
        }
    }
    fence_async_smem();                                           // the staging reads above precede the TMA write below
    __syncthreads();
    if (nid >= 0) { tc_prefetch_bwd(m, tile, tc, nid); tc.pre_id = nid; }
    if (threadIdx.x < TC_H) {
        const int u = threadIdx.x;
        auto tot = [&](int f) { return red[u * (1 + TC_NLMAX) + f] + red[(TC_H + u) * (1 + TC_NLMAX) + f]; };
        g[m.boff[0] + u] += tot(0);
        for (int j = 0; j < nL; ++j) g[m.woff[1] + j * TC_H + u] += tot(1 + j);
    }
    __syncthreads();
    if (threadIdx.x < TC_TR * nL) red[threadIdx.x] = e.db2;       // db2[j] = sum over rows r of the per-(r, j) sums
    __syncthreads();
    if (threadIdx.x < 32) {
        for (int j = 0; j < nL; ++j) {
            const float sj = warp_sum(red[threadIdx.x * nL + j] + red[(threadIdx.x + 32) * nL + j]);
            if (threadIdx.x == 0) g[m.boff[1] + j] += sj;
        }
    }
    __syncthreads();
    TC_MARK(13);
}

// g += d ll_split / dq over this rank's tiles of the rows [r_begin, r_end)  (g must already hold the prior part / zeros)
__device__ __forceinline__ void mlp_backprop_rows(const MlpDev& m, const float* q, float* g, float* tile, int r_begin,
                                                  int r_end, ClusterCtx cc) {
    int ti = 0;
    for (int r0 = r_begin; r0 < r_end; r0 += m.T, ++ti) {
        if (ti % cc.size != cc.rank) continue;
        const int cnt = min(m.T, r_end - r0);
        mlp_forward_tile(m, q, tile, r0, cnt);
        float* dz = tile + m.dzoff[m.L & 1];
        mlp_loss_tile(m, tile + m.aoff[m.L], dz, r0, cnt, r_end - r_begin);
        __syncthreads();
        for (int l = m.L - 1; l >= 0; --l) {
            float* dz_prev = tile + m.dzoff[l & 1];
            mlp_weight_grad(tile + m.aoff[l], dz, g + m.woff[l], g + m.boff[l], m.n[l], m.n[l + 1], m.T);
            if (l > 0)
                mlp_input_grad(dz, q + m.woff[l], tile + m.aoff[l], dz_prev, m.n[l], m.n[l + 1], m.act[l - 1], m.T);
            __syncthreads();
            dz = dz_prev;
        }
    }
}

// prior part of the gradient: d(prior/prior_scale)/dw = -(coef_i * (2w))   (pow/div backward order, DESIGN.md 3.4)
__device__ __forceinline__ void mlp_prior_grad(const MlpDev& m, const float* q, float* g) {
    for (int l = 0; l < m.L; ++l) {
        const int nw = m.n[l] * m.n[l + 1];
        const float cw = m.gcoef[2 * l], cb = m.gcoef[2 * l + 1];
        if (((m.woff[l] | nw) & 3) == 0) {                         // 16-byte aligned tensor: four weights per access
            const float4* q4 = reinterpret_cast<const float4*>(q + m.woff[l]);
            float4* g4 = reinterpret_cast<float4*>(g + m.woff[l]);
            for (int i = threadIdx.x; i < (nw >> 2); i += MLP_THREADS) {
                const float4 w = q4[i];
                g4[i] = make_float4(-mul(cw, mul(2.0f, w.x)), -mul(cw, mul(2.0f, w.y)), -mul(cw, mul(2.0f, w.z)),
                                    -mul(cw, mul(2.0f, w.w)));
            }
        } else {
            for (int i = threadIdx.x; i < nw; i += MLP_THREADS) g[m.woff[l] + i] = -mul(cw, mul(2.0f, q[m.woff[l] + i]));
        }
        for (int i = threadIdx.x; i < m.n[l + 1]; i += MLP_THREADS)
            g[m.boff[l] + i] = -mul(cb, mul(2.0f, q[m.boff[l] + i]));
    }
}

// g = d log p_split / dq for split s (s < 0: all rows as one potential)
template <int CS>
__device__ __forceinline__ void mlp_grad_split(const MlpDev& m, const float* q, float* g, float* tile, int s,
                                               ClusterCtx cc, TcCtx& tc, bool leave_partials = false, int next_s = -2) {
    TC_MARK(1);
    if (cc.rank == 0) mlp_prior_grad(m, q, g);                 // the prior part enters the rank-ordered sum once
    else for (int i = threadIdx.x; i < m.Dp; i += MLP_THREADS) g[i] = 0.0f;
    if (m.tc) fence_async_smem();                              // (generic accesses of the operand buffers precede the TMA writes)
    __syncthreads();
    TC_MARK(2);
    if (m.has_data) {
        const int rb = s < 0 ? 0 : m.sb[s], re = s < 0 ? m.N : m.sb[s + 1];
        if (m.tc) tc_backprop_rows(m, q, g, tile, tc, rb, re, s < 0 ? m.flat_base : m.tb[s], cc, next_s);
        else mlp_backprop_rows(m, q, g, tile, rb, re, cc);
        TC_MARK(14);
        // leave_partials: the caller's kick adds the ranks' partial gradients itself (one DSMEM pass instead of reduce +
        // write back + kick); all it needs here is that every rank's partial is complete
        if (!leave_partials) cluster_sum_vector<CS>(g, m.D);
        else if (CS > 1) cg::this_cluster().sync();
        TC_MARK(15);
    }
}

// l_prior = sum_i Normal(0, scale_i).log_prob(w_i).sum(), accumulated tensor by tensor (samplers.py:1153-1157)
__device__ __forceinline__ float mlp_log_prior(const MlpDev& m, const float* q, float* sred) {
    float l_prior = 0.0f;
    for (int t = 0; t < 2 * m.L; ++t) {
        const int l = t >> 1;
        const int off = (t & 1) ? m.boff[l] : m.woff[l];
        const int cnt = (t & 1) ? m.n[l + 1] : m.n[l] * m.n[l + 1];
        float s[1] = {0.0f};
        for (int i = threadIdx.x; i < cnt; i += MLP_THREADS) {
            const float w = q[off + i];
            // -((w - 0)**2) / (2*var) - log_scale - log(sqrt(2*pi))
            const float v = sub(sub(__fdiv_rn(-mul(w, w), m.two_var[t]), m.log_scale[t]), 0.9189385332046727f);
            s[0] = add(s[0], v);
        }
        block_sum<1>(s, sred);
        __syncthreads();
        l_prior = add(s[0], l_prior);
    }
    return l_prior;
}

// log p(q) = sum over splits of (ll_m + l_prior/prior_scale)  (hamiltonian's split loop, samplers.py:787-796);
// with s >= 0 only that split.  Optionally writes the network outputs (predict_model) and, to every thread's *lsum_out,
// the sum over splits of ll_m / c_ll added in fp64 in split order: the untempered log-likelihood over c_ll, and for
// regression the SSE the tau_out Gibbs step needs.
template <int CS>
__device__ __forceinline__ float mlp_log_prob(const MlpDev& m, const float* q, float* tile, float* sred, int s,
                                              float* pred_out, ClusterCtx cc, float* xslot, TcCtx& tc,
                                              double* lsum_out = nullptr) {
    const float prior_term = __fdiv_rn(mlp_log_prior(m, q, sred), m.prior_scale);
    if (lsum_out) *lsum_out = 0.0;
    if (!m.has_data) return prior_term;
    TcEpi te;
    if (m.tc) {
        tc_epi_begin(m, q, te);
        fence_async_smem();
        __syncthreads();
    }
    float lp = 0.0f;
    const int s0 = s < 0 ? 0 : s, s1 = s < 0 ? m.M : s + 1;
    for (int sp = s0; sp < s1; ++sp) {
        float sse[1] = {0.0f};
        int ti = 0;
        for (int r0 = m.sb[sp]; r0 < m.sb[sp + 1]; r0 += m.T, ++ti) {
            if (ti % cc.size != cc.rank) continue;
            const int cnt = min(m.T, m.sb[sp + 1] - r0);
            if (m.tc) {
                float act[16];
                tc_prefetch_fwd(m, tile, tc, m.tb[sp] + ti, 0);
                tc_prefetch_y(m, tile, r0, cnt);
                tc_forward_tile(m, q, tile, tc, te, act, 0);
            } else {
                mlp_forward_tile(m, q, tile, r0, cnt);
            }
            sse[0] = add(sse[0], mlp_loss_tile(m, tile + m.aoff[m.L], nullptr, r0, cnt, m.sb[sp + 1] - m.sb[sp],
                                               pred_out != nullptr && m.loss == HMCX_LOSS_MULTICLASS_LOGSOFTMAX,
                                               m.tc ? tile + m.tc_yraw : nullptr));
            if (pred_out) {
                __syncthreads();
                const int nL = m.n[m.L];
                for (int i = threadIdx.x; i < cnt * nL; i += MLP_THREADS)
                    pred_out[(size_t)r0 * nL + i] = tile[m.aoff[m.L] + i];
            }
            __syncthreads();
        }
        block_sum<1>(sse, sred);
        __syncthreads();
        sse[0] = cluster_sum_scalar<CS>(sse[0], xslot);
        // (the log-softmax loss is a per-split mean)
        if (lsum_out)
            *lsum_out += m.loss == HMCX_LOSS_MULTICLASS_LOGSOFTMAX ? (double)sse[0] / (double)(m.sb[sp + 1] - m.sb[sp])
                                                                   : (double)sse[0];
        const float ll = mlp_ll_from_sum(m, sse[0], m.sb[sp + 1] - m.sb[sp]);
        lp = (sp == s0) ? add(ll, prior_term) : add(lp, add(ll, prior_term));
    }
    return lp;
}

// ---------------------------------------------------------------------------------------------------------
// persistent sample() kernel for the BNN path
// ---------------------------------------------------------------------------------------------------------
constexpr int HYPER_GROUPS = 2 * HMCX_MLP_MAX_LAYERS + 1;     // the parameter tensors, then tau_out

// Gamma hyperpriors on the precisions (hmcx_hyper_t), read by the PER_CHAIN instantiations only (tau == NULL: none).
// Group k < 2L is parameter tensor k (tau_list order), group 2L the regression likelihood's tau_out.
struct MlpHyperDev {
    int sampled;                  // bit k: group k is Gibbs-updated
    double a[HYPER_GROUPS], b[HYPER_GROUPS];
    double n_obs;                 // N * O, the Gaussian likelihood's observation count
    float* tau;                   // [C, 2L] in/out
    float* tau_out;               // [C] in/out
    float* tau_trace;             // [C, keep, 2L] or NULL
    float* tau_out_trace;         // [C, keep] or NULL
    const double* gammas;         // INJECTED: standard-gamma draws [it1 - it0, C, 2L + 1]
};

// A PER_CHAIN kernel reads the model descriptor from a shared-memory copy whose constants are the chain's own: the prior
// constants and c_ll of its current precisions, or its rung's tau_out and c_ll (the constant bank holds the launch-wide
// ones).
struct ChainModelSm {
    MlpDev m;
    double red[MLP_THREADS / 32];
    double ssq[2 * HMCX_MLP_MAX_LAYERS];
    float tau[2 * HMCX_MLP_MAX_LAYERS];
    float tau_out;
};
__device__ __forceinline__ ChainModelSm& chain_model_sm() {
    __shared__ ChainModelSm s;
    return s;
}
// Replica exchange (hmcx_temper_t), read by the PER_CHAIN instantiations only: row c runs rung c % T, whose likelihood
// precision tau_out[c % T] replaces the target's (the power posterior at beta_t, DESIGN.md 3.17)
struct MlpTemperDev {
    int T;                        // 0: no replica exchange
    float tau_out[HMCX_TEMPER_MAX_TEMPS];
    double* ll_out;               // [C] or NULL: the untempered log-likelihood at q_cur when the launch ends
};

// The prior constants of the sampled tensors and c_ll from the precisions, in fp32 with the host's operation order
// (targets.MLPTarget.__init__: scale = tau ** -0.5, two_var = 2 * scale ** 2, log_scale = log(scale),
// grad_coef = (1 / prior_scale) / two_var; c_ll = fp32(-0.5 * tau_out)).  Unsampled groups keep the host's constants.
__device__ __forceinline__ void hyper_constants(MlpDev& m, const float* tau, float tau_out, int sampled) {
    for (int t = 0; t < 2 * m.L; ++t) {
        if (!((sampled >> t) & 1)) continue;
        const float sc = __fdiv_rn(1.0f, __fsqrt_rn(tau[t]));
        const float tv = mul(2.0f, mul(sc, sc));
        m.two_var[t] = tv;
        m.log_scale[t] = logf(sc);
        m.gcoef[t] = __fdiv_rn(__fdiv_rn(1.0f, m.prior_scale), tv);
    }
    if ((sampled >> (2 * m.L)) & 1) {
        m.tau_out = tau_out;
        m.c_ll = (float)(-0.5 * (double)tau_out);
    }
}

// sum over the CTA in fp64, in a fixed order (xor butterflies, then the warps in order): every thread returns the same bits
__device__ __forceinline__ double block_sum_d(double v, double* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double s = 0.0;
    for (int w = 0; w < MLP_THREADS / 32; ++w) s += red[w];
    __syncthreads();
    return s;
}

struct MlpRunArgs {
    MlpDev m;
    int scheme, mk, C, ld;
    const float* im;
    const float* sd;
    int rng_mode;
    uint64_t seed, chain_offset;
    const float* normals;
    const float* logu;
    const int32_t* perms;
    int nuts;
    double delta, mu;
    const double* table;
    double* h_bar;
    double* eps_bar;
    const float* eps_schedule;
    double eps0;                  // hmcx_nuts_t.step_size_init (0 = not given)
    float* eps_trace;
    const float* q_init;
    float* q_cur;
    float* eps;
    int L, S, burn, it0, it1;
    float* samples;
    uint8_t* accept;
    uint8_t* diverged;
    float* ham;
    int32_t* num_rejected;
    // stand-alone samplers.leapfrog with a SPLITTING integrator (:494-603): the momentum is given, the trajectory recorded
    const float* p_given;         // [C, ld] or NULL
    float* q_traj;                // [L, C, ld]: params after every step (ret_params)
    float* p_traj;                // [L, C, ld]: momentum after every step (ret_momenta)
    // sample sink (hmcx_sink_t; {thin = 1} when the caller gives none): thinning + running moments of the post-burn states
    int thin;
    float* msum;
    float* msumsq;
    float* msum_lo;               // optional compensation terms (true sum = hi + lo)
    float* msumsq_lo;
    // mass adaptation (ABI v11): moments over every iteration of the launch; per-chain mu (may be null)
    int moments_all;
    const double* mu_chain;
    MlpHyperDev hy;               // PER_CHAIN instantiations only
    MlpTemperDev tp;              // PER_CHAIN instantiations only
    int folds;                    // K-fold (PLAIN only, 0 = off): global chain g's whole potential is split g % folds
};

// One sink accumulator [C, ld] (sum, or sum of squares when `squares`) += the float4 x at element offset `off`, read and
// written in place: the chain state fills shared memory, so the running sums stay in the caller's arrays (in L2 at the
// sizes this kernel runs).  Without a compensation array the term is folded into the sum every time, i.e. the sum is a
// plain fp32 running sum.
__device__ __forceinline__ void sink_accumulate(float* hi, float* lo, size_t off, float4 x, bool squares) {
    float4 s = *reinterpret_cast<const float4*>(hi + off);
    float4 e = lo ? *reinterpret_cast<const float4*>(lo + off) : make_float4(0.f, 0.f, 0.f, 0.f);
    float* sp = &s.x;
    float* ep = &e.x;
    const float* xp = &x.x;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        if (squares) {
            const float xx = mul(xp[j], xp[j]);
            comp_add(sp[j], ep[j], xx);
            ep[j] = add(ep[j], fmaf(xp[j], xp[j], -xx));      // the rounding error of x*x itself (exact)
        } else {
            comp_add(sp[j], ep[j], xp[j]);
        }
    }
    if (lo) *reinterpret_cast<float4*>(lo + off) = e;
    else s = make_float4(add(s.x, e.x), add(s.y, e.y), add(s.z, e.z), add(s.w, e.w));
    *reinterpret_cast<float4*>(hi + off) = s;
}

// The sample() loop with the sample sink, its row work divided over the cluster's ranks (see sink_row below).  PER_CHAIN:
// the chain's model constants live in a shared-memory copy of the descriptor, which the launch's settings fill.
// Hyperpriors (a.hy.tau != NULL) add the Gibbs updates of the Gamma hyperpriors on the precisions after every MH step
// (DESIGN.md 3.15).  Replica exchange (a.tp.T > 0) runs row c at rung c % T of a ladder: its descriptor copy carries the
// rung's tau_out, it tracks the untempered log-likelihood at q_cur, and only rung 0 (beta = 1) rows store samples, to row
// c / T of samples_out (DESIGN.md 3.17).  Both are tested once per launch or per iteration, never inside the trajectory.
template <int CS, bool PER_CHAIN>
__global__ void __launch_bounds__(MLP_THREADS, 1) mlp_run_kernel(const MlpRunArgs a) {
    extern __shared__ __align__(128) float sm[];
    __shared__ float sred[64];
    __shared__ float s_bcast[4];
    __shared__ float s_xchg;
    __shared__ int s_perm[HMCX_MLP_MAX_SPLITS];
    __shared__ __align__(8) uint64_t s_bars[3];

    const bool hyper = PER_CHAIN && a.hy.tau, temper = PER_CHAIN && a.tp.T > 0;
    if constexpr (PER_CHAIN) {
        ChainModelSm& cm = chain_model_sm();
        if (threadIdx.x == 0) {
            const int c0 = blockIdx.x / CS, K = 2 * a.m.L;
            cm.m = a.m;
            if (hyper) {                                       // this chain's precisions and the constants they give
                for (int k = 0; k < K; ++k) cm.tau[k] = a.hy.tau[(size_t)c0 * K + k];
                cm.tau_out = a.hy.tau_out[c0];
                hyper_constants(cm.m, cm.tau, cm.tau_out, a.hy.sampled);
            }
            if (temper) {                                      // the rung's tau_out and c_ll, as fill_mlp derives them
                const float tau = a.tp.tau_out[c0 % a.tp.T];
                cm.m.tau_out = tau;
                cm.m.c_ll = (a.m.loss == HMCX_LOSS_REGRESSION) ? (float)(-0.5 * (double)tau) : (float)(-(double)tau);
            }
        }
        __syncthreads();
    }
    const MlpDev& m = PER_CHAIN ? chain_model_sm().m : a.m;
    ClusterCtx cc = {0, 1};
    if (CS > 1) { cc.rank = (int)cg::this_cluster().block_rank(); cc.size = CS; }
    const bool lead = cc.rank == 0;                            // rank 0 owns every global-memory output but the sink rows
    const int c = blockIdx.x / CS, tid = threadIdx.x, D = m.D, M = m.M;
    float* q = sm;
    float* p = q + m.Dp;
    float* g = p + m.Dp;
    float* tile = sm + m.tile_base;
    const size_t row = (size_t)c * a.ld;
    const uint64_t chain_id = a.chain_offset + (uint64_t)c;
    // the data split that is this chain's whole PLAIN potential: -1 (every split) unless a K-fold run gives the chain
    // fold k = g mod K's training rows, split k (DESIGN.md 3.18).  The host refuses folds with hyperpriors or tempering:
    // the PER_CHAIN form keeps a constant -1 (one more live value there raises its spills).
    const int psp = (!PER_CHAIN && a.folds) ? (int)(chain_id % (uint64_t)a.folds) : -1;
    TcCtx tc = {};
    if (m.tc) tc_init(tc, s_bars);

    for (int i = tid; i < m.Dp; i += MLP_THREADS) { q[i] = i < D ? a.q_cur[row + i] : 0.0f; p[i] = 0.0f; g[i] = 0.0f; }
    __syncthreads();
    double ls_cur = 0.0, ls_new = 0.0;                        // PER_CHAIN: log-likelihood / c_ll at q_cur / the proposal
    float lp_cur = a.p_given ? 0.0f : mlp_log_prob<CS>(m, q, tile, sred, psp, nullptr, cc, &s_xchg, tc,
                                                       PER_CHAIN ? &ls_cur : nullptr);

    float eps = a.eps[c];
    double h_bar = 0.0, eps_bar = 1.0;
    if (a.nuts && tid == 0) { h_bar = a.h_bar[c]; eps_bar = a.eps_bar[c]; }
    double mu_sink = 0.0;                                      // this chain's mu (the restarted dual averaging's)
    if (a.nuts && tid == 0) mu_sink = a.mu_chain ? a.mu_chain[c] : a.mu;
    int rejected = 0;
    const int keep = 1 + (a.S - a.burn - 1) / a.thin;                      // slots per chain in samples_out
    float* const my_samples = temper ? ((a.samples && c % a.tp.T == 0) ? a.samples + (size_t)(c / a.tp.T) * keep * a.ld
                                                                       : nullptr)
                                     : (a.samples ? a.samples + (size_t)c * keep * a.ld : nullptr);
    // Sink: rank r owns the float4 vectors [sv0, sv1) of the row -- their thinned stores (16-byte streaming stores, which is
    // what lets rows leave over PCIe when samples_out is pinned host memory) and their moment updates.  Every rank holds a
    // bit-identical replica of q, so this needs no DSMEM traffic and no barrier beyond the loop's own.
    const int sv_rank = ((a.ld >> 2) + CS - 1) / CS;
    const int sv0 = cc.rank * sv_rank, sv1 = min(a.ld >> 2, sv0 + sv_rank);
    auto sink_row = [&](float* dst, bool moments) {
        const float4* q4 = reinterpret_cast<const float4*>(q);
        for (int v = sv0 + tid; v < sv1; v += MLP_THREADS) {
            const float4 x = 4 * v < m.Dp ? q4[v] : make_float4(0.f, 0.f, 0.f, 0.f);   // q's padding lanes are zero
            if (dst) __stcs(reinterpret_cast<float4*>(dst) + v, x);
            if (moments && a.msum) sink_accumulate(a.msum, a.msum_lo, row + 4 * v, x, false);
            if (moments && a.msumsq) sink_accumulate(a.msumsq, a.msumsq_lo, row + 4 * v, x, true);
        }
    };
    if (a.it0 == 0 && my_samples) sink_row(my_samples, false);
    // hyperpriors: the precisions of retained slot j (the slots of samples_out, thinned alike); slot 0 = the initial values
    auto hyper_store = [&](int slot) {
        if (tid == 0 && lead) {
            const ChainModelSm& cm = chain_model_sm();
            const int K = 2 * m.L;
            if (a.hy.tau_trace)
                for (int k = 0; k < K; ++k) a.hy.tau_trace[((size_t)c * keep + slot) * K + k] = cm.tau[k];
            if (a.hy.tau_out_trace) a.hy.tau_out_trace[(size_t)c * keep + slot] = cm.tau_out;
        }
    };
    if (hyper && a.it0 == 0) hyper_store(0);

    auto kinetic = [&]() {                                    // 2*K: p.p or p.(im*p)   (samplers.py:801, :814)
        float s[1] = {0.0f};
        for (int i = tid; i < D; i += MLP_THREADS)
            s[0] = add(s[0], a.mk == HMCX_MASS_DIAG ? mul(p[i], mul(a.im[i], p[i])) : mul(p[i], p[i]));
        block_sum<1>(s, sred);
        __syncthreads();
        return s[0];
    };
    // element-wise passes over the state: 16-byte accesses, VPT independent vectors per thread in flight (the inverse-mass
    // read of a drift comes from L2 and the partial gradients of a fused kick from a peer SM: latency-bound otherwise).
    // The padding lanes [D, Dp) of q / p / g are zero and stay zero (inv_mass lanes past D are read as 0).
    constexpr int VPT = 5;                                     // Dp/4 <= 512 * 5 vectors covers D <= 10240 in one round
    const int nvec = m.Dp >> 2;
    const bool im_aligned = (reinterpret_cast<size_t>(a.im) & 15) == 0;
    auto ld_im4 = [&](int v) {
        const int i = 4 * v;
        if (i + 3 < D && im_aligned) return __ldg(reinterpret_cast<const float4*>(a.im) + v);
        float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
        if (i < D) r.x = a.im[i];
        if (i + 1 < D) r.y = a.im[i + 1];
        if (i + 2 < D) r.z = a.im[i + 2];
        if (i + 3 < D) r.w = a.im[i + 3];
        return r;
    };
    // momentum += coef * grad; `twice`: the NEXT schedule position re-uses this gradient with no drift in between, its
    // kick (a second, separately rounded `+= coef2 * grad`) is applied in the same pass
    auto kick = [&](float coef, bool twice = false, float coef2 = 0.0f) {
        float4* p4 = reinterpret_cast<float4*>(p);
        const float4* g4 = reinterpret_cast<const float4*>(g);
        for (int v = tid; v < nvec; v += MLP_THREADS) {
            float4 pv = p4[v];
            const float4 gv = g4[v];
            pv.x = add(pv.x, mul(coef, gv.x)); pv.y = add(pv.y, mul(coef, gv.y));
            pv.z = add(pv.z, mul(coef, gv.z)); pv.w = add(pv.w, mul(coef, gv.w));
            if (twice) {
                pv.x = add(pv.x, mul(coef2, gv.x)); pv.y = add(pv.y, mul(coef2, gv.y));
                pv.z = add(pv.z, mul(coef2, gv.z)); pv.w = add(pv.w, mul(coef2, gv.w));
            }
            p4[v] = pv;
        }
        __syncthreads();
    };
    // momentum += coef * (g_rank0 + g_rank1 + ...): the cluster reduction of the split gradient FUSED into the kick -- every
    // rank reads all partials through distributed shared memory (16-byte loads), adds them in rank order (the same bits as
    // reduce-then-kick) and updates its replica of p.  The peers may overwrite their g only after everybody has read it:
    // barrier.cluster arrive here, wait after the drift that follows (its latency hides behind the drift).
    // `drift_cd` != 0: the drift that follows this kick (params += drift_cd * M^-1 momentum, the same operations as drift()
    // below on the just-updated momentum) in the same pass -- one sweep over the state and one barrier less per position
    auto kick_partials = [&](float coef, bool twice = false, float coef2 = 0.0f, float drift_cd = 0.0f) {
        cg::cluster_group cluster = cg::this_cluster();
        const float4* gr[CS];
#pragma unroll
        for (int r = 0; r < CS; ++r) gr[r] = reinterpret_cast<const float4*>(r == cc.rank ? g : cluster.map_shared_rank(g, r));
        float4* p4 = reinterpret_cast<float4*>(p);
        float4* q4 = reinterpret_cast<float4*>(q);
        const bool with_drift = drift_cd != 0.0f, with_im = with_drift && a.mk == HMCX_MASS_DIAG;
        constexpr int KV = CS >= 4 ? 2 : VPT;                  // (register budget: KV * CS vectors live)
        for (int v0 = tid; v0 < nvec; v0 += MLP_THREADS * KV) {
            float4 part[KV][CS], imv[KV];
#pragma unroll
            for (int k = 0; k < KV; ++k) {                     // all remote (and L2) loads of the round in flight together
                const int v = v0 + k * MLP_THREADS;
#pragma unroll
                for (int r = 0; r < CS; ++r) part[k][r] = v < nvec ? gr[r][v] : make_float4(0.f, 0.f, 0.f, 0.f);
                imv[k] = (with_im && v < nvec) ? ld_im4(v) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int k = 0; k < KV; ++k) {
                const int v = v0 + k * MLP_THREADS;
                if (v < nvec) {
                    float4 sg = part[k][0];
#pragma unroll
                    for (int r = 1; r < CS; ++r) {
                        sg.x = add(sg.x, part[k][r].x); sg.y = add(sg.y, part[k][r].y);
                        sg.z = add(sg.z, part[k][r].z); sg.w = add(sg.w, part[k][r].w);
                    }
                    float4 pv = p4[v];
                    pv.x = add(pv.x, mul(coef, sg.x)); pv.y = add(pv.y, mul(coef, sg.y));
                    pv.z = add(pv.z, mul(coef, sg.z)); pv.w = add(pv.w, mul(coef, sg.w));
                    if (twice) {
                        pv.x = add(pv.x, mul(coef2, sg.x)); pv.y = add(pv.y, mul(coef2, sg.y));
                        pv.z = add(pv.z, mul(coef2, sg.z)); pv.w = add(pv.w, mul(coef2, sg.w));
                    }
                    p4[v] = pv;
                    if (with_drift) {
                        float4 qv = q4[v];
                        if (with_im) {
                            qv.x = add(qv.x, mul(mul(drift_cd, imv[k].x), pv.x)); qv.y = add(qv.y, mul(mul(drift_cd, imv[k].y), pv.y));
                            qv.z = add(qv.z, mul(mul(drift_cd, imv[k].z), pv.z)); qv.w = add(qv.w, mul(mul(drift_cd, imv[k].w), pv.w));
                        } else {
                            qv.x = add(qv.x, mul(drift_cd, pv.x)); qv.y = add(qv.y, mul(drift_cd, pv.y));
                            qv.z = add(qv.z, mul(drift_cd, pv.z)); qv.w = add(qv.w, mul(drift_cd, pv.w));
                        }
                        q4[v] = qv;
                    }
                }
            }
        }
        asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
        __syncthreads();
    };
    const bool fused_kick = CS > 1 && m.has_data;
    auto drift = [&](float coef) {                             // params += coef * M^-1 momentum
        float4* q4 = reinterpret_cast<float4*>(q);
        const float4* p4 = reinterpret_cast<const float4*>(p);
        if (a.mk == HMCX_MASS_DIAG) {
            for (int v0 = tid; v0 < nvec; v0 += MLP_THREADS * VPT) {
                float4 im[VPT];
#pragma unroll
                for (int k = 0; k < VPT; ++k) {                // the L2 reads of the round in flight together
                    const int v = v0 + k * MLP_THREADS;
                    im[k] = v < nvec ? ld_im4(v) : make_float4(0.f, 0.f, 0.f, 0.f);
                }
#pragma unroll
                for (int k = 0; k < VPT; ++k) {
                    const int v = v0 + k * MLP_THREADS;
                    if (v < nvec) {
                        float4 qv = q4[v];
                        const float4 pv = p4[v];
                        qv.x = add(qv.x, mul(mul(coef, im[k].x), pv.x)); qv.y = add(qv.y, mul(mul(coef, im[k].y), pv.y));
                        qv.z = add(qv.z, mul(mul(coef, im[k].z), pv.z)); qv.w = add(qv.w, mul(mul(coef, im[k].w), pv.w));
                        q4[v] = qv;
                    }
                }
            }
        } else {
            for (int v = tid; v < nvec; v += MLP_THREADS) {
                float4 qv = q4[v];
                const float4 pv = p4[v];
                qv.x = add(qv.x, mul(coef, pv.x)); qv.y = add(qv.y, mul(coef, pv.y));
                qv.z = add(qv.z, mul(coef, pv.z)); qv.w = add(qv.w, mul(coef, pv.w));
                q4[v] = qv;
            }
        }
        __syncthreads();
    };

    // split drifts divide the step size as a DOUBLE (step_size/K_div, samplers.py:513, :558): the run's initial Python
    // double while the chain still uses it, the fp32 value once dual averaging produced one (:668)
    auto eps_double = [&](float e) { return (a.eps0 != 0.0 && e == (float)a.eps0) ? a.eps0 : (double)e; };

    int g_last_sp = -3;
    bool g_fresh = false;
    for (int n = a.it0; n < a.it1; ++n) {
        if (a.eps_schedule) eps = a.eps_schedule[(size_t)n * a.C + c];
        const float half = mul(0.5f, eps);
        // ---- gibbs (or the caller's momentum) ----
        if (a.p_given) for (int i = tid; i < D; i += MLP_THREADS) p[i] = a.p_given[row + i];
        else for (int v = tid; 4 * v < a.ld; v += MLP_THREADS) {
            float z[4];
            if (a.rng_mode == HMCX_RNG_INJECTED) ld4_stream(a.normals + ((size_t)(n - a.it0) * a.C + c) * a.ld + 4 * v, z);
            else philox_normal4(a.seed, chain_id, (uint64_t)n, (uint32_t)v, z);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int i = 4 * v + j;
                if (i < D) p[i] = a.mk == HMCX_MASS_DIAG ? mul(z[j], a.sd[i]) : z[j];
            }
        }
        if (a.scheme == HMCX_SCHEME_SPLIT_RAND && tid == 0) {            // idx = randperm(M), once per trajectory (:550)
            if (a.rng_mode == HMCX_RNG_INJECTED) {
                for (int s = 0; s < M; ++s) s_perm[s] = a.perms[((size_t)(n - a.it0) * a.C + c) * M + s];
            } else {
                for (int s = 0; s < M; ++s) s_perm[s] = s;
                for (int s = M - 1; s > 0; --s) {                        // Fisher-Yates on the PERM stream
                    const uint4 r = philox_draw(a.seed, chain_id, (uint64_t)n, (uint32_t)s, STREAM_PERM);
                    const int j = (int)(r.x % (uint32_t)(s + 1));
                    const int t = s_perm[s]; s_perm[s] = s_perm[j]; s_perm[j] = t;
                }
            }
        }
        __syncthreads();
        const float kin0 = a.p_given ? 0.0f : kinetic();
        // ---- trajectory: every integrator schedule is a sequence of steps [drift] grad(split) kick [drift] ----
        // ONE loop around ONE inlined copy of the gradient evaluation (nine call sites, one per schedule position, made
        // each instantiation of this kernel ~100k instructions = 1.6 MB of code and minutes of ptxas; an out-of-line copy
        // was measured 1.6x slower: the model descriptor then lives behind a pointer instead of in the constant bank).
        //   PLAIN (:281-302)      t = 0: grad, kick(eps/2); t = 1..L: drift(eps), grad, kick(eps); finally kick(-eps/2)
        //   SPLITTING (:499-540)  per step j = 0..2M-1: s = j < M ? j : 2M-1-j; grad(s), kick(eps/2), drift(eps/(2(M-1))) unless
        //                         the sweep's last split
        //   SPLITTING_RAND (:551-568)  per step, split s = perm[j/2]: grad, kick(eps/2), drift(eps/M) | grad, kick(eps/2)
        //   SPLITTING_KMID (:579-598)  M kicks up, drift(eps), M kicks down
        {
            const int twoM = 2 * M;
            const bool plain = a.scheme == HMCX_SCHEME_PLAIN;
            const int T = plain ? a.L + 1 : a.L * twoM;
            float cd = 0.0f;
            if (a.scheme == HMCX_SCHEME_SPLIT_SYM) cd = (float)(eps_double(eps) / (double)((M - 1) * 2));
            else if (a.scheme == HMCX_SCHEME_SPLIT_RAND) cd = (float)(eps_double(eps) / (double)M);
            else if (a.scheme == HMCX_SCHEME_SPLIT_KMID) cd = eps;
            int jj = 0;
            auto split_at = [&](int j) {                                  // the data split of schedule position j
                const int up = j < M ? j : twoM - 1 - j;
                return a.scheme == HMCX_SCHEME_SPLIT_RAND ? s_perm[j >> 1] : up;
            };
            auto post_at = [&](int j) {                                   // a drift follows the kick of schedule position j
                const int up = j < M ? j : twoM - 1 - j;
                if (a.scheme == HMCX_SCHEME_SPLIT_SYM) return j < M ? (up < M - 1) : (up > 0);
                if (a.scheme == HMCX_SCHEME_SPLIT_RAND) return (j & 1) == 0;
                return j == M - 1;
            };
            // Two consecutive schedule positions with the SAME split and NO drift between them differentiate the same function
            // at the same parameters: the turning point of the symmetric sweep (m = M-1 up, then M-1 down, :501-:523) and the
            // step boundary (m = 0 down, then m = 0 up of the next step); SPLITTING_KMID has the latter.  The reference calls
            // autograd twice and gets the same tensor twice; here the second evaluation is skipped and g (per-rank partials
            // included) is kicked again -- the same bits, 2 of the 2M evaluations of a symmetric step saved.
            // The same across iterations: a trajectory ends with an evaluation at its final parameters and no drift after it;
            // when the proposal is accepted the next trajectory starts by differentiating the same split (the whole potential
            // for PLAIN) at those parameters -- g_last_sp / g_fresh carry the gradient over (1 of L+1 evaluations of
            // sample_model's plain leapfrog at high acceptance).
            int prev_sp = g_fresh ? g_last_sp : -3;
            bool prev_post = !g_fresh, kicked_ahead = false;
#pragma unroll 1
            for (int t = 0; t < T; ++t) {
                int sp = psp, sp_next = psp;
                float kc = half;
                bool post = false, reuse = false, kick_twice = false, drift_done = false;
                if (plain) {
                    if (t > 0) { drift(eps); kc = eps; }
                    else reuse = g_fresh && g_last_sp == -1;
                } else {
                    sp = split_at(jj);
                    post = post_at(jj);
                    reuse = sp == prev_sp && !prev_post;
                    if (++jj == twoM) jj = 0;
                    sp_next = split_at(jj);
                    int ahead = 1;
                    if (sp_next == sp && !post) {                         // the next position re-uses this gradient: prefetch for
                        sp_next = split_at(jj + 1 == twoM ? 0 : jj + 1);  // the one after it
                        ahead = 2;
                        // ... and its kick joins this one -- unless a trajectory is being recorded and a leapfrog step
                        // ends between the two (the recorded momentum is the one after the first kick only)
                        kick_twice = !reuse && t + 1 < T && !(a.q_traj && jj == 0);
                    }
                    if (t + ahead >= T) sp_next = -2;
                    prev_sp = sp; prev_post = post;
                }
                if (t + 1 == T) sp_next = -2;                             // the Hamiltonian evaluation follows: nothing to prefetch
                if (!reuse) mlp_grad_split<CS>(m, q, g, tile, sp, cc, tc, fused_kick, sp_next);
                if (kicked_ahead) {                                       // this position's kick was applied with the previous one
                    kicked_ahead = false;
                    if (fused_kick) asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
                } else if (fused_kick) {
                    // (plain: the drift belongs to the NEXT position and takes its own pass; a recorded trajectory keeps the
                    // separate pass too -- nothing to gain there)
                    drift_done = post && !plain && cd != 0.0f;
                    kick_partials(kc, kick_twice, half, drift_done ? cd : 0.0f);
                } else {
                    kick(kc, kick_twice, half);
                }
                kicked_ahead = kick_twice;
                TC_MARK(16);
                if (post && !drift_done) drift(cd);
                if (fused_kick) asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
                TC_MARK(17);
                if (a.q_traj && !plain && jj == 0 && lead) {              // a leapfrog step just ended (:546-547, :570-571, :600-601)
                    const size_t o = ((size_t)(t / twoM) * a.C + c) * a.ld;
                    for (int i = tid; i < a.ld; i += MLP_THREADS) {
                        a.q_traj[o + i] = i < D ? q[i] : 0.0f;
                        a.p_traj[o + i] = i < D ? p[i] : 0.0f;
                    }
                }
            }
            if (plain) {                                                  // p - half*g == p + (-half)*g exactly
                if (fused_kick) { kick_partials(-half); asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
                else kick(-half);
            }
            // g now holds the gradient of the last schedule position's split at the proposal, unless a drift followed it
            g_last_sp = plain ? -1 : prev_sp;
            g_fresh = plain || !prev_post;
        }
        if (a.p_given) break;                                             // stand-alone leapfrog: no Hamiltonian, no MH
        // ---- Hamiltonians + MH ----
        const float lp_new = mlp_log_prob<CS>(m, q, tile, sred, psp, nullptr, cc, &s_xchg, tc,
                                              PER_CHAIN ? &ls_new : nullptr);
        const float kin1 = kinetic();
        const float h_old = add(-lp_cur, mul(0.5f, kin0));
        const float h_new = add(-lp_new, mul(0.5f, kin1));
        const bool bad = !finite_f(lp_cur) || !finite_f(lp_new);
        const float x = add(-h_new, h_old);
        const float rho = (x < 0.0f) ? x : 0.0f;
        if (tid == 0)
            s_bcast[0] = (a.rng_mode == HMCX_RNG_INJECTED) ? a.logu[(size_t)(n - a.it0) * a.C + c]
                                                           : philox_log_uniform(a.seed, chain_id, (uint64_t)n);
        __syncthreads();
        const float logu = s_bcast[0];
        const bool acc = !bad && (rho >= logu);
        if (acc) {
            lp_cur = lp_new;
            if constexpr (PER_CHAIN) ls_cur = ls_new;
            if (lead) for (int i = tid; i < D; i += MLP_THREADS) a.q_cur[row + i] = q[i];
        } else {
            ++rejected;
            g_fresh = false;                                              // q goes back: g belongs to the rejected proposal
            const float* src = (n == a.burn + 1) ? a.q_init : a.q_cur;    // the first-stored-iteration quirk (:1018)
            for (int i = tid; i < D; i += MLP_THREADS) q[i] = src[row + i];
            __syncthreads();
            if (n == a.burn + 1) {
                lp_cur = mlp_log_prob<CS>(m, q, tile, sred, psp, nullptr, cc, &s_xchg, tc,
                                          PER_CHAIN ? &ls_cur : nullptr);
                if (lead) for (int i = tid; i < D; i += MLP_THREADS) a.q_cur[row + i] = q[i];
            }
        }
        if (CS > 1) cg::this_cluster().sync();                 // q_cur is stable before any rank re-reads it
        if (hyper) {
            // Gibbs step of the precisions given q_n: tau_k ~ Gamma(a_k + n_k/2, b_k + |w_k|^2/2), tau_out ~ Gamma(a_o + N O/2,
            // b_o + SSE(q_n)/2).  |w_k|^2 is a fixed-order fp64 sum over every rank's identical replica of q, SSE (ls_cur, a
            // regression run's) the cluster sum of the MH evaluation at q_cur, so every rank draws the same precisions.
            ChainModelSm& cm = chain_model_sm();
            const int K = 2 * m.L;
            __syncthreads();                                   // nobody reads the constants thread 0 rewrites below
            for (int t = 0; t < K; ++t) {
                if (!((a.hy.sampled >> t) & 1)) continue;
                const int l = t >> 1, off = (t & 1) ? m.boff[l] : m.woff[l];
                const int cnt = (t & 1) ? m.n[l + 1] : m.n[l] * m.n[l + 1];
                double ss = 0.0;
                for (int i = tid; i < cnt; i += MLP_THREADS) { const double w = (double)q[off + i]; ss = fma(w, w, ss); }
                ss = block_sum_d(ss, cm.red);
                if (tid == 0) cm.ssq[t] = ss;
            }
            if (tid == 0) {
                for (int k = 0; k <= K; ++k) {
                    if (!((a.hy.sampled >> k) & 1)) continue;
                    const int l = k >> 1;
                    const double nk = k < K ? (double)((k & 1) ? m.n[l + 1] : m.n[l] * m.n[l + 1]) : a.hy.n_obs;
                    const double shape = a.hy.a[k] + 0.5 * nk, rate = a.hy.b[k] + 0.5 * (k < K ? cm.ssq[k] : ls_cur);
                    const double g = a.rng_mode == HMCX_RNG_INJECTED
                                         ? a.hy.gammas[((size_t)(n - a.it0) * a.C + c) * (K + 1) + k]
                                         : philox_std_gamma(a.seed, chain_id, (uint64_t)n, (uint32_t)k, shape);
                    const float tau = (float)(g / rate);
                    if (k < K) cm.tau[k] = tau;
                    else cm.tau_out = tau;
                }
                hyper_constants(cm.m, cm.tau, cm.tau_out, a.hy.sampled);
            }
            __syncthreads();
            // log p(q_cur) and any carried gradient belong to the old precisions: re-evaluate the former, drop the latter
            lp_cur = mlp_log_prob<CS>(m, q, tile, sred, -1, nullptr, cc, &s_xchg, tc);
            g_fresh = false;
            if (n > a.burn && (n - a.burn) % a.thin == 0) hyper_store((n - a.burn) / a.thin);
        }
        if (n > a.burn)
            sink_row((my_samples && (n - a.burn) % a.thin == 0) ? my_samples + (size_t)((n - a.burn) / a.thin) * a.ld
                                                                : nullptr, true);
        else if (a.moments_all)
            sink_row(nullptr, true);                                       // a warm-up window's moments
        if (tid == 0 && lead) {
            const size_t o = (size_t)c * a.S + n;
            if (a.accept) a.accept[o] = acc ? 1 : 0;
            if (a.diverged) a.diverged[o] = bad ? 1 : 0;
            if (a.ham) { a.ham[2 * o] = h_old; a.ham[2 * o + 1] = h_new; }
        }
        if (a.nuts && n <= a.burn) {                                       // dual averaging, as hmc_run_kernel
            if (tid == 0) {
                float e = eps;
                if (n < a.burn || bad) {
                    const double* T = a.table + 5 * (size_t)n;
                    const double alpha = bad ? 0.0 : (double)expf(rho);
                    h_bar = __dadd_rn(__dmul_rn(T[0], h_bar), __dmul_rn(T[1], a.delta - alpha));
                    const double x_new = mu_sink - __dmul_rn(T[2], h_bar);
                    e = expf((float)x_new);
                    const float xb = add((float)__dmul_rn(T[3], x_new), mul((float)T[4], logf((float)eps_bar)));
                    eps_bar = (double)expf(xb);
                }
                if (n == a.burn) e = (float)eps_bar;
                s_bcast[1] = e;
                if (a.eps_trace && lead) a.eps_trace[(size_t)c * a.S + n] = e;
            }
            __syncthreads();
            eps = s_bcast[1];
        } else if (a.eps_trace && tid == 0 && lead) {
            a.eps_trace[(size_t)c * a.S + n] = eps;
        }
        __syncthreads();
    }
    if (hyper && tid == 0 && lead) {
        const ChainModelSm& cm = chain_model_sm();
        for (int k = 0; k < 2 * m.L; ++k) a.hy.tau[(size_t)c * 2 * m.L + k] = cm.tau[k];
        a.hy.tau_out[c] = cm.tau_out;
    }
    if (temper && tid == 0 && lead && a.tp.ll_out)           // the untempered c_ll is the constant bank's
        a.tp.ll_out[c] = (double)a.m.c_ll * ls_cur;
    if (tid == 0 && lead && !a.p_given) {
        a.eps[c] = eps;
        if (a.nuts) { a.h_bar[c] = h_bar; a.eps_bar[c] = eps_bar; }
        if (a.num_rejected) a.num_rejected[c] += rejected;
    }
}

// gradient / log-prob of C parameter vectors (collect_gradients mirror, also the unit-test hook of the backward pass)
__global__ void __launch_bounds__(MLP_THREADS, 1)
mlp_grad_kernel(const MlpDev m, const float* __restrict__ qin, int ld, int split, float* __restrict__ gout,
                float* __restrict__ lpout) {
    extern __shared__ __align__(128) float sm[];
    __shared__ float sred[64];
    __shared__ __align__(8) uint64_t s_bars[3];
    float* q = sm;
    float* g = q + m.Dp;
    float* tile = sm + m.tile_base;
    const size_t row = (size_t)blockIdx.x * ld;
    TcCtx tc = {};
    if (m.tc) tc_init(tc, s_bars);
    for (int i = threadIdx.x; i < m.Dp; i += MLP_THREADS) { q[i] = i < m.D ? qin[row + i] : 0.0f; g[i] = 0.0f; }
    __syncthreads();
    if (gout) {
        mlp_grad_split<1>(m, q, g, tile, split, ClusterCtx{0, 1}, tc);
        __syncthreads();
        for (int i = threadIdx.x; i < ld; i += MLP_THREADS) gout[row + i] = i < m.D ? g[i] : 0.0f;
    }
    if (lpout) {
        const float lp = mlp_log_prob<1>(m, q, tile, sred, split, nullptr, ClusterCtx{0, 1}, nullptr, tc);
        if (threadIdx.x == 0) lpout[blockIdx.x] = lp;
    }
}

// predict_model: one CTA per posterior sample
__global__ void __launch_bounds__(MLP_THREADS, 1)
mlp_predict_kernel(const MlpDev m, const float* __restrict__ samples, int ld, float* __restrict__ pred,
                   float* __restrict__ lpout) {
    extern __shared__ __align__(128) float sm[];
    __shared__ float sred[64];
    __shared__ __align__(8) uint64_t s_bars[3];
    float* q = sm;
    float* tile = sm + m.tile_base;
    const size_t row = (size_t)blockIdx.x * ld;
    for (int i = threadIdx.x; i < m.Dp; i += MLP_THREADS) q[i] = i < m.D ? samples[row + i] : 0.0f;
    __syncthreads();
    float* my_pred = pred + (size_t)blockIdx.x * m.N * m.n[m.L];
    TcCtx tc = {};
    if (m.tc) tc_init(tc, s_bars);
    const float lp = mlp_log_prob<1>(m, q, tile, sred, -1, my_pred, ClusterCtx{0, 1}, nullptr, tc);
    if (threadIdx.x == 0 && lpout) lpout[blockIdx.x] = lp;
}

// Pointwise log-likelihood of the rows [r_begin, r_end) of a forwarded tile (rows r0 .. r0 + cnt - 1), one thread per row:
//   regression   ll_const + c_ll * sum_o (f_o - y_o)^2       (c_ll = -0.5 tau_out, ll_const = 0.5 O log(tau_out / 2 pi))
//   binary       -sum_o BCEWithLogits(f_o, y_o) in torch's stable form
//   multi-class  log_softmax(f)[y];  LogSoftmax output: f[y], the same value of the logits
// tau_out tempers the classification likelihoods during sampling only; it does not enter these densities.
__device__ __forceinline__ void mlp_ll_rows(const MlpDev& m, const float* out, const float* ytile, int r0, int cnt,
                                            int r_begin, int r_end, float ll_const, float tau_out, float* llrow) {
    const int nL = m.n[m.L];
    for (int r = threadIdx.x; r < cnt; r += MLP_THREADS) {
        const int i = r0 + r;
        if (i < r_begin || i >= r_end) continue;
        const float* z = out + r * nL;
        float v = 0.0f;
        if (m.loss == HMCX_LOSS_REGRESSION || m.loss == HMCX_LOSS_BINARY) {
            for (int o = 0; o < nL; ++o) {
                const float yv = ytile ? ytile[r * nL + o] : __ldg(m.y + (size_t)i * nL + o), f = z[o];
                if (m.loss == HMCX_LOSS_REGRESSION) {
                    const float d = f - yv;
                    v += d * d;
                } else {
                    v -= (1.0f - yv) * f + fmaxf(-f, 0.0f) + log1pf(expf(-fabsf(f)));
                }
            }
            if (m.loss == HMCX_LOSS_REGRESSION) v = ll_const + (-0.5f * tau_out) * v;
        } else {
            // both multi-class losses: the tile holds the logits (a LogSoftmax output layer is applied here, as in the
            // loss stage), so f[y] of a LogSoftmax network is log_softmax(logits)[y]
            int label = (int)(ytile ? ytile[r] : __ldg(m.y + i));
            label = label < 0 ? 0 : (label >= nL ? nL - 1 : label);
            float mx = z[0];
            for (int k = 1; k < nL; ++k) mx = fmaxf(mx, z[k]);
            float se = 0.0f;
            for (int k = 0; k < nL; ++k) se += expf(z[k] - mx);
            v = (z[label] - mx) - logf(se);
        }
        llrow[i] = v;
    }
}

// The draw pass of the pointwise kernels: one CTA per draw loads it (qin) into shared memory and forwards the rows
// [r_begin, r_end) tile by tile with the code of mlp_predict_kernel, over the target's own tiles split by split, so x, y
// and the packed tensor-core operands are read in place.  pro() runs once, after the draw's loads are issued and before
// the barrier that publishes it, so a kernel's per-draw set-up overlaps them.  Tiles that straddle the slab's edges are
// forwarded whole; epi(tile, sp, r0, cnt) then sees the outputs of the rows r0 .. r0 + cnt - 1 of split sp at
// tile + m.aoff[m.L] (and, on the tensor-core path, their y at tile + m.tc_yraw) and handles the rows inside the slab.
template <typename Pro, typename Epi>
__device__ __forceinline__ void mlp_draw_pass(const MlpDev& m, const float* qin, int r_begin, int r_end, Pro pro,
                                              Epi epi) {
    extern __shared__ __align__(128) float sm[];
    __shared__ __align__(8) uint64_t s_bars[3];
    float* q = sm;
    float* tile = sm + m.tile_base;
    for (int i = threadIdx.x; i < m.Dp; i += MLP_THREADS) q[i] = i < m.D ? qin[i] : 0.0f;
    pro();
    __syncthreads();
    TcCtx tc = {};
    TcEpi te;
    if (m.tc) {
        tc_init(tc, s_bars);
        tc_epi_begin(m, q, te);
        fence_async_smem();
        __syncthreads();
    }
    for (int sp = 0; sp < m.M; ++sp) {
        if (m.sb[sp + 1] <= r_begin || m.sb[sp] >= r_end) continue;
        int ti = 0;
        for (int r0 = m.sb[sp]; r0 < m.sb[sp + 1] && r0 < r_end; r0 += m.T, ++ti) {
            if (r0 + m.T <= r_begin) continue;
            const int cnt = min(m.T, m.sb[sp + 1] - r0);
            if (m.tc) {
                float act[16];
                tc_prefetch_fwd(m, tile, tc, m.tb[sp] + ti, 0);
                tc_prefetch_y(m, tile, r0, cnt);
                tc_forward_tile(m, q, tile, tc, te, act, 0);
            } else {
                mlp_forward_tile(m, q, tile, r0, cnt);
            }
            epi(tile, sp, r0, cnt);
            __syncthreads();
        }
    }
}

// ll[c, s, i - r_begin] = log p(y_i | theta_{c,s}) for the rows [r_begin, r_end), one CTA per draw; the network outputs
// never leave shared memory.  tau == NULL: the target's tau_out and the host's ll_const.  Otherwise draw (c, s) reads
// its own tau_out at tau[c * tcs + s * tds] (the draws of a run with a tau_out hyperprior, DESIGN.md 3.15) and
// evaluates its constant as the host does (fp64 log, then the fp32 rounding).
__global__ void __launch_bounds__(MLP_THREADS, 1)
mlp_ll_kernel(const MlpDev m, const float* __restrict__ samples, long long cs, long long ds, int n, int r_begin,
              int r_end, float ll_const, const float* __restrict__ tau, long long tcs, long long tds,
              float* __restrict__ ll, long long lcs, long long lds) {
    const int c = blockIdx.x / n, s = blockIdx.x - c * n;
    float tau_out = m.tau_out;
    float* llrow = ll + (long long)c * lcs + (long long)s * lds - r_begin;
    mlp_draw_pass(m, samples + (long long)c * cs + (long long)s * ds, r_begin, r_end,
                  [&] {
                      if (!tau) return;
                      tau_out = tau[(long long)c * tcs + (long long)s * tds];
                      ll_const = (float)(0.5 * m.n[m.L] * log((double)tau_out / (2.0 * 3.14159265358979323846)));
                  },
                  [&](const float* tile, int, int r0, int cnt) {
                      mlp_ll_rows(m, tile + m.aoff[m.L], m.tc ? tile + m.tc_yraw : nullptr, r0, cnt, r_begin, r_end,
                                  ll_const, tau_out, llrow);
                  });
}

// out[c, s, i - r_begin, :] = the network outputs of draw (c, s) at the rows [r_begin, r_end) (held-out evaluation,
// DESIGN.md 3.16): the forward of mlp_predict_kernel, and a LogSoftmax output layer applied by the loss stage of
// mlp_log_prob, so the values are predict_model's, bit for bit.
__global__ void __launch_bounds__(MLP_THREADS, 1)
mlp_out_kernel(const MlpDev m, const float* __restrict__ samples, long long cs, long long ds, int n, int r_begin,
               int r_end, float* __restrict__ out, long long ocs, long long ods) {
    const int c = blockIdx.x / n, s = blockIdx.x - c * n;
    int nL;
    float* orow;
    mlp_draw_pass(m, samples + (long long)c * cs + (long long)s * ds, r_begin, r_end,
                  [&] {
                      nL = m.n[m.L];
                      orow = out + (long long)c * ocs + (long long)s * ods - (long long)r_begin * nL;
                  },
                  [&](float* tile, int sp, int r0, int cnt) {
                      if (m.loss == HMCX_LOSS_MULTICLASS_LOGSOFTMAX) {
                          mlp_loss_tile(m, tile + m.aoff[m.L], nullptr, r0, cnt, m.sb[sp + 1] - m.sb[sp], true,
                                        m.tc ? tile + m.tc_yraw : nullptr);
                          __syncthreads();
                      }
                      const int lo = max(r0, r_begin) - r0, hi = min(r0 + cnt, r_end) - r0;
                      for (int e = lo * nL + threadIdx.x; e < hi * nL; e += MLP_THREADS)
                          orow[(long long)r0 * nL + e] = tile[m.aoff[m.L] + e];
                  });
}

// ---------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------
static void mlp_layout_tiles(MlpDev& m, int T) {
    int aoff = 0, maxw = 0;
    for (int l = 0; l <= m.L; ++l) {
        m.aoff[l] = aoff;
        aoff += T * m.n[l];
        if (m.n[l] > maxw) maxw = m.n[l];
    }
    m.dzoff[0] = aoff;
    m.dzoff[1] = aoff + T * maxw;
    m.tile_floats = aoff + 2 * T * maxw;
    m.T = T;
}

static bool mlp_tc_shape(const MlpDev& m) {
    return m.L == 2 && m.n[1] == TC_H && m.n[0] >= 16 && m.n[0] <= 64 && (m.n[0] & 15) == 0 && m.n[2] <= TC_NLMAX && m.has_data;
}

// tensor-core layout of the tile area (one-hidden-layer stacks n0 -> 128 -> nL, see the tensor-core section above);
// `reserve`: static shared memory a kernel form holds beyond the common headroom (ChainModelSm for the PER_CHAIN forms)
static bool mlp_layout_tc(MlpDev& m, int state_vectors, size_t reserve) {
    if (!mlp_tc_shape(m) || !m.xp) return false;
    const int n0 = m.n[0];
    int off = 0;
    m.tc_f0 = off; off += 2 * TC_TR * n0;       // forward X operand (hi|lo), double-buffered; f0 | f1 also stage dW1
    m.tc_f1 = off; off += 2 * TC_TR * n0;       //   (128 rows, pitch n0 + 4) at the end of an evaluation
    m.tc_b = off; off += 2 * TC_TR * n0;        // backward X operand (hi|lo)
    m.tc_part = off; off += 4 * TC_H * (1 + TC_NLMAX);
    m.tc_yraw = off; off += TC_TR * TC_NLMAX;
    m.aoff[0] = m.aoff[1] = 0;
    m.aoff[2] = off; off += TC_TR * TC_NLMAX;
    m.dzoff[0] = m.dzoff[1] = off; off += TC_TR * TC_NLMAX;
    m.tile_floats = off;
    m.tile_base = (state_vectors * m.Dp + 31) / 32 * 32;      // 128-byte aligned operand buffers
    m.T = TC_TR;
    m.tc = 1;
    return (size_t)(m.tile_base + m.tile_floats) * sizeof(float) + reserve <= 227 * 1024 - 2048;
}

// pick the largest tile height whose buffers fit next to `state_vectors` copies of the parameter vector
static bool mlp_pick_tile(MlpDev& m, int state_vectors, bool allow_tc = false, size_t reserve = 0) {
    if (allow_tc && mlp_layout_tc(m, state_vectors, reserve)) return true;
    m.tc = 0;
    m.tile_base = state_vectors * m.Dp;
    for (int T = MLP_T_MAX; T >= 8; T >>= 1) {
        mlp_layout_tiles(m, T);
        if ((size_t)(state_vectors * m.Dp + m.tile_floats) * sizeof(float) + reserve <= 227 * 1024 - 4096) return true;
    }
    return false;
}

// packed-operand tile numbering (see mlp_pack_x_kernel): the tiles of every split, then -- only when some interior split
// boundary is not a multiple of the tile height -- the tiles of the all-rows tiling; returns the number of tiles
static int mlp_packed_tiles(MlpDev& m) {
    int t = 0;
    bool aligned = true;
    for (int s = 0; s < m.M; ++s) {
        m.tb[s] = t;
        t += (m.sb[s + 1] - m.sb[s] + TC_TR - 1) / TC_TR;
        if (s > 0 && (m.sb[s] % TC_TR) != 0) aligned = false;
    }
    m.tb[m.M] = t;
    if (aligned) { m.flat_base = 0; return t; }
    m.flat_base = t;
    return t + (m.N + TC_TR - 1) / TC_TR;
}

static int fill_mlp(const hmcx_target_t* target, MlpDev& m) {
    if (!target || target->kind != HMCX_TARGET_MLP || !target->mlp) return HMCX_ERR_INVALID_ARG;
    const hmcx_mlp_t& h = *target->mlp;
    if (h.num_layers < 1 || h.num_layers > HMCX_MLP_MAX_LAYERS) return HMCX_ERR_INVALID_ARG;
    if (h.loss < HMCX_LOSS_REGRESSION || h.loss > HMCX_LOSS_MULTICLASS_LOGSOFTMAX) return HMCX_ERR_UNSUPPORTED;
    m.loss = h.loss;
    if (h.activation[h.num_layers - 1] != HMCX_ACT_NONE) return HMCX_ERR_INVALID_ARG;
    m.L = h.num_layers;
    int off = 0;
    for (int l = 0; l <= m.L; ++l) {
        if (h.widths[l] < 1) return HMCX_ERR_INVALID_ARG;
        m.n[l] = h.widths[l];
    }
    for (int l = 0; l < m.L; ++l) {
        m.act[l] = h.activation[l];
        if (m.act[l] < 0 || m.act[l] > HMCX_ACT_SIGMOID) return HMCX_ERR_INVALID_ARG;
        m.woff[l] = off; off += m.n[l] * m.n[l + 1];
        m.boff[l] = off; off += m.n[l + 1];
    }
    m.D = off;
    if (m.D != target->dim) return HMCX_ERR_INVALID_ARG;
    m.Dp = (m.D + 3) / 4 * 4;
    mlp_layout_tiles(m, 8);
    m.tau_out = h.tau_out;
    m.prior_scale = h.prior_scale;
    m.c_ll = (h.loss == HMCX_LOSS_REGRESSION) ? (float)(-0.5 * (double)h.tau_out) : (float)(-(double)h.tau_out);
    for (int t = 0; t < 2 * m.L; ++t) {
        m.two_var[t] = h.prior_two_var[t]; m.log_scale[t] = h.prior_log_scale[t]; m.gcoef[t] = h.prior_grad_coef[t];
    }
    m.x = h.x; m.y = h.y; m.N = h.num_rows;
    m.has_data = (h.x != nullptr) ? 1 : 0;
    m.M = h.num_splits;
    if (m.M < 1 || m.M > HMCX_MLP_MAX_SPLITS) return HMCX_ERR_INVALID_ARG;
    if (m.has_data) {
        if (!h.y || h.num_rows < 1) return HMCX_ERR_INVALID_ARG;
        if (h.split_begin[0] != 0 || h.split_begin[m.M] != h.num_rows) return HMCX_ERR_INVALID_ARG;
        for (int s = 0; s <= m.M; ++s) {
            m.sb[s] = h.split_begin[s];
            if (s && m.sb[s] <= m.sb[s - 1]) return HMCX_ERR_INVALID_ARG;
        }
    } else {
        for (int s = 0; s <= m.M; ++s) m.sb[s] = 0;
    }
    mlp_packed_tiles(m);
    m.xp = h.x_packed;
    return HMCX_OK;
}

static inline int cuda_status() { return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA; }

template <typename Kern>
static int prepare_smem(Kern kern, size_t bytes) {
    if (bytes > 227 * 1024) return HMCX_ERR_UNSUPPORTED;       // the chain state does not fit one SM's shared memory
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes) != cudaSuccess) {
        cudaGetLastError();
        return HMCX_ERR_UNSUPPORTED;
    }
    return HMCX_OK;
}

int mlp_split_run(const hmcx_target_t* target, const hmcx_mass_t* mass, const hmcx_rng_t* rng, const hmcx_nuts_t* nuts,
                  int scheme, const float* q_init, float* q_cur, float* eps, int C, int ld, int L, int S, int burn,
                  int it0, int it1, float* samples, uint8_t* accept, uint8_t* diverged, float* ham,
                  int32_t* num_rejected, cudaStream_t st, const float* p_given, float* q_traj, float* p_traj,
                  const hmcx_sink_t* sink, const hmcx_hyper_t* hyper, const hmcx_temper_t* temper, int folds) {
    MlpRunArgs a = {};
    hmcx_sink_t thin1 = {};
    if (!sink) { thin1.thin = 1; sink = &thin1; }              // every run is a sink run: no sink = {thin = 1}
    a.p_given = p_given; a.q_traj = q_traj; a.p_traj = p_traj;
    a.thin = sink->thin; a.msum = sink->sum; a.msumsq = sink->sumsq;
    a.msum_lo = sink->sum_lo; a.msumsq_lo = sink->sumsq_lo;
    a.moments_all = sink->moments_all;
    if (nuts && nuts->enabled) a.mu_chain = nuts->mu_chain;
    int rc = fill_mlp(target, a.m);
    if (rc != HMCX_OK) return rc;
    const int mk = mass ? mass->kind : HMCX_MASS_NONE;
    if (mk != HMCX_MASS_NONE && mk != HMCX_MASS_DIAG) return HMCX_ERR_UNSUPPORTED;
    if (mk == HMCX_MASS_DIAG && (!mass->inv_mass || !mass->mass_factor)) return HMCX_ERR_INVALID_ARG;
    if (!rng || !q_init || !q_cur || !eps || C < 1 || ld < a.m.D || (ld & 3) || L < 1 || S < 1 || burn < 0 || burn >= S ||
        it0 < 0 || it1 > S || it0 > it1)
        return HMCX_ERR_INVALID_ARG;
    if (scheme < HMCX_SCHEME_PLAIN || scheme > HMCX_SCHEME_SPLIT_KMID) return HMCX_ERR_INVALID_ARG;
    if ((scheme == HMCX_SCHEME_SPLIT_SYM || scheme == HMCX_SCHEME_SPLIT_KMID) && a.m.M < 2) return HMCX_ERR_INVALID_ARG;  // :497-498
    if (rng->mode == HMCX_RNG_INJECTED) {
        if (!p_given && (!rng->normals || !rng->log_uniforms)) return HMCX_ERR_INVALID_ARG;
        if (scheme == HMCX_SCHEME_SPLIT_RAND && !rng->perms) return HMCX_ERR_INVALID_ARG;
    } else if (rng->mode != HMCX_RNG_PHILOX) {
        return HMCX_ERR_INVALID_ARG;
    }
    if (hyper) {
        const int K = 2 * a.m.L;
        if (!hyper->tau || !hyper->tau_out || p_given) return HMCX_ERR_INVALID_ARG;
        if (rng->mode == HMCX_RNG_INJECTED && !hyper->gammas) return HMCX_ERR_INVALID_ARG;
        for (int k = 0; k < HMCX_HYPER_GROUPS; ++k) {
            if (!hyper->sampled[k]) continue;
            if (k > K || !(hyper->a[k] > 0.0) || !(hyper->b[k] > 0.0) || !(hyper->a[k] <= DBL_MAX) || !(hyper->b[k] <= DBL_MAX))
                return HMCX_ERR_INVALID_ARG;
            a.hy.sampled |= 1 << k;
            a.hy.a[k] = hyper->a[k]; a.hy.b[k] = hyper->b[k];
        }
        if (hyper->sampled[K] && !a.m.has_data) return HMCX_ERR_INVALID_ARG;
        if (hyper->sampled[K] && a.m.loss != HMCX_LOSS_REGRESSION) return HMCX_ERR_UNSUPPORTED;
        a.hy.n_obs = (double)a.m.N * (double)a.m.n[a.m.L];
        a.hy.tau = hyper->tau; a.hy.tau_out = hyper->tau_out;
        a.hy.tau_trace = hyper->tau_trace; a.hy.tau_out_trace = hyper->tau_out_trace;
        a.hy.gammas = hyper->gammas;
    }
    if (temper) {
        if (hyper) return HMCX_ERR_UNSUPPORTED;
        const int T = temper->num_temps;
        if (p_given || T < 1 || T > HMCX_TEMPER_MAX_TEMPS || C % T != 0) return HMCX_ERR_INVALID_ARG;
        a.tp.T = T;
        for (int t = 0; t < T; ++t) {
            const float v = temper->tau_out[t];
            if (!(v >= 0.0f) || !(v <= FLT_MAX) || (t > 0 && !(v <= temper->tau_out[t - 1]))) return HMCX_ERR_INVALID_ARG;
            a.tp.tau_out[t] = v;
        }
        a.tp.ll_out = temper->ll_out;
    }
    if (folds) {                                               // K-fold: one split per fold, each chain on its own
        if (hyper || temper) return HMCX_ERR_UNSUPPORTED;
        if (scheme != HMCX_SCHEME_PLAIN) return HMCX_ERR_UNSUPPORTED;
        if (p_given || folds < 2 || folds > HMCX_MLP_MAX_SPLITS || a.m.M != folds || !a.m.has_data)
            return HMCX_ERR_INVALID_ARG;
        a.folds = folds;
    }
    a.scheme = scheme; a.mk = mk; a.C = C; a.ld = ld;
    a.im = mass ? mass->inv_mass : nullptr; a.sd = mass ? mass->mass_factor : nullptr;
    a.rng_mode = rng->mode; a.seed = rng->seed; a.chain_offset = rng->chain_offset;
    a.normals = rng->normals; a.logu = rng->log_uniforms; a.perms = rng->perms;
    a.nuts = (nuts && nuts->enabled) ? 1 : 0;
    a.eps0 = nuts ? nuts->step_size_init : 0.0;
    if (a.nuts) {
        if (!nuts->table || !nuts->h_bar || !nuts->eps_bar || burn < 1) return HMCX_ERR_INVALID_ARG;
        a.delta = nuts->desired_accept_rate; a.mu = nuts->mu; a.table = nuts->table;
        a.h_bar = nuts->h_bar; a.eps_bar = nuts->eps_bar;
        a.eps_schedule = nuts->eps_schedule; a.eps_trace = nuts->eps_trace;
    }
    a.q_init = q_init; a.q_cur = q_cur; a.eps = eps; a.L = L; a.S = S; a.burn = burn; a.it0 = it0; a.it1 = it1;
    a.samples = samples; a.accept = accept; a.diverged = diverged; a.ham = ham; a.num_rejected = num_rejected;
    if (!mlp_pick_tile(a.m, 3, target->mlp->tensor_cores != HMCX_MLP_TC_OFF, (hyper || temper) ? sizeof(ChainModelSm) : 0))
        return HMCX_ERR_UNSUPPORTED;                            // q, p, g do not fit one SM's shared memory
    const size_t smem = (size_t)(a.m.tile_base + a.m.tile_floats) * sizeof(float);
    // CTAs per chain (thread-block cluster size): at most the tiles of the smallest split, at most 4, and -- unless the
    // caller pins it (hmcx_mlp_t.cluster_size) -- no more than keeps every chain's cluster resident at once.  The
    // partial gradients are associated per cluster rank, so low-order bits depend on this number: pin it to make
    // chains bit-reproducible across launches with different chain counts (e.g. different multi-GPU shardings).
    int cs = 1;
    if (a.m.has_data && a.m.D <= MLP_THREADS * 36) {
        int min_tiles = 1 << 30;
        for (int s = 0; s < a.m.M; ++s) min_tiles = min(min_tiles, (a.m.sb[s + 1] - a.m.sb[s] + a.m.T - 1) / a.m.T);
        int dev = 0, sms = 132;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        const int pinned = target->mlp->cluster_size;
        while (cs * 2 <= 4 && cs * 2 <= min_tiles && (pinned ? cs * 2 <= pinned : C * cs * 2 <= sms)) cs *= 2;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(C * cs);
    cfg.blockDim = dim3(MLP_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = cs; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    void (*kern)(MlpRunArgs);
    if (hyper || temper) kern = cs == 4 ? mlp_run_kernel<4, true> : cs == 2 ? mlp_run_kernel<2, true> : mlp_run_kernel<1, true>;
    else kern = cs == 4 ? mlp_run_kernel<4, false> : cs == 2 ? mlp_run_kernel<2, false> : mlp_run_kernel<1, false>;
    rc = prepare_smem(kern, smem);
    if (rc != HMCX_OK) return rc;
    if (cudaLaunchKernelEx(&cfg, kern, a) != cudaSuccess) { cudaGetLastError(); return HMCX_ERR_CUDA; }
    return cuda_status();
}

int mlp_grad_log_prob(const hmcx_target_t* target, const float* q, int C, int ld, int split, float* grad_out,
                      float* log_prob_out, cudaStream_t st) {
    MlpDev m = {};
    int rc = fill_mlp(target, m);
    if (rc != HMCX_OK) return rc;
    if (!q || C < 1 || ld < m.D || (ld & 3) || split < -1 || split >= m.M || (!grad_out && !log_prob_out))
        return HMCX_ERR_INVALID_ARG;
    if (!mlp_pick_tile(m, 2, target->mlp->tensor_cores != HMCX_MLP_TC_OFF)) return HMCX_ERR_UNSUPPORTED;
    const size_t smem = (size_t)(m.tile_base + m.tile_floats) * sizeof(float);
    rc = prepare_smem(mlp_grad_kernel, smem);
    if (rc != HMCX_OK) return rc;
    mlp_grad_kernel<<<C, MLP_THREADS, smem, st>>>(m, q, ld, split, grad_out, log_prob_out);
    return cuda_status();
}

int mlp_predict(const hmcx_target_t* target, const float* samples, int S, int ld, float* pred_out, float* log_prob_out,
                cudaStream_t st) {
    MlpDev m = {};
    int rc = fill_mlp(target, m);
    if (rc != HMCX_OK) return rc;
    if (!samples || !pred_out || S < 1 || ld < m.D || (ld & 3) || !m.has_data) return HMCX_ERR_INVALID_ARG;
    if (!mlp_pick_tile(m, 1, target->mlp->tensor_cores != HMCX_MLP_TC_OFF)) return HMCX_ERR_UNSUPPORTED;
    const size_t smem = (size_t)(m.tile_base + m.tile_floats) * sizeof(float);
    rc = prepare_smem(mlp_predict_kernel, smem);
    if (rc != HMCX_OK) return rc;
    mlp_predict_kernel<<<S, MLP_THREADS, smem, st>>>(m, samples, ld, pred_out, log_prob_out);
    return cuda_status();
}

// fill_mlp, the argument checks, the tile pick and the shared-memory opt-in of the pointwise entries: C x n draws, one
// CTA each, over the rows [r_begin, r_end) into a strided block; args_ok: the entry's own checks
template <typename Kern>
static int mlp_draw_pass_setup(const hmcx_target_t* target, MlpDev& m, Kern kern, const float* samples, long long cs,
                               long long ds, int C, int n, int r_begin, int r_end, const float* out, long long ocs,
                               long long ods, bool args_ok, size_t& smem) {
    const int rc = fill_mlp(target, m);
    if (rc != HMCX_OK) return rc;
    if (!samples || !out || C < 1 || n < 1 || (long long)C * n > 0x7fffffffLL || cs < 0 || ds < 0 || ocs < 0 ||
        ods < 0 || !m.has_data || r_begin < 0 || r_end > m.N || r_begin >= r_end || !args_ok)
        return HMCX_ERR_INVALID_ARG;
    if (!mlp_pick_tile(m, 1, target->mlp->tensor_cores != HMCX_MLP_TC_OFF)) return HMCX_ERR_UNSUPPORTED;
    smem = (size_t)(m.tile_base + m.tile_floats) * sizeof(float);
    return prepare_smem(kern, smem);
}

int mlp_pointwise_ll(const hmcx_target_t* target, const float* samples, long long cs, long long ds, int C, int n,
                     int r_begin, int r_end, float* ll, long long lcs, long long lds, cudaStream_t st,
                     const float* tau, long long tcs, long long tds) {
    MlpDev m = {};
    size_t smem = 0;
    const int rc = mlp_draw_pass_setup(target, m, mlp_ll_kernel, samples, cs, ds, C, n, r_begin, r_end, ll, lcs, lds,
                                       tcs >= 0 && tds >= 0, smem);
    if (rc != HMCX_OK) return rc;
    // the target's constant is evaluated here once, a per-draw block's by the kernel
    const float ll_const =
        tau ? 0.0f : (float)(0.5 * m.n[m.L] * log((double)m.tau_out / (2.0 * 3.14159265358979323846)));
    mlp_ll_kernel<<<C * n, MLP_THREADS, smem, st>>>(m, samples, cs, ds, n, r_begin, r_end, ll_const, tau, tcs, tds, ll,
                                                    lcs, lds);
    return cuda_status();
}

int mlp_pointwise_out(const hmcx_target_t* target, const float* samples, long long cs, long long ds, int C, int n,
                      int r_begin, int r_end, float* out, long long ocs, long long ods, cudaStream_t st) {
    MlpDev m = {};
    size_t smem = 0;
    const int rc = mlp_draw_pass_setup(target, m, mlp_out_kernel, samples, cs, ds, C, n, r_begin, r_end, out, ocs, ods,
                                       true, smem);
    if (rc != HMCX_OK) return rc;
    mlp_out_kernel<<<C * n, MLP_THREADS, smem, st>>>(m, samples, cs, ds, n, r_begin, r_end, out, ocs, ods);
    return cuda_status();
}

// stand-alone samplers.leapfrog with Integrator.SPLITTING / _RAND / _KMID (:494-603) over C chains: one "iteration" of the run
// kernel with the momentum given, no Hamiltonian and no MH; q_traj / p_traj [L, C, ld] take the state after every step
int mlp_leapfrog(const hmcx_target_t* target, const hmcx_mass_t* mass, const hmcx_rng_t* rng, int scheme, double step_size,
                 const float* q_in, const float* p_in, float* eps, int C, int ld, int L, float* q_traj, float* p_traj,
                 cudaStream_t st) {
    if (!p_in || !q_traj || !p_traj || scheme == HMCX_SCHEME_PLAIN) return HMCX_ERR_INVALID_ARG;
    hmcx_nuts_t no_nuts = {};
    no_nuts.step_size_init = step_size;                        // the Python double the drifts divide (:513, :558)
    return mlp_split_run(target, mass, rng, &no_nuts, scheme, q_in, const_cast<float*>(q_in), eps, C, ld, L, 1, 0, 0, 1,
                         nullptr, nullptr, nullptr, nullptr, nullptr, st, p_in, q_traj, p_traj, nullptr, nullptr, nullptr,
                         0);
}

// hmcx_hyper_gamma_draws: one thread per (iteration, chain, group), the device function of the hyperprior runs
struct GammaShapes { double v[HYPER_GROUPS]; };
__global__ void __launch_bounds__(256) hyper_gamma_kernel(uint64_t seed, uint64_t chain_offset, int C, int it0, int n_it,
                                                          int K, const GammaShapes shapes, double* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)n_it * C * K) return;
    const int k = (int)(i % K), c = (int)((i / K) % C), n = it0 + (int)(i / ((long long)K * C));
    out[i] = philox_std_gamma(seed, chain_offset + (uint64_t)c, (uint64_t)n, (uint32_t)k, shapes.v[k]);
}

int hyper_gamma_draws(uint64_t seed, uint64_t chain_offset, int C, int it0, int it1, int K, const double* shapes,
                      double* out, cudaStream_t st) {
    if (C < 1 || it0 < 0 || it1 <= it0 || K < 1 || K > HYPER_GROUPS || !shapes || !out) return HMCX_ERR_INVALID_ARG;
    GammaShapes sh = {};
    for (int k = 0; k < K; ++k) {
        if (!(shapes[k] > 0.0) || !(shapes[k] <= DBL_MAX)) return HMCX_ERR_INVALID_ARG;
        sh.v[k] = shapes[k];
    }
    const long long total = (long long)(it1 - it0) * C * K;
    hyper_gamma_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(seed, chain_offset, C, it0, it1 - it0, K, sh, out);
    return cuda_status();
}

// packed X operands of the tensor-core path (hmcx_mlp_t.x_packed): size in floats (0: the stack does not use it) / build
size_t mlp_packed_x_floats(const hmcx_target_t* target) {
    MlpDev m = {};
    if (fill_mlp(target, m) != HMCX_OK || !mlp_tc_shape(m)) return 0;
    return (size_t)mlp_packed_tiles(m) * 4 * TC_TR * m.n[0];
}

int mlp_pack_x(const hmcx_target_t* target, float* out, cudaStream_t st) {
    MlpDev m = {};
    const int rc = fill_mlp(target, m);
    if (rc != HMCX_OK) return rc;
    if (!out) return HMCX_ERR_INVALID_ARG;
    if (!mlp_tc_shape(m)) return HMCX_ERR_UNSUPPORTED;
    mlp_pack_x_kernel<<<mlp_packed_tiles(m), 256, 0, st>>>(m, out);
    return cuda_status();
}

#ifdef HMCX_TC_PROF
extern "C" int hmcx_debug_tc_prof(long long* out) {           // developer build only (scripts/prof_tc_phases.py)
    int n = 0;
    cudaDeviceSynchronize();
    cudaMemcpyFromSymbol(&n, g_tc_prof_n, sizeof(int));
    cudaMemcpyFromSymbol(out, g_tc_prof, sizeof(long long) * 512);
    int zero = 0;
    cudaMemcpyToSymbol(g_tc_prof_n, &zero, sizeof(int));
    return n;
}
#endif

}  // namespace hmcx
