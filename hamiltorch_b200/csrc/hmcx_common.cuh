// hmcx_common.cuh -- device helpers shared by the sm_90a HMC kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/hmcx.h"

#define HMCX_CHECK_ARG(cond) do { if (!(cond)) return HMCX_ERR_INVALID_ARG; } while (0)

namespace hmcx {

// ---------------------------------------------------------------------------------------------------------
// fp32 arithmetic in the reference's operation order: every product and sum is rounded separately
// (__fmul_rn/__fadd_rn are never contracted into FMA), because the reference evaluates e.g.
// ``params + step_size * momentum`` (samplers.py:284) as two ATen kernels.
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }

__device__ __forceinline__ bool finite_f(float x) { return fabsf(x) <= 3.402823466e+38f; }

// Neumaier's compensated accumulation: s + c carries the running sum to ~2^-46 relative whatever the number of terms
// (the sample sink exists for LONG runs: a naive fp32 running sum of x^2 loses the variance once |mean| >> std).  Plain
// fp32 adds, never contracted or re-associated.
__device__ __forceinline__ void comp_add(float& s, float& c, float x) {
    const float t = add(s, x);
    const float e = (fabsf(s) >= fabsf(x)) ? add(sub(s, t), x) : add(sub(x, t), s);
    c = add(c, e);
    s = t;
}

// ---------------------------------------------------------------------------------------------------------
// Philox4x32-10 counter RNG (Salmon et al. 2011).  Counter = (element-vector index, iteration lo, iteration hi
// | stream<<24, chain lo), key = seed ^ (chain hi).  One call yields the 4 normals of one float4 vector.
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(M0, c.x), lo0 = M0 * c.x;
        const uint32_t hi1 = __umulhi(M1, c.z), lo1 = M1 * c.z;
        c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
        k.x += W0; k.y += W1;
    }
    return c;
}

enum { STREAM_MOMENTUM = 0, STREAM_ACCEPT = 1, STREAM_JITTER = 2, STREAM_PERM = 3, STREAM_HYPER = 4, STREAM_SWAP = 5,
       STREAM_SBC_PRIOR = 6, STREAM_SBC_DATA = 7, STREAM_PPC = 8 };

// The key schedule k_r = k_0 + r*(W0, W1) depends on (seed, chain) only: a persistent kernel that owns one chain computes it
// once and keeps the 20 words in registers (the asm makes them opaque, otherwise the compiler re-derives each with an
// IADD3 per round and iteration: 20 of the ~60 instructions of a Philox call).
struct PhiloxKeys { uint32_t x[10], y[10]; };
__device__ __forceinline__ void philox_make_keys(uint64_t seed, uint64_t chain, PhiloxKeys& K) {
    uint32_t kx = (uint32_t)seed, ky = (uint32_t)(seed >> 32) ^ (uint32_t)(chain >> 32);
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        K.x[r] = kx; K.y[r] = ky;
        asm volatile("" : "+r"(K.x[r]), "+r"(K.y[r]));
        kx += 0x9E3779B9u; ky += 0xBB67AE85u;
    }
}
__device__ __forceinline__ uint4 philox_draw(const PhiloxKeys& K, uint64_t chain, uint64_t iter, uint32_t vec,
                                             uint32_t stream) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u;
    uint4 c = make_uint4(vec, (uint32_t)iter, (uint32_t)(iter >> 32) | (stream << 24), (uint32_t)chain);
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(M0, c.x), lo0 = M0 * c.x;
        const uint32_t hi1 = __umulhi(M1, c.z), lo1 = M1 * c.z;
        c = make_uint4(hi1 ^ c.y ^ K.x[r], lo1, hi0 ^ c.w ^ K.y[r], lo0);
    }
    return c;
}

// A persistent kernel draws the same (vec, stream, chain) counter at every iteration: only the iteration's low word
// changes (iter < 2^32, so the high word is 0).  Everything of rounds 1-3 that does not depend on it is computed once per
// thread: in round 1 all but the XOR with iter, in round 2 the product of word z, in round 3 the product of word x and
// the XORs with the key.  philox_draw(K, PhiloxFixed, iter) then yields the bits of philox_draw(K, chain, iter, vec, stream).
struct PhiloxFixed { uint32_t x1, w1k, y2k, z3k, w3; };
__device__ __forceinline__ void philox_fix(const PhiloxKeys& K, uint64_t chain, uint32_t vec, uint32_t stream,
                                           PhiloxFixed& F) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u;
    const uint32_t cz = stream << 24;
    const uint32_t x1 = __umulhi(M1, cz) ^ K.x[0], y1 = M1 * cz;              // round 1 (x1 ^ iter is the real x)
    const uint32_t z1 = __umulhi(M0, vec) ^ (uint32_t)chain ^ K.y[0], w1 = M0 * vec;
    const uint32_t x2 = __umulhi(M1, z1) ^ y1 ^ K.x[1], y2 = M1 * z1;        // round 2
    F.x1 = x1;
    F.w1k = w1 ^ K.y[1];
    F.y2k = y2 ^ K.x[2];                                                      // round 3
    F.z3k = __umulhi(M0, x2) ^ K.y[2];
    F.w3 = M0 * x2;
}
__device__ __forceinline__ uint4 philox_draw(const PhiloxKeys& K, const PhiloxFixed& F, uint32_t iter) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u;
    const uint32_t x1 = F.x1 ^ iter;
    const uint32_t z2 = __umulhi(M0, x1) ^ F.w1k, w2 = M0 * x1;
    uint4 c = make_uint4(__umulhi(M1, z2) ^ F.y2k, M1 * z2, F.z3k ^ w2, F.w3);
#pragma unroll
    for (int r = 3; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(M0, c.x), lo0 = M0 * c.x;
        const uint32_t hi1 = __umulhi(M1, c.z), lo1 = M1 * c.z;
        c = make_uint4(hi1 ^ c.y ^ K.x[r], lo1, hi0 ^ c.w ^ K.y[r], lo0);
    }
    return c;
}

__device__ __forceinline__ uint4 philox_draw(uint64_t seed, uint64_t chain, uint64_t iter, uint32_t vec,
                                             uint32_t stream) {
    uint4 c = make_uint4(vec, (uint32_t)iter, (uint32_t)(iter >> 32) | (stream << 24), (uint32_t)chain);
    uint2 k = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32) ^ (uint32_t)(chain >> 32));
    return philox4x32_10(c, k);
}

// uniform in (0,1]: never 0, so log() is finite
__device__ __forceinline__ float u01(uint32_t x) { return fmaf((float)x, 2.3283064365386963e-10f, 1.1641532182693481e-10f); }

// Box-Muller: two uniforms -> two independent N(0,1).  The kernel is fp32-issue bound, so the transform is written for
// instruction count: MUFU.LG2 / MUFU.SQRT / MUFU.SIN / MUFU.COS through the .approx.ftz PTX forms (u >= 2^-33 is never
// denormal, so the range checks of logf / sqrtf are dead weight), -2 ln 2 folded into one constant, and the angle
// 2 pi (u - 1/2) produced by a single FFMA from the raw 32-bit draw.  Absolute error of a normal ~1e-6.
__device__ __forceinline__ float lg2_approx(float x) { float y; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float sqrt_approx(float x) { float y; asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ void box_muller(uint32_t a, uint32_t b, float& z0, float& z1) {
    const float r = sqrt_approx(lg2_approx(u01(a)) * -1.3862943611198906f);          // sqrt(-2 ln u)
    float s, c;
    __sincosf(fmaf((float)b, 1.4629180792671596e-09f, -3.1415926521268f), &s, &c);   // 2 pi (b + 1/2) 2^-32 - pi
    z0 = r * c;
    z1 = r * s;
}

// ---------------------------------------------------------------------------------------------------------
// One data element simulated from a Bayesian NN's likelihood at the network output f: the definitions hmcx_sbc_simulate
// (prior predictive) and hmcx_ppc_pass (posterior predictive) share, so both give the same bits for the same words.
// ---------------------------------------------------------------------------------------------------------
// regression: f + z sd, sd = 1 / sqrt(tau_out) rounded to fp32 (noise_sd)
__device__ __forceinline__ float noise_sd(float tau) { return (float)(1.0 / sqrt((double)tau)); }
__device__ __forceinline__ float sim_gaussian(float f, float z, float sd) { return add(f, mul(z, sd)); }
// binary: 1 when the uniform word is below sigmoid(f) (fp64), else 0
__device__ __forceinline__ float sim_bernoulli(float f, uint32_t w) {
    const double p = 1.0 / (1.0 + exp(-(double)f));
    return (double)u01(w) < p ? 1.0f : 0.0f;
}
// multi-class: Categorical(softmax f) over O classes, e_c = exp(f_c - max f) in class order (fp64); the label is the first
// class c with u * sum_c' e_c' <= e_0 + ... + e_c (the last class if rounding leaves none)
__device__ __forceinline__ int sim_categorical(const float* fr, int O, uint32_t w) {
    double mx = (double)fr[0];
    for (int c = 1; c < O; ++c) mx = fmax(mx, (double)fr[c]);
    double tot = 0.0;
    for (int c = 0; c < O; ++c) tot += exp((double)fr[c] - mx);
    const double t = (double)u01(w) * tot;
    double cum = 0.0;
    for (int c = 0; c < O - 1; ++c) {
        cum += exp((double)fr[c] - mx);
        if (t <= cum) return c;
    }
    return O - 1;
}

// Canonical momentum stream (identical for every kernel geometry): one Philox call per float4 VECTOR of the chain
// and per iteration; r = (x,y,z,w): elements 4v,4v+1 <- Box-Muller(x,y), elements 4v+2,4v+3 <- Box-Muller(z,w).
__device__ __forceinline__ void philox_normal4(uint64_t seed, uint64_t chain, uint64_t iter, uint32_t vec,
                                               float z[4]) {
    const uint4 r = philox_draw(seed, chain, iter, vec, STREAM_MOMENTUM);
    box_muller(r.x, r.y, z[0], z[1]);
    box_muller(r.z, r.w, z[2], z[3]);
}
// the two normals of element pair `pair` (= elements 2*pair, 2*pair+1): half of vector pair>>1
__device__ __forceinline__ void philox_normal2(uint64_t seed, uint64_t chain, uint64_t iter, uint32_t pair,
                                               float z[2]) {
    const uint4 r = philox_draw(seed, chain, iter, pair >> 1, STREAM_MOMENTUM);
    if (pair & 1) box_muller(r.z, r.w, z[0], z[1]);
    else box_muller(r.x, r.y, z[0], z[1]);
}
// the same streams from a precomputed key schedule and the thread's fixed rounds (F from philox_fix with
// vec = E == 4 ? grp : grp >> 1, STREAM_MOMENTUM)
template <int E> __device__ __forceinline__ void philox_normals(const PhiloxKeys& K, const PhiloxFixed& F, uint32_t iter,
                                                                uint32_t grp, float* z) {
    const uint4 r = philox_draw(K, F, iter);
    if (E == 4) {
        box_muller(r.x, r.y, z[0], z[1]);
        box_muller(r.z, r.w, z[2], z[3]);
    } else if (grp & 1) {
        box_muller(r.z, r.w, z[0], z[1]);
    } else {
        box_muller(r.x, r.y, z[0], z[1]);
    }
}
template <int E> __device__ __forceinline__ void philox_normals(uint64_t seed, uint64_t chain, uint64_t iter,
                                                                uint32_t grp, float* z);
template <> __device__ __forceinline__ void philox_normals<4>(uint64_t seed, uint64_t chain, uint64_t iter,
                                                              uint32_t grp, float* z) {
    philox_normal4(seed, chain, iter, grp, z);
}
template <> __device__ __forceinline__ void philox_normals<2>(uint64_t seed, uint64_t chain, uint64_t iter,
                                                              uint32_t grp, float* z) {
    philox_normal2(seed, chain, iter, grp, z);
}

__device__ __forceinline__ float philox_log_uniform(const PhiloxKeys& K, uint64_t chain, uint64_t iter) {
    const uint4 r = philox_draw(K, chain, iter, 0xFFFFFFFFu, STREAM_ACCEPT);
    return logf(u01(r.x));
}
__device__ __forceinline__ float philox_log_uniform(uint64_t seed, uint64_t chain, uint64_t iter) {
    const uint4 r = philox_draw(seed, chain, iter, 0xFFFFFFFFu, STREAM_ACCEPT);
    return logf(u01(r.x));
}

// Jitter stream: the torch.rand(D) that fisher() call `call` of an iteration draws (samplers.py:115).  Each call owns
// JITTER_VECS_PER_CALL counter vectors, one Philox call per 4 elements, so a row of up to 64 elements never reaches the
// next call's counters (hmcx_rmhmc_cta.cu ties this to its largest D).  Element 4*vec+j <- (word j >> 8) * 2^-24 in [0, 1).
constexpr int JITTER_VECS_PER_CALL = 16;
__device__ __forceinline__ void philox_jitter4(uint64_t seed, uint64_t chain, uint64_t iter, int call, int vec,
                                               float u[4]) {
    const uint4 r = philox_draw(seed, chain, iter, (uint32_t)(call * JITTER_VECS_PER_CALL + vec), STREAM_JITTER);
    u[0] = (float)(r.x >> 8) * 5.9604645e-8f;
    u[1] = (float)(r.y >> 8) * 5.9604645e-8f;
    u[2] = (float)(r.z >> 8) * 5.9604645e-8f;
    u[3] = (float)(r.w >> 8) * 5.9604645e-8f;
}

// Standard Gamma(alpha) draw of the hyperprior Gibbs step (Marsaglia & Tsang 2000), in fp64.  Attempt t of group k reads
// the Philox block (seed, chain, iter, k << 16 | t) of STREAM_HYPER: a 53-bit uniform from words x, y and a 32-bit one from
// z give the normal (Box-Muller), w the acceptance uniform.  Shapes below 1 draw G(alpha + 1) U^(1/alpha), U from the block
// k << 16 | 0xFFFF.  The counters depend on (seed, global chain, iteration, group) only, never on the launch geometry.
__device__ __forceinline__ double u01_53(uint32_t hi, uint32_t lo) {          // (0, 1)
    return ((double)(((uint64_t)hi << 21) | (lo >> 11)) + 0.5) * 1.1102230246251565e-16;
}
static __device__ __noinline__ double philox_std_gamma(uint64_t seed, uint64_t chain, uint64_t iter, uint32_t group, double alpha) {
    const bool boost = alpha < 1.0;
    const double d = (boost ? alpha + 1.0 : alpha) - 1.0 / 3.0, c = 1.0 / sqrt(9.0 * d);
    double g = 0.0;
    for (uint32_t t = 0; t < 0xFFFFu; ++t) {
        const uint4 r = philox_draw(seed, chain, iter, (group << 16) | t, STREAM_HYPER);
        const double u1 = u01_53(r.x, r.y), u2 = ((double)r.z + 0.5) * 2.3283064365386963e-10;
        const double u3 = ((double)r.w + 0.5) * 2.3283064365386963e-10;
        const double z = sqrt(-2.0 * log(u1)) * cospi(2.0 * u2);
        double v = 1.0 + c * z;
        if (v <= 0.0) continue;
        v = v * v * v;
        if (log(u3) < 0.5 * z * z + d - d * v + d * log(v)) { g = d * v; break; }
    }
    if (boost) {
        const uint4 r = philox_draw(seed, chain, iter, (group << 16) | 0xFFFFu, STREAM_HYPER);
        g *= pow(u01_53(r.x, r.y), 1.0 / alpha);
    }
    return g;
}

// ---------------------------------------------------------------------------------------------------------
// reductions.  xor-butterflies: every lane ends with the same bits (fp add is commutative and each level pairs
// identical operands), so all threads of a CTA take identical decisions without a broadcast.
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = add(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// Three sums over a warp with a packed butterfly: 9 shuffles instead of 15.  After the xor-16 / xor-8 exchange
// lanes [0,8) own a, [8,16) own b, [16,24) own c; three more levels finish each, then the totals are broadcast, so
// every lane returns the same bits.
__device__ __forceinline__ void warp_sum3(float& a, float& b, float& c, bool broadcast) {
    const int lane = threadIdx.x & 31;
    const bool h16 = lane & 16, h8 = lane & 8;
    float k0 = h16 ? c : a, k1 = h16 ? 0.0f : b;
    const float s0 = h16 ? a : c, s1 = h16 ? b : 0.0f;
    k0 = add(k0, __shfl_xor_sync(0xffffffffu, s0, 16));
    k1 = add(k1, __shfl_xor_sync(0xffffffffu, s1, 16));
    float k = h8 ? k1 : k0;
    const float s = h8 ? k0 : k1;
    k = add(k, __shfl_xor_sync(0xffffffffu, s, 8));
    k = add(k, __shfl_xor_sync(0xffffffffu, k, 4));
    k = add(k, __shfl_xor_sync(0xffffffffu, k, 2));
    k = add(k, __shfl_xor_sync(0xffffffffu, k, 1));
    if (broadcast) {
        a = __shfl_sync(0xffffffffu, k, 0);
        b = __shfl_sync(0xffffffffu, k, 8);
        c = __shfl_sync(0xffffffffu, k, 16);
    } else {
        a = k;          // valid in lane 0 (a), lane 8 (b), lane 16 (c)
    }
}

// Sum 3 values over the CTA and hand every thread one extra scalar produced by thread 0 (`extra`, e.g. the
// iteration's log-uniform) through the same shared buffer and the same single barrier.
// `sbuf` holds 3*32+1 floats; callers alternate between two buffers on consecutive calls.
__device__ __forceinline__ void block_sum3(float& a, float& b, float& c, float& extra, float* sbuf) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = (blockDim.x + 31) >> 5;
    if (nwarp == 1) {
        warp_sum3(a, b, c, true);
        extra = __shfl_sync(0xffffffffu, extra, 0);
        return;
    }
    warp_sum3(a, b, c, false);
    if ((lane & 7) == 0 && lane < 24) sbuf[(lane >> 3) * 32 + warp] = a;
    if (threadIdx.x == 0) sbuf[96] = extra;
    __syncthreads();
    a = lane < nwarp ? sbuf[lane] : 0.0f;
    b = lane < nwarp ? sbuf[32 + lane] : 0.0f;
    c = lane < nwarp ? sbuf[64 + lane] : 0.0f;
    extra = sbuf[96];
    warp_sum3(a, b, c, true);
}

// Sum N values over the CTA (generic, used off the hot loop).  `sbuf` holds 32*N floats.
template <int N>
__device__ __forceinline__ void block_sum(float (&v)[N], float* sbuf) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = (blockDim.x + 31) >> 5;
#pragma unroll
    for (int i = 0; i < N; ++i) v[i] = warp_sum(v[i]);
    if (nwarp == 1) return;
    if (lane == 0) {
#pragma unroll
        for (int i = 0; i < N; ++i) sbuf[warp * N + i] = v[i];
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < N; ++i) v[i] = warp_sum(lane < nwarp ? sbuf[lane * N + i] : 0.0f);
}

// 16-byte vector access helpers
__device__ __forceinline__ void ld4(const float* p, float v[4]) {
    const float4 t = *reinterpret_cast<const float4*>(p);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
__device__ __forceinline__ void ld4_stream(const float* p, float v[4]) {   // read-once data: don't keep in L1
    const float4 t = __ldcs(reinterpret_cast<const float4*>(p));
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
__device__ __forceinline__ void st4(float* p, const float v[4]) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
}
__device__ __forceinline__ void st4_stream(float* p, const float v[4]) {   // write-once data: evict first
    __stcs(reinterpret_cast<float4*>(p), make_float4(v[0], v[1], v[2], v[3]));
}


// E-wide (E = 2 or 4) contiguous element groups
template <int E> __device__ __forceinline__ void ldE(const float* p, float* v);
template <> __device__ __forceinline__ void ldE<4>(const float* p, float* v) { ld4(p, v); }
template <> __device__ __forceinline__ void ldE<2>(const float* p, float* v) {
    const float2 t = *reinterpret_cast<const float2*>(p); v[0] = t.x; v[1] = t.y;
}
template <int E> __device__ __forceinline__ void ldE_stream(const float* p, float* v);
template <> __device__ __forceinline__ void ldE_stream<4>(const float* p, float* v) { ld4_stream(p, v); }
template <> __device__ __forceinline__ void ldE_stream<2>(const float* p, float* v) {
    const float2 t = __ldcs(reinterpret_cast<const float2*>(p)); v[0] = t.x; v[1] = t.y;
}
template <int E> __device__ __forceinline__ void stE(float* p, const float* v);
template <> __device__ __forceinline__ void stE<4>(float* p, const float* v) { st4(p, v); }
template <> __device__ __forceinline__ void stE<2>(float* p, const float* v) {
    *reinterpret_cast<float2*>(p) = make_float2(v[0], v[1]);
}
template <int E> __device__ __forceinline__ void stE_stream(float* p, const float* v);
template <> __device__ __forceinline__ void stE_stream<4>(float* p, const float* v) { st4_stream(p, v); }
template <> __device__ __forceinline__ void stE_stream<2>(float* p, const float* v) {
    __stcs(reinterpret_cast<float2*>(p), make_float2(v[0], v[1]));
}

}  // namespace hmcx
