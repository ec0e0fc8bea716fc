// hmcx_hmc.cu -- plain-HMC hot path for element-wise targets (isotropic / diagonal Gaussians) on sm_90a (H100).
//
// Replaces, for a batch of C independent chains, the reference's per-chain Python loop
//   samplers.py:965-1067  (sample: gibbs -> hamiltonian -> leapfrog -> hamiltonian -> MH -> bookkeeping -> adaptation)
//   samplers.py:269-304   (leapfrog, plain HMC branch)      samplers.py:779-815 (hamiltonian, HMC branch)
//   samplers.py:185-202   (gibbs)                           samplers.py:629-674 (adaptation)
//
// Kernels
//   hmc_run_kernel<TK,MK,E,K>  persistent: one CTA owns one chain for ALL iterations of the launch.  The chain's
//       position, proposal and momentum live in registers (K groups of E contiguous elements per thread,
//       D <= E*K*blockDim), the whole L-step trajectory is thread-private for these targets, the only cross-thread
//       traffic per iteration is ONE fused block reduction of (p0.M^-1.p0, U(q_L) terms, p_L.M^-1.p_L) that also
//       carries the iteration's log-uniform, and HBM sees one coalesced store of the retained sample (+ one read
//       of injected normals in parity mode).
//   leapfrog_kernel<TK,MK>   streaming form of samplers.leapfrog for (C, ld) state arrays in HBM (grid-stride
//       float4; 16 B/element moved once, all L steps in registers).  This is the HBM-roofline kernel.
//   hamiltonian_kernel<TK,MK>, gibbs_kernel<MK>   the remaining stand-alone pieces of the reference surface.
#include <cstdlib>
#include "hmcx_common.cuh"

namespace hmcx {

struct ElemTarget {           // element-wise target + mass description, passed by value
    int tk, mk;
    int D, ld, C;
    const float* mean;
    const float* ivar;
    const float* im;          // inv_mass [D]
    const float* sd;          // sqrt(mass) [D]
    float log_norm;
    uint32_t vpr_magic;       // ceil(2^vpr_shift / (ld/4)): row = (v * magic) >> shift for v < 2^31 (Granlund-Montgomery)
    int vpr_shift;
};

// per-group constants kept in registers (dead members are eliminated for ISO / MASS_NONE)
template <int E>
struct VecConst { float mean[E], ivar[E], im[E], sd[E]; };

template <int TK, int MK, int E>
__device__ __forceinline__ void load_consts(const ElemTarget& t, int e0, VecConst<E>& c) {
#pragma unroll
    for (int j = 0; j < E; ++j) {
        const bool ok = (e0 + j) < t.D;
        if (TK == HMCX_TARGET_GAUSS_DIAG) {
            c.mean[j] = (ok && t.mean) ? t.mean[e0 + j] : 0.0f;
            c.ivar[j] = ok ? t.ivar[e0 + j] : 0.0f;
        }
        if (MK == HMCX_MASS_DIAG) {
            c.im[j] = ok ? t.im[e0 + j] : 0.0f;
            c.sd[j] = ok ? t.sd[e0 + j] : 0.0f;
        }
    }
}

// g = d log p / dq_i in the op order autograd produces for targets.py (GaussianIso: -x; GaussianDiag: -(iv*(x-m)))
template <int TK>
__device__ __forceinline__ float grad1(float q, float mean, float ivar) {
    if (TK == HMCX_TARGET_GAUSS_ISO) return -q;
    return -mul(ivar, sub(q, mean));
}
// -grad1, exactly
template <int TK>
__device__ __forceinline__ float neg_grad1(float q, float mean, float ivar) {
    if (TK == HMCX_TARGET_GAUSS_ISO) return q;
    return mul(ivar, sub(q, mean));
}
// summand of -2*(log p - log_norm)
template <int TK>
__device__ __forceinline__ float uterm1(float q, float mean, float ivar) {
    if (TK == HMCX_TARGET_GAUSS_ISO) return mul(q, q);
    const float y = sub(q, mean);
    return mul(mul(y, y), ivar);
}
// samplers.py:284 / :296
template <int MK>
__device__ __forceinline__ float drift1(float q, float eps, float im, float p) {
    if (MK == HMCX_MASS_NONE) return add(q, mul(eps, p));
    return add(q, mul(mul(eps, im), p));
}
// summand of 2*kinetic, samplers.py:801 / :814
template <int MK>
__device__ __forceinline__ float kterm1(float p, float im) {
    if (MK == HMCX_MASS_NONE) return mul(p, p);
    return mul(p, mul(im, p));
}
// s + x for the terms of a per-thread partial sum (s = 0 before the first).  A first term that is a square is never -0,
// so 0 + x == x bit for bit and the sum starts with it: the ISO potential and the kinetic term without a mass matrix.
template <bool SQUARE>
__device__ __forceinline__ float sum_in(float s, float x, bool first) { return (SQUARE && first) ? x : add(s, x); }

// log p from the reduced sum, targets.py op order: -0.5*sum (+ log_norm)
__device__ __forceinline__ float log_prob_from_sum(float s, float log_norm) { return add(mul(-0.5f, s), log_norm); }

// One group of E elements through a whole trajectory (samplers.py:281-302).  Optionally records the L clones.
// The gradient is recomputed for the final half-kick rather than carried out of the step loop: the same value, and a
// loop-carried g would have to be materialised (one negation or more per element and step) on every trip.
template <int TK, int MK, int E, bool TRAJ>
__device__ __forceinline__ void trajectory(float* q, float* p, const VecConst<E>& c, float eps, float half, int L,
                                           float* q_traj, float* p_traj, size_t traj_stride) {
#pragma unroll
    for (int j = 0; j < E; ++j) p[j] = add(p[j], mul(half, grad1<TK>(q[j], c.mean[j], c.ivar[j])));   // :281
    auto one_step = [&](int l) {
#pragma unroll
        for (int j = 0; j < E; ++j) {
            q[j] = drift1<MK>(q[j], eps, c.im[j], p[j]);                     // :284 / :296
            p[j] = add(p[j], mul(eps, grad1<TK>(q[j], c.mean[j], c.ivar[j])));   // :297-298
        }
        if (TRAJ) {
            if (l + 1 < L) {                                                 // :299-300
                stE_stream<E>(q_traj + (size_t)l * traj_stride, q);
                stE_stream<E>(p_traj + (size_t)l * traj_stride, p);
            }
        }
    };
    int l = 0;
#pragma unroll 1
    for (; l + 2 <= L; l += 2) { one_step(l); one_step(l + 1); }             // halve the loop overhead; no deeper
                                                                             // unrolling: the sample() loop body must stay
                                                                             // inside the instruction cache
    if (l < L) one_step(l);
#pragma unroll
    for (int j = 0; j < E; ++j) p[j] = sub(p[j], mul(half, grad1<TK>(q[j], c.mean[j], c.ivar[j])));   // :302
    if (TRAJ) {
        stE_stream<E>(q_traj + (size_t)(L - 1) * traj_stride, q);
        stE_stream<E>(p_traj + (size_t)(L - 1) * traj_stride, p);
    }
}

// The same trajectory for NG groups of one thread in one step loop: every trip advances all NG*E elements, so a thread
// with two groups runs 8 independent element chains per step instead of two loops of 4.  Element-wise, so the bits are
// those of trajectory<> on each group.
// `side()` is independent work (the next iteration's normals) placed after the first half-kick and the first step,
// which are peeled out of the step loop (L >= 1) so that the three share one basic block: the side work's dependent
// chains then interleave with 8 independent element chains instead of standing alone in the iteration's serial tail.
template <int TK, int MK, int E, int NG, typename F>
__device__ __forceinline__ void trajectory_groups(float (*q)[E], float (*p)[E], const VecConst<E>* c, float eps,
                                                  float half, int L, F&& side) {
#pragma unroll
    for (int g = 0; g < NG; ++g)
#pragma unroll
        for (int j = 0; j < E; ++j) p[g][j] = add(p[g][j], mul(half, grad1<TK>(q[g][j], c[g].mean[j], c[g].ivar[j])));
    auto one_step = [&]() {
#pragma unroll
        for (int g = 0; g < NG; ++g)
#pragma unroll
            for (int j = 0; j < E; ++j) {
                q[g][j] = drift1<MK>(q[g][j], eps, c[g].im[j], p[g][j]);
                p[g][j] = add(p[g][j], mul(eps, grad1<TK>(q[g][j], c[g].mean[j], c[g].ivar[j])));
            }
    };
    one_step();
    side();
    int l = 1;
#pragma unroll 1
    for (; l + 2 <= L; l += 2) { one_step(); one_step(); }
    if (l < L) one_step();
    // p - half*g as p + half*(-g): half*(-g) == -(half*g) and p - (-y) == p + y in round-to-nearest, bit for bit.  With
    // -g the compiler materialised the negation of every element where the odd and even step counts join (8 FADDs).
#pragma unroll
    for (int g = 0; g < NG; ++g)
#pragma unroll
        for (int j = 0; j < E; ++j) p[g][j] = add(p[g][j], mul(half, neg_grad1<TK>(q[g][j], c[g].mean[j], c[g].ivar[j])));
}

// ---------------------------------------------------------------------------------------------------------
// persistent sample() kernel
// ---------------------------------------------------------------------------------------------------------
struct RunArgs {
    ElemTarget t;
    // rng
    int rng_mode;
    uint64_t seed, chain_offset;
    const float* normals;
    const float* logu;
    // nuts.  The mass-adaptation fields of the SINK instantiations (ABI v11) sit in what was alignment padding, so that
    // every other instantiation keeps its parameter layout and code: mu_per_chain = 1 selects the per-chain mu of the
    // restarted dual averaging (hmcx_nuts_t.mu_chain), which then shares the storage of the scalar mu
    int nuts;
    int mu_per_chain;
    double delta;
    union {
        double mu;
        const double* mu_chain;
    };
    const double* table;
    double* h_bar;
    double* eps_bar;
    const float* eps_schedule;   // [S, C] teacher forcing (parity tests), may be null
    float* eps_trace;            // [C, S] the kernel's own step size for iteration n+1, may be null
    // state / outputs
    const float* q_init;
    float* q_cur;
    float* eps;
    int L, S, burn, it0, it1;
    float* samples;
    uint8_t* accept;
    uint8_t* diverged;
    float* ham;
    int32_t* num_rejected;
    // sample sink (hmcx_sink_t): thinning + running first / second moments of the post-burn states (of every iteration of
    // the launch with moments_all: a mass-adaptation window)
    int thin;
    int moments_all;
    float* msum;
    float* msumsq;
    float* msum_lo;           // optional: the compensation terms of the running sums (true sum = hi + lo)
    float* msumsq_lo;
    // windows of iterations: [C] log p(q_cur) left by the launch that ended at iter_begin (the loop carries it in a register
    // and its fused 3-value reduction does not associate like the prologue's recomputation: without the carry a run cut into
    // windows differs from a single launch in the last bit of H_old at every window start)
    float* lp_carry;
};

// block_sum3 for CTAs of at most 8 warps: the second level reads the warps' partials with broadcast LDS.128 and adds them
// in warp order (3 independent 8-term chains) instead of a second shuffle butterfly: ~90 cycles less latency on the
// per-iteration critical path, same instruction count, every thread ends with the same bits.
// `sbuf` holds 4*8+1 floats; callers alternate between two buffers on consecutive calls.  The slots of the warps the CTA
// does not have hold -0.0f (block_sum3_small_init): x + -0 == x for every x, so the second level adds all 8 slots
// without re-deriving from blockDim which warps exist.  `groups` = partial sums per thread (block_sum3_pair: 2).
__device__ __forceinline__ void block_sum3_small_init(float (*sbuf)[100], int groups = 1) {
    const int nwarp = (blockDim.x + 31) >> 5;
    if ((int)threadIdx.x >= 4 * groups * nwarp && threadIdx.x < 32) sbuf[0][threadIdx.x] = sbuf[1][threadIdx.x] = -0.0f;
}
// second level: every thread adds the 8 slots in warp order
__device__ __forceinline__ void block_sum3_slots(float& a, float& b, float& c, float& extra, const float* sbuf) {
    float4 v = *reinterpret_cast<const float4*>(sbuf);
    a = v.x; b = v.y; c = v.z;
#pragma unroll
    for (int w = 1; w < 8; ++w) {
        v = *reinterpret_cast<const float4*>(sbuf + 4 * w);
        a = add(a, v.x); b = add(b, v.y); c = add(c, v.z);
    }
    extra = sbuf[32];
}
__device__ __forceinline__ void block_sum3_small(float& a, float& b, float& c, float& extra, float* sbuf) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = (blockDim.x + 31) >> 5;
    if (nwarp == 1) {
        warp_sum3(a, b, c, true);
        extra = __shfl_sync(0xffffffffu, extra, 0);
        return;
    }
    warp_sum3(a, b, c, false);
    if ((lane & 7) == 0 && lane < 24) sbuf[4 * warp + (lane >> 3)] = a;
    if (threadIdx.x == 0) sbuf[32] = extra;
    __syncthreads();
    block_sum3_slots(a, b, c, extra, sbuf);
}

// The same sums for a CTA of at most 4 warps whose threads hold two element groups (K=2), each with its own partial
// (a[k], b[k], c[k]).  Group k of thread t takes the place of lane t&31 of warp (t>>5) + k*nwarp in the CTA of twice
// as many threads with one group each, so the sums have that CTA's block_sum3_small tree and bits.
// publish: one packed butterfly over both groups' 6 values with warp_sum3's xor pairing (16, 8, 4, 2, 1) for each,
// 8 shuffles instead of 2 x 6; lanes 0/4/8 end with group 0's a/b/c, lanes 16/20/24 with group 1's.  Then the 6 slots
// and the extra scalar are stored.
__device__ __forceinline__ void block_sum3_pair_publish(const float (&a)[2], const float (&b)[2], const float (&c)[2],
                                                        float extra, float* sbuf) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = (blockDim.x + 31) >> 5;
    const bool h16 = lane & 16, h8 = lane & 8, h4 = lane & 4;
    // xor 16: lanes [0,16) keep group 0's three values, lanes [16,32) group 1's
    const float x0 = add(h16 ? a[1] : a[0], __shfl_xor_sync(0xffffffffu, h16 ? a[0] : a[1], 16));
    float x1 = add(h16 ? b[1] : b[0], __shfl_xor_sync(0xffffffffu, h16 ? b[0] : b[1], 16));
    const float x2 = add(h16 ? c[1] : c[0], __shfl_xor_sync(0xffffffffu, h16 ? c[0] : c[1], 16));
    // xor 8: lanes with bit 8 clear finish a, set finish c; both halves finish b
    float k = add(h8 ? x2 : x0, __shfl_xor_sync(0xffffffffu, h8 ? x0 : x2, 8));
    x1 = add(x1, __shfl_xor_sync(0xffffffffu, x1, 8));
    // xor 4: lanes with bit 4 clear keep a / c, set keep b
    k = add(h4 ? x1 : k, __shfl_xor_sync(0xffffffffu, h4 ? k : x1, 4));
    k = add(k, __shfl_xor_sync(0xffffffffu, k, 2));
    k = add(k, __shfl_xor_sync(0xffffffffu, k, 1));
    if ((lane & 3) == 0 && (lane & 12) != 12) sbuf[4 * (warp + (lane >> 4) * nwarp) + ((lane >> 2) & 3)] = k;
    if (threadIdx.x == 0) sbuf[32] = extra;
}
__device__ __forceinline__ void block_sum3_pair_collect(float& a, float& b, float& c, float& extra, const float* sbuf) {
    __syncthreads();
    block_sum3_slots(a, b, c, extra, sbuf);
}
// The producer form's publish: the kinetic sums of the momentum come from the producer warps (hmc_produce), so only
// (b[k], c[k]) are reduced here, with the same xor pairing and into the same slot positions (.y, .z) as
// block_sum3_pair_publish.  Lanes 0/8 end with group 0's b/c, lanes 16/24 with group 1's; 6 shuffles.
__device__ __forceinline__ void block_sum2_pair_publish(const float (&b)[2], const float (&c)[2], float* sbuf, int nwarp) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const bool h16 = lane & 16, h8 = lane & 8;
    const float x1 = add(h16 ? b[1] : b[0], __shfl_xor_sync(0xffffffffu, h16 ? b[0] : b[1], 16));
    const float x2 = add(h16 ? c[1] : c[0], __shfl_xor_sync(0xffffffffu, h16 ? c[0] : c[1], 16));
    // xor 8: lanes with bit 8 clear finish b, set finish c
    float k = add(h8 ? x2 : x1, __shfl_xor_sync(0xffffffffu, h8 ? x1 : x2, 8));
    k = add(k, __shfl_xor_sync(0xffffffffu, k, 4));
    k = add(k, __shfl_xor_sync(0xffffffffu, k, 2));
    k = add(k, __shfl_xor_sync(0xffffffffu, k, 1));
    if ((lane & 7) == 0) sbuf[4 * (warp + (lane >> 4) * nwarp) + 1 + ((lane >> 3) & 1)] = k;
}

// Named barriers of the producer form (PW > 0): 0 is __syncthreads, 1 the compute threads' own barrier.  The momentum
// slot has a "full" barrier (producers arrive once the slot holds iteration n, compute threads wait) and an "empty" one
// (compute threads arrive when iteration n's trajectory is done, by which time they hold the slot's contents in
// registers; producers wait before they draw iteration n+1 into it).
constexpr int BAR_CHAIN = 1, BAR_SLOT_FULL = 2, BAR_SLOT_EMPTY = 3;
__device__ __forceinline__ void bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" :: "r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void bar_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" :: "r"(id), "r"(n) : "memory"); }
// the barrier of the threads that hold the chain's state: the whole CTA, or the G compute threads of the producer form
template <int PW>
__device__ __forceinline__ void chain_sync(int G) {
    if constexpr (PW == 0) __syncthreads();
    else bar_sync(BAR_CHAIN, G);
}

// block_sum<1> with the same correspondence for a thread holding K partials: partial k is lane t&31 of warp
// (t>>5) + k*nwarp.  `sbuf` holds 32 floats.  PW = the CTA's producer warps, which do not take part.
template <int K, int PW = 0>
__device__ __forceinline__ float block_sum1_groups(float (&v)[K], float* sbuf) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = ((blockDim.x + 31) >> 5) - PW;
#pragma unroll
    for (int k = 0; k < K; ++k) v[k] = warp_sum(v[k]);
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < K; ++k) sbuf[warp + k * nwarp] = v[k];
    }
    chain_sync<PW>(nwarp * 32);
    return warp_sum(lane < K * nwarp ? sbuf[lane] : 0.0f);
}

// ---------------------------------------------------------------------------------------------------------
// Thread-block clusters: one chain spread over CS CTAs (SMs) -- finer-grained work units for launches with few chains
// (BASELINE config 2: 256 chains on 132 SMs), so that every SM holds several independent CTAs whose latencies overlap.
// At config 2 the cluster barrier + DSMEM round trip per iteration costs more than the finer granularity buys, so this
// form is opt-in (tuning 41 / 42), kept as the tested starting point for single-chain / few-chain launches where one
// SM per chain leaves the GPU idle.
// The chain's only cross-thread traffic, the per-iteration reduction, goes through DISTRIBUTED SHARED MEMORY: every
// warp publishes its partial sums in its CTA's slot, one cluster barrier (arrive ... independent work ... wait), then
// every thread adds all CS x nwarp partials in rank / warp order -- identical bits, hence identical decisions, in every
// CTA of the cluster.  Slots are double-buffered by iteration parity: one cluster barrier per iteration.
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ float4 ld_dsmem_f4(const void* smem_ptr, uint32_t rank) {
    const uint32_t local = (uint32_t)__cvta_generic_to_shared(smem_ptr);
    uint32_t remote;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local), "r"(rank));
    float4 v;
    asm volatile("ld.shared::cluster.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(remote) : "memory");
    return v;
}
// phase 1: warp-level sums -> this CTA's slot; signal the cluster
__device__ __forceinline__ void cluster_sum3_publish(float a, float b, float c, float extra, float4* slot) {
    warp_sum3(a, b, c, true);
    if ((threadIdx.x & 31) == 0) slot[threadIdx.x >> 5] = make_float4(a, b, c, extra);
    cluster_arrive();
}
// phase 2: wait for every CTA's slot, add all partials in (rank, warp) order; `extra` is rank 0 / warp 0's
template <int CS>
__device__ __forceinline__ void cluster_sum3_collect(float& a, float& b, float& c, float& extra, const float4* slot) {
    cluster_wait();
    const int nwarp = (blockDim.x + 31) >> 5;
    a = 0.0f; b = 0.0f; c = 0.0f;
#pragma unroll
    for (int r = 0; r < CS; ++r) {
        for (int w = 0; w < nwarp; ++w) {
            const float4 v = ld_dsmem_f4(slot + w, (uint32_t)r);
            if (r == 0 && w == 0) { a = v.x; b = v.y; c = v.z; extra = v.w; }
            else { a = add(a, v.x); b = add(b, v.y); c = add(c, v.z); }
        }
    }
}
// one value, off the hot loop (initial log p, the :1018 quirk): full barrier on both sides
template <int CS>
__device__ __forceinline__ float cluster_sum1(float v, float4* slot) {
    float z0 = 0.0f, z1 = 0.0f, z2 = 0.0f;
    cluster_sum3_publish(v, z0, z1, 0.0f, slot);
    cluster_sum3_collect<CS>(v, z0, z1, z2, slot);
    cluster_arrive();
    cluster_wait();                        // everyone has read: the slot may be reused
    return v;
}

constexpr int run_max_threads(int E, int K) { return (E * K <= 4) ? 1024 : (E * K <= 8 ? 512 : 256); }

// Developer build only (-DHMCX_HMC_PROF, scripts/prof_hmc_phases.py): clock64() stamps of the paired loop, lane 0 of every
// warp of the first HMC_PROF_CTAS CTAs, iterations [HMC_PROF_IT0, HMC_PROF_IT0 + HMC_PROF_ITS) of the launch, 8 stamp ids
// per iteration, and each CTA's SM id so that the co-resident chains can be matched.  The producer form also stamps, per
// iteration, when producer warp 0 published the iteration's momentum slot.
#ifdef HMCX_HMC_PROF
constexpr int HMC_PROF_CTAS = 256, HMC_PROF_WARPS = 4, HMC_PROF_IT0 = 256, HMC_PROF_ITS = 64, HMC_PROF_IDS = 8;
__device__ long long g_hmc_prof[HMC_PROF_CTAS * HMC_PROF_WARPS * HMC_PROF_ITS * HMC_PROF_IDS];
__device__ long long g_hmc_prof_pub[HMC_PROF_CTAS * HMC_PROF_ITS];
__device__ int g_hmc_prof_sm[HMC_PROF_CTAS];
__device__ __forceinline__ void hmc_prof_publish(int n, int it0, int pt) {
    const int i = n - it0 - HMC_PROF_IT0;
    if (pt == 0 && blockIdx.x < HMC_PROF_CTAS && i >= 0 && i < HMC_PROF_ITS)
        g_hmc_prof_pub[blockIdx.x * HMC_PROF_ITS + i] = clock64();
}
__device__ __forceinline__ long long* hmc_prof_row(int n, int it0) {
    const int i = n - it0 - HMC_PROF_IT0, w = threadIdx.x >> 5;
    if ((threadIdx.x & 31) || blockIdx.x >= HMC_PROF_CTAS || w >= HMC_PROF_WARPS || i < 0 || i >= HMC_PROF_ITS) return nullptr;
    return g_hmc_prof + ((size_t)(blockIdx.x * HMC_PROF_WARPS + w) * HMC_PROF_ITS + i) * HMC_PROF_IDS;
}
#define HMC_MARK(row, id) do { if (row) (row)[id] = clock64(); } while (0)
#else
#define HMC_MARK(row, id) do {} while (0)
#endif

// The producer form of the paired loop (PW > 0): PW producer warps behind the G compute threads draw each iteration's
// momentum, its kinetic sums and the MH log-uniform into one shared-memory slot.  None of that work depends on the
// chain's state, so it leaves the compute warps' instruction stream.  The producers draw iteration n once iteration
// n-1's trajectory is done, i.e. while the compute warps sit in the serial tail (butterfly, barrier, MH, row store),
// where a scheduler has idle issue slots; drawing further ahead competes with the trajectory for them and measured
// slower (DESIGN §3.1), and since the compute threads have read the slot before their trajectory, one slot suffices.
// Producer thread pt mirrors compute threads pt + u*32*PW: the same groups, Philox counters and normals, and for each
// virtual warp of block_sum3_pair_publish the same 32 lanes, so the kinetic sums (a plain xor butterfly, the pairing
// warp_sum3 gives every value) have that tree's bits.
struct MomentumSlot {
    float4 p[2][128];     // the momentum of group k of compute thread t
    float kin[8];         // the kinetic sum of virtual warp w (slot .x of block_sum3_pair_publish)
    float logu;
};

template <int TK, int MK, int PW, int MAXT>
__device__ __forceinline__ void hmc_produce(const RunArgs& a, int pt, int G, uint64_t chain_id, MomentumSlot& r) {
    constexpr int NT = MAXT / (32 * PW);             // compute threads per producer thread
    const int lane = pt & 31, nwarp = G >> 5, nthr = G + 32 * PW;
    PhiloxKeys keys;
    philox_make_keys(a.seed, chain_id, keys);
    VecConst<4> vc[NT][2];
    PhiloxFixed pfix[NT][2];
    uint32_t zmask[NT][2][4];
#pragma unroll
    for (int u = 0; u < NT; ++u)
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const int grp = pt + 32 * PW * u + k * G;
            load_consts<TK, MK, 4>(a.t, 4 * grp, vc[u][k]);
            philox_fix(keys, chain_id, grp, STREAM_MOMENTUM, pfix[u][k]);
#pragma unroll
            for (int j = 0; j < 4; ++j) zmask[u][k][j] = 4 * grp + j < a.t.D ? 0xFFFFFFFFu : 0u;
        }
    float logu_lanes = 0.0f;
    for (int n = a.it0, m = 0; n < a.it1; ++n, ++m) {
        if (m > 0) bar_sync(BAR_SLOT_EMPTY, nthr);        // the compute warps have finished iteration n-1's trajectory
        float4 pv[NT][2];
        float kin[NT][2];
#pragma unroll
        for (int u = 0; u < NT; ++u)
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                float z[4], p[4];
                philox_normals<4>(keys, pfix[u][k], (uint32_t)n, (uint32_t)(pt + 32 * PW * u + k * G), z);
                kin[u][k] = 0.0f;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    z[j] = __uint_as_float(__float_as_uint(z[j]) & zmask[u][k][j]);
                    p[j] = (MK == HMCX_MASS_DIAG) ? mul(z[j], vc[u][k].sd[j]) : z[j];
                    kin[u][k] = sum_in<MK == HMCX_MASS_NONE>(kin[u][k], kterm1<MK>(p[j], vc[u][k].im[j]), j == 0);
                }
                pv[u][k] = make_float4(p[0], p[1], p[2], p[3]);
            }
#pragma unroll
        for (int u = 0; u < NT; ++u) {                // both groups in one butterfly: lanes [0,16) group 0, [16,32) 1
            const bool h16 = lane & 16;
            float x = add(h16 ? kin[u][1] : kin[u][0], __shfl_xor_sync(0xffffffffu, h16 ? kin[u][0] : kin[u][1], 16));
#pragma unroll
            for (int o = 8; o > 0; o >>= 1) x = add(x, __shfl_xor_sync(0xffffffffu, x, o));
            kin[u][0] = x;
        }
        float logu = 0.0f;
        if (pt < 32) {                                // 32 iterations per Philox call, lane l for iteration n + l
            const int phase = m & 31;
            if (phase == 0) logu_lanes = philox_log_uniform(keys, chain_id, (uint64_t)(n + lane));
            logu = __shfl_sync(0xffffffffu, logu_lanes, phase);
        }
#pragma unroll
        for (int u = 0; u < NT; ++u) {
            const int tt = pt + 32 * PW * u;            // < 32 * PW * NT = MAXT = G: every mirrored thread exists
            r.p[0][tt] = pv[u][0];
            r.p[1][tt] = pv[u][1];
            if ((lane & 15) == 0) r.kin[(tt >> 5) + (lane >> 4) * nwarp] = kin[u][0];
        }
        if (pt == 0) r.logu = logu;
        bar_arrive(BAR_SLOT_FULL, nthr);
#ifdef HMCX_HMC_PROF
        hmc_prof_publish(n, a.it0, pt);
#endif
    }
}

// MAXT = CTA size the instantiation is compiled for (register budget 64K/MAXT): chains of D <= 1024 run with <= 256
// threads and get a generous budget, which lets the compiler software-pipeline the next iteration's RNG.
// SINK = true adds the sample sink to the bookkeeping step (thinned stores, register-resident moment accumulators); it is
// a separate instantiation so that the plain sample() loop keeps its register allocation and schedule.
// PHILOX = true compiles the in-kernel counter RNG branch-free (no memory access, so dead lanes just compute and are
// masked): the Philox / Box-Muller arithmetic of iteration n+1 and the shuffle chain of iteration n's reduction then
// sit in one basic block and the scheduler interleaves them.
// CS > 1: the chain is owned by a cluster of CS CTAs (see above); CTA `rank` holds float4 groups [rank*G, (rank+1)*G).
// NUTS = false compiles the dual-averaging path out (the plain sample() loop then carries no trace of it), and with it
// the step-size schedule and trace, which elem_hmc_run sets only for NUTS: their per-iteration null tests and the
// reload of eps were ~20 warp-instructions of the paired loop's 1,023.
// K = 2 with MAXT <= 128 (PAIR): every group keeps its own partial sums and enters the reductions in the place it has
// in the K = 1 CTA of twice the threads (block_sum3_pair_*, block_sum1_groups), so the run is bit-identical to that
// geometry; the other K > 1 forms sum their groups per thread first (a different tree).
// PW > 0 (paired Philox loop only): the CTA is G compute threads followed by PW producer warps (hmc_produce).
template <int TK, int MK, int E, int K, int MAXT, bool SINK = false, bool PHILOX = false, int CS = 1, bool NUTS = true,
          int PW = 0>
__global__ void __launch_bounds__(MAXT + 32 * PW)
hmc_run_kernel(const RunArgs a) {
    static_assert(CS == 1 || (K == 1 && !SINK), "cluster form: one group per thread, no sink");
    constexpr bool PAIR = K == 2 && MAXT <= 128 && CS == 1;
    constexpr int KP = PAIR ? K : 1;                          // partial sums per thread
    static_assert(!PAIR || E == 4, "the paired form mirrors the float4 (K = 1) geometry");
    static_assert(PW == 0 || (PAIR && PHILOX && !SINK && !NUTS && MAXT % (32 * PW) == 0),
                  "producer warps: the paired Philox loop only");
    __shared__ __align__(16) float s_red[2][100];
    __shared__ __align__(16) float4 s_part[3][8];           // CS > 1: per-warp partials (two iteration parities + misc)
    __shared__ float s_eps[2];
    __shared__ MomentumSlot s_slot;                        // PW > 0 only (unreferenced, and dropped, otherwise)

    // the producer form always runs MAXT compute threads (elem_hmc_run): a compile-time G makes its barrier counts, warp
    // count and slot offsets immediates instead of values re-derived from blockDim on every iteration
    const int c = blockIdx.x / CS, rank = blockIdx.x % CS, G = PW > 0 ? MAXT : blockDim.x - 32 * PW;
    const int tid = threadIdx.x, gt = rank * G + tid;       // thread index within the CTA / within the chain
    const bool lead = tid == 0 && rank == 0;                // writes the chain's scalar outputs
    const bool nuts = NUTS && a.nuts;
    const ElemTarget& t = a.t;
    const int ld = t.ld, D = t.D;
    const size_t row = (size_t)c * ld;
    const uint64_t chain_id = a.chain_offset + (uint64_t)c;
    if constexpr (PW > 0) {
        if (tid >= G) {
            hmc_produce<TK, MK, PW, MAXT>(a, tid - G, G, chain_id, s_slot);
            return;
        }
    }

    VecConst<E> vc[K];
    float qc[K][E], q[K][E], p[K][E];
    bool live[K];                 // group lies inside the padded row
    uint32_t zmask[K][E];         // ~0 for an element of the chain, 0 for padding (whose normals are zeroed)
#pragma unroll
    for (int k = 0; k < K; ++k) {
        const int e0 = E * (gt + k * G);
        live[k] = e0 < ld;
        load_consts<TK, MK, E>(t, e0, vc[k]);
        if (live[k]) ldE<E>(a.q_cur + row + e0, qc[k]);
#pragma unroll
        for (int j = 0; j < E; ++j) {
            if (!live[k] || e0 + j >= D) qc[k][j] = 0.0f;
            zmask[k][j] = e0 + j < D ? 0xFFFFFFFFu : 0u;
        }
    }
    // PW > 0 stores the .y / .z of all 8 slots and uses nothing else from them (.x comes from the producers)
    if (CS == 1 && MAXT <= 256 && PW == 0) block_sum3_small_init(s_red, KP);
#ifdef HMCX_HMC_PROF
    if (PAIR && tid == 0 && blockIdx.x < HMC_PROF_CTAS) {
        int sm;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(sm));
        g_hmc_prof_sm[blockIdx.x] = sm;
    }
#endif

    // U(q_cur) once; afterwards it is carried (the reference recomputes the identical value, :971)
    float lp_cur;
    {
        float r[KP];
#pragma unroll
        for (int i = 0; i < KP; ++i) r[i] = 0.0f;
#pragma unroll
        for (int k = 0; k < K; ++k)
#pragma unroll
            for (int j = 0; j < E; ++j)
                r[PAIR ? k : 0] = add(r[PAIR ? k : 0], uterm1<TK>(qc[k][j], vc[k].mean[j], vc[k].ivar[j]));
        if constexpr (PAIR) r[0] = block_sum1_groups<KP, PW>(r, s_red[1]);
        else if (CS > 1) r[0] = cluster_sum1<CS>(r[0], s_part[2]);
        else block_sum<1>(r, s_red[1]);
        lp_cur = log_prob_from_sum(r[0], t.log_norm);
        chain_sync<PW>(G);
    }
    if (a.lp_carry && a.it0 > 0) lp_cur = a.lp_carry[c];

    float eps = a.eps[c];
    double h_bar = 0.0, eps_bar = 1.0;
    if (nuts && tid == 0) { h_bar = a.h_bar[c]; eps_bar = a.eps_bar[c]; }
    double mu_sink = 0.0;                                   // SINK: this chain's mu (the restarted dual averaging's)
    if constexpr (SINK) {
        if (nuts && tid == 0) mu_sink = a.mu_per_chain ? a.mu_chain[c] : a.mu;
    }
    int rejected = 0;
    const int thin = SINK ? a.thin : 1;
    const int keep = SINK ? 1 + (a.S - a.burn - 1) / thin : a.S - a.burn;    // slots per chain in samples_out
    float* const my_samples = a.samples ? a.samples + (size_t)c * keep * ld : nullptr;
    float msum[K][E], msq[K][E], csum[K][E], csq[K][E];
    if (SINK) {
#pragma unroll
        for (int k = 0; k < K; ++k) {
#pragma unroll
            for (int j = 0; j < E; ++j) { msum[k][j] = 0.0f; msq[k][j] = 0.0f; csum[k][j] = 0.0f; csq[k][j] = 0.0f; }
            if (live[k] && a.msum) ldE<E>(a.msum + row + E * (gt + k * G), msum[k]);
            if (live[k] && a.msumsq) ldE<E>(a.msumsq + row + E * (gt + k * G), msq[k]);
            if (live[k] && a.msum && a.msum_lo) ldE<E>(a.msum_lo + row + E * (gt + k * G), csum[k]);
            if (live[k] && a.msumsq && a.msumsq_lo) ldE<E>(a.msumsq_lo + row + E * (gt + k * G), csq[k]);
        }
    }

    // the plain sample() loop stores one row per post-burn iteration: keep a running row pointer (one 64-bit add per
    // iteration instead of re-deriving the address from n)
    float* row_ptr = nullptr;
    if (!SINK && my_samples) {
        const int first = (a.it0 > a.burn + 1 ? a.it0 : a.burn + 1) - a.burn;
        row_ptr = my_samples + (size_t)first * ld + E * gt;
    }

    if (a.it0 == 0 && my_samples) {                // ret_params = [params_init] (:959)
#pragma unroll
        for (int k = 0; k < K; ++k)
            if (live[k]) stE_stream<E>(my_samples + E * (gt + k * G), qc[k]);
    }

    // the standard normals of iteration n: produced one iteration AHEAD (they do not depend on the MH decision), so
    // that the Philox/Box-Muller arithmetic of iteration n+1 overlaps the shuffle/barrier latency of iteration n, or, in
    // the paired form, the first leapfrog step of iteration n
    float zn[K][E];
    PhiloxKeys keys;
    PhiloxFixed pfix[K];
    if (PHILOX && PW == 0) {
        philox_make_keys(a.seed, chain_id, keys);
#pragma unroll
        for (int k = 0; k < K; ++k) {
            const uint32_t grp = gt + k * G;
            philox_fix(keys, chain_id, E == 4 ? grp : grp >> 1, STREAM_MOMENTUM, pfix[k]);
        }
    }
    auto draw = [&](int n) {
#pragma unroll
        for (int k = 0; k < K; ++k) {
            const int grp = gt + k * G, e0 = E * grp;
#pragma unroll
            for (int j = 0; j < E; ++j) zn[k][j] = 0.0f;
            if (PHILOX) {
                philox_normals<E>(keys, pfix[k], (uint32_t)n, (uint32_t)grp, zn[k]);
            } else if (live[k]) {
                if (a.rng_mode == HMCX_RNG_INJECTED) ldE_stream<E>(a.normals + ((size_t)(n - a.it0) * t.C + c) * ld + e0, zn[k]);
                else philox_normals<E>(a.seed, chain_id, (uint64_t)n, (uint32_t)grp, zn[k]);
            }
#pragma unroll
            for (int j = 0; j < E; ++j) zn[k][j] = __uint_as_float(__float_as_uint(zn[k][j]) & zmask[k][j]);
        }
    };
    if (PW == 0 && a.it0 < a.it1) draw(a.it0);

    // the MH test's log-uniforms: warp 0 produces them 32 iterations at a time, lane l for iteration n+l, so the ~70
    // dependent instructions of Philox + logf leave the per-iteration critical path (every other warp waits for warp 0 at
    // the reduction's barrier) and cost 1/32 of the issue slots.  The producer form draws them in its producer warps.
    float logu_lanes = 0.0f;
    const bool warp0 = PW == 0 && tid < 32 && rank == 0;

    for (int n = a.it0; n < a.it1; ++n) {
#ifdef HMCX_HMC_PROF
        long long* const prow = PAIR ? hmc_prof_row(n, a.it0) : nullptr;
#endif
        // producer form: this iteration's momentum, kinetic sum (the 8 virtual warps' slots added in warp order, as
        // block_sum3_slots adds them) and log-uniform from the producers' slot
        float slot_kin = 0.0f, slot_logu = 0.0f;
        if constexpr (PW > 0) {
            HMC_MARK(prow, 6);              // before the slot-full wait
            bar_sync(BAR_SLOT_FULL, G + 32 * PW);
            HMC_MARK(prow, 7);
            const MomentumSlot& r = s_slot;
#pragma unroll
            for (int k = 0; k < K; ++k) {
                const float4 v = r.p[k][tid];
                p[k][0] = v.x; p[k][1] = v.y; p[k][2] = v.z; p[k][3] = v.w;
            }
            const float4 k0 = *reinterpret_cast<const float4*>(r.kin), k1 = *reinterpret_cast<const float4*>(r.kin + 4);
            slot_kin = add(add(add(add(add(add(add(k0.x, k0.y), k0.z), k0.w), k1.x), k1.y), k1.z), k1.w);
            slot_logu = r.logu;
        }
        HMC_MARK(prow, 0);                  // the iteration starts
        if (NUTS && a.eps_schedule) eps = a.eps_schedule[(size_t)n * t.C + c];
        const float half = mul(0.5f, eps);
        if (nuts && tid == 0 && n <= a.burn) {
            // dual averaging is a serial scalar recurrence on the critical path (all other threads wait for the new step
            // size): pull this iteration's five table constants towards the SM now, a whole trajectory ahead of their use
            const double* T = a.table + 5 * (size_t)n;
            asm volatile("prefetch.global.L1 [%0];" :: "l"(T));
            asm volatile("prefetch.global.L1 [%0];" :: "l"(T + 4));
        }
        // the iteration's log-uniform (warp 0; rides the reduction's shared buffer)
        float logu = 0.0f;
        if (warp0) {
            const int phase = (n - a.it0) & 31;
            if (phase == 0) {
                const int m = n + tid;
                if (a.rng_mode == HMCX_RNG_INJECTED) logu_lanes = m < a.it1 ? a.logu[(size_t)(m - a.it0) * t.C + c] : 0.0f;
                else if (PHILOX) logu_lanes = philox_log_uniform(keys, chain_id, (uint64_t)m);
                else logu_lanes = philox_log_uniform(a.seed, chain_id, (uint64_t)m);
            }
            logu = __shfl_sync(0xffffffffu, logu_lanes, phase);
        }
        // ---- gibbs (:969): p = z (*sqrt(mass)) ----
        // partial sums: index k for group k in the paired form, index 0 for all groups otherwise
        float r0[KP], r1[KP], r2[KP];
#pragma unroll
        for (int i = 0; i < KP; ++i) { r0[i] = 0.0f; r1[i] = 0.0f; r2[i] = 0.0f; }
#pragma unroll
        for (int k = 0; k < K; ++k) {
            const int i = PAIR ? k : 0;
            const bool first = i == k;                               // the partial's first group
#pragma unroll
            for (int j = 0; j < E; ++j) {
                if (PW == 0) {
                    p[k][j] = (MK == HMCX_MASS_DIAG) ? mul(zn[k][j], vc[k].sd[j]) : zn[k][j];
                    r0[i] = sum_in<MK == HMCX_MASS_NONE>(r0[i], kterm1<MK>(p[k][j], vc[k].im[j]), first && j == 0);
                }
                q[k][j] = qc[k][j];
            }
        }
        // ---- leapfrog (:973) : thread-private ----
        if (PW > 0) {
            trajectory_groups<TK, MK, E, K>(q, p, vc, eps, half, a.L, []() {});
            // the producers draw iteration n+1 while this iteration is in its serial tail
            if (n + 1 < a.it1) bar_arrive(BAR_SLOT_EMPTY, G + 32 * PW);
        } else if (PAIR) {
            // the normals of iteration n+1 (zn is consumed above; branch-free, one unused draw after the last iteration)
            trajectory_groups<TK, MK, E, K>(q, p, vc, eps, half, a.L, [&]() { draw(n + 1); });
        } else {
#pragma unroll
            for (int k = 0; k < K; ++k)
                trajectory<TK, MK, E, false>(q[k], p[k], vc[k], eps, half, a.L, nullptr, nullptr, 0);
        }
        // ---- both Hamiltonians with one fused reduction (:971, :995) ----
#pragma unroll
        for (int k = 0; k < K; ++k) {
            const int i = PAIR ? k : 0;
            const bool first = i == k;
#pragma unroll
            for (int j = 0; j < E; ++j) {
                r1[i] = sum_in<TK == HMCX_TARGET_GAUSS_ISO>(r1[i], uterm1<TK>(q[k][j], vc[k].mean[j], vc[k].ivar[j]),
                                                            first && j == 0);
                r2[i] = sum_in<MK == HMCX_MASS_NONE>(r2[i], kterm1<MK>(p[k][j], vc[k].im[j]), first && j == 0);
            }
        }
        // next iteration's normals: independent work.  In Philox mode the draw is branch-free and unconditional (one
        // unused draw after the last iteration) so that it shares a basic block with the reduction's shuffle chain.
        // The cluster form publishes its partials first: the draw then sits between the stores and the barrier.
        HMC_MARK(prow, 1);                  // trajectory and per-thread sums done
        if constexpr (PW > 0) block_sum2_pair_publish(r1, r2, s_red[n & 1], G >> 5);
        else if constexpr (PAIR) block_sum3_pair_publish(r0, r1, r2, logu, s_red[n & 1]);
        else if (CS > 1) cluster_sum3_publish(r0[0], r1[0], r2[0], logu, s_part[n & 1]);
        HMC_MARK(prow, 2);                  // slots stored
        if (!PAIR && (PHILOX || n + 1 < a.it1)) draw(n + 1);     // the paired form draws inside the trajectory
        HMC_MARK(prow, 3);                  // next normals drawn
        if (PW > 0) {
            chain_sync<PW>(G);
            HMC_MARK(prow, 4);
            // .x and sbuf[32] are never stored in this form: their sums are dead code, which the compiler drops
            float unused_a, unused_extra;
            block_sum3_slots(unused_a, r1[0], r2[0], unused_extra, s_red[n & 1]);
            r0[0] = slot_kin;
            logu = slot_logu;
        } else if (PAIR) {
            __syncthreads();                // block_sum3_pair_collect, with a stamp after its barrier
            HMC_MARK(prow, 4);
            block_sum3_slots(r0[0], r1[0], r2[0], logu, s_red[n & 1]);
        }
        else if (CS > 1) cluster_sum3_collect<CS>(r0[0], r1[0], r2[0], logu, s_part[n & 1]);
        else if (MAXT <= 256) block_sum3_small(r0[0], r1[0], r2[0], logu, s_red[n & 1]);
        else block_sum3(r0[0], r1[0], r2[0], logu, s_red[n & 1]);
        const float lp_new = log_prob_from_sum(r1[0], t.log_norm);
        const float h_old = add(-lp_cur, mul(0.5f, r0[0]));                  // potential + kinetic (:815)
        const float h_new = add(-lp_new, mul(0.5f, r2[0]));
        const bool bad = !finite_f(lp_cur) || !finite_f(lp_new);            // LogProbError (:783-785)
        // ---- MH (:1000-1004) ----
        const float x = add(-h_new, h_old);                                  // acceptance(), :626
        const float rho = (x < 0.0f) ? x : 0.0f;                             // Python min(0., x): nan -> 0.
        const bool acc = !bad && (rho >= logu);
        if (acc) {
            lp_cur = lp_new;
#pragma unroll
            for (int k = 0; k < K; ++k)
#pragma unroll
                for (int j = 0; j < E; ++j) qc[k][j] = q[k][j];
        } else {
            ++rejected;
            if (n == a.burn + 1) {
                // reference quirk (:1018): the first stored iteration restores ret_params[-1] == params_init,
                // not the pre-trajectory state.  Rare path: re-read params_init and recompute its log p.
                float s[KP];
#pragma unroll
                for (int i = 0; i < KP; ++i) s[i] = 0.0f;
#pragma unroll
                for (int k = 0; k < K; ++k) {
                    const int e0 = E * (gt + k * G);
                    if (live[k]) ldE<E>(a.q_init + row + e0, qc[k]);
#pragma unroll
                    for (int j = 0; j < E; ++j) {
                        if (!live[k] || e0 + j >= D) qc[k][j] = 0.0f;
                        s[PAIR ? k : 0] = add(s[PAIR ? k : 0], uterm1<TK>(qc[k][j], vc[k].mean[j], vc[k].ivar[j]));
                    }
                }
                if constexpr (PAIR) s[0] = block_sum1_groups<KP, PW>(s, s_red[(n & 1) ^ 1]);
                else if (CS > 1) s[0] = cluster_sum1<CS>(s[0], s_part[2]);  // every CTA of the cluster takes this branch
                else block_sum<1>(s, s_red[(n & 1) ^ 1]);
                lp_cur = log_prob_from_sum(s[0], t.log_norm);
                chain_sync<PW>(G);        // the next iteration reduces through the same buffer
            }
        }
        // ---- bookkeeping (:1007-1026): store only for n > burn ----
        if (SINK) {
            if (n > a.burn || a.moments_all) {
#pragma unroll
                for (int k = 0; k < K; ++k)
#pragma unroll
                    for (int j = 0; j < E; ++j) {
                        const float x = qc[k][j], xx = mul(x, x);
                        comp_add(msum[k][j], csum[k][j], x);
                        comp_add(msq[k][j], csq[k][j], xx);
                        csq[k][j] = add(csq[k][j], fmaf(x, x, -xx));      // the rounding error of x*x itself (exact)
                    }
            }
            if (n > a.burn) {
                if (my_samples && (n - a.burn) % thin == 0) {
                    float* dst = my_samples + (size_t)((n - a.burn) / thin) * ld;
#pragma unroll
                    for (int k = 0; k < K; ++k)
                        if (live[k]) stE_stream<E>(dst + E * (gt + k * G), qc[k]);
                }
            }
        } else if (n > a.burn && my_samples) {
#pragma unroll
            for (int k = 0; k < K; ++k)
                if (live[k]) stE_stream<E>(row_ptr + E * k * G, qc[k]);
            row_ptr += ld;
        }
        HMC_MARK(prow, 5);                  // MH decided, state selected, row stored
        if (lead) {
            const size_t o = (size_t)c * a.S + n;
            if (a.accept) a.accept[o] = acc ? 1 : 0;
            if (a.diverged) a.diverged[o] = bad ? 1 : 0;
            if (a.ham) { a.ham[2 * o] = h_old; a.ham[2 * o + 1] = h_new; }
        }
        // ---- dual averaging (:1030-1035, exception path :1060-1067) ----
        if (nuts && n <= a.burn) {
            if (tid == 0) {
                float e = eps;
                if (n < a.burn || bad) {
                    const double* T = a.table + 5 * (size_t)n;               // t = n+1
                    const double alpha = bad ? 0.0 : (double)expf(rho);      // min(1, exp(rho)), rho <= 0
                    h_bar = __dadd_rn(__dmul_rn(T[0], h_bar), __dmul_rn(T[1], a.delta - alpha));
                    const double x_new = (SINK ? mu_sink : a.mu) - __dmul_rn(T[2], h_bar);
                    e = expf((float)x_new);
                    const float xb = add((float)__dmul_rn(T[3], x_new), mul((float)T[4], logf((float)eps_bar)));
                    eps_bar = (double)expf(xb);
                }
                if (n == a.burn) e = (float)eps_bar;                          // freeze (:1033-1034)
                s_eps[n & 1] = e;
                if (a.eps_trace && lead) a.eps_trace[(size_t)c * a.S + n] = e;
            }
            __syncthreads();
            eps = s_eps[n & 1];
        } else if (NUTS && a.eps_trace && lead) {
            a.eps_trace[(size_t)c * a.S + n] = eps;
        }
    }
    if (CS > 1) { cluster_arrive(); cluster_wait(); }       // no CTA leaves while a peer may still read its slots

    // final state for resumption
#pragma unroll
    for (int k = 0; k < K; ++k)
        if (live[k]) stE<E>(a.q_cur + row + E * (gt + k * G), qc[k]);
    if (SINK) {
#pragma unroll
        for (int k = 0; k < K; ++k) {
            if (!a.msum_lo) {
#pragma unroll
                for (int j = 0; j < E; ++j) msum[k][j] = add(msum[k][j], csum[k][j]);
            }
            if (!a.msumsq_lo) {
#pragma unroll
                for (int j = 0; j < E; ++j) msq[k][j] = add(msq[k][j], csq[k][j]);
            }
            if (live[k] && a.msum) stE<E>(a.msum + row + E * (gt + k * G), msum[k]);
            if (live[k] && a.msumsq) stE<E>(a.msumsq + row + E * (gt + k * G), msq[k]);
            if (live[k] && a.msum && a.msum_lo) stE<E>(a.msum_lo + row + E * (gt + k * G), csum[k]);
            if (live[k] && a.msumsq && a.msumsq_lo) stE<E>(a.msumsq_lo + row + E * (gt + k * G), csq[k]);
        }
    }
    if (lead) {
        a.eps[c] = eps;
        if (nuts) { a.h_bar[c] = h_bar; a.eps_bar[c] = eps_bar; }
        if (a.num_rejected) a.num_rejected[c] += rejected;
        if (a.lp_carry) a.lp_carry[c] = lp_cur;
    }
}


// ---------------------------------------------------------------------------------------------------------
// large-D form of the persistent kernel (D > 4096): same per-iteration logic, but the chain's state does not fit the
// register file of one CTA, so it is streamed.  One CTA of 1024 threads per chain walks the chain's float4 vectors:
//   pass A  load q_cur, draw p, integrate the (thread-private) trajectory, accumulate the three Hamiltonian sums,
//           park the proposal in `work` (caller-provided (C, ld) scratch);
//   decide  one fused block reduction + MH, exactly as hmc_run_kernel;
//   pass B  commit proposal / keep / restore params_init (the :1018 quirk), write the retained row.
// Pass B touches only vectors the same thread wrote in pass A: no extra barrier.  Traffic: 20*D bytes per iteration
// and chain (L2-resident while C*ld*8 B < ~100 MB), i.e. HBM/L2-bound like the streaming leapfrog kernel.
// ---------------------------------------------------------------------------------------------------------
template <int TK, int MK>
__global__ void __launch_bounds__(1024)
hmc_run_big_kernel(const RunArgs a, float* __restrict__ work) {
    __shared__ float s_red[2][100];
    __shared__ float s_eps[2];
    const int c = blockIdx.x, tid = threadIdx.x, G = blockDim.x;
    const ElemTarget& t = a.t;
    const int ld = t.ld, D = t.D, nvec = ld >> 2;
    const size_t row = (size_t)c * ld;
    const uint64_t chain_id = a.chain_offset + (uint64_t)c;
    float* const qcur = a.q_cur + row;
    float* const prop = work + row;
    const float* const qinit = a.q_init + row;

    auto log_prob_of = [&](const float* src, float* sbuf) {     // full pass over a state row
        float r[1] = {0.0f};
        for (int v = tid; v < nvec; v += G) {
            VecConst<4> vc;
            load_consts<TK, MK, 4>(t, 4 * v, vc);
            float x[4];
            ld4(src + 4 * v, x);
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (4 * v + j < D) r[0] = add(r[0], uterm1<TK>(x[j], vc.mean[j], vc.ivar[j]));
        }
        block_sum<1>(r, sbuf);
        __syncthreads();
        return log_prob_from_sum(r[0], t.log_norm);
    };
    float lp_cur = log_prob_of(qcur, s_red[1]);

    float eps = a.eps[c];
    double h_bar = 0.0, eps_bar = 1.0;
    if (a.nuts && tid == 0) { h_bar = a.h_bar[c]; eps_bar = a.eps_bar[c]; }
    int rejected = 0;
    const int keep = a.S - a.burn;
    float* const my_samples = a.samples ? a.samples + (size_t)c * keep * ld : nullptr;
    if (a.it0 == 0 && my_samples)
        for (int v = tid; v < nvec; v += G) { float x[4]; ld4(qcur + 4 * v, x); st4_stream(my_samples + 4 * v, x); }

    for (int n = a.it0; n < a.it1; ++n) {
        if (a.eps_schedule) eps = a.eps_schedule[(size_t)n * t.C + c];
        const float half = mul(0.5f, eps);
        float r0 = 0.0f, r1 = 0.0f, r2 = 0.0f;
        for (int v = tid; v < nvec; v += G) {                   // ---- pass A ----
            const int e0 = 4 * v;
            VecConst<4> vc;
            load_consts<TK, MK, 4>(t, e0, vc);
            float q[4], p[4], z[4];
            ld4(qcur + e0, q);
            if (a.rng_mode == HMCX_RNG_INJECTED) ld4_stream(a.normals + ((size_t)(n - a.it0) * t.C + c) * ld + e0, z);
            else philox_normal4(a.seed, chain_id, (uint64_t)n, (uint32_t)v, z);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (e0 + j >= D) { z[j] = 0.0f; q[j] = 0.0f; }
                p[j] = (MK == HMCX_MASS_DIAG) ? mul(z[j], vc.sd[j]) : z[j];
                r0 = add(r0, kterm1<MK>(p[j], vc.im[j]));
            }
            trajectory<TK, MK, 4, false>(q, p, vc, eps, half, a.L, nullptr, nullptr, 0);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                r1 = add(r1, uterm1<TK>(q[j], vc.mean[j], vc.ivar[j]));
                r2 = add(r2, kterm1<MK>(p[j], vc.im[j]));
            }
            st4(prop + e0, q);
        }
        float logu = 0.0f;
        if (tid == 0)
            logu = (a.rng_mode == HMCX_RNG_INJECTED) ? a.logu[(size_t)(n - a.it0) * t.C + c]
                                                     : philox_log_uniform(a.seed, chain_id, (uint64_t)n);
        block_sum3(r0, r1, r2, logu, s_red[n & 1]);
        const float lp_new = log_prob_from_sum(r1, t.log_norm);
        const float h_old = add(-lp_cur, mul(0.5f, r0));
        const float h_new = add(-lp_new, mul(0.5f, r2));
        const bool bad = !finite_f(lp_cur) || !finite_f(lp_new);
        const float x = add(-h_new, h_old);
        const float rho = (x < 0.0f) ? x : 0.0f;
        const bool acc = !bad && (rho >= logu);
        const bool quirk = !acc && (n == a.burn + 1);
        if (!acc) ++rejected;
        if (acc) lp_cur = lp_new;
        const bool store = (n > a.burn) && my_samples;
        if (acc || quirk || store) {                            // ---- pass B ----
            float* dst = store ? my_samples + (size_t)(n - a.burn) * ld : nullptr;
            const float* src = acc ? prop : (quirk ? qinit : qcur);
            for (int v = tid; v < nvec; v += G) {
                float xq[4];
                ld4(src + 4 * v, xq);
                if (acc || quirk) st4(qcur + 4 * v, xq);
                if (dst) st4_stream(dst + 4 * v, xq);
            }
        }
        if (quirk) {
            __syncthreads();
            lp_cur = log_prob_of(qcur, s_red[(n & 1) ^ 1]);
        }
        if (tid == 0) {
            const size_t o = (size_t)c * a.S + n;
            if (a.accept) a.accept[o] = acc ? 1 : 0;
            if (a.diverged) a.diverged[o] = bad ? 1 : 0;
            if (a.ham) { a.ham[2 * o] = h_old; a.ham[2 * o + 1] = h_new; }
        }
        if (a.nuts && n <= a.burn) {
            if (tid == 0) {
                float e = eps;
                if (n < a.burn || bad) {
                    const double* T = a.table + 5 * (size_t)n;
                    const double alpha = bad ? 0.0 : (double)expf(rho);
                    h_bar = __dadd_rn(__dmul_rn(T[0], h_bar), __dmul_rn(T[1], a.delta - alpha));
                    const double x_new = a.mu - __dmul_rn(T[2], h_bar);
                    e = expf((float)x_new);
                    const float xb = add((float)__dmul_rn(T[3], x_new), mul((float)T[4], logf((float)eps_bar)));
                    eps_bar = (double)expf(xb);
                }
                if (n == a.burn) e = (float)eps_bar;
                s_eps[n & 1] = e;
                if (a.eps_trace && tid == 0) a.eps_trace[(size_t)c * a.S + n] = e;
            }
            __syncthreads();
            eps = s_eps[n & 1];
        } else if (a.eps_trace && tid == 0) {
            a.eps_trace[(size_t)c * a.S + n] = eps;
        }
    }
    if (tid == 0) {
        a.eps[c] = eps;
        if (a.nuts) { a.h_bar[c] = h_bar; a.eps_bar[c] = eps_bar; }
        if (a.num_rejected) a.num_rejected[c] += rejected;
    }
}

// ---------------------------------------------------------------------------------------------------------
// streaming kernels
// ---------------------------------------------------------------------------------------------------------
template <int TK, int MK, bool TRAJ>
__global__ void __launch_bounds__(256)
leapfrog_kernel(const ElemTarget t, const float* __restrict__ q_in, const float* __restrict__ p_in,
                const float* __restrict__ eps_c, int L, float* __restrict__ q_out, float* __restrict__ p_out,
                float* q_traj, float* p_traj) {
    const int vpr = t.ld >> 2;                                  // float4 vectors per row
    const size_t nvec = (size_t)t.C * vpr;
    const size_t traj_stride = (size_t)t.C * t.ld;
    // row of a vector: one multiply-high by a host-computed reciprocal (exact for v < 2^31) instead of a 64-bit division --
    // the division alone was ~45 of the ~70 instructions per float4 and kept this kernel issue-bound below the HBM roofline
    const bool fast = nvec < (1ull << 31);
    for (size_t v = (size_t)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += (size_t)gridDim.x * blockDim.x) {
        const int c = fast ? (int)(((uint64_t)(uint32_t)v * t.vpr_magic) >> t.vpr_shift) : (int)(v / vpr);
        const int e0 = 4 * (int)(v - (size_t)c * vpr);
        VecConst<4> vc;
        load_consts<TK, MK, 4>(t, e0, vc);
        float q[4], p[4];
        ld4_stream(q_in + 4 * v, q);
        ld4_stream(p_in + 4 * v, p);
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (e0 + j >= t.D) { q[j] = 0.0f; p[j] = 0.0f; }
        const float eps = eps_c[c];
        trajectory<TK, MK, 4, TRAJ>(q, p, vc, eps, mul(0.5f, eps), L, TRAJ ? q_traj + 4 * v : nullptr,
                                    TRAJ ? p_traj + 4 * v : nullptr, traj_stride);
        st4_stream(q_out + 4 * v, q);
        st4_stream(p_out + 4 * v, p);
    }
}

template <int TK, int MK>
__global__ void __launch_bounds__(256)
hamiltonian_kernel(const ElemTarget t, const float* __restrict__ q, const float* __restrict__ p,
                   float* __restrict__ H, uint8_t* __restrict__ flags) {
    __shared__ float s_red[32 * 2];
    const int c = blockIdx.x;
    const size_t row = (size_t)c * t.ld;
    float r[2] = {0.0f, 0.0f};
    for (int e0 = 4 * threadIdx.x; e0 < t.ld; e0 += 4 * blockDim.x) {
        VecConst<4> vc;
        load_consts<TK, MK, 4>(t, e0, vc);
        float qv[4], pv[4];
        ld4_stream(q + row + e0, qv);
        ld4_stream(p + row + e0, pv);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (e0 + j < t.D) {
                r[0] = add(r[0], uterm1<TK>(qv[j], vc.mean[j], vc.ivar[j]));
                r[1] = add(r[1], kterm1<MK>(pv[j], vc.im[j]));
            }
        }
    }
    block_sum<2>(r, s_red);
    if (threadIdx.x == 0) {
        const float lp = log_prob_from_sum(r[0], t.log_norm);
        H[c] = add(-lp, mul(0.5f, r[1]));
        if (flags) flags[c] = finite_f(lp) ? 0 : 1;
    }
}

template <int MK>
__global__ void __launch_bounds__(256)
gibbs_kernel(const ElemTarget t, uint64_t seed, uint64_t chain_offset, uint64_t iter, float* __restrict__ p_out) {
    const int ppr = t.ld >> 1;                                  // element pairs per row
    const size_t npair = (size_t)t.C * ppr;
    for (size_t v = (size_t)blockIdx.x * blockDim.x + threadIdx.x; v < npair; v += (size_t)gridDim.x * blockDim.x) {
        const int c = (int)(v / ppr), pi = (int)(v - (size_t)c * ppr), e0 = 2 * pi;
        float z[2];
        philox_normal2(seed, chain_offset + (uint64_t)c, iter, (uint32_t)pi, z);
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            if (e0 + j >= t.D) z[j] = 0.0f;
            else if (MK == HMCX_MASS_DIAG) z[j] = mul(z[j], t.sd[e0 + j]);
        }
        stE<2>(p_out + 2 * v, z);
    }
}

// ---------------------------------------------------------------------------------------------------------
// host-side dispatch
// ---------------------------------------------------------------------------------------------------------
static int fill_elem_target(const hmcx_target_t* target, const hmcx_mass_t* mass, int C, int ld, ElemTarget& t) {
    if (!target) return HMCX_ERR_INVALID_ARG;
    if (target->kind != HMCX_TARGET_GAUSS_ISO && target->kind != HMCX_TARGET_GAUSS_DIAG) return HMCX_ERR_UNSUPPORTED;
    const int mk = mass ? mass->kind : HMCX_MASS_NONE;
    if (mk != HMCX_MASS_NONE && mk != HMCX_MASS_DIAG) return HMCX_ERR_UNSUPPORTED;
    if (target->dim < 1 || C < 1 || ld < target->dim || (ld & 3)) return HMCX_ERR_INVALID_ARG;
    if (target->kind == HMCX_TARGET_GAUSS_DIAG && !target->inv_var) return HMCX_ERR_INVALID_ARG;
    if (mk == HMCX_MASS_DIAG && (!mass->inv_mass || !mass->mass_factor)) return HMCX_ERR_INVALID_ARG;
    t.tk = target->kind; t.mk = mk; t.D = target->dim; t.ld = ld; t.C = C;
    {
        const uint32_t d = (uint32_t)(ld >> 2);                 // vectors per row, d >= 1
        int s = 0;
        while ((1u << s) < d) ++s;                              // s = ceil(log2 d)
        t.vpr_shift = 31 + s;
        t.vpr_magic = (uint32_t)((((uint64_t)1 << t.vpr_shift) + d - 1) / d);      // < 2^32 because 2^s < 2 d
    }
    t.mean = target->mean; t.ivar = target->inv_var; t.log_norm = target->log_norm;
    t.im = mass ? mass->inv_mass : nullptr; t.sd = mass ? mass->mass_factor : nullptr;
    return HMCX_OK;
}

static inline int cuda_status() { return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA; }

static int sm_count() {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    return sms;
}

static int stream_grid(size_t nvec, int block) {
    const size_t want = (nvec + block - 1) / block;
    const size_t cap = (size_t)sm_count() * 8;                 // 8 resident CTAs of 256 threads per SM
    return (int)(want < cap ? (want ? want : 1) : cap);
}

#define DISPATCH_TK_MK(t, CALL)                                                                         \
    do {                                                                                                \
        if ((t).tk == HMCX_TARGET_GAUSS_ISO) {                                                          \
            if ((t).mk == HMCX_MASS_NONE) { CALL(HMCX_TARGET_GAUSS_ISO, HMCX_MASS_NONE); }              \
            else { CALL(HMCX_TARGET_GAUSS_ISO, HMCX_MASS_DIAG); }                                       \
        } else {                                                                                        \
            if ((t).mk == HMCX_MASS_NONE) { CALL(HMCX_TARGET_GAUSS_DIAG, HMCX_MASS_NONE); }             \
            else { CALL(HMCX_TARGET_GAUSS_DIAG, HMCX_MASS_DIAG); }                                      \
        }                                                                                               \
    } while (0)

int elem_leapfrog(const hmcx_target_t* target, const hmcx_mass_t* mass, const float* q_in, const float* p_in,
                  const float* eps, int C, int ld, int L, float* q_out, float* p_out, float* q_traj,
                  float* p_traj, cudaStream_t st) {
    ElemTarget t;
    const int rc = fill_elem_target(target, mass, C, ld, t);
    if (rc != HMCX_OK) return rc;
    if (!q_in || !p_in || !eps || !q_out || !p_out || L < 1 || ((q_traj == nullptr) != (p_traj == nullptr)))
        return HMCX_ERR_INVALID_ARG;
    const int grid = stream_grid((size_t)C * (ld >> 2), 256);
#define CALL(TK, MK)                                                                                    \
    if (q_traj) leapfrog_kernel<TK, MK, true><<<grid, 256, 0, st>>>(t, q_in, p_in, eps, L, q_out, p_out, q_traj, p_traj); \
    else leapfrog_kernel<TK, MK, false><<<grid, 256, 0, st>>>(t, q_in, p_in, eps, L, q_out, p_out, nullptr, nullptr)
    DISPATCH_TK_MK(t, CALL);
#undef CALL
    return cuda_status();
}

int elem_hamiltonian(const hmcx_target_t* target, const hmcx_mass_t* mass, const float* q, const float* p, int C,
                     int ld, float* H, uint8_t* flags, cudaStream_t st) {
    ElemTarget t;
    const int rc = fill_elem_target(target, mass, C, ld, t);
    if (rc != HMCX_OK) return rc;
    if (!q || !p || !H) return HMCX_ERR_INVALID_ARG;
    int block = ((ld >> 2) + 31) / 32 * 32;
    if (block > 256) block = 256;
#define CALL(TK, MK) hamiltonian_kernel<TK, MK><<<C, block, 0, st>>>(t, q, p, H, flags)
    DISPATCH_TK_MK(t, CALL);
#undef CALL
    return cuda_status();
}

int elem_gibbs(const hmcx_mass_t* mass, const hmcx_rng_t* rng, int D, int C, int ld, int64_t iter, float* p_out,
               cudaStream_t st) {
    if (!rng || rng->mode != HMCX_RNG_PHILOX || !p_out || iter < 0) return HMCX_ERR_INVALID_ARG;
    hmcx_target_t dummy = {};
    dummy.kind = HMCX_TARGET_GAUSS_ISO; dummy.dim = D;
    ElemTarget t;
    const int rc = fill_elem_target(&dummy, mass, C, ld, t);
    if (rc != HMCX_OK) return rc;
    const int grid = stream_grid((size_t)C * (ld >> 1), 256);
    if (t.mk == HMCX_MASS_NONE) gibbs_kernel<HMCX_MASS_NONE><<<grid, 256, 0, st>>>(t, rng->seed, rng->chain_offset, (uint64_t)iter, p_out);
    else gibbs_kernel<HMCX_MASS_DIAG><<<grid, 256, 0, st>>>(t, rng->seed, rng->chain_offset, (uint64_t)iter, p_out);
    return cuda_status();
}

// Register-resident geometry (one CTA per chain): each thread owns K groups of E contiguous elements.
//   tuning 0 (auto): one float4 per thread (E=4,K=1), except
//                    * 768 < ld <= 1024 in the plain Philox loop (pair_ok): two float4 per thread in CTAs of <= 128
//                      threads (the paired form, bit-identical to K=1).  The loop is issue-bound there, and every warp
//                      pays the iteration's fixed cost (reduction, barrier, MH, loop) once: half the warps, ~20 % fewer
//                      instructions per chain.  Measured at 256 chains (2 CTAs per SM; H100 80GB HBM3, 400 W), launch
//                      time paired / K=1: 1.05 at ld 512, 1.12 at 768, 0.98 at 832 and 896, 0.94 at 960 and 1024.  Below
//                      ~7 warps per K=1 CTA the halved warp count leaves the schedulers short of warps and latency wins.
//                      Up to 2 chains per SM it runs with two producer warps per CTA (PW = 2, hmc_produce);
//                    * D > 2560: K=2 in CTAs of <= 512 threads (at config 5, D=4096, CTAs of 768-1024 threads x 1 are
//                      slower).
//   tuning 1: E=4, K=1 forced.
//   tuning 2 / 4: E=4 with K = 2 / 4 groups per thread, each thread's groups summed first (the tree of neither the
//                 paired form nor K=1);  21: E=2,K=1 (D <= 2048);  22: E=2,K=2.
static bool pick_geometry(int ld, int tuning, bool pair_ok, int& E, int& K, int& G) {
    if (ld > 4096) return false;
    if (tuning == 0) { E = 4; K = (ld > 2560 || (pair_ok && ld > 768 && ld <= 1024)) ? 2 : 1; }
    else if (tuning == 1) { E = 4; K = 1; }
    else if (tuning == 21) { E = 2; K = 1; }
    else if (tuning == 2 || tuning == 4) { E = 4; K = tuning; }
    else if (tuning == 22) { E = 2; K = 2; }
    else return false;
    const int groups = ld / E;
    G = ((groups + K - 1) / K + 31) / 32 * 32;
    return G <= run_max_threads(E, K);
}

int elem_hmc_run(const hmcx_target_t* target, const hmcx_mass_t* mass, const hmcx_rng_t* rng,
                 const hmcx_nuts_t* nuts, const float* q_init, float* q_cur, float* eps, int C, int ld, int L,
                 int S, int burn, int it0, int it1, float* samples, uint8_t* accept, uint8_t* diverged,
                 float* ham, int32_t* num_rejected, int tuning, float* workspace, const hmcx_sink_t* sink,
                 cudaStream_t st) {
    RunArgs a = {};
    const int rc = fill_elem_target(target, mass, C, ld, a.t);
    if (rc != HMCX_OK) return rc;
    if (!rng || !q_init || !q_cur || !eps || L < 1 || S < 1 || burn < 0 || burn >= S || it0 < 0 || it1 > S || it0 > it1)
        return HMCX_ERR_INVALID_ARG;
    if (rng->mode == HMCX_RNG_INJECTED) {
        if (!rng->normals || !rng->log_uniforms) return HMCX_ERR_INVALID_ARG;
    } else if (rng->mode != HMCX_RNG_PHILOX) {
        return HMCX_ERR_INVALID_ARG;
    }
    a.rng_mode = rng->mode; a.seed = rng->seed; a.chain_offset = rng->chain_offset;
    a.normals = rng->normals; a.logu = rng->log_uniforms;
    a.nuts = (nuts && nuts->enabled) ? 1 : 0;
    if (a.nuts) {
        if (!nuts->table || !nuts->h_bar || !nuts->eps_bar || burn < 1) return HMCX_ERR_INVALID_ARG;
        a.delta = nuts->desired_accept_rate; a.mu = nuts->mu; a.table = nuts->table;
        a.h_bar = nuts->h_bar; a.eps_bar = nuts->eps_bar;
        a.eps_schedule = nuts->eps_schedule; a.eps_trace = nuts->eps_trace;
    }
    a.q_init = q_init; a.q_cur = q_cur; a.eps = eps; a.L = L; a.S = S; a.burn = burn; a.it0 = it0; a.it1 = it1;
    a.samples = samples; a.accept = accept; a.diverged = diverged; a.ham = ham; a.num_rejected = num_rejected;

    int E, K, G;
    if (tuning == 41 || tuning == 42) {                    // one chain per cluster of 4 / 2 CTAs (DSMEM reduction)
        if (sink) return HMCX_ERR_UNSUPPORTED;
        const int CS = tuning == 41 ? 4 : 2;
        const int groups = (ld / 4 + CS - 1) / CS;
        G = (groups + 31) / 32 * 32;
        if (G > 256) return HMCX_ERR_UNSUPPORTED;
        const bool philox = a.rng_mode == HMCX_RNG_PHILOX;
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3((unsigned)(C * CS)); cfg.blockDim = dim3((unsigned)G); cfg.stream = st;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = (unsigned)CS; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
        cfg.attrs = attr; cfg.numAttrs = 1;
#define CALLCL(TK, MK)                                                                                  \
        if (CS == 4 && philox) cudaLaunchKernelEx(&cfg, hmc_run_kernel<TK, MK, 4, 1, 256, false, true, 4>, a);   \
        else if (CS == 4) cudaLaunchKernelEx(&cfg, hmc_run_kernel<TK, MK, 4, 1, 256, false, false, 4>, a);       \
        else if (philox) cudaLaunchKernelEx(&cfg, hmc_run_kernel<TK, MK, 4, 1, 256, false, true, 2>, a);         \
        else cudaLaunchKernelEx(&cfg, hmc_run_kernel<TK, MK, 4, 1, 256, false, false, 2>, a)
        DISPATCH_TK_MK(a.t, CALLCL);
#undef CALLCL
        return cuda_status();
    }
    if (sink) {                                            // thinning / moments: float4-per-thread geometry only
        if (ld > 4096 || (tuning != 0 && tuning != 1)) return HMCX_ERR_UNSUPPORTED;
        a.thin = sink->thin; a.msum = sink->sum; a.msumsq = sink->sumsq;
        a.msum_lo = sink->sum_lo; a.msumsq_lo = sink->sumsq_lo;
        a.moments_all = sink->moments_all;
        if (a.nuts && nuts->mu_chain) { a.mu_per_chain = 1; a.mu_chain = nuts->mu_chain; }
        a.lp_carry = workspace;                            // windows of a sink run chain bit for bit, as the plain loop's
        pick_geometry(ld, 1, false, E, K, G);
#define CALLSINK(TK, MK)                                                                                \
        if (G <= 256) hmc_run_kernel<TK, MK, 4, 1, 256, true><<<C, G, 0, st>>>(a);                      \
        else hmc_run_kernel<TK, MK, 4, 1, 1024, true><<<C, G, 0, st>>>(a)
        DISPATCH_TK_MK(a.t, CALLSINK);
#undef CALLSINK
        return cuda_status();
    }
    if (ld > 4096 && tuning == 0) {                        // state does not fit one CTA's registers: streamed form
        if (!workspace) return HMCX_ERR_INVALID_ARG;       // needs hmcx_hmc_workspace_bytes() of scratch
#define CALLBIG(TK, MK) hmc_run_big_kernel<TK, MK><<<C, 1024, 0, st>>>(a, workspace)
        DISPATCH_TK_MK(a.t, CALLBIG);
#undef CALLBIG
        return cuda_status();
    }
    const bool philox = a.rng_mode == HMCX_RNG_PHILOX;
    const bool pair_ok = philox && !a.nuts;                // the paired K = 2 form is compiled for this loop only
    if (!pick_geometry(ld, tuning, pair_ok, E, K, G)) return tuning ? HMCX_ERR_INVALID_ARG : HMCX_ERR_UNSUPPORTED;
    a.lp_carry = workspace;                                // [C] floats (hmcx_hmc_workspace_bytes) or NULL
    const bool pair = tuning == 0 && K == 2 && G <= 128 && pair_ok;
    // the producer form's CTAs have 1.5x the threads and ~1.5x the registers per thread: it runs while every chain's CTA
    // finds an SM beside at most one other, and the plain paired form above that (measured at 512 chains, DESIGN §3.1)
    const bool producers = pair && G == 128 && C <= 2 * sm_count();     // G is 128 whenever 768 < ld <= 1024
#define CALL(TK, MK)                                                                                    \
    if (producers) hmc_run_kernel<TK, MK, 4, 2, 128, false, true, 1, false, 2><<<C, G + 64, 0, st>>>(a);  \
    else if (pair) hmc_run_kernel<TK, MK, 4, 2, 128, false, true, 1, false><<<C, G, 0, st>>>(a);        \
    else if (E == 2 && K == 1) hmc_run_kernel<TK, MK, 2, 1, 1024><<<C, G, 0, st>>>(a);                  \
    else if (E == 2) hmc_run_kernel<TK, MK, 2, 2, 1024><<<C, G, 0, st>>>(a);                            \
    else if (K == 1 && G <= 256 && philox && !a.nuts)                                                   \
        hmc_run_kernel<TK, MK, 4, 1, 256, false, true, 1, false><<<C, G, 0, st>>>(a);                   \
    else if (K == 1 && G <= 256 && philox) hmc_run_kernel<TK, MK, 4, 1, 256, false, true><<<C, G, 0, st>>>(a); \
    else if (K == 1 && G <= 256) hmc_run_kernel<TK, MK, 4, 1, 256><<<C, G, 0, st>>>(a);                 \
    else if (K == 1 && philox) hmc_run_kernel<TK, MK, 4, 1, 1024, false, true><<<C, G, 0, st>>>(a);     \
    else if (K == 1) hmc_run_kernel<TK, MK, 4, 1, 1024><<<C, G, 0, st>>>(a);                            \
    else if (K == 2 && philox) hmc_run_kernel<TK, MK, 4, 2, 512, false, true><<<C, G, 0, st>>>(a);      \
    else if (K == 2) hmc_run_kernel<TK, MK, 4, 2, 512><<<C, G, 0, st>>>(a);                             \
    else hmc_run_kernel<TK, MK, 4, 4, 256><<<C, G, 0, st>>>(a)
    DISPATCH_TK_MK(a.t, CALL);
#undef CALL
    return cuda_status();
}

#ifdef HMCX_HMC_PROF
// developer build only (scripts/prof_hmc_phases.py): copies out and clears the stamps (and the producer form's
// publication stamps, [CTA][iteration]); returns the number of stamps
extern "C" int hmcx_debug_hmc_prof(long long* stamps, int* sm, long long* pub) {
    const int n = HMC_PROF_CTAS * HMC_PROF_WARPS * HMC_PROF_ITS * HMC_PROF_IDS;
    cudaDeviceSynchronize();
    cudaMemcpyFromSymbol(stamps, g_hmc_prof, sizeof(long long) * n);
    cudaMemcpyFromSymbol(sm, g_hmc_prof_sm, sizeof(int) * HMC_PROF_CTAS);
    cudaMemcpyFromSymbol(pub, g_hmc_prof_pub, sizeof(long long) * HMC_PROF_CTAS * HMC_PROF_ITS);
    void* p = nullptr;
    cudaGetSymbolAddress(&p, g_hmc_prof);
    cudaMemset(p, 0, sizeof(long long) * n);
    cudaGetSymbolAddress(&p, g_hmc_prof_pub);
    cudaMemset(p, 0, sizeof(long long) * HMC_PROF_CTAS * HMC_PROF_ITS);
    cudaDeviceSynchronize();
    return n;
}
#endif

}  // namespace hmcx
