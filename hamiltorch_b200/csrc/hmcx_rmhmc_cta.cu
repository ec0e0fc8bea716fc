// hmcx_rmhmc_cta.cu -- Riemannian-manifold HMC with the metric assembled, eigen-decomposed and solved IN the kernel for
// 2 <= D <= 64: one CTA per chain, the D x D metric, its eigenvectors and one work matrix in shared memory.
//
//   fisher (HESSIAN / SOFTABS / JACOBIAN_DIAG, jitter)   samplers.py:69-127    -> rc_eval_metric()
//   cholesky_inverse                                      samplers.py:130-149   -> G~^-1 p = Q diag(1/lam~) Q^T p
//   rm_hamiltonian                                        samplers.py:677-736   -> rc_hamiltonian()
//   gibbs (RMHMC)                                         samplers.py:183-184   -> rc_gibbs(): in-kernel Cholesky of G~
//   explicit / implicit leapfrog                          samplers.py:389-462, :305-387
//   sample() loop                                         samplers.py:965-1067  -> rmhmc_cta_kernel
//   stand-alone leapfrog() / hamiltonian(), sampler=RMHMC  samplers.py:305-462, :817-829 -> the same kernel with the
//                                                         momentum supplied (`p_given`) and per-step trajectory outputs
//
// This is the general-D form of hmcx_rmhmc.cu (which keeps D <= 16 in one thread's registers): position-dependent
// metrics (Funnel) and per-call random metrics (Gaussian targets with jitter) beyond D = 16, where the round-1 engine
// had only the constant-metric tensor-core path.  The eigensolver is a two-sided cyclic Jacobi in PARALLEL ORDER: a
// round-robin schedule gives D/2 disjoint rotations per step; with both rotations of a (row pair, column pair) known, the
// 2x2 block A[P_i, P_j] <- J_i^T A[P_i, P_j] J_j is independent of every other block, so a step is "compute D/2 rotations,
// barrier, update (D/2)^2 blocks of A and D*D/2 column pairs of Q in place, barrier" -- two barriers per step, D-1 steps
// per sweep.  dH/dtheta is the closed form of hmcx_rmhmc.cu (Betancourt's softabs derivative); for the Funnel only
// row 0 and the diagonal of Z = Q B Q^T enter the contraction with dG/dtheta, so one D^3 product (Q B) suffices.
// Bound: barrier latency and shared-memory traffic of a tiny dense eigenproblem per metric evaluation (8L+3 per
// iteration) -- neither HBM nor tensor cores; many chains run concurrently (several CTAs per SM).
#include "hmcx_rm.cuh"

namespace hmcx {

constexpr int RC_T = 256;                 // threads per chain
constexpr int RC_DMAX = 64;
static_assert(4 * JITTER_VECS_PER_CALL >= RC_DMAX, "a fisher() call's jitter row would overlap the next call's counters");

struct RcArgs {
    RmTarget t;
    RmCfg cfg;
    int integrator;               // 1 explicit, 2 implicit
    float cosw, sinw, fp_threshold;
    int fp_max_iter, jitter_max_tries;
    int C, ld, rng_mode;
    uint64_t seed, chain_offset;
    const float* normals;         // [S, C, ld]
    const float* logu;            // [S, C]
    const float* uniforms;        // [S, C, J, ld]
    int J;
    const float* q_init;
    float* q_cur;
    const float* eps;
    int L, S, burn, it0, it1;
    float* samples;
    uint8_t* accept;
    uint8_t* diverged;
    float* ham;
    int32_t* num_rejected;
    // stand-alone leapfrog() / hamiltonian(): one "iteration" with the momentum given, no MH
    const float* p_given;         // [C, ld] or NULL
    float* q_traj;                // [L, C, ld] or NULL: theta after every step (ret_params)
    float* p_traj;                // [L, C, ld] or NULL: p after every step (ret_momenta)
    float* qt_out;                // [C, ld] or NULL: explicit integrator's params_copy after the last step (:462)
    float* pt_out;                // [C, ld] or NULL: momentum_copy
    int only_h;                   // 1: evaluate H(theta, p_given) only (hamiltonian())
    float* h_out;                 // [C] or NULL: that H
};

// ---------------------------------------------------------------------------------------------------------
// per-CTA context: shared-memory views
// ---------------------------------------------------------------------------------------------------------
struct Rc {
    int D, DP, tid;
    float* A;        // D x DP   metric / Jacobi work matrix; afterwards Q.B
    float* Q;        // D x DP   eigenvectors in columns
    float* W;        // D x DP   work: B, G~ for the Cholesky, the Hessian for JACOBIAN_DIAG
    float* lam; float* lt; float* dlt; float* w; float* u; float* ub; float* glp; float* t0; float* t1;
    float* cs;       // D floats: (c, s) of the D/2 rotations of a step
    int* pr;         // D ints: the pairs (p, q) of a step
    float* red;      // 40 floats: block reductions
    int* flag;
};

__device__ __forceinline__ float rc_block_sum(const Rc& c, float v) {
    v = warp_sum(v);
    const int lane = c.tid & 31, warp = c.tid >> 5;
    __syncthreads();                                   // red[] may still be read from the previous reduction
    if (lane == 0) c.red[warp] = v;
    __syncthreads();
    float s = c.red[0];
#pragma unroll
    for (int wv = 1; wv < RC_T / 32; ++wv) s = add(s, c.red[wv]);
    return s;                                          // same bits in every thread
}

// Code size: rc_eval_metric / rc_hamiltonian / rc_grad_* are OUT-OF-LINE (one copy each).  Inlined at the iteration's 15 call
// sites the kernel was 91k instructions (1.4 MB) and ran at the instruction-fetch rate; all threads of the CTA call them
// convergently (they contain barriers).
// ---- targets (same closed forms as hmcx_rmhmc.cu, vectorised over the CTA) ------------------------------------------
// sum of x_i^2 over i >= 1 (Funnel) -- every thread gets the value
__device__ __forceinline__ float rc_funnel_s(const Rc& c, const float* th) {
    float v = 0.0f;
    for (int i = 1 + c.tid; i < c.D; i += RC_T) v = add(v, mul(th[i], th[i]));
    return rc_block_sum(c, v);
}

__device__ float rc_log_prob(const Rc& c, const RmTarget& t, const float* th) {
    const int d = c.D;
    if (t.kind == HMCX_TARGET_FUNNEL) {
        const float s = rc_funnel_s(c, th);
        const float v = th[0];
        const float t1 = mul((float)(-0.5 * (double)t.inv_var_v), mul(v, v));
        const float t2 = mul(0.5f * (float)(d - 1), v);
        const float t3 = mul(mul(0.5f, expf(v)), s);
        return add(sub(add(t1, t2), t3), t.log_norm);
    }
    float part = 0.0f;
    if (t.kind == HMCX_TARGET_GAUSS_FULL) {
        for (int a = c.tid; a < d; a += RC_T) {
            float r = 0.0f;
            for (int b = 0; b < d; ++b) r += t.prec[a * d + b] * (th[b] - (t.mean ? t.mean[b] : 0.0f));
            part += (th[a] - (t.mean ? t.mean[a] : 0.0f)) * r;
        }
    } else {
        for (int i = c.tid; i < d; i += RC_T) {
            if (t.kind == HMCX_TARGET_GAUSS_ISO) part = add(part, mul(th[i], th[i]));
            else { const float y = sub(th[i], t.mean ? t.mean[i] : 0.0f); part = add(part, mul(mul(y, y), t.ivar[i])); }
        }
    }
    return add(mul(-0.5f, rc_block_sum(c, part)), t.log_norm);
}

// g (shared, D) = grad log p(th); callers barrier before reading
__device__ void rc_grad_log_prob(const Rc& c, const RmTarget& t, const float* th, float* g) {
    const int d = c.D;
    if (t.kind == HMCX_TARGET_FUNNEL) {
        float v = 0.0f;
        for (int i = 1 + c.tid; i < d; i += RC_T) v += th[i] * th[i];
        const float s = rc_block_sum(c, v);
        const float E = expf(th[0]);
        for (int i = 1 + c.tid; i < d; i += RC_T) g[i] = -(E * th[i]);
        if (c.tid == 0) g[0] = -(t.inv_var_v * th[0]) + 0.5f * (float)(d - 1) - 0.5f * E * s;
        return;
    }
    for (int a = c.tid; a < d; a += RC_T) {
        if (t.kind == HMCX_TARGET_GAUSS_FULL) {
            float r = 0.0f;
            for (int b = 0; b < d; ++b) r += t.prec[a * d + b] * (th[b] - (t.mean ? t.mean[b] : 0.0f));
            g[a] = -r;
        } else {
            g[a] = (t.kind == HMCX_TARGET_GAUSS_ISO) ? -th[a] : -(t.ivar[a] * (th[a] - (t.mean ? t.mean[a] : 0.0f)));
        }
    }
}

// M (shared, D x DP) = -Hessian(log p)(th); callers barrier before reading
__device__ void rc_fill_metric(const Rc& c, const RmTarget& t, const float* th, float* M) {
    const int d = c.D, DP = c.DP;
    float s = 0.0f, E = 0.0f;
    if (t.kind == HMCX_TARGET_FUNNEL) { s = rc_funnel_s(c, th); E = expf(th[0]); }
    for (int e = c.tid; e < d * d; e += RC_T) {
        const int a = e / d, b = e - a * d;
        float v = 0.0f;
        if (t.kind == HMCX_TARGET_FUNNEL) {
            if (a == 0 && b == 0) v = t.inv_var_v + 0.5f * E * s;
            else if (a == 0) v = E * th[b];
            else if (b == 0) v = E * th[a];
            else if (a == b) v = E;
        } else if (t.kind == HMCX_TARGET_GAUSS_FULL) {
            v = t.prec[a * d + b];
        } else if (a == b) {
            v = (t.kind == HMCX_TARGET_GAUSS_ISO) ? 1.0f : t.ivar[a];
        }
        M[a * DP + b] = v;
    }
}

// ---- parallel-order cyclic Jacobi: A (symmetric, destroyed) -> eigenvalues on its diagonal, Q = eigenvectors ---------
__device__ void rc_jacobi(const Rc& c) {
    const int d = c.D, DP = c.DP, tid = c.tid;
    const int m = (d + 1) & ~1;                         // players of the round-robin (a dummy when D is odd)
    const int np = m >> 1;
    for (int e = tid; e < d * d; e += RC_T) { const int a = e / d, b = e - a * d; c.Q[a * DP + b] = (a == b) ? 1.0f : 0.0f; }
    __syncthreads();
    // e / np for e < 16384, np <= 64 as one multiply-shift (ncu: the two integer divisions of the update loops were 23 % of
    // the kernel's instructions)
    const unsigned magic = ((1u << 20) + (unsigned)np - 1u) / (unsigned)np;
    for (int sweep = 0; sweep < 14; ++sweep) {
        float off = 0.0f, dg = 0.0f;
        for (int e = tid; e < d * d; e += RC_T) {
            const int a = e / d, b = e - a * d;
            const float v = c.A[a * DP + b];
            if (a == b) dg += v * v; else if (b > a) off += v * v;
        }
        off = rc_block_sum(c, off);
        dg = rc_block_sum(c, dg);
        if (!(off > 1e-14f * dg)) break;               // uniform: every thread holds the same sums
        for (int r = 0; r < m - 1; ++r) {
            if (tid < np) {                            // pair k of round r (circle method, player m-1 fixed)
                int p, q;
                if (tid == 0) { p = m - 1; q = r; }
                else { p = r + tid; if (p >= m - 1) p -= m - 1; q = r - tid; if (q < 0) q += m - 1; }   // tid, r < m - 1
                if (p > q) { const int x = p; p = q; q = x; }
                float cc = 1.0f, ss = 0.0f;
                if (q < d) {                           // (a pair with the dummy player of an odd D is skipped)
                    const float apq = c.A[p * DP + q];
                    if (fabsf(apq) >= 1e-30f) {
                        const float theta = (c.A[q * DP + q] - c.A[p * DP + p]) / (2.0f * apq);
                        const float tt = (theta >= 0.0f ? 1.0f : -1.0f) / (fabsf(theta) + sqrtf(theta * theta + 1.0f));
                        cc = rsqrtf(tt * tt + 1.0f);
                        ss = tt * cc;
                    }
                } else { q = -1; }
                reinterpret_cast<int2*>(c.pr)[tid] = make_int2(p, q);          // (8-byte aligned: every carve-out before is even)
                reinterpret_cast<float2*>(c.cs)[tid] = make_float2(cc, ss);
            }
            __syncthreads();
            for (int e = tid; e < np * np; e += RC_T) {         // A[P_i, P_j] <- J_i^T A[P_i, P_j] J_j
                const int i = (int)(((unsigned)e * magic) >> 20), j = e - i * np;
                const int2 pi = reinterpret_cast<const int2*>(c.pr)[i], pj = reinterpret_cast<const int2*>(c.pr)[j];
                const float2 ri = reinterpret_cast<const float2*>(c.cs)[i], rj = reinterpret_cast<const float2*>(c.cs)[j];
                const int p1 = pi.x, q1 = pi.y, p2 = pj.x, q2 = pj.y;
                const float c1 = ri.x, s1 = ri.y, c2 = rj.x, s2 = rj.y;
                if (q1 < 0 && q2 < 0) continue;
                if (q1 < 0) {                          // row p1 (the dummy's partner) only sees the column rotation
                    const float a = c.A[p1 * DP + p2], b = c.A[p1 * DP + q2];
                    c.A[p1 * DP + p2] = c2 * a - s2 * b; c.A[p1 * DP + q2] = s2 * a + c2 * b;
                } else if (q2 < 0) {
                    const float a = c.A[p1 * DP + p2], b = c.A[q1 * DP + p2];
                    c.A[p1 * DP + p2] = c1 * a - s1 * b; c.A[q1 * DP + p2] = s1 * a + c1 * b;
                } else {
                    const float a = c.A[p1 * DP + p2], b = c.A[p1 * DP + q2], cq = c.A[q1 * DP + p2], dd = c.A[q1 * DP + q2];
                    const float t1 = c2 * a - s2 * b, t2 = s2 * a + c2 * b, t3 = c2 * cq - s2 * dd, t4 = s2 * cq + c2 * dd;
                    c.A[p1 * DP + p2] = c1 * t1 - s1 * t3; c.A[q1 * DP + p2] = s1 * t1 + c1 * t3;
                    c.A[p1 * DP + q2] = c1 * t2 - s1 * t4; c.A[q1 * DP + q2] = s1 * t2 + c1 * t4;
                }
            }
            for (int e = tid; e < d * np; e += RC_T) {          // Q <- Q J
                const int k = (int)(((unsigned)e * magic) >> 20), j = e - k * np;
                const int2 pj = reinterpret_cast<const int2*>(c.pr)[j];
                const int p = pj.x, q = pj.y;
                if (q < 0) continue;
                const float2 rj = reinterpret_cast<const float2*>(c.cs)[j];
                const float cc = rj.x, ss = rj.y;
                const float a = c.Q[k * DP + p], b = c.Q[k * DP + q];
                c.Q[k * DP + p] = cc * a - ss * b; c.Q[k * DP + q] = ss * a + cc * b;
            }
            __syncthreads();
        }
    }
    for (int i = tid; i < d; i += RC_T) c.lam[i] = c.A[i * DP + i];
    __syncthreads();
}

// fisher(): false <=> the reference raises LogProbError (:110-112, :717).  Leaves Q, lam, lt, dlt.  urow = this call's
// jitter uniforms (shared, D) or NULL.
__device__ __noinline__ bool rc_eval_metric(const Rc& c, const RmTarget& t, const RmCfg& cfg, const float* th, const float* urow) {
    const int d = c.D, DP = c.DP, tid = c.tid;
    int bad = 0;
    if (cfg.jacdiag) {                                 // G = diag(g_i^2 (+ jitter)): already diagonal
        rc_grad_log_prob(c, t, th, c.glp);
        __syncthreads();
        for (int e = tid; e < d * d; e += RC_T) { const int a = e / d, b = e - a * d; c.Q[a * DP + b] = (a == b) ? 1.0f : 0.0f; }
        for (int i = tid; i < d; i += RC_T) {
            float v = mul(c.glp[i], c.glp[i]);
            if (urow) v = add(v, mul(urow[i], cfg.jitter));
            c.lam[i] = v; c.lt[i] = v; c.dlt[i] = 1.0f;
            bad |= !finite_f(v);
        }
        return !__syncthreads_or(bad);
    }
    rc_fill_metric(c, t, th, c.A);
    __syncthreads();
    for (int i = tid; i < d; i += RC_T)
        if (urow) c.A[i * DP + i] = add(c.A[i * DP + i], mul(urow[i], cfg.jitter));
    __syncthreads();
    for (int e = tid; e < d * d; e += RC_T) { const int a = e / d, b = e - a * d; bad |= !finite_f(c.A[a * DP + b]); }
    if (__syncthreads_or(bad)) return false;
    rc_jacobi(c);
    bad = 0;
    for (int i = tid; i < d; i += RC_T) {
        const float l = c.lam[i];
        if (cfg.softabs) {
            const float x = cfg.alpha * l;
            if (fabsf(x) >= 20.0f && finite_f(x)) {    // saturated softabs: exactly the bits of the general branch
                const float sg = x > 0.0f ? 1.0f : -1.0f;
                c.lt[i] = sg * l; c.dlt[i] = sg;
            } else {
                const float th_ = tanhf(x);
                c.lt[i] = (1.0f / th_) * l;
                const float sh = sinhf(x);
                float dv = 1.0f / th_ - x / (sh * sh);
                if (!finite_f(dv)) dv = (l >= 0.0f) ? 1.0f : -1.0f;
                c.dlt[i] = dv;
            }
        } else { c.lt[i] = l; c.dlt[i] = 1.0f; }
        bad |= !finite_f(c.lt[i]);
    }
    return !__syncthreads_or(bad);
}

// rm_hamiltonian (:710-736) given the metric; leaves w = Q^T p (shared).  ok=false <=> LogProbError.
__device__ __noinline__ float rc_hamiltonian(const Rc& c, const RmTarget& t, const RmCfg& cfg, const float* th, const float* p, bool& ok) {
    const int d = c.D, DP = c.DP, tid = c.tid;
    const float lp = rc_log_prob(c, t, th);
    float ld_part = 0.0f, q_part = 0.0f;
    int bad = 0;
    for (int i = tid; i < d; i += RC_T) {
        float wi = 0.0f;
        for (int a = 0; a < d; ++a) wi += c.Q[a * DP + i] * p[a];
        c.w[i] = wi;
        const float l = c.lt[i];
        if (cfg.softabs) ld_part += logf(l);
        else { ld_part += logf(fabsf(l)); bad |= !(l > 0.0f); }           // Cholesky of a non-PD metric
        q_part += wi * wi / l;
    }
    const float logdet = rc_block_sum(c, ld_part);
    const float quad = rc_block_sum(c, q_part);
    const float H = add(add(add(-lp, mul(0.5f, cfg.pi_term)), mul(0.5f, logdet)), mul(0.5f, quad));
    bad |= !finite_f(lp) || !finite_f(H);
    if (__syncthreads_or(bad)) ok = false;
    return H;
}

// dH/dp = G~^-1 p -> out (shared); needs w from rc_hamiltonian.  Callers barrier before reading out.
__device__ __noinline__ void rc_grad_momentum(const Rc& c, float* out) {
    const int d = c.D, DP = c.DP, tid = c.tid;
    for (int i = tid; i < d; i += RC_T) c.u[i] = c.w[i] / c.lt[i];
    __syncthreads();
    for (int a = tid; a < d; a += RC_T) {
        float s = 0.0f;
        for (int i = 0; i < d; ++i) s += c.Q[a * DP + i] * c.u[i];
        out[a] = s;
    }
}

// dH/dtheta -> out (shared); needs w.  Returns false when a component is non-finite (the NaN-retry test, :402).
__device__ __noinline__ bool rc_grad_params(const Rc& c, const RmTarget& t, const RmCfg& cfg, const float* th, const float* p, float* out) {
    const int d = c.D, DP = c.DP, tid = c.tid;
    rc_grad_log_prob(c, t, th, c.glp);
    __syncthreads();
    if (cfg.jacdiag) {
        // dH/dtheta_k = -g_k + sum_i (1/(2 d_i) - p_i^2/(2 d_i^2)) 2 g_i Hess_ik,  Hess = -(rc_fill_metric's matrix)
        rc_fill_metric(c, t, th, c.W);
        for (int i = tid; i < d; i += RC_T) {
            const float ui = p[i] / c.lt[i];
            c.t0[i] = (0.5f / c.lt[i] - 0.5f * ui * ui) * 2.0f * c.glp[i];
        }
        __syncthreads();
        for (int k = tid; k < d; k += RC_T) {
            float s = 0.0f;
            for (int i = 0; i < d; ++i) s += c.t0[i] * (-c.W[i * DP + k]);
            out[k] = s - c.glp[k];
        }
    } else if (t.kind != HMCX_TARGET_FUNNEL) {
        for (int k = tid; k < d; k += RC_T) out[k] = 0.0f - c.glp[k];     // constant Hessian: the metric term vanishes
    } else {
        for (int i = tid; i < d; i += RC_T) c.u[i] = c.w[i] / c.lt[i];
        __syncthreads();
        for (int e = tid; e < d * d; e += RC_T) {                        // B_ij
            const int i = e / d, j = e - i * d;
            float F;
            if (i == j) F = c.dlt[i];
            else {
                const float dl = c.lam[i] - c.lam[j];
                F = (fabsf(dl) > 1e-12f * (fabsf(c.lam[i]) + fabsf(c.lam[j]))) ? (c.lt[i] - c.lt[j]) / dl : c.dlt[i];
            }
            c.W[i * DP + j] = -0.5f * c.u[i] * c.u[j] * F + ((i == j) ? 0.5f * c.dlt[i] / c.lt[i] : 0.0f);
        }
        __syncthreads();
        for (int e = tid; e < d * d; e += RC_T) {                        // A <- Q B   (A is free after the eigensolve)
            const int a = e / d, j = e - a * d;
            float s = 0.0f;
            for (int i = 0; i < d; ++i) s += c.Q[a * DP + i] * c.W[i * DP + j];
            c.A[a * DP + j] = s;
        }
        __syncthreads();
        for (int b = tid; b < d; b += RC_T) {                            // Z_0b and Z_bb of Z = Q B Q^T
            float z0 = 0.0f, zb = 0.0f;
            for (int j = 0; j < d; ++j) { z0 += c.A[j] * c.Q[b * DP + j]; zb += c.A[b * DP + j] * c.Q[b * DP + j]; }
            c.t0[b] = z0; c.t1[b] = zb;
        }
        __syncthreads();
        float sp = 0.0f, zxp = 0.0f, trp = 0.0f;
        for (int i = 1 + tid; i < d; i += RC_T) { sp += th[i] * th[i]; zxp += c.t0[i] * th[i]; trp += c.t1[i]; }
        const float s = rc_block_sum(c, sp), zx = rc_block_sum(c, zxp), tr = rc_block_sum(c, trp);
        const float E = expf(th[0]), z00 = c.t0[0];
        for (int i = 1 + tid; i < d; i += RC_T) out[i] = (z00 * E * th[i] + 2.0f * c.t0[i] * E) - c.glp[i];
        if (tid == 0) out[0] = (z00 * (0.5f * E * s) + 2.0f * E * zx + E * tr) - c.glp[0];
    }
    __syncthreads();
    int bad = 0;
    for (int i = tid; i < d; i += RC_T) bad |= !finite_f(out[i]);
    return !__syncthreads_or(bad);
}

// gibbs (:183-184): p = chol(G~) z,  G~ = Q diag(lam~) Q^T  (MultivariateNormal's scale_tril)
__device__ __noinline__ bool rc_gibbs(const Rc& c, const float* z, float* p) {
    const int d = c.D, DP = c.DP, tid = c.tid;
    for (int e = tid; e < d * d; e += RC_T) {
        const int a = e / d, b = e - a * d;
        if (b > a) continue;
        float s = 0.0f;
        for (int i = 0; i < d; ++i) s += c.Q[a * DP + i] * c.lt[i] * c.Q[b * DP + i];
        c.W[a * DP + b] = s;
    }
    __syncthreads();
    int bad = 0;
    for (int j = 0; j < d; ++j) {                      // right-looking Cholesky, lower, in place
        if (tid == 0) {
            float s = c.W[j * DP + j];
            for (int k = 0; k < j; ++k) s -= c.W[j * DP + k] * c.W[j * DP + k];
            if (!(s > 0.0f)) bad = 1;
            c.W[j * DP + j] = sqrtf(s);
        }
        __syncthreads();
        const float ljj = c.W[j * DP + j];
        for (int i = j + 1 + tid; i < d; i += RC_T) {
            float v = c.W[i * DP + j];
            for (int k = 0; k < j; ++k) v -= c.W[i * DP + k] * c.W[j * DP + k];
            c.W[i * DP + j] = v / ljj;
        }
        __syncthreads();
    }
    for (int a = tid; a < d; a += RC_T) {
        float s = 0.0f;
        for (int b = 0; b <= a; ++b) s += c.W[a * DP + b] * z[b];
        p[a] = s;
    }
    const bool ok = !__syncthreads_or(bad);
    return ok;
}

// ---------------------------------------------------------------------------------------------------------
// the kernel: one CTA = one chain
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(RC_T) rmhmc_cta_kernel(const RcArgs a) {
    extern __shared__ __align__(16) float smem[];
    const int c_ = blockIdx.x, tid = threadIdx.x;
    const RmTarget& t = a.t;
    Rc c;
    c.D = t.D; c.DP = t.D + 1; c.tid = tid;
    const int d = c.D, MS = d * c.DP;
    float* f = smem;
    c.A = f; f += MS; c.Q = f; f += MS; c.W = f; f += MS;
    c.lam = f; f += RC_DMAX; c.lt = f; f += RC_DMAX; c.dlt = f; f += RC_DMAX; c.w = f; f += RC_DMAX; c.u = f; f += RC_DMAX;
    c.ub = f; f += RC_DMAX; c.glp = f; f += RC_DMAX; c.t0 = f; f += RC_DMAX; c.t1 = f; f += RC_DMAX;
    float* qc = f; f += RC_DMAX; float* q = f; f += RC_DMAX; float* p = f; f += RC_DMAX;
    float* qt = f; f += RC_DMAX; float* pt = f; f += RC_DMAX; float* g = f; f += RC_DMAX; float* g2 = f; f += RC_DMAX;
    float* zz = f; f += RC_DMAX;
    c.cs = f; f += RC_DMAX; c.red = f; f += 40;
    c.pr = reinterpret_cast<int*>(f); f += RC_DMAX;
    c.flag = reinterpret_cast<int*>(f);

    const size_t row = (size_t)c_ * a.ld;
    const uint64_t chain_id = a.chain_offset + (uint64_t)c_;
    for (int i = tid; i < d; i += RC_T) qc[i] = a.p_given ? a.q_init[row + i] : a.q_cur[row + i];
    const float eps = a.eps ? a.eps[c_] : 0.0f;
    const float half = mul(0.5f, eps);
    int rejected = 0;
    const int keep = a.S - a.burn;
    float* const my_samples = a.samples ? a.samples + (size_t)c_ * keep * a.ld : nullptr;
    if (a.it0 == 0 && my_samples)
        for (int i = tid; i < a.ld; i += RC_T) my_samples[i] = i < d ? qc[i] : 0.0f;
    __syncthreads();
    const bool jit_on = a.cfg.jitter >= 0.0f;

    for (int n = a.it0; n < a.it1; ++n) {
        int idx = 0;
        bool ok = true;
        float h_old = nanf(""), h_new = nanf("");
        // the jitter row of the next fisher() call -> c.ub (shared); NULL without jitter
        auto next_jitter = [&]() -> const float* {
            if (!jit_on) return nullptr;
            const int k = idx++;
            __syncthreads();                                     // previous readers of ub are done
            if (a.rng_mode == HMCX_RNG_INJECTED) {
                const int j = k < a.J ? k : a.J - 1;
                const float* src = a.uniforms + (((size_t)(n - a.it0) * a.C + c_) * a.J + j) * a.ld;
                for (int i = tid; i < d; i += RC_T) c.ub[i] = src[i];
            } else {
                for (int v = tid; 4 * v < d; v += RC_T) {
                    float u[4];
                    philox_jitter4(a.seed, chain_id, (uint64_t)n, k, v, u);
                    for (int j = 0; j < 4 && 4 * v + j < d; ++j) c.ub[4 * v + j] = u[j];
                }
            }
            __syncthreads();
            return c.ub;
        };
        // dH/dtheta with the reference's NaN-retry loop (:402-410) -> out; dH/dp (:415-422) -> out
        auto dHdq = [&](const float* th, const float* pp, float* out) {
            for (int tries = 0; ok; ++tries) {
                if (!rc_eval_metric(c, t, a.cfg, th, next_jitter())) { ok = false; break; }
                bool okh = true;
                rc_hamiltonian(c, t, a.cfg, th, pp, okh);
                if (!okh) { ok = false; break; }
                if (rc_grad_params(c, t, a.cfg, th, pp, out)) break;
                if (tries + 1 > a.jitter_max_tries) { ok = false; break; }
            }
        };
        auto dHdp = [&](const float* th, const float* pp, float* out) {
            if (!ok) return;
            if (!rc_eval_metric(c, t, a.cfg, th, next_jitter())) { ok = false; return; }
            bool okh = true;
            rc_hamiltonian(c, t, a.cfg, th, pp, okh);
            if (!okh) { ok = false; return; }
            rc_grad_momentum(c, out);
            __syncthreads();
        };
        auto axpy = [&](float* y, float coef, const float* x, bool minus) {      // y = y -/+ coef * x (reference roundings)
            if (ok)
                for (int i = tid; i < d; i += RC_T) y[i] = minus ? sub(y[i], mul(coef, x[i])) : add(y[i], mul(coef, x[i]));
            __syncthreads();
        };

        // ---- momentum: gibbs (:969 -> :183-184), or the caller's (stand-alone leapfrog / hamiltonian) ----
        if (a.p_given) {
            for (int i = tid; i < d; i += RC_T) p[i] = a.p_given[row + i];
        } else {
            ok = rc_eval_metric(c, t, a.cfg, qc, next_jitter());
            if (a.rng_mode == HMCX_RNG_INJECTED) {
                for (int i = tid; i < d; i += RC_T) zz[i] = a.normals[((size_t)(n - a.it0) * a.C + c_) * a.ld + i];
            } else {
                for (int v = tid; 4 * v < d; v += RC_T) {
                    float z4[4];
                    philox_normal4(a.seed, chain_id, (uint64_t)n, (uint32_t)v, z4);
                    for (int j = 0; j < 4 && 4 * v + j < d; ++j) zz[4 * v + j] = z4[j];
                }
            }
            __syncthreads();
            if (ok) ok = rc_gibbs(c, zz, p);
        }
        for (int i = tid; i < d; i += RC_T) q[i] = qc[i];
        __syncthreads();
        // ---- H(theta, p) (:971) ----
        if (!a.p_given || a.only_h) {
            if (ok && rc_eval_metric(c, t, a.cfg, q, next_jitter())) h_old = rc_hamiltonian(c, t, a.cfg, q, p, ok);
            else ok = false;
        }
        // ---- trajectory ----
        if (!a.only_h && a.integrator == 1) {                                       // explicit (:423-461)
            for (int i = tid; i < d; i += RC_T) { qt[i] = q[i]; pt[i] = p[i]; }
            __syncthreads();
            for (int l = 0; l < a.L && ok; ++l) {
                dHdq(q, pt, g);  axpy(p, half, g, true);                              // A
                dHdp(q, pt, g);  axpy(qt, half, g, false);
                dHdp(qt, p, g);  axpy(q, half, g, false);                             // B
                dHdq(qt, p, g);  axpy(pt, half, g, true);
                if (!ok) break;
                for (int i = tid; i < d; i += RC_T) {                                 // C, sequential (:447-450)
                    const float cw = a.cosw, sw = a.sinw;
                    const float qn = mul(0.5f, add(add(add(q[i], qt[i]), mul(cw, sub(q[i], qt[i]))), mul(sw, sub(p[i], pt[i]))));
                    const float pn = mul(0.5f, add(sub(add(p[i], pt[i]), mul(sw, sub(qn, qt[i]))), mul(cw, sub(p[i], pt[i]))));
                    const float qtn = mul(0.5f, sub(sub(add(qn, qt[i]), mul(cw, sub(qn, qt[i]))), mul(sw, sub(pn, pt[i]))));
                    const float ptn = mul(0.5f, sub(add(add(pn, pt[i]), mul(sw, sub(qn, qtn))), mul(cw, sub(pn, pt[i]))));
                    q[i] = qn; p[i] = pn; qt[i] = qtn; pt[i] = ptn;
                }
                __syncthreads();
                dHdp(qt, p, g);  axpy(q, half, g, false);                             // B
                dHdq(qt, p, g);  axpy(pt, half, g, true);
                dHdq(q, pt, g);  axpy(p, half, g, true);                              // A
                dHdp(q, pt, g);  axpy(qt, half, g, false);
                if (ok && a.q_traj) for (int i = tid; i < a.ld; i += RC_T) a.q_traj[((size_t)l * a.C + c_) * a.ld + i] = i < d ? q[i] : 0.0f;
                if (ok && a.p_traj) for (int i = tid; i < a.ld; i += RC_T) a.p_traj[((size_t)l * a.C + c_) * a.ld + i] = i < d ? p[i] : 0.0f;
            }
            if (a.qt_out) for (int i = tid; i < a.ld; i += RC_T) a.qt_out[row + i] = (ok && i < d) ? qt[i] : (i < d ? nanf("") : 0.0f);
            if (a.pt_out) for (int i = tid; i < a.ld; i += RC_T) a.pt_out[row + i] = (ok && i < d) ? pt[i] : (i < d ? nanf("") : 0.0f);
        } else if (!a.only_h) {                                                      // implicit (:363-386)
            for (int l = 0; l < a.L && ok; ++l) {
                for (int i = tid; i < d; i += RC_T) pt[i] = p[i];                     // momentum_old
                __syncthreads();
                for (int it = 0; it < a.fp_max_iter && ok; ++it) {                    // fixed_point_momentum
                    dHdq(q, p, g);
                    if (!ok) break;
                    float diff = 0.0f;
                    for (int i = tid; i < d; i += RC_T) {
                        const float pn = sub(pt[i], mul(half, g[i]));
                        const float e = sub(p[i], pn);
                        diff = fmaxf(diff, mul(e, e));
                        p[i] = pn;
                    }
                    if (!__syncthreads_or(diff >= a.fp_threshold || diff != diff)) break;   // max diff < threshold
                }
                if (!ok) break;
                for (int i = tid; i < d; i += RC_T) qt[i] = q[i];                     // params_old
                __syncthreads();
                dHdp(q, p, g2);                                                       // the (theta_old, p) term
                for (int it = 0; it < a.fp_max_iter && ok; ++it) {                    // fixed_point_params
                    dHdp(q, p, g);
                    if (!ok) break;
                    float diff = 0.0f;
                    for (int i = tid; i < d; i += RC_T) {
                        const float qn = add(add(qt[i], mul(half, g[i])), mul(half, g2[i]));
                        const float e = sub(q[i], qn);
                        diff = fmaxf(diff, mul(e, e));
                        q[i] = qn;
                    }
                    if (!__syncthreads_or(diff >= a.fp_threshold || diff != diff)) break;
                }
                if (!ok) break;
                dHdq(q, p, g);  axpy(p, half, g, true);
                if (ok && a.q_traj) for (int i = tid; i < a.ld; i += RC_T) a.q_traj[((size_t)l * a.C + c_) * a.ld + i] = i < d ? q[i] : 0.0f;
                if (ok && a.p_traj) for (int i = tid; i < a.ld; i += RC_T) a.p_traj[((size_t)l * a.C + c_) * a.ld + i] = i < d ? p[i] : 0.0f;
            }
        }
        const size_t o = (size_t)c_ * a.S + n;
        if (a.p_given) {                                                             // stand-alone call: no MH
            if (tid == 0) {
                if (a.diverged) a.diverged[o] = ok ? 0 : 1;
                if (a.ham) { a.ham[2 * o] = h_old; a.ham[2 * o + 1] = h_new; }
                if (a.h_out) a.h_out[c_] = h_old;
            }
            for (int i = tid; i < d; i += RC_T) qc[i] = q[i];
            __syncthreads();
            continue;
        }
        // ---- H(theta_L, p_L) on the un-augmented Hamiltonian (:989) ----
        if (ok && rc_eval_metric(c, t, a.cfg, q, next_jitter())) h_new = rc_hamiltonian(c, t, a.cfg, q, p, ok);
        else ok = false;
        // ---- MH + bookkeeping ----
        const float x = add(-h_new, h_old);
        const float rho = (x < 0.0f) ? x : 0.0f;
        const float logu = (a.rng_mode == HMCX_RNG_INJECTED) ? a.logu[(size_t)(n - a.it0) * a.C + c_]
                                                             : philox_log_uniform(a.seed, chain_id, (uint64_t)n);
        const bool acc = ok && (rho >= logu);
        __syncthreads();
        if (acc) {
            for (int i = tid; i < d; i += RC_T) qc[i] = q[i];
        } else {
            ++rejected;
            if (n == a.burn + 1) for (int i = tid; i < d; i += RC_T) qc[i] = a.q_init[row + i];   // :1018 quirk
        }
        __syncthreads();
        if (n > a.burn && my_samples) {
            float* dst = my_samples + (size_t)(n - a.burn) * a.ld;
            for (int i = tid; i < a.ld; i += RC_T) dst[i] = i < d ? qc[i] : 0.0f;
        }
        if (tid == 0) {
            if (a.accept) a.accept[o] = acc ? 1 : 0;
            if (a.diverged) a.diverged[o] = ok ? 0 : 1;
            if (a.ham) { a.ham[2 * o] = h_old; a.ham[2 * o + 1] = h_new; }
        }
    }
    if (!a.p_given) for (int i = tid; i < d; i += RC_T) a.q_cur[row + i] = qc[i];
    if (tid == 0 && a.num_rejected) a.num_rejected[c_] += rejected;
}

static size_t rc_smem_bytes(int D) {
    return ((size_t)3 * D * (D + 1) + 19 * RC_DMAX + 40 + 8) * sizeof(float);
}

int rmhmc_cta_run(const hmcx_target_t* target, const hmcx_rmhmc_t* cfg, const hmcx_rng_t* rng, const float* q_init,
                  float* q_cur, const float* eps, int C, int ld, int L, int S, int burn, int it0, int it1, float* samples,
                  uint8_t* accept, uint8_t* diverged, float* ham, int32_t* num_rejected, const float* p_given,
                  float* q_traj, float* p_traj, float* qt_out, float* pt_out, int only_h, float* h_out, cudaStream_t st) {
    if (!target || !cfg || !rng || !q_init || (!q_cur && !p_given) || (!eps && !only_h)) return HMCX_ERR_INVALID_ARG;
    if (target->kind != HMCX_TARGET_FUNNEL && target->kind != HMCX_TARGET_GAUSS_ISO &&
        target->kind != HMCX_TARGET_GAUSS_DIAG && target->kind != HMCX_TARGET_GAUSS_FULL)
        return HMCX_ERR_UNSUPPORTED;
    const int D = target->dim;
    if (D < 1 || C < 1 || ld < D || (ld & 3) || L < 1 || S < 1 || burn < 0 || burn >= S || it0 < 0 || it1 > S || it0 > it1)
        return HMCX_ERR_INVALID_ARG;
    if (D > RC_DMAX) return HMCX_ERR_UNSUPPORTED;
    if (target->kind == HMCX_TARGET_FUNNEL && D < 2) return HMCX_ERR_INVALID_ARG;
    if (target->kind == HMCX_TARGET_GAUSS_DIAG && !target->inv_var) return HMCX_ERR_INVALID_ARG;
    if (target->kind == HMCX_TARGET_GAUSS_FULL && !target->prec) return HMCX_ERR_INVALID_ARG;
    if (cfg->integrator != 1 && cfg->integrator != 2) return HMCX_ERR_UNSUPPORTED;
    if (cfg->metric < 1 || cfg->metric > 3) return HMCX_ERR_UNSUPPORTED;
    RcArgs a = {};
    a.t.kind = target->kind; a.t.D = D; a.t.log_norm = target->log_norm; a.t.inv_var_v = target->funnel_inv_var_v;
    a.t.mean = target->mean; a.t.ivar = target->inv_var; a.t.prec = target->prec;
    a.cfg.softabs = cfg->metric == 2; a.cfg.jacdiag = cfg->metric == 3; a.cfg.alpha = cfg->softabs_const;
    a.cfg.jitter = cfg->jitter; a.cfg.pi_term = cfg->pi_term;
    a.integrator = cfg->integrator; a.cosw = cfg->cos_2we; a.sinw = cfg->sin_2we;
    a.fp_threshold = cfg->fixed_point_threshold; a.fp_max_iter = cfg->fixed_point_max_iterations;
    a.jitter_max_tries = cfg->jitter_max_tries;
    a.C = C; a.ld = ld;
    a.rng_mode = rng->mode; a.seed = rng->seed; a.chain_offset = rng->chain_offset;
    a.normals = rng->normals; a.logu = rng->log_uniforms; a.uniforms = rng->uniforms; a.J = rng->uniforms_per_iter;
    if (rng->mode == HMCX_RNG_INJECTED) {
        if (!p_given && (!rng->normals || !rng->log_uniforms)) return HMCX_ERR_INVALID_ARG;
        if (cfg->jitter >= 0.0f && (!rng->uniforms || rng->uniforms_per_iter < 1)) return HMCX_ERR_INVALID_ARG;
    } else if (rng->mode != HMCX_RNG_PHILOX) {
        return HMCX_ERR_INVALID_ARG;
    }
    a.q_init = q_init; a.q_cur = q_cur; a.eps = eps; a.L = L; a.S = S; a.burn = burn; a.it0 = it0; a.it1 = it1;
    a.samples = samples; a.accept = accept; a.diverged = diverged; a.ham = ham; a.num_rejected = num_rejected;
    a.p_given = p_given; a.q_traj = q_traj; a.p_traj = p_traj; a.qt_out = qt_out; a.pt_out = pt_out; a.only_h = only_h; a.h_out = h_out;
    const size_t smem = rc_smem_bytes(D);
    if (cudaFuncSetAttribute(rmhmc_cta_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
        return HMCX_ERR_CUDA;
    rmhmc_cta_kernel<<<C, RC_T, smem, st>>>(a);
    return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA;
}

}  // namespace hmcx
