// hmcx_flow.cu -- persistent kernel for the LINEAR flows of the path at small dimension (16 < D <= 128):
//   * plain HMC / HMC_NUTS with a full (2-D) inv_mass on Gaussian targets (samplers.py:199 gibbs p = chol(M) z, :294 drift
//     q += eps*(M^-1 p), :812 kinetic 0.5 p.(M^-1 p)) and GaussianFull targets with no / diagonal mass (:281-302);
//   * sampler=RMHMC on Gaussian targets without jitter, whose metric is ONE matrix: explicit integrator (:389-462, the
//     A-B-C-B-A flows on the augmented state) and implicit integrator (:305-387), with dH/dp = G^-1 p and
//     dH/dtheta = -grad log p(theta).
// Every flow of these samplers is y = M x with M one of at most three D x D matrices (precision, M^-1 / G^-1, chol).  At
// D <= 128 all three fit in ONE SM's shared memory (3 * 64 KB), and a whole sample() run -- gibbs, both Hamiltonians, the
// L leapfrog steps, MH, bookkeeping, dual averaging -- stays inside one launch: a warp owns R chains (state in registers,
// lane j holds elements j, j+32, ...), reads each matrix row once from shared memory for its R chains (conflict-free:
// the matrices are stored transposed, lane <-> column) and accumulates in exact fp32 FMAs.  This replaces, for small D,
// the step-synchronous tensor-core path of hmcx_tc.cu (8L+3 GEMM launches of ~9 us per iteration at D = 64: launch-latency
// bound, tensor pipe 3 %) -- the contraction is 128 x 64 x 64 per tile, far below what feeds a tensor core, so the honest
// roofline here is shared-memory bandwidth (each warp-matvec streams the D*D*4-byte matrix once: 128 B/clk/SM).
// Same random streams (Philox keyed by global chain id / iteration, or injected), same bookkeeping and the same
// element-wise operation order as the tensor-core path, so both give the same chains up to the summation order of the
// contractions.
#include <cstdlib>
#include "hmcx_common.cuh"

namespace hmcx {

enum { FLOW_HMC = 0, FLOW_RM_EXPLICIT = 1, FLOW_RM_IMPLICIT = 2 };

struct FlowArgs {
    int C, D, ld, L, S, burn, it0, it1;
    int tk, mk, mode;
    const float* prec;  const float* mean;  const float* ivar;     // target (GAUSS_FULL: prec; GAUSS_DIAG: ivar)
    const float* minv;  const float* chol;                          // mk == FULL: M^-1 (G^-1) and chol(M) (chol(G)), [D, D]
    const float* im;    const float* sd;                            // mk == DIAG: inverse mass, sqrt(mass)
    float log_norm, ham_c1, ham_c2, cw, sw;
    int rng_mode;
    uint64_t seed, chain_offset;
    const float* normals;  const float* logu;
    int nuts;
    double delta, mu;
    const double* table;  double* h_bar;  double* eps_bar;
    const float* eps_schedule;  float* eps_trace;
    const float* q_init;  float* q_cur;  float* eps;  int eps_writable;
    float* samples;  uint8_t* accept;  uint8_t* diverged;  float* ham;  int32_t* num_rejected;
};

__device__ __forceinline__ float f4c(const float4& v, int i) { return i == 0 ? v.x : i == 1 ? v.y : i == 2 ? v.z : v.w; }

// NJ = ceil(D / 32) register slots per vector and lane; R = chains per warp
template <int NJ, int R>
__global__ void __launch_bounds__(256, 1) flow_small_kernel(const FlowArgs a) {
    constexpr int DP = NJ * 32;
    // partial sums per output element (independent FMA chains in flight).  A function of D only, never of R: a chain's
    // bits must not depend on how many chains share its warp (the launch picks R from the batch size)
    constexpr int NACC = (NJ >= 4) ? 1 : (NJ >= 3 ? 2 : 4);
    extern __shared__ __align__(16) float smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarp = blockDim.x >> 5;
    const int D = a.D, K4 = (D + 3) & ~3, ld = a.ld;
    const bool full_t = a.tk == HMCX_TARGET_GAUSS_FULL, full_m = a.mk == HMCX_MASS_FULL, diag_m = a.mk == HMCX_MASS_DIAG;
    const bool rm = a.mode != FLOW_HMC;

    // ---- shared memory: the transposed matrices (row k = column k of M, zero-padded to DP columns) + one staging row per chain
    float* mt_prec = smem;
    float* mt_minv = mt_prec + (full_t ? K4 * DP : 0);
    float* mt_chol = mt_minv + (full_m ? K4 * DP : 0);
    float* xs = mt_chol + (full_m ? K4 * DP : 0) + warp * (2 * R * DP);           // two staging rows per chain (paired matvecs)
    float* xs2 = xs + R * DP;
    {
        const float* src[3] = {full_t ? a.prec : nullptr, full_m ? a.minv : nullptr, full_m ? a.chol : nullptr};
        float* dst[3] = {mt_prec, mt_minv, mt_chol};
        for (int m = 0; m < 3; ++m) {
            if (!src[m]) continue;
            for (int idx = threadIdx.x; idx < K4 * DP; idx += blockDim.x) {
                const int k = idx / DP, j = idx - k * DP;
                dst[m][idx] = (k < D && j < D) ? __ldg(src[m] + (size_t)j * D + k) : 0.0f;       // MT[k][j] = M[j][k]
            }
        }
    }
    __syncthreads();

    // ---- this warp's chains
    const int c0 = (blockIdx.x * nwarp + warp) * R;
    if (c0 >= a.C) return;                                         // no CTA-wide barrier below
    bool live[R];
    int ch[R];
#pragma unroll
    for (int r = 0; r < R; ++r) { live[r] = c0 + r < a.C; ch[r] = live[r] ? c0 + r : a.C - 1; }   // dead slots shadow the last chain, never store

    float meanv[NJ], ivarv[NJ], imv[NJ], sdv[NJ];
#pragma unroll
    for (int jj = 0; jj < NJ; ++jj) {
        const int i = jj * 32 + lane;
        const bool in = i < D;
        meanv[jj] = (in && a.mean) ? a.mean[i] : 0.0f;
        ivarv[jj] = (in && a.ivar) ? a.ivar[i] : 0.0f;
        imv[jj] = (in && diag_m) ? a.im[i] : 0.0f;
        sdv[jj] = (in && diag_m) ? a.sd[i] : 0.0f;
    }

    auto stage = [&](const float (&x)[R][NJ]) {
#pragma unroll
        for (int r = 0; r < R; ++r)
#pragma unroll
            for (int jj = 0; jj < NJ; ++jj) xs[r * DP + jj * 32 + lane] = x[r][jj];
        __syncwarp();
    };
    // y[r] = M x[r] for the staged x (rows >= D of MT and columns >= D are zero, so the padding never contributes)
    auto matvec = [&](const float* __restrict__ MT, float (&y)[R][NJ]) {
        float acc[NACC][R][NJ];
#pragma unroll
        for (int t = 0; t < NACC; ++t)
#pragma unroll
            for (int r = 0; r < R; ++r)
#pragma unroll
                for (int jj = 0; jj < NJ; ++jj) acc[t][r][jj] = 0.0f;
#pragma unroll(R <= 2 ? 4 : 2)
        for (int k = 0; k < K4; k += 4) {
            float4 xv[R];
#pragma unroll
            for (int r = 0; r < R; ++r) xv[r] = *reinterpret_cast<const float4*>(xs + r * DP + k);
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
                for (int jj = 0; jj < NJ; ++jj) {
                    const float m = MT[(k + kk) * DP + jj * 32 + lane];
#pragma unroll
                    for (int r = 0; r < R; ++r) acc[kk % NACC][r][jj] = fmaf(m, f4c(xv[r], kk), acc[kk % NACC][r][jj]);
                }
            }
        }
#pragma unroll
        for (int r = 0; r < R; ++r)
#pragma unroll
            for (int jj = 0; jj < NJ; ++jj) {
                float s = acc[0][r][jj];
                if (NACC == 2) s = add(s, acc[1 % NACC][r][jj]);
                if (NACC == 4) s = add(add(s, acc[1 % NACC][r][jj]), add(acc[2 % NACC][r][jj], acc[3 % NACC][r][jj]));
                y[r][jj] = s;
            }
        __syncwarp();
    };
    auto dot = [&](const float (&x)[R][NJ], const float (&y)[R][NJ], float (&s)[R]) {
#pragma unroll
        for (int r = 0; r < R; ++r) {
            float t = 0.0f;
#pragma unroll
            for (int jj = 0; jj < NJ; ++jj) t = add(t, mul(x[r][jj], y[r][jj]));
            s[r] = warp_sum(t);
        }
    };
    // Two INDEPENDENT matvecs in one pass (the explicit integrator's dH/dtheta and G^-1 p of a flow): twice the FFMA chains in
    // flight for a warp that is alone on its scheduler.  Each product accumulates exactly as in matvec() -- the same bits.
    constexpr bool PAIR = R <= 2;                                  // (register budget; large batches hide latency with warps)
    auto stage2 = [&](const float (&x1)[R][NJ], const float (&x2)[R][NJ]) {
#pragma unroll
        for (int r = 0; r < R; ++r)
#pragma unroll
            for (int jj = 0; jj < NJ; ++jj) { xs[r * DP + jj * 32 + lane] = x1[r][jj]; xs2[r * DP + jj * 32 + lane] = x2[r][jj]; }
        __syncwarp();
    };
    auto matvec2 = [&](const float* __restrict__ MT1, const float* __restrict__ MT2, float (&y1)[R][NJ], float (&y2)[R][NJ]) {
        float a1[NACC][R][NJ], a2[NACC][R][NJ];
#pragma unroll
        for (int t = 0; t < NACC; ++t)
#pragma unroll
            for (int r = 0; r < R; ++r)
#pragma unroll
                for (int jj = 0; jj < NJ; ++jj) { a1[t][r][jj] = 0.0f; a2[t][r][jj] = 0.0f; }
#pragma unroll 2
        for (int k = 0; k < K4; k += 4) {
            float4 x1[R], x2[R];
#pragma unroll
            for (int r = 0; r < R; ++r) {
                x1[r] = *reinterpret_cast<const float4*>(xs + r * DP + k);
                x2[r] = *reinterpret_cast<const float4*>(xs2 + r * DP + k);
            }
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
                for (int jj = 0; jj < NJ; ++jj) {
                    const float m1 = MT1[(k + kk) * DP + jj * 32 + lane], m2 = MT2[(k + kk) * DP + jj * 32 + lane];
#pragma unroll
                    for (int r = 0; r < R; ++r) {
                        a1[kk % NACC][r][jj] = fmaf(m1, f4c(x1[r], kk), a1[kk % NACC][r][jj]);
                        a2[kk % NACC][r][jj] = fmaf(m2, f4c(x2[r], kk), a2[kk % NACC][r][jj]);
                    }
                }
            }
        }
#pragma unroll
        for (int r = 0; r < R; ++r)
#pragma unroll
            for (int jj = 0; jj < NJ; ++jj) {
                float s1 = a1[0][r][jj], s2 = a2[0][r][jj];
                if (NACC == 2) { s1 = add(s1, a1[1 % NACC][r][jj]); s2 = add(s2, a2[1 % NACC][r][jj]); }
                if (NACC == 4) {
                    s1 = add(add(s1, a1[1 % NACC][r][jj]), add(a1[2 % NACC][r][jj], a1[3 % NACC][r][jj]));
                    s2 = add(add(s2, a2[1 % NACC][r][jj]), add(a2[2 % NACC][r][jj], a2[3 % NACC][r][jj]));
                }
                y1[r][jj] = s1; y2[r][jj] = s2;
            }
        __syncwarp();
    };
    // (grad log p(x), G^-1 w) together: == grad(x, g, u, want_u); vel(w, vv)
    auto grad_vel = [&](const float (&x)[R][NJ], float (&g)[R][NJ], float (&u)[R], bool want_u, const float (&w)[R][NJ],
                        float (&vv)[R][NJ]) {
        float y[R][NJ];
#pragma unroll
        for (int r = 0; r < R; ++r)
#pragma unroll
            for (int jj = 0; jj < NJ; ++jj) y[r][jj] = sub(x[r][jj], meanv[jj]);
        stage2(y, w);
        matvec2(mt_prec, mt_minv, g, vv);
        if (want_u) dot(y, g, u);
#pragma unroll
        for (int r = 0; r < R; ++r)
#pragma unroll
            for (int jj = 0; jj < NJ; ++jj) g[r][jj] = -g[r][jj];
    };
    // g = grad log p(q); u = the U-terms of log p (log p = -0.5*u + log_norm) when want_u
    auto grad = [&](const float (&q)[R][NJ], float (&g)[R][NJ], float (&u)[R], bool want_u) {
        if (full_t) {
            float y[R][NJ];
#pragma unroll
            for (int r = 0; r < R; ++r)
#pragma unroll
                for (int jj = 0; jj < NJ; ++jj) y[r][jj] = sub(q[r][jj], meanv[jj]);
            stage(y);
            matvec(mt_prec, g);
            if (want_u) dot(y, g, u);
#pragma unroll
            for (int r = 0; r < R; ++r)
#pragma unroll
                for (int jj = 0; jj < NJ; ++jj) g[r][jj] = -g[r][jj];
        } else {
#pragma unroll
            for (int r = 0; r < R; ++r) {
                float t = 0.0f;
#pragma unroll
                for (int jj = 0; jj < NJ; ++jj) {
                    if (a.tk == HMCX_TARGET_GAUSS_ISO) {
                        g[r][jj] = -q[r][jj];
                        t = add(t, mul(q[r][jj], q[r][jj]));
                    } else {
                        const float y = sub(q[r][jj], meanv[jj]);
                        g[r][jj] = -mul(ivarv[jj], y);
                        t = add(t, mul(mul(y, y), ivarv[jj]));
                    }
                }
                if (want_u) u[r] = warp_sum(t);
            }
        }
    };
    // v = M^-1 p (G^-1 p)
    auto vel = [&](const float (&p)[R][NJ], float (&v)[R][NJ]) {
        if (full_m) {
            stage(p);
            matvec(mt_minv, v);
        } else {
#pragma unroll
            for (int r = 0; r < R; ++r)
#pragma unroll
                for (int jj = 0; jj < NJ; ++jj) v[r][jj] = diag_m ? mul(imv[jj], p[r][jj]) : p[r][jj];
        }
    };
    // x <- x + k*d
    auto axpy = [&](float (&x)[R][NJ], const float (&k)[R], const float (&d)[R][NJ]) {
#pragma unroll
        for (int r = 0; r < R; ++r)
#pragma unroll
            for (int jj = 0; jj < NJ; ++jj) x[r][jj] = add(x[r][jj], mul(k[r], d[r][jj]));
    };
    auto load_rows = [&](const float* base, float (&x)[R][NJ]) {
#pragma unroll
        for (int r = 0; r < R; ++r)
#pragma unroll
            for (int jj = 0; jj < NJ; ++jj) {
                const int i = jj * 32 + lane;
                x[r][jj] = i < D ? base[(size_t)ch[r] * ld + i] : 0.0f;
            }
    };

    float q[R][NJ], p[R][NJ], g[R][NJ], v[R][NJ];
    float U_init[R], U_cur[R], e[R];
    {
        float u[R];
        load_rows(a.q_init, q);
        grad(q, g, u, true);
#pragma unroll
        for (int r = 0; r < R; ++r) U_init[r] = add(mul(-0.5f, u[r]), a.log_norm);
        if (a.it0 == 0 && a.samples) {                                              // slot 0 = params_init (:959)
#pragma unroll
            for (int r = 0; r < R; ++r)
                for (int i = lane; i < ld && live[r]; i += 32)
                    a.samples[(size_t)ch[r] * (a.S - a.burn) * ld + i] = a.q_init[(size_t)ch[r] * ld + i];
        }
        load_rows(a.q_cur, q);
        grad(q, g, u, true);
#pragma unroll
        for (int r = 0; r < R; ++r) { U_cur[r] = add(mul(-0.5f, u[r]), a.log_norm); e[r] = a.eps[ch[r]]; }
    }

    for (int n = a.it0; n < a.it1; ++n) {
        float half[R];
#pragma unroll
        for (int r = 0; r < R; ++r) {
            if (a.eps_schedule) {
                e[r] = a.eps_schedule[(size_t)n * a.C + ch[r]];
                if (lane == 0 && live[r] && a.eps_writable) a.eps[ch[r]] = e[r];
            }
            half[r] = mul(0.5f, e[r]);
        }
        // ---- gibbs (:152-202): z ~ N(0, I) in the canonical stream, p = chol(M) z | z*sqrt(mass) | z
        float z[R][NJ];
        if (a.rng_mode == HMCX_RNG_INJECTED) {
            load_rows(a.normals + (size_t)(n - a.it0) * a.C * ld, z);
        } else {
#pragma unroll
            for (int r = 0; r < R; ++r) {
                if (4 * lane < DP) {
                    float t[4] = {0.f, 0.f, 0.f, 0.f};
                    if (4 * lane < ld) philox_normal4(a.seed, a.chain_offset + (uint64_t)ch[r], (uint64_t)n, (uint32_t)lane, t);
                    *reinterpret_cast<float4*>(xs + r * DP + 4 * lane) = make_float4(t[0], t[1], t[2], t[3]);
                }
            }
            __syncwarp();
#pragma unroll
            for (int r = 0; r < R; ++r)
#pragma unroll
                for (int jj = 0; jj < NJ; ++jj) z[r][jj] = (jj * 32 + lane < D) ? xs[r * DP + jj * 32 + lane] : 0.0f;
            __syncwarp();
        }
        if (full_m) {
            stage(z);
            matvec(mt_chol, p);
        } else {
#pragma unroll
            for (int r = 0; r < R; ++r)
#pragma unroll
                for (int jj = 0; jj < NJ; ++jj) p[r][jj] = diag_m ? mul(z[r][jj], sdv[jj]) : z[r][jj];
        }
        load_rows(a.q_cur, q);
        float kin_old[R], kin_new[R], u_new[R];
        vel(p, v);
        dot(p, v, kin_old);

        if (a.mode == FLOW_HMC) {                                                   // :281-302
            grad(q, g, u_new, false);
            axpy(p, half, g);
            for (int l = 1; l <= a.L; ++l) {
                vel(p, v);
                axpy(q, e, v);                                                      // :284 / :294 / :296 (diag: (eps*im)*p)
                grad(q, g, u_new, l == a.L);
                axpy(p, e, g);                                                      // :298
            }
#pragma unroll
            for (int r = 0; r < R; ++r)
#pragma unroll
                for (int jj = 0; jj < NJ; ++jj) p[r][jj] = sub(p[r][jj], mul(half[r], g[r][jj]));   // :302
        } else if (a.mode == FLOW_RM_IMPLICIT) {                                    // :363-386 with a constant metric
            grad(q, g, u_new, false);
            for (int l = 0; l < a.L; ++l) {
                axpy(p, half, g);
                vel(p, v);
                axpy(q, half, v);
                axpy(q, half, v);
                grad(q, g, u_new, l == a.L - 1);
                axpy(p, half, g);
            }
        } else {                                                                    // :425-458, augmented state (q, p, qc, pc)
            float qc[R][NJ], pc[R][NJ], vc[R][NJ];
#pragma unroll
            for (int r = 0; r < R; ++r)
#pragma unroll
                for (int jj = 0; jj < NJ; ++jj) { qc[r][jj] = q[r][jj]; pc[r][jj] = p[r][jj]; vc[r][jj] = v[r][jj]; }
            grad(q, g, u_new, false);
            for (int l = 0; l < a.L; ++l) {
                axpy(p, half, g);                                                   // A (:429-430): flows of H(theta, p~)
                axpy(qc, half, vc);
                for (int b = 0; b < 2; ++b) {                                       // B (:432-433), C (:435-450), B (:454-455)
                    if (PAIR && full_t && full_m) {
                        float gc[R][NJ];
                        grad_vel(qc, gc, u_new, false, p, v);
                        axpy(q, half, v);
                        axpy(pc, half, gc);
                    } else {
                        vel(p, v);
                        axpy(q, half, v);
                        grad(qc, v, u_new, false);
                        axpy(pc, half, v);
                    }
                    if (b == 0) {
#pragma unroll
                        for (int r = 0; r < R; ++r)
#pragma unroll
                            for (int jj = 0; jj < NJ; ++jj) {
                                const float q0 = q[r][jj], p0 = p[r][jj], qt = qc[r][jj], pt = pc[r][jj];
                                const float qn = mul(0.5f, add(add(add(q0, qt), mul(a.cw, sub(q0, qt))), mul(a.sw, sub(p0, pt))));
                                const float pn = mul(0.5f, add(sub(add(p0, pt), mul(a.sw, sub(qn, qt))), mul(a.cw, sub(p0, pt))));
                                const float qtn = mul(0.5f, sub(sub(add(qn, qt), mul(a.cw, sub(qn, qt))), mul(a.sw, sub(pn, pt))));
                                const float ptn = mul(0.5f, sub(add(add(pn, pt), mul(a.sw, sub(qn, qtn))), mul(a.cw, sub(pn, pt))));
                                q[r][jj] = qn; p[r][jj] = pn; qc[r][jj] = qtn; pc[r][jj] = ptn;
                            }
                    }
                }
                if (PAIR && full_t && full_m && l < a.L - 1) {                      // A (:457-458); g and vc also serve the next step's A
                    grad_vel(q, g, u_new, false, pc, vc);
                    axpy(p, half, g);
                    axpy(qc, half, vc);
                } else {
                    grad(q, g, u_new, l == a.L - 1);
                    axpy(p, half, g);
                    if (l < a.L - 1) {
                        vel(pc, vc);
                        axpy(qc, half, vc);
                    }
                }
            }
        }
        vel(p, v);
        dot(p, v, kin_new);

        // ---- Hamiltonians, MH, bookkeeping, dual averaging (:995-1067); every lane holds the same bits
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const int c = ch[r];
            const float lp_cur = U_cur[r], lp_new = add(mul(-0.5f, u_new[r]), a.log_norm);
            float h_old, h_new;
            if (rm) {
                h_old = add(add(add(-lp_cur, a.ham_c1), a.ham_c2), mul(0.5f, kin_old[r]));
                h_new = add(add(add(-lp_new, a.ham_c1), a.ham_c2), mul(0.5f, kin_new[r]));
            } else {
                h_old = add(-lp_cur, mul(0.5f, kin_old[r]));
                h_new = add(-lp_new, mul(0.5f, kin_new[r]));
            }
            const bool bad = !finite_f(lp_cur) || !finite_f(lp_new) || (rm && (!finite_f(h_old) || !finite_f(h_new)));
            const float x = add(-h_new, h_old);
            const float rho = (x < 0.0f) ? x : 0.0f;
            const float logu = (a.rng_mode == HMCX_RNG_INJECTED) ? a.logu[(size_t)(n - a.it0) * a.C + c]
                                                                 : philox_log_uniform(a.seed, a.chain_offset + (uint64_t)c, (uint64_t)n);
            const bool acc = !bad && (rho >= logu);
            const bool quirk = !acc && (n == a.burn + 1);
            if (acc) U_cur[r] = lp_new;
            else if (quirk) U_cur[r] = U_init[r];
            const size_t o = (size_t)c * a.S + n;
            float en = e[r];
            if (a.nuts && n <= a.burn) {                                            // :1030-1035, :1060-1067
                double h_bar = a.h_bar[c], eps_bar = a.eps_bar[c];
                if (n < a.burn || bad) {
                    const double* T = a.table + 5 * (size_t)n;
                    const double alpha = bad ? 0.0 : (double)expf(rho);
                    h_bar = __dadd_rn(__dmul_rn(T[0], h_bar), __dmul_rn(T[1], a.delta - alpha));
                    const double x_new = a.mu - __dmul_rn(T[2], h_bar);
                    en = expf((float)x_new);
                    const float xb = add((float)__dmul_rn(T[3], x_new), mul((float)T[4], logf((float)eps_bar)));
                    eps_bar = (double)expf(xb);
                }
                if (n == a.burn) en = (float)eps_bar;
                __syncwarp();
                if (lane == 0 && live[r]) { a.h_bar[c] = h_bar; a.eps_bar[c] = eps_bar; a.eps[c] = en; }
            }
            if (lane == 0 && live[r]) {
                if (!acc && a.num_rejected) a.num_rejected[c] += 1;
                if (a.accept) a.accept[o] = acc ? 1 : 0;
                if (a.diverged) a.diverged[o] = bad ? 1 : 0;
                if (a.ham) { a.ham[2 * o] = h_old; a.ham[2 * o + 1] = h_new; }
                if (a.eps_trace) a.eps_trace[o] = en;
            }
            e[r] = en;
            if (live[r]) {
                float* qcur = a.q_cur + (size_t)c * ld;
                float* dst = (n > a.burn && a.samples) ? a.samples + ((size_t)c * (a.S - a.burn) + (n - a.burn)) * ld : nullptr;
#pragma unroll
                for (int jj = 0; jj < NJ; ++jj) {
                    const int i = jj * 32 + lane;
                    if (i < ld) {
                        float val;
                        if (acc) val = i < D ? q[r][jj] : 0.0f;
                        else if (quirk) val = a.q_init[(size_t)c * ld + i];
                        else val = qcur[i];
                        if (acc || quirk) qcur[i] = val;
                        if (dst) dst[i] = val;
                    }
                }
            }
        }
        __syncwarp();
    }
}

// A test switch (HMCX_FLOW_R / HMCX_FLOW_W): -1 when unset, the value when it is a whole decimal number in [lo, hi], else 0
static int flow_env(const char* name, long lo, long hi) {
    const char* e = getenv(name);
    if (!e) return -1;
    char* end = nullptr;
    const long v = strtol(e, &end, 10);
    return (end != e && *end == '\0' && v >= lo && v <= hi) ? (int)v : 0;
}

// Launch geometry: R chains per warp, w = threads / 32 warps per CTA, `grid` CTAs and `smem` bytes of dynamic shared memory
// (the nmat transposed K4 x DP matrices, then two staging rows of DP floats per chain of every warp).  HMCX_FLOW_R = 1|2|4
// forces R and HMCX_FLOW_W = 1..8 caps w (tests and tuning: every instantiation reachable at any batch); both are read on
// every call.  Any other value of either, or a geometry whose shared memory exceeds the device's opt-in limit, is
// HMCX_ERR_INVALID_ARG: the run never launches a geometry nobody asked for, nor one that cannot launch.
// tests/test_flow_geometry_cpu.py restates this rule and checks it against the constants below.
static int flow_geometry(int C, int nmat, int K4, int DP, int& R, int& threads, int& grid, size_t& smem) {
    int dev = 0, sms = 0, optin = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess) {
        cudaGetLastError();
        return HMCX_ERR_CUDA;
    }
    const int fr = flow_env("HMCX_FLOW_R", 1, 4), fw = flow_env("HMCX_FLOW_W", 1, 8);
    if (fr == 0 || fr == 3 || fw == 0) return HMCX_ERR_INVALID_ARG;
    // chains per warp: every warp-matvec streams the whole matrix from shared memory once, so more chains per warp = less
    // shared-memory traffic per chain, fewer chains per warp = more warps (SMs) working on a small batch
    R = fr > 0 ? fr : (C <= 4 * sms) ? 1 : (C <= 12 * sms) ? 2 : 4;
    const int warps = (C + R - 1) / R;
    int w = (warps + sms - 1) / sms;
    // big batches: when two CTAs' matrices fit one SM, CTAs of 4 warps (finer waves, the same warps per SM); D = 128 with
    // three matrices fills the SM with one CTA of 8
    const size_t matrix_bytes = (size_t)nmat * K4 * DP * sizeof(float);
    const int wmax = fw > 0 ? fw : (matrix_bytes <= 100 * 1024 ? 4 : 8);
    if (w > wmax) w = wmax;
    if (w < 1) w = 1;
    threads = 32 * w;
    grid = (warps + w - 1) / w;
    smem = ((size_t)nmat * K4 * DP + (size_t)w * 2 * R * DP) * sizeof(float);
    return smem <= (size_t)optin ? HMCX_OK : HMCX_ERR_INVALID_ARG;
}

template <int NJ>
static int flow_launch_nj(const FlowArgs& a, int R, int threads, int grid, size_t smem, cudaStream_t st) {
    auto go = [&](auto kern) -> int {
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
            cudaGetLastError();
            return HMCX_ERR_CUDA;
        }
        kern<<<grid, threads, smem, st>>>(a);
        return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA;
    };
    if (R == 1) return go(flow_small_kernel<NJ, 1>);
    if (R == 2) return go(flow_small_kernel<NJ, 2>);
    return go(flow_small_kernel<NJ, 4>);
}

static int flow_launch(const FlowArgs& a, cudaStream_t st) {
    const int NJ = (a.D + 31) / 32, DP = NJ * 32, K4 = (a.D + 3) & ~3;
    int R, threads, grid;
    size_t smem;
    const int nmat = (a.tk == HMCX_TARGET_GAUSS_FULL ? 1 : 0) + (a.mk == HMCX_MASS_FULL ? 2 : 0);
    if (const int rc = flow_geometry(a.C, nmat, K4, DP, R, threads, grid, smem)) return rc;
    switch (NJ) {
        case 1: return flow_launch_nj<1>(a, R, threads, grid, smem, st);
        case 2: return flow_launch_nj<2>(a, R, threads, grid, smem, st);
        case 3: return flow_launch_nj<3>(a, R, threads, grid, smem, st);
        case 4: return flow_launch_nj<4>(a, R, threads, grid, smem, st);
    }
    return HMCX_ERR_UNSUPPORTED;
}

// The persistent kernel covers D <= 128 with the row stride inside its padded width; HMCX_FLOW_SMALL=0 keeps everything
// on the tensor-core path (A/B measurements, tests of that path at small D).
bool flow_small_ok(int D, int ld) {
    const char* s = getenv("HMCX_FLOW_SMALL");
    if (s && s[0] == '0') return false;
    return D >= 1 && D <= 128 && ld <= (D + 31) / 32 * 32;
}

static void flow_common(FlowArgs& a, const hmcx_target_t* target, const hmcx_rng_t* rng, const float* q_init, float* q_cur,
                        int C, int ld, int L, int S, int burn, int it0, int it1, float* samples, uint8_t* accept,
                        uint8_t* diverged, float* ham, int32_t* num_rejected) {
    a.C = C; a.D = target->dim; a.ld = ld; a.L = L; a.S = S; a.burn = burn; a.it0 = it0; a.it1 = it1;
    a.tk = target->kind; a.prec = target->prec; a.ivar = target->inv_var; a.log_norm = target->log_norm;
    a.mean = (target->kind == HMCX_TARGET_GAUSS_ISO) ? nullptr : target->mean;
    a.rng_mode = rng->mode; a.seed = rng->seed; a.chain_offset = rng->chain_offset;
    a.normals = rng->normals; a.logu = rng->log_uniforms;
    a.q_init = q_init; a.q_cur = q_cur;
    a.samples = samples; a.accept = accept; a.diverged = diverged; a.ham = ham; a.num_rejected = num_rejected;
}

// arguments validated by dense_hmc_run
int flow_small_hmc_run(const hmcx_target_t* target, const hmcx_mass_t* mass, const hmcx_rng_t* rng, const hmcx_nuts_t* nuts,
                       const float* q_init, float* q_cur, float* eps, int C, int ld, int L, int S, int burn, int it0, int it1,
                       float* samples, uint8_t* accept, uint8_t* diverged, float* ham, int32_t* num_rejected,
                       cudaStream_t st) {
    FlowArgs a = {};
    flow_common(a, target, rng, q_init, q_cur, C, ld, L, S, burn, it0, it1, samples, accept, diverged, ham, num_rejected);
    a.mode = FLOW_HMC;
    a.mk = mass ? mass->kind : HMCX_MASS_NONE;
    if (a.mk == HMCX_MASS_FULL) {
        if (!mass->inv_mass || !mass->mass_factor) return HMCX_ERR_INVALID_ARG;
        a.minv = mass->inv_mass; a.chol = mass->mass_factor;
    } else if (a.mk == HMCX_MASS_DIAG) {
        a.im = mass->inv_mass; a.sd = mass->mass_factor;
    }
    if (a.tk == HMCX_TARGET_GAUSS_DIAG && !target->inv_var) return HMCX_ERR_INVALID_ARG;
    a.nuts = (nuts && nuts->enabled) ? 1 : 0;
    if (a.nuts) {
        if (!nuts->table || !nuts->h_bar || !nuts->eps_bar || burn < 1) return HMCX_ERR_INVALID_ARG;
        a.delta = nuts->desired_accept_rate; a.mu = nuts->mu; a.table = nuts->table;
        a.h_bar = nuts->h_bar; a.eps_bar = nuts->eps_bar;
        a.eps_schedule = nuts->eps_schedule; a.eps_trace = nuts->eps_trace;
    }
    a.eps = eps; a.eps_writable = 1;
    return flow_launch(a, st);
}

// arguments validated by dense_rmhmc_run
int flow_small_rmhmc_run(const hmcx_target_t* target, const hmcx_rmhmc_t* cfg, const hmcx_const_metric_t* gm,
                         const hmcx_rng_t* rng, const float* q_init, float* q_cur, const float* eps, int C, int ld, int L,
                         int S, int burn, int it0, int it1, float* samples, uint8_t* accept, uint8_t* diverged, float* ham,
                         int32_t* num_rejected, float ham_c1, float ham_c2, cudaStream_t st) {
    FlowArgs a = {};
    flow_common(a, target, rng, q_init, q_cur, C, ld, L, S, burn, it0, it1, samples, accept, diverged, ham, num_rejected);
    a.mode = cfg->integrator == 1 ? FLOW_RM_EXPLICIT : FLOW_RM_IMPLICIT;
    a.mk = HMCX_MASS_FULL;
    a.minv = gm->metric_inv; a.chol = gm->metric_chol;
    a.ham_c1 = ham_c1; a.ham_c2 = ham_c2; a.cw = cfg->cos_2we; a.sw = cfg->sin_2we;
    a.eps = const_cast<float*>(eps); a.eps_writable = 0;
    return flow_launch(a, st);
}

}  // namespace hmcx
