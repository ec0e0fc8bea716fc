// hmcx_rmhmc.cu -- Riemannian-manifold HMC (sampler=RMHMC) on sm_90a (H100).
//
//   fisher + softabs          samplers.py:69-127      -> eval_metric()  (closed-form Hessian, Jacobi eigensolver)
//   cholesky_inverse          samplers.py:130-149     -> via the eigen-decomposition (G~^-1 p = Q diag(1/lam~) Q^T p)
//   rm_hamiltonian            samplers.py:677-736     -> rm_hamiltonian()
//   gibbs, RMHMC branch       samplers.py:183-184     -> p = chol(G~) z
//   leapfrog explicit         samplers.py:389-462     -> explicit_trajectory()  (A-B-C-B-A, sequential C update)
//   leapfrog implicit         samplers.py:305-387     -> implicit_trajectory()  (fixed-point iterations)
//   sample() loop             samplers.py:965-1067    -> rmhmc_run_kernel
//
// The reference obtains dH/dtheta by autograd THROUGH the Hessian, eigh and the Cholesky solve (third derivatives
// of log p by double backward).  Here it is the closed form (Betancourt 2013, softabs):
//     dH/dtheta_k = -d_k log p + sum_ab Z_ab (dG/dtheta_k)_ab ,     Z = Q B Q^T ,
//     B_ij = 1/2 delta_ij lam~'_i/lam~_i - 1/2 u_i u_j F_ij ,   u = diag(1/lam~) Q^T p ,
//     F_ij = (lam~_i - lam~_j)/(lam_i - lam_j)  (i != j),  F_ii = lam~'(lam_i) ,   lam~ = lam*coth(alpha*lam)
// with the target supplying G = -Hessian(log p) and the contraction with its third-derivative tensor in closed form.
// One THREAD owns one chain (D is small on this path: BASELINE config 3 has D=2; D <= 16 supported): every metric
// evaluation is thread-private, so 512 chains need no synchronisation at all; the arithmetic is latency/SFU bound
// (exp, tanh, sinh, sqrt, divisions), not a tensor-core or HBM problem at these sizes (DESIGN.md 3.5).
#include "hmcx_common.cuh"
#include "hmcx_rm.cuh"

namespace hmcx {

// DM is the capacity of the per-thread arrays.  The DM == 2 instantiation is launched only for D == 2 (BASELINE
// config 3), so there the dimension is a compile-time constant: every loop unrolls and the 2x2 metric algebra lives
// in registers instead of local memory.
template <int DM>
__device__ __forceinline__ int rm_dim(const RmTarget& t) { return DM == 2 ? 2 : t.D; }

// ---- targets: log p, its gradient, G = -Hessian, and the contraction of Z with dG/dtheta_k ----------------------
template <int DM>
__device__ __forceinline__ float rm_log_prob(const RmTarget& t, const float* th) {
    const int d = rm_dim<DM>(t);
    if (t.kind == HMCX_TARGET_FUNNEL) {                       // targets.Funnel.__call__
        const float v = th[0];
        float s = 0.0f;
        for (int i = 1; i < d; ++i) s = add(s, mul(th[i], th[i]));
        const float t1 = mul((float)(-0.5 * (double)t.inv_var_v), mul(v, v));
        const float t2 = mul(0.5f * (float)(d - 1), v);
        const float t3 = mul(mul(0.5f, expf(v)), s);
        return add(sub(add(t1, t2), t3), t.log_norm);
    }
    float s = 0.0f;
    if (t.kind == HMCX_TARGET_GAUSS_FULL) {                   // -0.5 * dot(y, P y) + log_norm
        for (int a = 0; a < d; ++a) {
            float r = 0.0f;
            for (int b = 0; b < d; ++b) r += t.prec[a * d + b] * (th[b] - (t.mean ? t.mean[b] : 0.0f));
            s += (th[a] - (t.mean ? t.mean[a] : 0.0f)) * r;
        }
        return add(mul(-0.5f, s), t.log_norm);
    }
    for (int i = 0; i < d; ++i) {
        if (t.kind == HMCX_TARGET_GAUSS_ISO) s = add(s, mul(th[i], th[i]));
        else { const float y = sub(th[i], t.mean ? t.mean[i] : 0.0f); s = add(s, mul(mul(y, y), t.ivar[i])); }
    }
    return add(mul(-0.5f, s), t.log_norm);
}

template <int DM>
__device__ __forceinline__ void rm_grad_log_prob(const RmTarget& t, const float* th, float* g) {
    const int d = rm_dim<DM>(t);
    if (t.kind == HMCX_TARGET_FUNNEL) {
        const float v = th[0], E = expf(v);
        float s = 0.0f;
        for (int i = 1; i < d; ++i) { s += th[i] * th[i]; g[i] = -(E * th[i]); }
        g[0] = -(t.inv_var_v * v) + 0.5f * (float)(d - 1) - 0.5f * E * s;
        return;
    }
    if (t.kind == HMCX_TARGET_GAUSS_FULL) {                   // -(P y)
        for (int a = 0; a < d; ++a) {
            float r = 0.0f;
            for (int b = 0; b < d; ++b) r += t.prec[a * d + b] * (th[b] - (t.mean ? t.mean[b] : 0.0f));
            g[a] = -r;
        }
        return;
    }
    for (int i = 0; i < d; ++i)
        g[i] = (t.kind == HMCX_TARGET_GAUSS_ISO) ? -th[i] : -(t.ivar[i] * (th[i] - (t.mean ? t.mean[i] : 0.0f)));
}

template <int DM>
__device__ __forceinline__ void rm_fill_metric(const RmTarget& t, const float* th, float (*G)[DM]) {
    const int d = rm_dim<DM>(t);
    for (int a = 0; a < d; ++a)
        for (int b = 0; b < d; ++b) G[a][b] = 0.0f;
    if (t.kind == HMCX_TARGET_FUNNEL) {
        const float E = expf(th[0]);
        float s = 0.0f;
        for (int i = 1; i < d; ++i) { s += th[i] * th[i]; G[0][i] = G[i][0] = E * th[i]; G[i][i] = E; }
        G[0][0] = t.inv_var_v + 0.5f * E * s;
        return;
    }
    if (t.kind == HMCX_TARGET_GAUSS_FULL) {
        for (int a = 0; a < d; ++a)
            for (int b = 0; b < d; ++b) G[a][b] = t.prec[a * d + b];
        return;
    }
    for (int i = 0; i < d; ++i) G[i][i] = (t.kind == HMCX_TARGET_GAUSS_ISO) ? 1.0f : t.ivar[i];
}

// out_k = sum_ab Z_ab (dG/dtheta_k)_ab ; Z symmetric
template <int DM>
__device__ __forceinline__ void rm_contract_dmetric(const RmTarget& t, const float* th, const float (*Z)[DM], float* out) {
    const int d = rm_dim<DM>(t);
    if (t.kind == HMCX_TARGET_FUNNEL) {
        const float E = expf(th[0]);
        float s = 0.0f, zx = 0.0f, tr = 0.0f;
        for (int i = 1; i < d; ++i) { s += th[i] * th[i]; zx += Z[0][i] * th[i]; tr += Z[i][i]; }
        out[0] = Z[0][0] * (0.5f * E * s) + 2.0f * E * zx + E * tr;
        for (int i = 1; i < d; ++i) out[i] = Z[0][0] * E * th[i] + 2.0f * Z[0][i] * E;
        return;
    }
    for (int i = 0; i < d; ++i) out[i] = 0.0f;            // Gaussian: constant metric
}

// ---- symmetric eigensolver (cyclic Jacobi), fp32 ------------------------------------------------------------------
template <int DM>
__device__ __forceinline__ void jacobi_eigh(int d_, float (*A)[DM], float (*Q)[DM], float* lam) {
    const int d = DM == 2 ? 2 : d_;
    for (int a = 0; a < d; ++a)
        for (int b = 0; b < d; ++b) Q[a][b] = (a == b) ? 1.0f : 0.0f;
    for (int sweep = 0; sweep < 16; ++sweep) {
        float off = 0.0f, diag = 0.0f;
        for (int a = 0; a < d; ++a) {
            diag += A[a][a] * A[a][a];
            for (int b = a + 1; b < d; ++b) off += A[a][b] * A[a][b];
        }
        if (!(off > 1e-14f * diag) ) break;
        for (int p = 0; p < d - 1; ++p)
            for (int q = p + 1; q < d; ++q) {
                const float apq = A[p][q];
                if (fabsf(apq) < 1e-30f) continue;
                const float theta = (A[q][q] - A[p][p]) / (2.0f * apq);
                const float tt = (theta >= 0.0f ? 1.0f : -1.0f) / (fabsf(theta) + sqrtf(theta * theta + 1.0f));
                const float c = rsqrtf(tt * tt + 1.0f), s = tt * c;
                for (int k = 0; k < d; ++k) {                 // A <- A J
                    const float akp = A[k][p], akq = A[k][q];
                    A[k][p] = c * akp - s * akq;
                    A[k][q] = s * akp + c * akq;
                }
                for (int k = 0; k < d; ++k) {                 // A <- J^T A
                    const float apk = A[p][k], aqk = A[q][k];
                    A[p][k] = c * apk - s * aqk;
                    A[q][k] = s * apk + c * aqk;
                }
                for (int k = 0; k < d; ++k) {                 // Q <- Q J
                    const float qkp = Q[k][p], qkq = Q[k][q];
                    Q[k][p] = c * qkp - s * qkq;
                    Q[k][q] = s * qkp + c * qkq;
                }
            }
    }
    for (int a = 0; a < d; ++a) lam[a] = A[a][a];
}

template <int DM>
struct Metric {
    float Q[DM][DM];      // eigenvectors in columns
    float lam[DM];        // eigenvalues of G (+ jitter)
    float lt[DM];         // lam~ = softabs(lam) (or lam for the HESSIAN metric)
    float dlt[DM];        // d lam~ / d lam
};

// fisher(): G = -Hess (+ diag(u*jitter)), eigh, softabs.  false <=> the reference raises LogProbError (:110-112, :717)
template <int DM>
__device__ __forceinline__ bool eval_metric(const RmTarget& t, const RmCfg& cfg, const float* th, const float* u,
                                            Metric<DM>& M) {
    const int d = rm_dim<DM>(t);
    if (cfg.jacdiag) {
        // fish = (jac jac^T).diag().diag() (:104-106) + diag(u * jitter): already diagonal -> Q = I, lam~ = lam
        float g[DM];
        rm_grad_log_prob<DM>(t, th, g);
        bool okd = true;
        for (int a = 0; a < d; ++a) {
            for (int b = 0; b < d; ++b) M.Q[a][b] = (a == b) ? 1.0f : 0.0f;
            float v = mul(g[a], g[a]);
            if (u) v = add(v, mul(u[a], cfg.jitter));
            M.lam[a] = v; M.lt[a] = v; M.dlt[a] = 1.0f;
            okd = okd && finite_f(v);
        }
        return okd;
    }
    float G[DM][DM];
    rm_fill_metric<DM>(t, th, G);
    bool ok = true;
    for (int a = 0; a < d; ++a) {
        if (u) G[a][a] = add(G[a][a], mul(u[a], cfg.jitter));
        for (int b = 0; b < d; ++b) ok = ok && finite_f(G[a][b]);
    }
    if (!ok) return false;
    jacobi_eigh<DM>(d, G, M.Q, M.lam);
    for (int i = 0; i < d; ++i) {
        const float l = M.lam[i];
        if (cfg.softabs) {
            const float x = cfg.alpha * l;
            if (fabsf(x) >= 20.0f && finite_f(x)) {
                // saturated softabs (alpha = 1e6: practically always).  tanhf(x) is exactly +-1 in fp32 beyond |x| = 9.1,
                // and x/sinh(x)^2 < 4e-16 vanishes against 1/tanh: the general branch below returns exactly these
                // bits, after ~110 more dependent instructions (tanhf, sinhf, two divisions) on the critical path.
                const float sg = x > 0.0f ? 1.0f : -1.0f;
                M.lt[i] = sg * l;                                             // (1/+-1) * lam
                M.dlt[i] = sg;
            } else {
                const float th_ = tanhf(x);
                M.lt[i] = (1.0f / th_) * l;                               // (1./tanh(alpha*lam))*lam   (:120)
                const float sh = sinhf(x);
                M.dlt[i] = 1.0f / th_ - x / (sh * sh);
                if (!finite_f(M.dlt[i])) M.dlt[i] = (l >= 0.0f) ? 1.0f : -1.0f;   // saturated: |lam|' = sign
            }
        } else {
            M.lt[i] = l;
            M.dlt[i] = 1.0f;
        }
        ok = ok && finite_f(M.lt[i]);
    }
    return ok;
}

// rm_hamiltonian (:710-736) given the metric; also leaves w = Q^T p for the gradients.  ok=false <=> LogProbError
template <int DM>
__device__ __forceinline__ float rm_hamiltonian(const RmTarget& t, const RmCfg& cfg, const float* th, const float* p,
                                                const Metric<DM>& M, float* w, bool& ok) {
    const int d = rm_dim<DM>(t);
    const float lp = rm_log_prob<DM>(t, th);
    if (!finite_f(lp)) ok = false;
    float logdet = 0.0f, quad = 0.0f;
    for (int i = 0; i < d; ++i) {
        float wi = 0.0f;
        for (int a = 0; a < d; ++a) wi += M.Q[a][i] * p[a];
        w[i] = wi;
        if (cfg.softabs) logdet += logf(M.lt[i]);
        else { logdet += logf(fabsf(M.lt[i])); if (!(M.lt[i] > 0.0f)) ok = false; }   // Cholesky of a non-PD metric
        quad += wi * wi / M.lt[i];
    }
    const float H = add(add(add(-lp, mul(0.5f, cfg.pi_term)), mul(0.5f, logdet)), mul(0.5f, quad));
    if (!finite_f(H)) ok = false;
    return H;
}

// dH/dp = G~^-1 p
template <int DM>
__device__ __forceinline__ void grad_momentum(const RmTarget& t, const Metric<DM>& M, const float* p, float* out) {
    const int d = rm_dim<DM>(t);
    float u[DM];
    for (int i = 0; i < d; ++i) {
        float wi = 0.0f;
        for (int a = 0; a < d; ++a) wi += M.Q[a][i] * p[a];
        u[i] = wi / M.lt[i];
    }
    for (int a = 0; a < d; ++a) {
        float s = 0.0f;
        for (int i = 0; i < d; ++i) s += M.Q[a][i] * u[i];
        out[a] = s;
    }
}

// dH/dtheta for Metric.JACOBIAN_DIAG: G = diag(g_i^2 (+ jitter)), g = grad log p, so
//   dH/dtheta_k = -g_k + sum_i Z_ii * d(g_i^2)/dtheta_k = -g_k + sum_i (1/(2 d_i) - p_i^2/(2 d_i^2)) * 2 g_i * Hess_ik
// with Hess = Hessian(log p) = -(the matrix rm_fill_metric returns).  (autograd through .diag().diag(), :104-106)
template <int DM>
__device__ __forceinline__ void grad_params_jacdiag(const RmTarget& t, const float* th, const Metric<DM>& M,
                                                    const float* p, float* out) {
    const int d = rm_dim<DM>(t);
    float g[DM], zz[DM], Gh[DM][DM];
    rm_grad_log_prob<DM>(t, th, g);
    rm_fill_metric<DM>(t, th, Gh);
    for (int i = 0; i < d; ++i) {
        const float ui = p[i] / M.lt[i];
        zz[i] = (0.5f / M.lt[i] - 0.5f * ui * ui) * 2.0f * g[i];
    }
    for (int k = 0; k < d; ++k) {
        float s = 0.0f;
        for (int i = 0; i < d; ++i) s += zz[i] * (-Gh[i][k]);
        out[k] = s - g[k];
    }
}

// dH/dtheta (closed form, see header)
template <int DM>
__device__ __forceinline__ void grad_params(const RmTarget& t, const float* th, const Metric<DM>& M, const float* p,
                                            float* out) {
    const int d = rm_dim<DM>(t);
    float u[DM], glp[DM];
    for (int i = 0; i < d; ++i) {
        float wi = 0.0f;
        for (int a = 0; a < d; ++a) wi += M.Q[a][i] * p[a];
        u[i] = wi / M.lt[i];
    }
    float B[DM][DM], Z[DM][DM];
    for (int i = 0; i < d; ++i)
        for (int j = 0; j < d; ++j) {
            float F;
            if (i == j) F = M.dlt[i];
            else {
                const float dl = M.lam[i] - M.lam[j];
                F = (fabsf(dl) > 1e-12f * (fabsf(M.lam[i]) + fabsf(M.lam[j]))) ? (M.lt[i] - M.lt[j]) / dl : M.dlt[i];
            }
            B[i][j] = -0.5f * u[i] * u[j] * F + ((i == j) ? 0.5f * M.dlt[i] / M.lt[i] : 0.0f);
        }
    // Z = Q B Q^T
    for (int a = 0; a < d; ++a)
        for (int j = 0; j < d; ++j) {
            float s = 0.0f;
            for (int i = 0; i < d; ++i) s += M.Q[a][i] * B[i][j];
            Z[a][j] = s;                                      // (Q B)[a][j]
        }
    for (int a = 0; a < d; ++a) {
        float row[DM];
        for (int b = 0; b < d; ++b) {
            float s = 0.0f;
            for (int j = 0; j < d; ++j) s += Z[a][j] * M.Q[b][j];
            row[b] = s;
        }
        for (int b = 0; b < d; ++b) B[a][b] = row[b];         // reuse B as Z = Q B Q^T
    }
    rm_contract_dmetric<DM>(t, th, B, out);
    rm_grad_log_prob<DM>(t, th, glp);
    for (int k = 0; k < d; ++k) out[k] = out[k] - glp[k];
}

// gibbs (:183-184): p = chol(G~) z,  G~ = Q diag(lam~) Q^T
template <int DM>
__device__ __forceinline__ bool gibbs_rm(const RmTarget& t, const Metric<DM>& M, const float* z, float* p) {
    const int d = rm_dim<DM>(t);
    float G[DM][DM];
    for (int a = 0; a < d; ++a)
        for (int b = 0; b <= a; ++b) {
            float s = 0.0f;
            for (int i = 0; i < d; ++i) s += M.Q[a][i] * M.lt[i] * M.Q[b][i];
            G[a][b] = s;
        }
    bool ok = true;
    for (int j = 0; j < d; ++j) {                             // Cholesky, lower, in place
        float s = G[j][j];
        for (int k = 0; k < j; ++k) s -= G[j][k] * G[j][k];
        if (!(s > 0.0f)) ok = false;
        const float ljj = sqrtf(s);
        G[j][j] = ljj;
        for (int i = j + 1; i < d; ++i) {
            float v = G[i][j];
            for (int k = 0; k < j; ++k) v -= G[i][k] * G[j][k];
            G[i][j] = v / ljj;
        }
    }
    for (int a = 0; a < d; ++a) {
        float s = 0.0f;
        for (int b = 0; b <= a; ++b) s += G[a][b] * z[b];
        p[a] = s;
    }
    return ok;
}

// ---------------------------------------------------------------------------------------------------------
// run kernel: one thread = one chain
// ---------------------------------------------------------------------------------------------------------
struct RmRunArgs {
    RmTarget t;
    RmCfg cfg;
    int integrator;               // 1 explicit, 2 implicit (Integrator enum values)
    float cosw, sinw;             // cos/sin(2*omega*eps) evaluated in fp32 like samplers.py:435-436
    float fp_threshold;
    int fp_max_iter, jitter_max_tries;
    int C, ld;
    int rng_mode;
    uint64_t seed, chain_offset;
    const float* normals;         // [S, C, ld]
    const float* logu;            // [S, C]
    const float* uniforms;        // [S, C, J, ld]  injected jitter draws
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
};

template <int DM>
struct JitterSrc {                // the jitter uniforms of fisher() (:115), one row of D per call
    const RmRunArgs& a;
    int c, n, idx;
    uint64_t chain_id;
    __device__ JitterSrc(const RmRunArgs& a_, int c_, int n_) : a(a_), c(c_), n(n_), idx(0),
                                                               chain_id(a_.chain_offset + (uint64_t)c_) {}
    __device__ const float* next(float* buf) {
        if (a.cfg.jitter < 0.0f) return nullptr;
        const int d = rm_dim<DM>(a.t);
        if (a.rng_mode == HMCX_RNG_INJECTED) {
            const int j = idx < a.J ? idx : a.J - 1;          // overflow (NaN retries) re-uses the last row
            const float* src = a.uniforms + (((size_t)(n - a.it0) * a.C + c) * a.J + j) * a.ld;
            for (int i = 0; i < d; ++i) buf[i] = src[i];
        } else {
            for (int v = 0; 4 * v < d; ++v) {
                float u[4];
                philox_jitter4(a.seed, chain_id, (uint64_t)n, idx, v, u);
                for (int j = 0; j < 4 && 4 * v + j < d; ++j) buf[4 * v + j] = u[j];
            }
        }
        ++idx;
        return buf;
    }
};

// Every metric evaluation of the thread-per-chain kernel goes through this ONE out-of-line function.  The first form
// inlined eval_metric / rm_hamiltonian / grad_* at each of the 15 call sites of an iteration (gibbs, 2 x H, 8 explicit +
// 4 implicit flows): 100k instructions (1.6 MB of code) for DM = 6 / 16, executed at the instruction-fetch rate.
//   RM_EVAL_METRIC  fisher() only (gibbs)                 RM_EVAL_H     + rm_hamiltonian -> *H_out (NaN if the metric failed)
//   RM_EVAL_DHDQ    dH/dtheta with the NaN-retry loop     RM_EVAL_DHDP  dH/dp
// Returns false <=> the reference raises LogProbError.
enum { RM_EVAL_METRIC = 0, RM_EVAL_H = 1, RM_EVAL_DHDQ = 2, RM_EVAL_DHDP = 3 };

template <int DM>
__device__ __noinline__ bool rm_eval(JitterSrc<DM>& jit, int kind, const float* th, const float* pp, Metric<DM>& M,
                                     float* w, float* ub, float* out, float* H_out) {
    const RmRunArgs& a = jit.a;
    const RmTarget& t = a.t;
    const int d = rm_dim<DM>(t);
    for (int tries = 0;; ++tries) {
        if (!eval_metric<DM>(t, a.cfg, th, jit.next(ub), M)) return false;
        if (kind == RM_EVAL_METRIC) return true;
        bool okh = true;
        const float H = rm_hamiltonian<DM>(t, a.cfg, th, pp, M, w, okh);
        if (kind == RM_EVAL_H) { *H_out = H; return okh; }
        if (!okh) return false;
        if (kind == RM_EVAL_DHDP) { grad_momentum<DM>(t, M, pp, out); return true; }
        if (a.cfg.jacdiag) grad_params_jacdiag<DM>(t, th, M, pp, out); else grad_params<DM>(t, th, M, pp, out);
        bool fin = true;
        for (int i = 0; i < d; ++i) fin = fin && finite_f(out[i]);
        if (fin) return true;
        if (tries + 1 > a.jitter_max_tries) return false;
    }
}

template <int DM>
__global__ void __launch_bounds__(128) rmhmc_run_kernel(const RmRunArgs a) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= a.C) return;
    const RmTarget& t = a.t;
    const int d = rm_dim<DM>(t);
    const size_t row = (size_t)c * a.ld;
    const uint64_t chain_id = a.chain_offset + (uint64_t)c;

    float qc[DM], q[DM], p[DM], qt[DM], pt[DM], g[DM], w[DM], ub[DM];
    for (int i = 0; i < d; ++i) qc[i] = a.q_cur[row + i];
    const float eps = a.eps[c];
    const float half = mul(0.5f, eps);
    int rejected = 0;
    const int keep = a.S - a.burn;
    float* const my_samples = a.samples ? a.samples + (size_t)c * keep * a.ld : nullptr;
    if (a.it0 == 0 && my_samples)
        for (int i = 0; i < a.ld; ++i) my_samples[i] = i < d ? qc[i] : 0.0f;

    Metric<DM> M;
    for (int n = a.it0; n < a.it1; ++n) {
        JitterSrc<DM> jit(a, c, n);
        bool ok = true;
        float h_old = nanf(""), h_new = nanf("");
        // dH/dtheta with the reference's NaN-retry loop (:402-410); dH/dp (:415-422): calls of the ONE out-of-line copy
        auto dHdq = [&](const float* th, const float* pp, float* out) {
            if (ok) ok = rm_eval<DM>(jit, RM_EVAL_DHDQ, th, pp, M, w, ub, out, nullptr);
        };
        auto dHdp = [&](const float* th, const float* pp, float* out) {
            if (ok) ok = rm_eval<DM>(jit, RM_EVAL_DHDP, th, pp, M, w, ub, out, nullptr);
        };

        // ---- gibbs (:969 -> :183-184) ----
        ok = rm_eval<DM>(jit, RM_EVAL_METRIC, qc, nullptr, M, w, ub, nullptr, nullptr);
        {
            float z[DM];
            if (a.rng_mode == HMCX_RNG_INJECTED) {
                for (int i = 0; i < d; ++i) z[i] = a.normals[((size_t)(n - a.it0) * a.C + c) * a.ld + i];
            } else {
                for (int v = 0; 4 * v < d; ++v) {
                    float z4[4];
                    philox_normal4(a.seed, chain_id, (uint64_t)n, (uint32_t)v, z4);
                    for (int j = 0; j < 4 && 4 * v + j < d; ++j) z[4 * v + j] = z4[j];
                }
            }
            if (ok) ok = gibbs_rm<DM>(t, M, z, p);
        }
        for (int i = 0; i < d; ++i) q[i] = qc[i];
        // ---- H(theta, p) (:971; the explicit branch's 2*H ... /2 is exact) ----
        if (ok) ok = rm_eval<DM>(jit, RM_EVAL_H, q, p, M, w, ub, nullptr, &h_old);
        // ---- trajectory ----
        if (ok && a.integrator == 1) {                                              // explicit (:423-461)
            for (int i = 0; i < d; ++i) { qt[i] = q[i]; pt[i] = p[i]; }
            for (int l = 0; l < a.L && ok; ++l) {
                dHdq(q, pt, g);  if (ok) for (int i = 0; i < d; ++i) p[i] = sub(p[i], mul(half, g[i]));      // A
                dHdp(q, pt, g);  if (ok) for (int i = 0; i < d; ++i) qt[i] = add(qt[i], mul(half, g[i]));
                dHdp(qt, p, g);  if (ok) for (int i = 0; i < d; ++i) q[i] = add(q[i], mul(half, g[i]));       // B
                dHdq(qt, p, g);  if (ok) for (int i = 0; i < d; ++i) pt[i] = sub(pt[i], mul(half, g[i]));
                if (!ok) break;
                for (int i = 0; i < d; ++i) {                                                                  // C, sequential
                    const float cw = a.cosw, sw = a.sinw;
                    const float qn = mul(0.5f, add(add(add(q[i], qt[i]), mul(cw, sub(q[i], qt[i]))), mul(sw, sub(p[i], pt[i]))));
                    const float pn = mul(0.5f, add(sub(add(p[i], pt[i]), mul(sw, sub(qn, qt[i]))), mul(cw, sub(p[i], pt[i]))));
                    const float qtn = mul(0.5f, sub(sub(add(qn, qt[i]), mul(cw, sub(qn, qt[i]))), mul(sw, sub(pn, pt[i]))));
                    const float ptn = mul(0.5f, sub(add(add(pn, pt[i]), mul(sw, sub(qn, qtn))), mul(cw, sub(pn, pt[i]))));
                    q[i] = qn; p[i] = pn; qt[i] = qtn; pt[i] = ptn;
                }
                dHdp(qt, p, g);  if (ok) for (int i = 0; i < d; ++i) q[i] = add(q[i], mul(half, g[i]));       // B
                dHdq(qt, p, g);  if (ok) for (int i = 0; i < d; ++i) pt[i] = sub(pt[i], mul(half, g[i]));
                dHdq(q, pt, g);  if (ok) for (int i = 0; i < d; ++i) p[i] = sub(p[i], mul(half, g[i]));      // A
                dHdp(q, pt, g);  if (ok) for (int i = 0; i < d; ++i) qt[i] = add(qt[i], mul(half, g[i]));
            }
        } else if (ok) {                                                            // implicit (:363-386)
            for (int l = 0; l < a.L && ok; ++l) {
                for (int i = 0; i < d; ++i) pt[i] = p[i];                           // momentum_old
                for (int it = 0; it < a.fp_max_iter && ok; ++it) {                  // fixed_point_momentum
                    dHdq(q, p, g);
                    if (!ok) break;
                    float diff = 0.0f;
                    for (int i = 0; i < d; ++i) {
                        const float pn = sub(pt[i], mul(half, g[i]));
                        const float e = sub(p[i], pn);
                        diff = fmaxf(diff, mul(e, e));
                        p[i] = pn;
                    }
                    if (diff < a.fp_threshold) break;
                }
                if (!ok) break;
                float g_old[DM];
                for (int i = 0; i < d; ++i) qt[i] = q[i];                           // params_old
                dHdp(q, p, g_old);
                for (int it = 0; it < a.fp_max_iter && ok; ++it) {                  // fixed_point_params
                    dHdp(q, p, g);
                    if (!ok) break;
                    float diff = 0.0f;
                    for (int i = 0; i < d; ++i) {
                        const float qn = add(add(qt[i], mul(half, g[i])), mul(half, g_old[i]));
                        const float e = sub(q[i], qn);
                        diff = fmaxf(diff, mul(e, e));
                        q[i] = qn;
                    }
                    if (diff < a.fp_threshold) break;
                }
                if (!ok) break;
                dHdq(q, p, g);
                if (ok) for (int i = 0; i < d; ++i) p[i] = sub(p[i], mul(half, g[i]));
            }
        }
        // ---- H(theta_L, p_L) on the un-augmented Hamiltonian (:989) ----
        if (ok) ok = rm_eval<DM>(jit, RM_EVAL_H, q, p, M, w, ub, nullptr, &h_new);
        // ---- MH + bookkeeping ----
        const float x = add(-h_new, h_old);
        const float rho = (x < 0.0f) ? x : 0.0f;
        const float logu = (a.rng_mode == HMCX_RNG_INJECTED) ? a.logu[(size_t)(n - a.it0) * a.C + c]
                                                             : philox_log_uniform(a.seed, chain_id, (uint64_t)n);
        const bool acc = ok && (rho >= logu);
        if (acc) {
            for (int i = 0; i < d; ++i) qc[i] = q[i];
        } else {
            ++rejected;
            if (n == a.burn + 1) for (int i = 0; i < d; ++i) qc[i] = a.q_init[row + i];   // :1018 quirk
        }
        if (n > a.burn && my_samples) {
            float* dst = my_samples + (size_t)(n - a.burn) * a.ld;
            for (int i = 0; i < a.ld; ++i) dst[i] = i < d ? qc[i] : 0.0f;
        }
        const size_t o = (size_t)c * a.S + n;
        if (a.accept) a.accept[o] = acc ? 1 : 0;
        if (a.diverged) a.diverged[o] = ok ? 0 : 1;
        if (a.ham) { a.ham[2 * o] = h_old; a.ham[2 * o + 1] = h_new; }
    }
    for (int i = 0; i < d; ++i) a.q_cur[row + i] = qc[i];
    if (a.num_rejected) a.num_rejected[c] += rejected;
}


// ---------------------------------------------------------------------------------------------------------
// BASELINE config 3 form: D == 2, explicit integrator.  A chain is a serial recurrence of 8L+3 metric evaluations per
// iteration, ~600 dependent instructions each, so the run time is the LATENCY of that recurrence, not throughput.
// Independent evaluations are therefore run CONCURRENTLY by different warps (= different schedulers of the SM); a chain
// is owned by one lane of each of the CTA's 4 warps:
//   * the two evaluations of every A / B flow of the explicit step (samplers.py:429-430, :432-433, :454-455, :457-458) take
//     the SAME arguments and differ only in the jitter row and in what is differentiated: warp 0 dH/dtheta, warp 1 dH/dp;
//   * the LAST A flow of step l and the FIRST A flow of step l+1 both act on (theta, p~) and update only (p, theta~): their
//     four evaluations are independent -> one stage of 4 warps ("AA");
//   * H(theta, p) before the trajectory (:971) and the first A flow see the same (theta, p~ = p): one stage (warp 2 takes H).
// Results cross through a double-buffered shared mailbox with one barrier per stage, and every warp applies all updates
// to its replica of (theta, p, theta~, p~) with the reference's roundings, so the replicas stay bit-identical and every
// scalar decision is taken four times, identically.  Serial stages per iteration: 3L+3 instead of 8L+3 evaluations
// (4L+3 for the two-warp form of this kernel).  32 chains per CTA -> 512 chains = 16 CTAs.
//
// Jitter rows (fisher's torch.rand(D), :115) are consumed in the reference's order.  The NaN-retry loop of a dH/dtheta
// (:402-410) may take extra rows, which shifts the rows of every later evaluation of the stage: each warp first assumes
// no retries and is re-run (rare) when the retry counts that precede it turn out non-zero.
//
// Code layout: the iteration is ONE loop over its stages around a SINGLE inlined copy of eval_metric / rm_hamiltonian /
// grad_params / grad_momentum (~2k instructions).  The first form of this kernel inlined a copy per call site -- 14.5k
// instructions, 11k of them in the iteration loop = 180 KB of code streamed through the instruction cache once per
// iteration -- and ran at the instruction-fetch rate (ncu: no_instruction was the top stall reason).
// ---------------------------------------------------------------------------------------------------------
struct PairMail { float g0, g1; int ok, retries; };

__device__ __forceinline__ const float* rm2_jitter_row(const RmRunArgs& a, int c, int n, uint64_t chain_id, int idx,
                                                       float* buf) {
    if (a.cfg.jitter < 0.0f) return nullptr;
    if (a.rng_mode == HMCX_RNG_INJECTED) {
        const int j = idx < a.J ? idx : a.J - 1;              // overflow (NaN retries) re-uses the last row
        const float* src = a.uniforms + (((size_t)(n - a.it0) * a.C + c) * a.J + j) * a.ld;
        buf[0] = src[0]; buf[1] = src[1];
    } else {
        float u[4];
        philox_jitter4(a.seed, chain_id, (uint64_t)n, idx, 0, u);
        buf[0] = u[0];
        buf[1] = u[1];
    }
    return buf;
}

enum { RQ_GIBBS = 0, RQ_HOLD_A = 1, RQ_B = 2, RQ_AA = 3, RQ_A = 4, RQ_HNEW = 5 };     // stage kinds
enum { RQ_EV_METRIC = 0, RQ_EV_H = 1, RQ_EV_DHDQ = 2, RQ_EV_DHDP = 3 };

__global__ void __launch_bounds__(128) rmhmc2_quad_kernel(const RmRunArgs a) {
    __shared__ PairMail mail[2][4][32];
    const int lane = threadIdx.x & 31, role = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + lane;
    const bool live = c < a.C;
    const int cc = live ? c : a.C - 1;                        // idle lanes shadow the last chain (no stores)
    const RmTarget& t = a.t;
    const size_t row = (size_t)cc * a.ld;
    const uint64_t chain_id = a.chain_offset + (uint64_t)cc;
    const bool writer = live && role == 0;

    float qc[2], q[2], p[2], qt[2], pt[2], g[2], w[2], ub[2];
    qc[0] = a.q_cur[row]; qc[1] = a.q_cur[row + 1];
    const float eps = a.eps[cc];
    const float half = mul(0.5f, eps);
    int rejected = 0;
    const int keep = a.S - a.burn;
    float* const my_samples = (a.samples && writer) ? a.samples + (size_t)cc * keep * a.ld : nullptr;
    if (a.it0 == 0 && my_samples)
        for (int i = 0; i < a.ld; ++i) my_samples[i] = i < 2 ? qc[i] : 0.0f;
    const bool jit_on = a.cfg.jitter >= 0.0f;
    int phase = 0;
    Metric<2> M;
    const int nst = 3 * a.L + 3;
    q[0] = q[1] = p[0] = p[1] = qt[0] = qt[1] = pt[0] = pt[1] = g[0] = g[1] = 0.0f;

    for (int n = a.it0; n < a.it1; ++n) {
        int idx = 0;                                          // jitter rows consumed so far in this iteration
        bool ok = true;
        float h_old = nanf(""), h_new = nanf("");
        q[0] = qc[0]; q[1] = qc[1];
#pragma unroll 1
        for (int st = 0; st < nst; ++st) {
            // ---- what this stage is, and what this warp evaluates in it ----
            int kind;
            bool first_b = false;
            if (st == 0) kind = RQ_GIBBS;
            else if (st == 1) kind = RQ_HOLD_A;
            else if (st == nst - 1) kind = RQ_HNEW;
            else {
                const int l = (st - 2) / 3, k = (st - 2) - 3 * l;
                kind = k < 2 ? RQ_B : (l == a.L - 1 ? RQ_A : RQ_AA);
                first_b = k == 0;
            }
            if (kind == RQ_HOLD_A) { qt[0] = q[0]; qt[1] = q[1]; pt[0] = p[0]; pt[1] = p[1]; }    // :423-424
            const bool mailed = kind != RQ_GIBBS && kind != RQ_HNEW;
            int ev, off;                                      // evaluation kind, jitter-row offset before retry shifts
            bool active = true;
            if (kind == RQ_GIBBS) { ev = RQ_EV_METRIC; off = 0; }
            else if (kind == RQ_HNEW) { ev = RQ_EV_H; off = 0; }
            else if (kind == RQ_HOLD_A) {                     // H(theta, p) row 0 | first A flow: dH/dtheta row 1, dH/dp row 2
                ev = role == 0 ? RQ_EV_DHDQ : (role == 1 ? RQ_EV_DHDP : RQ_EV_H);
                off = role == 0 ? 1 : (role == 1 ? 2 : 0);
                active = role < 3;
            } else if (kind == RQ_B) {                        // the reference calls dH/dp first in B flows
                ev = role == 0 ? RQ_EV_DHDQ : RQ_EV_DHDP;
                off = role == 0 ? 1 : 0;
                active = role < 2;
            } else {                                          // A / AA: dH/dtheta first
                ev = (role & 1) ? RQ_EV_DHDP : RQ_EV_DHDQ;
                off = role;
                active = kind == RQ_AA || role < 2;
            }
            const bool useB = kind == RQ_B, useA = kind == RQ_AA || kind == RQ_A;     // B: (theta~, p); A: (theta, p~)
            float th[2], pp[2];
            th[0] = useB ? qt[0] : q[0]; th[1] = useB ? qt[1] : q[1];
            pp[0] = useA ? pt[0] : p[0]; pp[1] = useA ? pt[1] : p[1];
            const int b = phase & 1;
            if (mailed) ++phase;
            PairMail m0 = PairMail{0.0f, 0.0f, 1, 0}, m1 = m0, m2 = m0, m3 = m0;
            float H = nanf("");
            bool good = true;
            int used_shift = 0;
            for (int pass = 0;; ++pass) {
                // retries of the dH/dtheta evaluations that precede this warp's in the reference's order shift its row
                int shift = 0;
                if (pass > 0) {
                    if (kind == RQ_AA) shift = role == 0 ? 0 : (role == 3 ? m0.retries + m2.retries : m0.retries);
                    else if (kind != RQ_B) shift = role == 1 ? m0.retries : 0;
                }
                if (ok && active && (pass == 0 || shift != used_shift)) {
                    used_shift = shift;
                    const int first_row = idx + off + shift;
                    good = true;
                    int tries = 0;
                    for (;; ++tries) {                        // the NaN-retry loop of dH/dtheta (:402-410); one trip otherwise
                        if (!eval_metric<2>(t, a.cfg, th, rm2_jitter_row(a, cc, n, chain_id, first_row + tries, ub), M)) { good = false; break; }
                        if (ev == RQ_EV_METRIC) break;
                        bool okh = true;
                        H = rm_hamiltonian<2>(t, a.cfg, th, pp, M, w, okh);
                        if (!okh) { good = false; break; }
                        if (ev == RQ_EV_H) break;
                        if (ev == RQ_EV_DHDP) { grad_momentum<2>(t, M, pp, g); break; }
                        if (a.cfg.jacdiag) grad_params_jacdiag<2>(t, th, M, pp, g); else grad_params<2>(t, th, M, pp, g);
                        if (finite_f(g[0]) && finite_f(g[1])) break;
                        if (tries + 1 > a.jitter_max_tries) { good = false; break; }
                    }
                    if (mailed) mail[b][role][lane] = PairMail{ev == RQ_EV_H ? H : g[0], g[1], good ? 1 : 0, ev == RQ_EV_DHDQ ? tries : 0};
                }
                if (!mailed) break;
                __syncthreads();
                m0 = mail[b][0][lane]; m1 = mail[b][1][lane]; m2 = mail[b][2][lane]; m3 = mail[b][3][lane];
                if (!jit_on || kind == RQ_B || pass == 2) break;
                int want = 0;
                if (kind == RQ_AA) want = role == 0 ? 0 : (role == 3 ? m0.retries + m2.retries : m0.retries);
                else want = role == 1 ? m0.retries : 0;
                if (!__syncthreads_or(ok && active && want != used_shift)) break;
            }
            // ---- apply the stage (every warp, identically) ----
            if (kind == RQ_GIBBS) {
                ++idx;
                ok = good;
                float z[2];
                if (a.rng_mode == HMCX_RNG_INJECTED) {
                    const float* zp = a.normals + ((size_t)(n - a.it0) * a.C + cc) * a.ld;
                    z[0] = zp[0]; z[1] = zp[1];
                } else {
                    float z4[4];
                    philox_normal4(a.seed, chain_id, (uint64_t)n, 0u, z4);
                    z[0] = z4[0]; z[1] = z4[1];
                }
                if (ok) ok = gibbs_rm<2>(t, M, z, p);
            } else if (kind == RQ_HNEW) {
                if (ok) { ++idx; h_new = H; ok = good; }       // NaN when the metric itself failed
            } else if (ok) {
                auto flow_a = [&](const PairMail& mq, const PairMail& mp) {
                    for (int i = 0; i < 2; ++i) {
                        const float gq = i ? mq.g1 : mq.g0, gp = i ? mp.g1 : mp.g0;
                        p[i] = sub(p[i], mul(half, gq)); qt[i] = add(qt[i], mul(half, gp));
                    }
                };
                if (kind == RQ_HOLD_A) {                       // reference order: H_old, then the flow (:971, :429-430)
                    ++idx;
                    h_old = m2.g0;
                    ok = m2.ok != 0;
                }
                if (ok) {
                    // the first call's LogProbError aborts before the second call is made
                    ok = m0.ok && m1.ok;
                    idx += 2 + m0.retries;
                    if (ok) {
                        if (kind != RQ_B) {
                            flow_a(m0, m1);
                            if (kind == RQ_AA) {               // the next step's first A flow: same arguments, next rows
                                ok = m2.ok && m3.ok;
                                idx += 2 + m2.retries;
                                if (ok) flow_a(m2, m3);
                            }
                        } else {
                            for (int i = 0; i < 2; ++i) {
                                const float gq = i ? m0.g1 : m0.g0, gp = i ? m1.g1 : m1.g0;
                                q[i] = add(q[i], mul(half, gp)); pt[i] = sub(pt[i], mul(half, gq));
                            }
                            if (first_b) {
                                for (int i = 0; i < 2; ++i) {                                           // C, sequential
                                    const float cw = a.cosw, sw = a.sinw;
                                    const float qn = mul(0.5f, add(add(add(q[i], qt[i]), mul(cw, sub(q[i], qt[i]))), mul(sw, sub(p[i], pt[i]))));
                                    const float pn = mul(0.5f, add(sub(add(p[i], pt[i]), mul(sw, sub(qn, qt[i]))), mul(cw, sub(p[i], pt[i]))));
                                    const float qtn = mul(0.5f, sub(sub(add(qn, qt[i]), mul(cw, sub(qn, qt[i]))), mul(sw, sub(pn, pt[i]))));
                                    const float ptn = mul(0.5f, sub(add(add(pn, pt[i]), mul(sw, sub(qn, qtn))), mul(cw, sub(pn, pt[i]))));
                                    q[i] = qn; p[i] = pn; qt[i] = qtn; pt[i] = ptn;
                                }
                            }
                        }
                    }
                }
            }
        }
        // ---- MH + bookkeeping (all warps decide identically; warp 0 stores) ----
        const float x = add(-h_new, h_old);
        const float rho = (x < 0.0f) ? x : 0.0f;
        const float logu = (a.rng_mode == HMCX_RNG_INJECTED) ? a.logu[(size_t)(n - a.it0) * a.C + cc]
                                                             : philox_log_uniform(a.seed, chain_id, (uint64_t)n);
        const bool acc = ok && (rho >= logu);
        if (acc) {
            qc[0] = q[0]; qc[1] = q[1];
        } else {
            ++rejected;
            if (n == a.burn + 1) { qc[0] = a.q_init[row]; qc[1] = a.q_init[row + 1]; }                 // :1018 quirk
        }
        if (writer) {
            if (n > a.burn && my_samples) {
                float* dst = my_samples + (size_t)(n - a.burn) * a.ld;
                for (int i = 0; i < a.ld; ++i) dst[i] = i < 2 ? qc[i] : 0.0f;
            }
            const size_t o = (size_t)cc * a.S + n;
            if (a.accept) a.accept[o] = acc ? 1 : 0;
            if (a.diverged) a.diverged[o] = ok ? 0 : 1;
            if (a.ham) { a.ham[2 * o] = h_old; a.ham[2 * o + 1] = h_new; }
        }
    }
    if (writer) {
        a.q_cur[row] = qc[0]; a.q_cur[row + 1] = qc[1];
        if (a.num_rejected) a.num_rejected[cc] += rejected;
    }
}


// ---------------------------------------------------------------------------------------------------------
// plain HMC / HMC_NUTS for small coupled problems (D <= 16): one thread per chain
//   targets GAUSS_FULL and FUNNEL (whose gradients couple the coordinates) and the full (2-D) inv_mass of
//   samplers.py:293-294 (drift), :811-812 (kinetic), :198-199 (gibbs: MultivariateNormal(0, inverse(inv_mass)))
//   -- e.g. the correlated variant of BASELINE config 1 and the notebook funnel under HMC / NUTS.
// ---------------------------------------------------------------------------------------------------------
struct SmallRunArgs {
    RmTarget t;
    int mk, C, ld;
    const float* im;              // inv_mass: [D] or [D,D]
    const float* mf;              // sqrt(mass) [D] or lower Cholesky factor of mass [D,D]
    int rng_mode;
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
    int L, S, burn, it0, it1;
    float* samples;
    uint8_t* accept;
    uint8_t* diverged;
    float* ham;
    int32_t* num_rejected;
};

template <int DM>
__global__ void __launch_bounds__(128) hmc_small_kernel(const SmallRunArgs a) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= a.C) return;
    const RmTarget& t = a.t;
    const int d = rm_dim<DM>(t);
    const size_t row = (size_t)c * a.ld;
    const uint64_t chain_id = a.chain_offset + (uint64_t)c;
    float qc[DM], q[DM], p[DM], g[DM], v[DM];
    for (int i = 0; i < d; ++i) qc[i] = a.q_cur[row + i];
    float eps = a.eps[c];
    double h_bar = 0.0, eps_bar = 1.0;
    if (a.nuts) { h_bar = a.h_bar[c]; eps_bar = a.eps_bar[c]; }
    int rejected = 0;
    const int keep = a.S - a.burn;
    float* const my_samples = a.samples ? a.samples + (size_t)c * keep * a.ld : nullptr;
    if (a.it0 == 0 && my_samples)
        for (int i = 0; i < a.ld; ++i) my_samples[i] = i < d ? qc[i] : 0.0f;

    auto minv = [&](const float* pp, float* out) {            // M^-1 p
        for (int i = 0; i < d; ++i) {
            if (a.mk == HMCX_MASS_FULL) {
                float s = 0.0f;
                for (int j = 0; j < d; ++j) s += a.im[i * d + j] * pp[j];
                out[i] = s;
            } else {
                out[i] = a.mk == HMCX_MASS_DIAG ? mul(a.im[i], pp[i]) : pp[i];
            }
        }
    };
    auto kinetic2 = [&](const float* pp) {                    // p . M^-1 p
        float s = 0.0f;
        minv(pp, v);
        for (int i = 0; i < d; ++i) s = add(s, mul(pp[i], v[i]));
        return s;
    };
    float lp_cur = rm_log_prob<DM>(t, qc);

    for (int n = a.it0; n < a.it1; ++n) {
        if (a.eps_schedule) eps = a.eps_schedule[(size_t)n * a.C + c];
        const float half = mul(0.5f, eps);
        float z[DM];
        if (a.rng_mode == HMCX_RNG_INJECTED) {
            for (int i = 0; i < d; ++i) z[i] = a.normals[((size_t)(n - a.it0) * a.C + c) * a.ld + i];
        } else {
            for (int vv = 0; 4 * vv < d; ++vv) {
                float z4[4];
                philox_normal4(a.seed, chain_id, (uint64_t)n, (uint32_t)vv, z4);
                for (int j = 0; j < 4 && 4 * vv + j < d; ++j) z[4 * vv + j] = z4[j];
            }
        }
        for (int i = 0; i < d; ++i) {                         // gibbs
            if (a.mk == HMCX_MASS_FULL) {
                float s = 0.0f;
                for (int j = 0; j <= i; ++j) s += a.mf[i * d + j] * z[j];
                p[i] = s;
            } else {
                p[i] = a.mk == HMCX_MASS_DIAG ? mul(z[i], a.mf[i]) : z[i];
            }
            q[i] = qc[i];
        }
        const float kin0 = kinetic2(p);
        rm_grad_log_prob<DM>(t, q, g);                                                          // :281
        for (int i = 0; i < d; ++i) p[i] = add(p[i], mul(half, g[i]));
        for (int l = 0; l < a.L; ++l) {
            minv(p, v);
            for (int i = 0; i < d; ++i) q[i] = add(q[i], a.mk == HMCX_MASS_DIAG ? mul(mul(eps, a.im[i]), p[i])
                                                                                 : mul(eps, v[i]));   // :284/:294/:296
            rm_grad_log_prob<DM>(t, q, g);
            for (int i = 0; i < d; ++i) p[i] = add(p[i], mul(eps, g[i]));                          // :298
        }
        for (int i = 0; i < d; ++i) p[i] = sub(p[i], mul(half, g[i]));                             // :302
        const float lp_new = rm_log_prob<DM>(t, q);
        const float kin1 = kinetic2(p);
        const float h_old = add(-lp_cur, mul(0.5f, kin0));
        const float h_new = add(-lp_new, mul(0.5f, kin1));
        const bool bad = !finite_f(lp_cur) || !finite_f(lp_new);
        const float x = add(-h_new, h_old);
        const float rho = (x < 0.0f) ? x : 0.0f;
        const float logu = (a.rng_mode == HMCX_RNG_INJECTED) ? a.logu[(size_t)(n - a.it0) * a.C + c]
                                                             : philox_log_uniform(a.seed, chain_id, (uint64_t)n);
        const bool acc = !bad && (rho >= logu);
        if (acc) {
            lp_cur = lp_new;
            for (int i = 0; i < d; ++i) qc[i] = q[i];
        } else {
            ++rejected;
            if (n == a.burn + 1) {                                                                // :1018 quirk
                for (int i = 0; i < d; ++i) qc[i] = a.q_init[row + i];
                lp_cur = rm_log_prob<DM>(t, qc);
            }
        }
        if (n > a.burn && my_samples) {
            float* dst = my_samples + (size_t)(n - a.burn) * a.ld;
            for (int i = 0; i < a.ld; ++i) dst[i] = i < d ? qc[i] : 0.0f;
        }
        const size_t o = (size_t)c * a.S + n;
        if (a.accept) a.accept[o] = acc ? 1 : 0;
        if (a.diverged) a.diverged[o] = bad ? 1 : 0;
        if (a.ham) { a.ham[2 * o] = h_old; a.ham[2 * o + 1] = h_new; }
        if (a.nuts && n <= a.burn) {                                                             // :1030-1035, :1060-1067
            if (n < a.burn || bad) {
                const double* T = a.table + 5 * (size_t)n;
                const double alpha = bad ? 0.0 : (double)expf(rho);
                h_bar = __dadd_rn(__dmul_rn(T[0], h_bar), __dmul_rn(T[1], a.delta - alpha));
                const double x_new = a.mu - __dmul_rn(T[2], h_bar);
                eps = expf((float)x_new);
                const float xb = add((float)__dmul_rn(T[3], x_new), mul((float)T[4], logf((float)eps_bar)));
                eps_bar = (double)expf(xb);
            }
            if (n == a.burn) eps = (float)eps_bar;
        }
        if (a.eps_trace) a.eps_trace[(size_t)c * a.S + n] = eps;
    }
    for (int i = 0; i < d; ++i) a.q_cur[row + i] = qc[i];
    a.eps[c] = eps;
    if (a.nuts) { a.h_bar[c] = h_bar; a.eps_bar[c] = eps_bar; }
    if (a.num_rejected) a.num_rejected[c] += rejected;
}

int small_hmc_run(const hmcx_target_t* target, const hmcx_mass_t* mass, const hmcx_rng_t* rng, const hmcx_nuts_t* nuts,
                  const float* q_init, float* q_cur, float* eps, int C, int ld, int L, int S, int burn, int it0,
                  int it1, float* samples, uint8_t* accept, uint8_t* diverged, float* ham, int32_t* num_rejected,
                  cudaStream_t st) {
    if (!target || !rng || !q_init || !q_cur || !eps) return HMCX_ERR_INVALID_ARG;
    const int D = target->dim;
    if (D < 1 || C < 1 || ld < D || (ld & 3) || L < 1 || S < 1 || burn < 0 || burn >= S || it0 < 0 || it1 > S || it0 > it1)
        return HMCX_ERR_INVALID_ARG;
    if (D > 16) return HMCX_ERR_UNSUPPORTED;      // large dense targets / mass matrices run on the tensor cores (hmcx_tc.cu)
    SmallRunArgs a = {};
    a.t.kind = target->kind; a.t.D = D; a.t.log_norm = target->log_norm; a.t.inv_var_v = target->funnel_inv_var_v;
    a.t.mean = target->mean; a.t.ivar = target->inv_var; a.t.prec = target->prec;
    if (target->kind == HMCX_TARGET_GAUSS_DIAG && !target->inv_var) return HMCX_ERR_INVALID_ARG;
    if (target->kind == HMCX_TARGET_GAUSS_FULL && !target->prec) return HMCX_ERR_INVALID_ARG;
    if (target->kind == HMCX_TARGET_FUNNEL && D < 2) return HMCX_ERR_INVALID_ARG;
    a.mk = mass ? mass->kind : HMCX_MASS_NONE;
    if (a.mk != HMCX_MASS_NONE && (!mass->inv_mass || !mass->mass_factor)) return HMCX_ERR_INVALID_ARG;
    a.im = mass ? mass->inv_mass : nullptr; a.mf = mass ? mass->mass_factor : nullptr;
    a.C = C; a.ld = ld;
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
    const int block = 128, grid = (C + block - 1) / block;
    if (D == 2) hmc_small_kernel<2><<<grid, block, 0, st>>>(a);
    else if (D <= 6) hmc_small_kernel<6><<<grid, block, 0, st>>>(a);
    else hmc_small_kernel<16><<<grid, block, 0, st>>>(a);
    return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA;
}

int rmhmc_run(const hmcx_target_t* target, const hmcx_rmhmc_t* cfg, const hmcx_rng_t* rng, const float* q_init,
              float* q_cur, const float* eps, int C, int ld, int L, int S, int burn, int it0, int it1, float* samples,
              uint8_t* accept, uint8_t* diverged, float* ham, int32_t* num_rejected, cudaStream_t st) {
    if (!target || !cfg || !rng || !q_init || !q_cur || !eps) return HMCX_ERR_INVALID_ARG;
    if (target->kind != HMCX_TARGET_FUNNEL && target->kind != HMCX_TARGET_GAUSS_ISO &&
        target->kind != HMCX_TARGET_GAUSS_DIAG && target->kind != HMCX_TARGET_GAUSS_FULL)
        return HMCX_ERR_UNSUPPORTED;
    if (target->kind == HMCX_TARGET_GAUSS_FULL && !target->prec) return HMCX_ERR_INVALID_ARG;
    const int D = target->dim;
    if (D < 1 || C < 1 || ld < D || (ld & 3) || L < 1 || S < 1 || burn < 0 || burn >= S || it0 < 0 || it1 > S || it0 > it1)
        return HMCX_ERR_INVALID_ARG;
    if (D > 16) return HMCX_ERR_UNSUPPORTED;
    if (target->kind == HMCX_TARGET_FUNNEL && D < 2) return HMCX_ERR_INVALID_ARG;
    if (target->kind == HMCX_TARGET_GAUSS_DIAG && !target->inv_var) return HMCX_ERR_INVALID_ARG;
    if (cfg->integrator != 1 && cfg->integrator != 2) return HMCX_ERR_UNSUPPORTED;      // S3: out of scope
    if (cfg->metric != 1 && cfg->metric != 2 && cfg->metric != 3) return HMCX_ERR_UNSUPPORTED;
    RmRunArgs a = {};
    a.t.kind = target->kind; a.t.D = D; a.t.log_norm = target->log_norm; a.t.inv_var_v = target->funnel_inv_var_v;
    a.t.mean = target->mean; a.t.ivar = target->inv_var; a.t.prec = target->prec;
    a.cfg.softabs = cfg->metric == 2; a.cfg.jacdiag = cfg->metric == 3; a.cfg.alpha = cfg->softabs_const;
    a.cfg.jitter = cfg->jitter;
    a.cfg.pi_term = cfg->pi_term;
    a.integrator = cfg->integrator; a.cosw = cfg->cos_2we; a.sinw = cfg->sin_2we;
    a.fp_threshold = cfg->fixed_point_threshold; a.fp_max_iter = cfg->fixed_point_max_iterations;
    a.jitter_max_tries = cfg->jitter_max_tries;
    a.C = C; a.ld = ld;
    a.rng_mode = rng->mode; a.seed = rng->seed; a.chain_offset = rng->chain_offset;
    a.normals = rng->normals; a.logu = rng->log_uniforms; a.uniforms = rng->uniforms; a.J = rng->uniforms_per_iter;
    if (rng->mode == HMCX_RNG_INJECTED) {
        if (!rng->normals || !rng->log_uniforms) return HMCX_ERR_INVALID_ARG;
        if (cfg->jitter >= 0.0f && (!rng->uniforms || rng->uniforms_per_iter < 1)) return HMCX_ERR_INVALID_ARG;
    } else if (rng->mode != HMCX_RNG_PHILOX) {
        return HMCX_ERR_INVALID_ARG;
    }
    a.q_init = q_init; a.q_cur = q_cur; a.eps = eps; a.L = L; a.S = S; a.burn = burn; a.it0 = it0; a.it1 = it1;
    a.samples = samples; a.accept = accept; a.diverged = diverged; a.ham = ham; a.num_rejected = num_rejected;
    const int block = 128, grid = (C + block - 1) / block;
    if (D == 2 && cfg->integrator == 1) rmhmc2_quad_kernel<<<(C + 31) / 32, 128, 0, st>>>(a);       // BASELINE config 3
    else if (D == 2) rmhmc_run_kernel<2><<<grid, block, 0, st>>>(a);
    else if (D <= 6) rmhmc_run_kernel<6><<<grid, block, 0, st>>>(a);
    else rmhmc_run_kernel<16><<<grid, block, 0, st>>>(a);
    return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA;
}

}  // namespace hmcx
