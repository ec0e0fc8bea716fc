// hmcx_pred.cu -- held-out evaluation of a Bayesian NN: the posterior predictive mixture of every data point over its
// S = C*n pooled draws, with the curves of the first t draws of every chain.  hamiltorch_b200/predictive.py drives it;
// tests/predictive_oracle.py is the numpy definition.
//
// The block is fp32 f[c, s, i, o] at f + c*chain_stride + s*draw_stride + i*O + o: the network outputs of draw (c, s) at
// data point i (hmcx_mlp_pointwise_out, or predict_model's outputs).  A call handles a slab of k points [i0, i0 + k):
//   pred_scan_kernel   one thread per point, 128-point CTAs aligned to the global point index.  For t = 1 .. n it adds the
//                      C draws (c, t) to the point's fp64 running sums (shared memory, one column per thread, so the
//                      block reads are coalesced across the CTA's points), then writes the point's curve terms for t to the
//                      workspace; after the scan, its per-point outputs and its terms of the totals.
//   pred_group_kernel  per (row, 128-point group) the slab's terms in point order, continuing the group's partial sum
//                      where an earlier slab left it: the additions are those of one left-to-right sum over the group,
//                      whatever the slab boundaries.
//   pred_totals_kernel per row the group partials in group order.
// No atomics: the outputs depend on the block alone, not on k or on how the points were split into slabs.
#include <cfloat>
#include "hmcx_common.cuh"

namespace hmcx {

constexpr int PRED_GROUP = 128;           // points per group = threads per scan CTA
constexpr int PRED_BINS = 15;             // equal-width confidence bins of the reliability table
constexpr int PRED_TOTAL_ROWS = 1 + 3 * PRED_BINS;

namespace {

constexpr double LOG_2PI = 1.8378770664093454836;

__device__ __forceinline__ void lse_add(double& m, double& s, double x) {
    if (x > m) { s = s * exp(m - x) + 1.0; m = x; }
    else s += exp(x - m);
}

// 0 log 0 = 0
__device__ __forceinline__ double xlogx(double p, double lp) { return p > 0.0 ? p * lp : 0.0; }

__device__ __forceinline__ int conf_bin(double conf) {
    const int b = (int)ceil(conf * PRED_BINS) - 1;
    return b < 0 ? 0 : (b >= PRED_BINS ? PRED_BINS - 1 : b);
}

struct PredArgs {
    const float* f; long long cs, ds;
    int C, n, O, N, i0, k;
    const float* y;
    const float* tau; long long tcs, tds;
    double* pw;           // [7, N]
    double* po;           // [1 or 4, N, O]
    int* nonfinite;       // [N]
    double* terms;        // [2n + PRED_TOTAL_ROWS, k]
    double* rec;          // [n, pred_rec_rows, k]: the sums over the C draws of each step
    const double* cw;     // [C] chain weights (pred_step_kernel<LOSS, true> only)
};

__host__ __device__ __forceinline__ int pred_rec_rows(int loss, int O) {
    return loss == HMCX_LOSS_REGRESSION ? 3 * O + 4 : loss == HMCX_LOSS_BINARY ? 3 * O + 2 : O + 4;
}

__device__ __forceinline__ void lse_merge(double& m, double& s, double m2, double s2) {
    if (m2 > m) { s = s * exp(m - m2) + s2; m = m2; }
    else s += s2 * exp(m2 - m);
}

constexpr int OC = 16;                    // outputs per register chunk of pred_step_kernel

// Step records: one thread per (draw index t, point) sums the C draws (c, t) of its point in chain order, the outputs in
// register chunks of OC (a draw's softmax normaliser is recomputed per chunk).  Rows of rec[t, :, point]:
//   multi-class  0..O-1 sum_c p_c[o], O / O+1 logsumexp (max, scaled sum) of log p_c[y], O+2 sum_c H[p_c], O+3 non-finite
//   binary       0..O-1 sum_c sigmoid, O..2O-1 / 2O..3O-1 logsumexp of log p_c(y_o), 3O sum of entropies, 3O+1 non-finite
//   regression   0..O-1 sum_c e, O..2O-1 sum_c e^2 (e = f - f of draw (0, 1)), 2O..3O-1 sum_c Phi, 3O / 3O+1 logsumexp
//                of ll_c, 3O+2 sum_c 1/tau, 3O+3 non-finite
// WEIGHTED: chain c's terms are scaled by C w_c (its log-densities shifted by log(C w_c)) and chains with w_c = 0 are
// skipped, so the sums are C times the w-weighted mixture of the chains' draws t, and pred_scan_kernel's divisions by
// S_t = C t turn them into the mixture of the first t draws of every chain, chain c weighted w_c.
template <int LOSS, bool WEIGHTED = false>
__global__ void __launch_bounds__(256) pred_step_kernel(const PredArgs a) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)a.n * a.k) return;
    const int t = (int)(idx / a.k), li = (int)(idx - (long long)t * a.k), i = a.i0 + li;
    const int O = a.O, C = a.C, k = a.k;
    double* rec = a.rec + (long long)t * pred_rec_rows(LOSS, O) * k + li;
    auto W = [&](int r, double v) { rec[(long long)r * k] = v; };
    const float* yi = a.y + (long long)i * (LOSS == HMCX_LOSS_MULTICLASS ? 1 : O);
    const float* base = a.f + (long long)t * a.ds + (long long)i * O;
    bool bad = false;
    double H = 0.0, m = -INFINITY, s = 0.0, alea = 0.0;
    for (int o0 = 0; o0 < O; o0 += OC) {
        double P[OC], Q[OC], R[OC];
#pragma unroll
        for (int j = 0; j < OC; ++j) { P[j] = 0.0; Q[j] = LOSS == HMCX_LOSS_BINARY ? -INFINITY : 0.0; R[j] = 0.0; }
        for (int c = 0; c < C; ++c) {
            double wc = 1.0, lwc = 0.0;
            if (WEIGHTED) {
                wc = (double)C * a.cw[c];
                if (wc == 0.0) continue;
                lwc = log(wc);
            }
            auto sc = [&](double v) { return WEIGHTED ? wc * v : v; };      // a scaled sum term
            auto sl = [&](double v) { return WEIGHTED ? v + lwc : v; };     // a shifted log term
            const float* z = base + (long long)c * a.cs;
            if (LOSS == HMCX_LOSS_MULTICLASS) {
                double mx = -INFINITY;
                for (int o = 0; o < O; ++o) mx = fmax(mx, (double)z[o]);
                double se = 0.0;
                for (int o = 0; o < O; ++o) se += exp((double)z[o] - mx);
                const double ls = log(se);
                if (o0 == 0) {
                    double h = 0.0;
                    for (int o = 0; o < O; ++o) {
                        const float v = z[o];
                        bad |= !isfinite(v);
                        const double lp = ((double)v - mx) - ls;
                        h -= xlogx(exp(lp), lp);
                    }
                    H += sc(h);
                    lse_add(m, s, sl(((double)z[(int)yi[0]] - mx) - ls));
                }
#pragma unroll
                for (int j = 0; j < OC; ++j)
                    if (o0 + j < O) P[j] += sc(exp(((double)z[o0 + j] - mx) - ls));
            } else if (LOSS == HMCX_LOSS_BINARY) {
#pragma unroll
                for (int j = 0; j < OC; ++j) {
                    if (o0 + j >= O) continue;
                    const float zv = z[o0 + j];
                    bad |= !isfinite(zv);
                    const double v = (double)zv, yv = (double)yi[o0 + j];
                    const double l1p = log1p(exp(-fabs(v)));
                    const double ls1 = -(fmax(-v, 0.0) + l1p), ls0 = -(fmax(v, 0.0) + l1p);   // log sigmoid(+-v)
                    const double p = exp(ls1), q = exp(ls0);
                    P[j] += sc(p);
                    H -= sc(xlogx(p, ls1) + xlogx(q, ls0));
                    lse_add(Q[j], R[j], sl(yv * ls1 + (1.0 - yv) * ls0));
                }
            } else {
                const double tau = (double)a.tau[(long long)c * a.tcs + (long long)t * a.tds];
                if (o0 == 0) {
                    double ll = 0.0;
                    for (int o = 0; o < O; ++o) {
                        const float v = z[o];
                        bad |= !isfinite(v);
                        const double d = (double)v - (double)yi[o];
                        ll -= 0.5 * tau * d * d;
                    }
                    lse_add(m, s, sl(ll + 0.5 * O * (log(tau) - LOG_2PI)));
                    alea += sc(1.0 / tau);
                }
                const double sq = sqrt(tau);
#pragma unroll
                for (int j = 0; j < OC; ++j) {
                    if (o0 + j >= O) continue;
                    const double v = (double)z[o0 + j], e = v - (double)a.f[(long long)i * O + o0 + j];
                    P[j] += sc(e);
                    Q[j] += sc(e * e);
                    R[j] += sc(normcdf(((double)yi[o0 + j] - v) * sq));
                }
            }
        }
#pragma unroll
        for (int j = 0; j < OC; ++j) {
            if (o0 + j >= O) continue;
            W(o0 + j, P[j]);
            if (LOSS != HMCX_LOSS_MULTICLASS) { W(O + o0 + j, Q[j]); W(2 * O + o0 + j, R[j]); }
        }
    }
    if (LOSS == HMCX_LOSS_MULTICLASS) { W(O, m); W(O + 1, s); W(O + 2, H); W(O + 3, bad ? 1.0 : 0.0); }
    else if (LOSS == HMCX_LOSS_BINARY) { W(3 * O, H); W(3 * O + 1, bad ? 1.0 : 0.0); }
    else { W(3 * O, m); W(3 * O + 1, s); W(3 * O + 2, alea); W(3 * O + 3, bad ? 1.0 : 0.0); }
}

// LOSS: HMCX_LOSS_REGRESSION, HMCX_LOSS_BINARY or HMCX_LOSS_MULTICLASS (both multi-class losses)
template <int LOSS>
__global__ void __launch_bounds__(PRED_GROUP) pred_scan_kernel(const PredArgs a) {
    extern __shared__ double sacc[];
    const int i = (a.i0 / PRED_GROUP + (int)blockIdx.x) * PRED_GROUP + (int)threadIdx.x;
    if (i < a.i0 || i >= a.i0 + a.k) return;
    const int O = a.O, n = a.n, C = a.C, N = a.N, k = a.k, li = i - a.i0;
    double* acc = sacc + threadIdx.x;                         // acc[(r * O + o) * PRED_GROUP]: running sums r of output o
    auto A = [&](int r, int o) -> double& { return acc[(size_t)(r * O + o) * PRED_GROUP]; };
    constexpr int NR = LOSS == HMCX_LOSS_REGRESSION ? 4 : LOSS == HMCX_LOSS_BINARY ? 3 : 1;
    for (int r = 0; r < NR; ++r)
        for (int o = 0; o < O; ++o) A(r, o) = (LOSS == HMCX_LOSS_BINARY && r == 1) ? -INFINITY : 0.0;
    if (LOSS == HMCX_LOSS_REGRESSION)
        for (int o = 0; o < O; ++o) A(0, o) = (double)a.f[(long long)i * O + o];   // shift of the moment sums
    const float* yi = a.y + (long long)i * (LOSS == HMCX_LOSS_MULTICLASS ? 1 : O);
    const int label = LOSS == HMCX_LOSS_MULTICLASS ? (int)yi[0] : 0;
    double m = -INFINITY, s = 0.0;                            // running logsumexp of the draws' log p(y_i)
    double H = 0.0;                                           // classification: sum of the draws' entropies
    double alea = 0.0;                                        // regression: sum of 1 / tau
    bool bad = false;
    const double nan = __longlong_as_double(0x7ff8000000000000LL);
    const int RR = pred_rec_rows(LOSS, O);
    for (int t = 0; t < n; ++t) {
        const double* rec = a.rec + (long long)t * RR * k + li;
        auto Rd = [&](int r) { return rec[(long long)r * k]; };
        if (LOSS == HMCX_LOSS_MULTICLASS) {
            for (int o = 0; o < O; ++o) A(0, o) += Rd(o);
            lse_merge(m, s, Rd(O), Rd(O + 1));
            H += Rd(O + 2);
            bad |= Rd(O + 3) != 0.0;
        } else if (LOSS == HMCX_LOSS_BINARY) {
            for (int o = 0; o < O; ++o) {
                A(0, o) += Rd(o);
                lse_merge(A(1, o), A(2, o), Rd(O + o), Rd(2 * O + o));
            }
            H += Rd(3 * O);
            bad |= Rd(3 * O + 1) != 0.0;
        } else {
            for (int o = 0; o < O; ++o) {
                A(1, o) += Rd(o);
                A(2, o) += Rd(O + o);
                A(3, o) += Rd(2 * O + o);
            }
            lse_merge(m, s, Rd(3 * O), Rd(3 * O + 1));
            alea += Rd(3 * O + 2);
            bad |= Rd(3 * O + 3) != 0.0;
        }
        // curve terms of the first t + 1 draws of every chain
        const double St = (double)C * (double)(t + 1), lSt = log(St);
        double r0 = 0.0, r1 = 0.0;
        if (LOSS == HMCX_LOSS_MULTICLASS) {
            int am = 0;
            for (int o = 1; o < O; ++o) if (A(0, o) > A(0, am)) am = o;
            r0 = am == label ? 1.0 : 0.0;
            r1 = -((m + log(s)) - lSt);
        } else if (LOSS == HMCX_LOSS_BINARY) {
            for (int o = 0; o < O; ++o) {
                r0 += ((A(0, o) / St > 0.5) == ((double)yi[o] > 0.5)) ? 1.0 : 0.0;
                r1 -= (A(1, o) + log(A(2, o))) - lSt;
            }
        } else {
            for (int o = 0; o < O; ++o) {
                const double d = (A(0, o) + A(1, o) / St) - (double)yi[o];
                r0 += d * d;
            }
            r1 = -((m + log(s)) - lSt);
        }
        a.terms[(long long)t * k + li] = bad ? nan : r0;
        a.terms[(long long)(n + t) * k + li] = bad ? nan : r1;
    }
    // per-point outputs over all S draws, and the point's terms of the totals
    const double S = (double)C * (double)n, lS = log(S);
    double out[7] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    double tot[PRED_TOTAL_ROWS];
    for (int r = 0; r < PRED_TOTAL_ROWS; ++r) tot[r] = 0.0;
    const long long NO = (long long)N * O;
    const double cover[4] = {0.5, 0.8, 0.9, 0.95};       // central PIT levels of the coverage totals
    if (LOSS == HMCX_LOSS_REGRESSION) {
        double se = 0.0;
        for (int o = 0; o < O; ++o) {
            const double mu1 = A(1, o) / S, epi = fmax(A(2, o) / S - mu1 * mu1, 0.0), mu = A(0, o) + mu1;
            const double u = A(3, o) / S, d = mu - (double)yi[o];
            se += d * d;
            const long long e = (long long)i * O + o;
            a.po[e] = bad ? nan : mu;
            a.po[NO + e] = bad ? nan : alea / S + epi;
            a.po[2 * NO + e] = bad ? nan : epi;
            a.po[3 * NO + e] = bad ? nan : u;
            for (int j = 0; j < 4; ++j) tot[j] += fabs(u - 0.5) <= 0.5 * cover[j] ? 1.0 : 0.0;
        }
        out[0] = -((m + log(s)) - lS);
        out[1] = se;
    } else {
        double nll = 0.0, brier = 0.0, Hp = 0.0, correct = 0.0;
        int am = 0;
        for (int o = 0; o < O; ++o) {
            const double p = A(0, o) / S;
            a.po[(long long)i * O + o] = bad ? nan : p;
            if (LOSS == HMCX_LOSS_MULTICLASS) {
                const double d = p - (o == label ? 1.0 : 0.0);
                brier += d * d;
                Hp -= xlogx(p, log(p));
                if (A(0, o) > A(0, am)) am = o;
            } else {
                const double yv = (double)yi[o], d = p - yv, q = 1.0 - p;
                brier += d * d;
                Hp -= xlogx(p, log(p)) + xlogx(q, log(q));
                nll -= (A(1, o) + log(A(2, o))) - lS;
                const bool ok = (p > 0.5) == (yv > 0.5);
                correct += ok ? 1.0 : 0.0;
                const double conf = fmax(p, q);
                const int b = conf_bin(conf);
                tot[1 + 3 * b] += 1.0;
                tot[2 + 3 * b] += conf;
                tot[3 + 3 * b] += ok ? 1.0 : 0.0;
            }
        }
        if (LOSS == HMCX_LOSS_MULTICLASS) {
            nll = -((m + log(s)) - lS);
            correct = am == label ? 1.0 : 0.0;
            const double conf = A(0, am) / S;
            const int b = conf_bin(conf);
            tot[1 + 3 * b] = 1.0;
            tot[2 + 3 * b] = conf;
            tot[3 + 3 * b] = correct;
            out[6] = (double)am;
        }
        tot[0] = brier;
        out[0] = nll; out[1] = brier; out[2] = Hp; out[3] = H / S; out[4] = Hp - H / S; out[5] = correct;
    }
    for (int r = 0; r < 7; ++r) a.pw[(long long)r * N + i] = bad ? nan : out[r];
    for (int r = 0; r < PRED_TOTAL_ROWS; ++r) a.terms[(long long)(2 * n + r) * k + li] = bad ? nan : tot[r];
    a.nonfinite[i] = bad ? 1 : 0;
}

// partials[row, g] += the slab's terms of group g, in point order (a group's first point starts its sum)
__global__ void __launch_bounds__(256) pred_group_kernel(const double* __restrict__ terms, int rows, int i0, int k, int G,
                                                         double* __restrict__ partials) {
    const int g0 = i0 / PRED_GROUP, ng = (i0 + k - 1) / PRED_GROUP - g0 + 1;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)rows * ng) return;
    const int row = (int)(idx / ng), g = g0 + (int)(idx % ng);
    const int p0 = max(i0, g * PRED_GROUP), p1 = min(i0 + k, (g + 1) * PRED_GROUP);
    const double* x = terms + (long long)row * k - i0;
    double* part = partials + (long long)row * G + g;
    double acc = p0 == g * PRED_GROUP ? x[p0] : *part + x[p0];
    for (int p = p0 + 1; p < p1; ++p) acc += x[p];
    *part = acc;
}

__global__ void __launch_bounds__(256) pred_totals_kernel(const double* __restrict__ partials, int rows, int G,
                                                          double* __restrict__ totals) {
    const int row = blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= rows) return;
    const double* p = partials + (long long)row * G;
    double acc = p[0];
    for (int g = 1; g < G; ++g) acc += p[g];
    totals[row] = acc;
}

int pred_sums(int loss) { return loss == HMCX_LOSS_REGRESSION ? 4 : loss == HMCX_LOSS_BINARY ? 3 : 1; }

}  // namespace

// loss: one of the three pass forms (HMCX_LOSS_MULTICLASS for both multi-class losses)
size_t pred_workspace_bytes(int n, int O, int loss, int k) {
    return ((size_t)n * pred_rec_rows(loss, O) + 2 * (size_t)n + PRED_TOTAL_ROWS) * (size_t)k * sizeof(double);
}

size_t pred_scan_smem(int loss, int O) { return (size_t)pred_sums(loss) * O * PRED_GROUP * sizeof(double); }

int pred_pass(const float* f, long long cs, long long ds, int C, int n, int O, int loss, const float* y, const float* tau,
              long long tcs, long long tds, int N, int i0, int k, double* pointwise, double* per_output, int* nonfinite,
              double* partials, void* ws, cudaStream_t st, const double* cw) {
    const size_t nterms = (2 * (size_t)n + PRED_TOTAL_ROWS) * (size_t)k;
    PredArgs a = {f, cs, ds, C, n, O, N, i0, k, y, tau, tcs, tds, pointwise, per_output, nonfinite, (double*)ws,
                  (double*)ws + nterms, cw};
    const size_t smem = pred_scan_smem(loss, O);
    if (smem > 227 * 1024) return HMCX_ERR_UNSUPPORTED;
    void (*kern)(PredArgs) = loss == HMCX_LOSS_REGRESSION ? pred_scan_kernel<HMCX_LOSS_REGRESSION>
                           : loss == HMCX_LOSS_BINARY ? pred_scan_kernel<HMCX_LOSS_BINARY>
                                                      : pred_scan_kernel<HMCX_LOSS_MULTICLASS>;
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
        cudaGetLastError();
        return HMCX_ERR_UNSUPPORTED;
    }
    const long long steps = (long long)n * k;
    const unsigned sb = (unsigned)((steps + 255) / 256);
    if (cw) {
        if (loss == HMCX_LOSS_REGRESSION) pred_step_kernel<HMCX_LOSS_REGRESSION, true><<<sb, 256, 0, st>>>(a);
        else if (loss == HMCX_LOSS_BINARY) pred_step_kernel<HMCX_LOSS_BINARY, true><<<sb, 256, 0, st>>>(a);
        else pred_step_kernel<HMCX_LOSS_MULTICLASS, true><<<sb, 256, 0, st>>>(a);
    } else if (loss == HMCX_LOSS_REGRESSION) pred_step_kernel<HMCX_LOSS_REGRESSION><<<(unsigned)((steps + 255) / 256), 256, 0, st>>>(a);
    else if (loss == HMCX_LOSS_BINARY) pred_step_kernel<HMCX_LOSS_BINARY><<<(unsigned)((steps + 255) / 256), 256, 0, st>>>(a);
    else pred_step_kernel<HMCX_LOSS_MULTICLASS><<<(unsigned)((steps + 255) / 256), 256, 0, st>>>(a);
    const int g0 = i0 / PRED_GROUP, ng = (i0 + k - 1) / PRED_GROUP - g0 + 1;
    kern<<<ng, PRED_GROUP, smem, st>>>(a);
    const int rows = 2 * n + PRED_TOTAL_ROWS, G = (N + PRED_GROUP - 1) / PRED_GROUP;
    const long long threads = (long long)rows * ng;
    pred_group_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(a.terms, rows, i0, k, G, partials);
    return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA;
}

int pred_totals(const double* partials, int n, int N, double* totals, cudaStream_t st) {
    const int rows = 2 * n + PRED_TOTAL_ROWS, G = (N + PRED_GROUP - 1) / PRED_GROUP;
    pred_totals_kernel<<<(rows + 255) / 256, 256, 0, st>>>(partials, rows, G, totals);
    return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA;
}

}  // namespace hmcx
