// hmcx_stack.cu -- stacking weights (Yao, Vehtari, Simpson & Gelman 2018; Yao, Vehtari & Gelman 2022): the simplex
// weights w of K rows of pointwise log predictive densities E[k, i] (models, or the chains of one run) that maximise the
// log score f(w) = sum_i log sum_k w_k exp(E_ki).  hamiltorch_b200/loo.py drives it; tests/stacking_oracle.py is the
// numpy definition.
//
// One evaluation of f and of its gradient g_k = sum_i exp(E_ki) / sum_j w_j exp(E_ji):
//   stack_point_kernel  one thread per point: m_i = max_k E_ki, s_i = sum_k w_k exp(E_ki - m_i) over the rows in order
//                       (rows with w_k = 0 add nothing), pointwise_i = m_i + log s_i, and the gradient terms
//                       exp(E_ki - m_i) / s_i to the workspace;
//   stack_sum_kernel    one CTA per row (0: f, 1 + k: g_k): the 128-point groups summed in point order, then the group
//                       partials in group order, as pred_group_kernel / pred_totals_kernel do.
// No atomics: the same E and w give the same bits on every call.
// The solver is the multiplicative (EM) update w_k <- w_k g_k / N from uniform w (stack_em_kernel, one CTA): since
// sum_k w_k g_k = N it stays on the simplex, f never decreases, and it needs no step size.  It stops once
// max_k g_k <= N (1 + tol); by concavity f(w*) - f(w) <= max_k g_k - sum_k w_k g_k = max_k g_k - N <= N tol.
#include <cfloat>
#include "hmcx_common.cuh"

namespace hmcx {
namespace {

constexpr int SG = 128;                   // points per fixed-order group
constexpr int ST = 256;                   // threads of the sum and EM CTAs

__global__ void __launch_bounds__(SG) stack_point_kernel(const double* __restrict__ E, int K, int N,
                                                         const double* __restrict__ w, double* __restrict__ pointwise,
                                                         double* __restrict__ terms, const int* __restrict__ state) {
    if (state && state[0]) return;
    const int i = blockIdx.x * SG + threadIdx.x;
    if (i >= N) return;
    double m = -DBL_MAX;
    for (int k = 0; k < K; ++k) m = fmax(m, E[(long long)k * N + i]);
    double s = 0.0;
    for (int k = 0; k < K; ++k) {
        const double wk = w[k];
        if (wk != 0.0) s += wk * exp(E[(long long)k * N + i] - m);
    }
    pointwise[i] = m + log(s);
    for (int k = 0; k < K; ++k) terms[(long long)k * N + i] = exp(E[(long long)k * N + i] - m) / s;
}

// row 0: objective = sum_i pointwise_i; row 1 + k: grad[k] = sum_i terms[k, i].  partials: G doubles per row.
__global__ void __launch_bounds__(ST) stack_sum_kernel(const double* __restrict__ pointwise,
                                                       const double* __restrict__ terms, int N,
                                                       double* __restrict__ partials, double* __restrict__ objective,
                                                       double* __restrict__ grad, const int* __restrict__ state) {
    if (state && state[0]) return;
    const int row = blockIdx.x, G = (N + SG - 1) / SG;
    const double* x = row == 0 ? pointwise : terms + (long long)(row - 1) * N;
    double* part = partials + (long long)row * G;
    for (int g = threadIdx.x; g < G; g += ST) {
        const int p0 = g * SG, p1 = min(N, p0 + SG);
        double acc = x[p0];
        for (int p = p0 + 1; p < p1; ++p) acc += x[p];
        part[g] = acc;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double acc = part[0];
        for (int g = 1; g < G; ++g) acc += part[g];
        if (row == 0) *objective = acc;
        else grad[row - 1] = acc;
    }
}

// state[0]: converged flag, state[1]: EM updates applied.  Skips once converged; otherwise checks the stopping rule on
// the gradient of the current w and, when it fails, applies one update.
__global__ void __launch_bounds__(ST) stack_em_kernel(int K, int N, double tol, double* __restrict__ w,
                                                      const double* __restrict__ grad, int* __restrict__ state) {
    __shared__ double sm[ST / 32];
    __shared__ int stop;
    if (state[0]) return;
    double mx = -DBL_MAX;
    for (int k = threadIdx.x; k < K; k += ST) mx = fmax(mx, grad[k]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = mx;
    __syncthreads();
    if (threadIdx.x == 0) {
        double g = sm[0];
        for (int j = 1; j < ST / 32; ++j) g = fmax(g, sm[j]);
        stop = g <= (double)N * (1.0 + tol);
        if (stop) state[0] = 1;
        else state[1] += 1;
    }
    __syncthreads();
    if (stop) return;
    for (int k = threadIdx.x; k < K; k += ST) w[k] = w[k] * grad[k] / (double)N;
}

}  // namespace

size_t stack_workspace_bytes(int K, int N) {
    const size_t G = ((size_t)N + SG - 1) / SG;
    return ((size_t)K * N + (size_t)(K + 1) * G) * sizeof(double);
}

static int stack_eval_launch(const double* E, int K, int N, const double* w, double* objective, double* grad,
                             double* pointwise, void* ws, const int* state, cudaStream_t st) {
    double* terms = (double*)ws;
    double* partials = terms + (size_t)K * N;
    stack_point_kernel<<<(N + SG - 1) / SG, SG, 0, st>>>(E, K, N, w, pointwise, terms, state);
    stack_sum_kernel<<<K + 1, ST, 0, st>>>(pointwise, terms, N, partials, objective, grad, state);
    return HMCX_OK;
}

int stack_eval(const double* E, int K, int N, const double* w, double* objective, double* grad, double* pointwise,
               void* ws, cudaStream_t st) {
    stack_eval_launch(E, K, N, w, objective, grad, pointwise, ws, nullptr, st);
    return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA;
}

int stack_em(const double* E, int K, int N, double tol, int iters, double* w, double* objective, double* grad,
             double* pointwise, int* state, void* ws, cudaStream_t st) {
    for (int it = 0; it < iters; ++it) {
        stack_eval_launch(E, K, N, w, objective, grad, pointwise, ws, state, st);
        stack_em_kernel<<<1, ST, 0, st>>>(K, N, tol, w, grad, state);
    }
    return cudaGetLastError() == cudaSuccess ? HMCX_OK : HMCX_ERR_CUDA;
}

}  // namespace hmcx
