// hmcx_api.cu -- the extern "C" surface declared in include/hmcx.h; validates and dispatches on target kind.
#include <cfloat>
#include <cstdlib>
#include "hmcx_common.cuh"

namespace hmcx {
int elem_leapfrog(const hmcx_target_t*, const hmcx_mass_t*, const float*, const float*, const float*, int, int, int,
                  float*, float*, float*, float*, cudaStream_t);
int elem_hamiltonian(const hmcx_target_t*, const hmcx_mass_t*, const float*, const float*, int, int, float*,
                     uint8_t*, cudaStream_t);
int elem_gibbs(const hmcx_mass_t*, const hmcx_rng_t*, int, int, int, int64_t, float*, cudaStream_t);
int elem_hmc_run(const hmcx_target_t*, const hmcx_mass_t*, const hmcx_rng_t*, const hmcx_nuts_t*, const float*,
                 float*, float*, int, int, int, int, int, int, int, float*, uint8_t*, uint8_t*, float*, int32_t*,
                 int, float*, const hmcx_sink_t*, cudaStream_t);
int coupled_leapfrog(const hmcx_target_t*, const hmcx_mass_t*, const float*, const float*, const float*, int, int, int,
                     float*, float*, float*, float*, cudaStream_t);
int coupled_hamiltonian(const hmcx_target_t*, const hmcx_mass_t*, const float*, const float*, int, int, float*, uint8_t*,
                        cudaStream_t);
size_t dense_rmhmc_workspace_floats(int, int);
int dense_rmhmc_run(const hmcx_target_t*, const hmcx_rmhmc_t*, const hmcx_const_metric_t*, const hmcx_rng_t*,
                    const float*, float*, const float*, int, int, int, int, int, int, int, float*, uint8_t*, uint8_t*,
                    float*, int32_t*, float*, cudaStream_t);
int mlp_split_run(const hmcx_target_t*, const hmcx_mass_t*, const hmcx_rng_t*, const hmcx_nuts_t*, int, const float*,
                  float*, float*, int, int, int, int, int, int, int, float*, uint8_t*, uint8_t*, float*, int32_t*,
                  cudaStream_t, const float*, float*, float*, const hmcx_sink_t*, const hmcx_hyper_t*,
                  const hmcx_temper_t*, int);
int temper_swap(float*, int, int, int, const double*, const double*, int, const hmcx_rng_t*, const double*, int8_t*,
                cudaStream_t);
int hyper_gamma_draws(uint64_t, uint64_t, int, int, int, int, const double*, double*, cudaStream_t);
int mlp_leapfrog(const hmcx_target_t*, const hmcx_mass_t*, const hmcx_rng_t*, int, double, const float*, const float*, float*,
                 int, int, int, float*, float*, cudaStream_t);
int mlp_grad_log_prob(const hmcx_target_t*, const float*, int, int, int, float*, float*, cudaStream_t);
int mlp_predict(const hmcx_target_t*, const float*, int, int, float*, float*, cudaStream_t);
int small_hmc_run(const hmcx_target_t*, const hmcx_mass_t*, const hmcx_rng_t*, const hmcx_nuts_t*, const float*, float*,
                  float*, int, int, int, int, int, int, int, float*, uint8_t*, uint8_t*, float*, int32_t*,
                  cudaStream_t);
int gemm_nt_tf32x3(const float*, const float*, float*, int, int, int, cudaStream_t);
size_t dense_workspace_floats(int, int, int);
int dense_hmc_run(const hmcx_target_t*, const hmcx_mass_t*, const hmcx_rng_t*, const hmcx_nuts_t*, const float*, float*,
                  float*, int, int, int, int, int, int, int, float*, uint8_t*, uint8_t*, float*, int32_t*, float*,
                  cudaStream_t);
int rmhmc_run(const hmcx_target_t*, const hmcx_rmhmc_t*, const hmcx_rng_t*, const float*, float*, const float*, int,
              int, int, int, int, int, int, float*, uint8_t*, uint8_t*, float*, int32_t*, cudaStream_t);
size_t mlp_packed_x_floats(const hmcx_target_t*);
int mlp_pack_x(const hmcx_target_t*, float*, cudaStream_t);
int rmhmc_cta_run(const hmcx_target_t*, const hmcx_rmhmc_t*, const hmcx_rng_t*, const float*, float*, const float*, int,
                  int, int, int, int, int, int, float*, uint8_t*, uint8_t*, float*, int32_t*, const float*, float*, float*,
                  float*, float*, int, float*, cudaStream_t);
int diag_means(const float*, long long, long long, int, int, int, double*, double*, cudaStream_t);
int diag_acov(const float*, long long, long long, int, int, int, const double*, const double*, int, double*, double*,
              cudaStream_t);
size_t rank_workspace_bytes(int, int, int);
int rank_pass(const float*, long long, long long, int, int, int, int, int, float*, long long, long long, float*,
              long long, long long, double*, int*, void*, cudaStream_t);
int rank_indicator(const float*, long long, long long, int, int, int, const double*, float*, long long, long long,
                   cudaStream_t);
int adapt_diag_mass(float*, float*, float*, float*, int, int, int, int, const float*, int, float*, float*, double*, double*,
                    double*, cudaStream_t);
int mlp_pointwise_ll(const hmcx_target_t*, const float*, long long, long long, int, int, int, int, float*, long long,
                     long long, cudaStream_t, const float*, long long, long long);
size_t loo_workspace_bytes(int, int, int);
int loo_pass(const float*, long long, long long, int, int, int, int, int, double, double*, int*, int*, void*,
             cudaStream_t);
int mlp_pointwise_out(const hmcx_target_t*, const float*, long long, long long, int, int, int, int, float*, long long,
                      long long, cudaStream_t);
size_t pred_workspace_bytes(int, int, int, int);
size_t pred_scan_smem(int, int);
int pred_pass(const float*, long long, long long, int, int, int, int, const float*, const float*, long long, long long,
              int, int, int, double*, double*, int*, double*, void*, cudaStream_t, const double*);
int pred_totals(const double*, int, int, double*, cudaStream_t);
int sbc_prior(const hmcx_target_t*, uint64_t, long long, int, int, int, float*, cudaStream_t);
int sbc_simulate(const hmcx_target_t*, const float*, uint64_t, long long, int, float*, cudaStream_t);
int sbc_rank(const float*, long long, long long, int, int, int, int, const float*, long long, int*, cudaStream_t);
int ppc_pass(const hmcx_target_t*, const float*, int, const long long*, uint64_t, const float*, float*, double*, double*,
             int*, cudaStream_t);
int loo_pit_pass(const float*, long long, long long, const float*, long long, long long, int, int, int, int, int, double,
                 const float*, const float*, long long, long long, double*, double*, int*, void*, cudaStream_t);
int loo_chain_pass(const float*, long long, long long, int, int, int, int, int, double, double*, int*, int*,
                   cudaStream_t);
size_t stack_workspace_bytes(int, int);
int stack_eval(const double*, int, int, const double*, double*, double*, double*, void*, cudaStream_t);
int stack_em(const double*, int, int, double, int, double*, double*, double*, double*, int*, void*, cudaStream_t);
int mlp_log_prior(const float*, long long, long long, int, int, int, const int*, const double*, double*, cudaStream_t);
int psens_ll_totals(const float*, long long, long long, int, int, int, int, const double*, double*, cudaStream_t);
size_t psens_workspace_bytes(int, int, int);
int psens_weights(const float*, long long, long long, int, int, int, double, double*, double*, int*, int*, void*,
                  cudaStream_t);
int psens_pass(const float*, long long, long long, int, int, int, int, int, const double*, double*, int*, void*,
               cudaStream_t);
}  // namespace hmcx

static inline bool has_mu_chain(const hmcx_nuts_t* nuts) { return nuts && nuts->enabled && nuts->mu_chain; }

static inline bool is_elem(const hmcx_target_t* t) {
    return t && (t->kind == HMCX_TARGET_GAUSS_ISO || t->kind == HMCX_TARGET_GAUSS_DIAG);
}

extern "C" {

int hmcx_abi_version(void) { return HMCX_ABI_VERSION; }

size_t hmcx_hmc_workspace_bytes(const hmcx_target_t* target, const hmcx_mass_t* mass, int32_t C, int32_t ld) {
    const bool full_mass = mass && mass->kind == HMCX_MASS_FULL;
    if (is_elem(target) && !full_mass && ld > 4096) return (size_t)C * (size_t)ld * sizeof(float);
    if (is_elem(target) && !full_mass) return (size_t)C * sizeof(float);      // log p(q_cur) carried between windows of iterations
    if (target && target->dim > 16 &&
        (target->kind == HMCX_TARGET_GAUSS_FULL || (full_mass && is_elem(target))))
        return hmcx::dense_workspace_floats(C, target->dim, full_mass ? 1 : 0) * sizeof(float);
    return 0;
}

const char* hmcx_status_string(int status) {
    switch (status) {
        case HMCX_OK: return "ok";
        case HMCX_ERR_INVALID_ARG: return "invalid argument";
        case HMCX_ERR_UNSUPPORTED: return "unsupported target / mass / dimension combination";
        case HMCX_ERR_CUDA: return "CUDA launch error";
        default: return "unknown status";
    }
}

int hmcx_leapfrog(const hmcx_target_t* target, const hmcx_mass_t* mass, const float* q_in, const float* p_in,
                  const float* eps, int32_t C, int32_t ld, int32_t L, float* q_out, float* p_out, float* q_traj,
                  float* p_traj, void* stream) {
    if (!target) return HMCX_ERR_INVALID_ARG;
    if (is_elem(target) && !(mass && mass->kind == HMCX_MASS_FULL))
        return hmcx::elem_leapfrog(target, mass, q_in, p_in, eps, C, ld, L, q_out, p_out, q_traj, p_traj,
                                   (cudaStream_t)stream);
    // coupled gradient (GAUSS_FULL, FUNNEL) or full mass matrix: one CTA per chain, any D (hmcx_coupled.cu)
    return hmcx::coupled_leapfrog(target, mass, q_in, p_in, eps, C, ld, L, q_out, p_out, q_traj, p_traj,
                                  (cudaStream_t)stream);
}

int hmcx_hamiltonian(const hmcx_target_t* target, const hmcx_mass_t* mass, const float* q, const float* p,
                     int32_t C, int32_t ld, float* H_out, uint8_t* flags_out, void* stream) {
    if (!target) return HMCX_ERR_INVALID_ARG;
    if (is_elem(target) && !(mass && mass->kind == HMCX_MASS_FULL))
        return hmcx::elem_hamiltonian(target, mass, q, p, C, ld, H_out, flags_out, (cudaStream_t)stream);
    return hmcx::coupled_hamiltonian(target, mass, q, p, C, ld, H_out, flags_out, (cudaStream_t)stream);
}

int hmcx_gibbs(const hmcx_mass_t* mass, const hmcx_rng_t* rng, int32_t D, int32_t C, int32_t ld, int64_t iter,
               float* p_out, void* stream) {
    return hmcx::elem_gibbs(mass, rng, D, C, ld, iter, p_out, (cudaStream_t)stream);
}

int hmcx_hmc_run(const hmcx_target_t* target, const hmcx_mass_t* mass, const hmcx_rng_t* rng,
                 const hmcx_nuts_t* nuts, const float* q_init, float* q_cur, float* eps, int32_t C, int32_t ld,
                 int32_t L, int32_t num_samples, int32_t burn, int32_t iter_begin, int32_t iter_end,
                 float* samples_out, uint8_t* accept_out, uint8_t* diverged_out, float* ham_out,
                 int32_t* num_rejected, int32_t tuning, float* workspace, void* stream) {
    if (has_mu_chain(nuts)) return HMCX_ERR_UNSUPPORTED;            // per-chain mu: the sink forms only
    return hmcx_hmc_run_sink(target, mass, rng, nuts, q_init, q_cur, eps, C, ld, L, num_samples, burn, iter_begin,
                             iter_end, samples_out, accept_out, diverged_out, ham_out, num_rejected, tuning, workspace,
                             nullptr, stream);
}

int hmcx_hmc_run_sink(const hmcx_target_t* target, const hmcx_mass_t* mass, const hmcx_rng_t* rng,
                      const hmcx_nuts_t* nuts, const float* q_init, float* q_cur, float* eps, int32_t C, int32_t ld,
                      int32_t L, int32_t num_samples, int32_t burn, int32_t iter_begin, int32_t iter_end,
                      float* samples_out, uint8_t* accept_out, uint8_t* diverged_out, float* ham_out,
                      int32_t* num_rejected, int32_t tuning, float* workspace, const hmcx_sink_t* sink, void* stream) {
    if (!target) return HMCX_ERR_INVALID_ARG;
    if (sink && sink->thin < 1) return HMCX_ERR_INVALID_ARG;
    if (sink && sink->thin == 1 && !sink->sum && !sink->sumsq && !has_mu_chain(nuts)) sink = nullptr;
    if (!sink && has_mu_chain(nuts)) return HMCX_ERR_UNSUPPORTED;
    const bool full_mass = mass && mass->kind == HMCX_MASS_FULL;
    if (is_elem(target) && !full_mass)
        return hmcx::elem_hmc_run(target, mass, rng, nuts, q_init, q_cur, eps, C, ld, L, num_samples, burn,
                                  iter_begin, iter_end, samples_out, accept_out, diverged_out, ham_out,
                                  num_rejected, tuning, workspace, sink, (cudaStream_t)stream);
    if (sink) return HMCX_ERR_UNSUPPORTED;
    if (target->dim > 16 && (target->kind == HMCX_TARGET_GAUSS_FULL || (full_mass && is_elem(target))))
        // dense target and / or full mass matrix at scale: tensor-core GEMMs over all chains per leapfrog step (hmcx_tc.cu)
        return hmcx::dense_hmc_run(target, mass, rng, nuts, q_init, q_cur, eps, C, ld, L, num_samples, burn,
                                   iter_begin, iter_end, samples_out, accept_out, diverged_out, ham_out,
                                   num_rejected, workspace, (cudaStream_t)stream);
    if (is_elem(target) || target->kind == HMCX_TARGET_GAUSS_FULL || target->kind == HMCX_TARGET_FUNNEL)
        // coupled gradient or full mass matrix: thread-per-chain kernel, D <= 16 (samplers.py:293-294, :811-812, :198-199)
        return hmcx::small_hmc_run(target, mass, rng, nuts, q_init, q_cur, eps, C, ld, L, num_samples, burn,
                                   iter_begin, iter_end, samples_out, accept_out, diverged_out, ham_out,
                                   num_rejected, (cudaStream_t)stream);
    if (target->kind == HMCX_TARGET_MLP)      // un-split Bayesian NN == sample_model (samplers.py:1261)
        return hmcx::mlp_split_run(target, mass, rng, nuts, HMCX_SCHEME_PLAIN, q_init, q_cur, eps, C, ld, L,
                                   num_samples, burn, iter_begin, iter_end, samples_out, accept_out, diverged_out,
                                   ham_out, num_rejected, (cudaStream_t)stream, nullptr, nullptr, nullptr, nullptr, nullptr,
                                   nullptr, 0);
    return HMCX_ERR_UNSUPPORTED;
}

int hmcx_split_run(const hmcx_target_t* target, const hmcx_mass_t* mass, const hmcx_rng_t* rng,
                   const hmcx_nuts_t* nuts, int32_t scheme, const float* q_init, float* q_cur, float* eps, int32_t C,
                   int32_t ld, int32_t L, int32_t num_samples, int32_t burn, int32_t iter_begin, int32_t iter_end,
                   float* samples_out, uint8_t* accept_out, uint8_t* diverged_out, float* ham_out,
                   int32_t* num_rejected, void* stream) {
    if (has_mu_chain(nuts)) return HMCX_ERR_UNSUPPORTED;            // per-chain mu: the sink form only
    return hmcx_split_run_sink(target, mass, rng, nuts, scheme, q_init, q_cur, eps, C, ld, L, num_samples, burn,
                               iter_begin, iter_end, samples_out, accept_out, diverged_out, ham_out, num_rejected,
                               nullptr, stream);
}

int hmcx_split_run_sink(const hmcx_target_t* target, const hmcx_mass_t* mass, const hmcx_rng_t* rng,
                        const hmcx_nuts_t* nuts, int32_t scheme, const float* q_init, float* q_cur, float* eps,
                        int32_t C, int32_t ld, int32_t L, int32_t num_samples, int32_t burn, int32_t iter_begin,
                        int32_t iter_end, float* samples_out, uint8_t* accept_out, uint8_t* diverged_out,
                        float* ham_out, int32_t* num_rejected, const hmcx_sink_t* sink, void* stream) {
    return hmcx_split_run_hyper(target, mass, rng, nuts, scheme, q_init, q_cur, eps, C, ld, L, num_samples, burn, iter_begin,
                                iter_end, samples_out, accept_out, diverged_out, ham_out, num_rejected, sink, nullptr,
                                stream);
}

int hmcx_split_run_hyper(const hmcx_target_t* target, const hmcx_mass_t* mass, const hmcx_rng_t* rng,
                         const hmcx_nuts_t* nuts, int32_t scheme, const float* q_init, float* q_cur, float* eps,
                         int32_t C, int32_t ld, int32_t L, int32_t num_samples, int32_t burn, int32_t iter_begin,
                         int32_t iter_end, float* samples_out, uint8_t* accept_out, uint8_t* diverged_out,
                         float* ham_out, int32_t* num_rejected, const hmcx_sink_t* sink, const hmcx_hyper_t* hyper,
                         void* stream) {
    if (!target) return HMCX_ERR_INVALID_ARG;
    if (sink && (sink->thin < 1 || (sink->sum_lo && !sink->sum) || (sink->sumsq_lo && !sink->sumsq)))
        return HMCX_ERR_INVALID_ARG;
    if (target->kind != HMCX_TARGET_MLP) return HMCX_ERR_UNSUPPORTED;
    if (!sink && !hyper && has_mu_chain(nuts)) return HMCX_ERR_UNSUPPORTED;
    return hmcx::mlp_split_run(target, mass, rng, nuts, scheme, q_init, q_cur, eps, C, ld, L, num_samples, burn,
                               iter_begin, iter_end, samples_out, accept_out, diverged_out, ham_out, num_rejected,
                               (cudaStream_t)stream, nullptr, nullptr, nullptr, sink, hyper, nullptr, 0);
}

int hmcx_split_run_temper(const hmcx_target_t* target, const hmcx_mass_t* mass, const hmcx_rng_t* rng,
                          const hmcx_nuts_t* nuts, int32_t scheme, const float* q_init, float* q_cur, float* eps,
                          int32_t C, int32_t ld, int32_t L, int32_t num_samples, int32_t burn, int32_t iter_begin,
                          int32_t iter_end, float* samples_out, uint8_t* accept_out, uint8_t* diverged_out,
                          float* ham_out, int32_t* num_rejected, const hmcx_sink_t* sink, const hmcx_temper_t* temper,
                          void* stream) {
    if (!target || !temper) return HMCX_ERR_INVALID_ARG;
    if (sink && (sink->thin < 1 || (sink->sum_lo && !sink->sum) || (sink->sumsq_lo && !sink->sumsq)))
        return HMCX_ERR_INVALID_ARG;
    if (target->kind != HMCX_TARGET_MLP) return HMCX_ERR_UNSUPPORTED;
    return hmcx::mlp_split_run(target, mass, rng, nuts, scheme, q_init, q_cur, eps, C, ld, L, num_samples, burn,
                               iter_begin, iter_end, samples_out, accept_out, diverged_out, ham_out, num_rejected,
                               (cudaStream_t)stream, nullptr, nullptr, nullptr, sink, nullptr, temper, 0);
}

int hmcx_split_run_folds(const hmcx_target_t* target, const hmcx_mass_t* mass, const hmcx_rng_t* rng,
                         const hmcx_nuts_t* nuts, int32_t scheme, const float* q_init, float* q_cur, float* eps,
                         int32_t C, int32_t ld, int32_t L, int32_t num_samples, int32_t burn, int32_t iter_begin,
                         int32_t iter_end, float* samples_out, uint8_t* accept_out, uint8_t* diverged_out,
                         float* ham_out, int32_t* num_rejected, const hmcx_sink_t* sink, int32_t num_folds,
                         void* stream) {
    if (!target || num_folds < 2 || num_folds > HMCX_MLP_MAX_SPLITS) return HMCX_ERR_INVALID_ARG;
    if (sink && (sink->thin < 1 || (sink->sum_lo && !sink->sum) || (sink->sumsq_lo && !sink->sumsq)))
        return HMCX_ERR_INVALID_ARG;
    if (target->kind != HMCX_TARGET_MLP || scheme != HMCX_SCHEME_PLAIN) return HMCX_ERR_UNSUPPORTED;
    if (!sink && has_mu_chain(nuts)) return HMCX_ERR_UNSUPPORTED;
    return hmcx::mlp_split_run(target, mass, rng, nuts, scheme, q_init, q_cur, eps, C, ld, L, num_samples, burn,
                               iter_begin, iter_end, samples_out, accept_out, diverged_out, ham_out, num_rejected,
                               (cudaStream_t)stream, nullptr, nullptr, nullptr, sink, nullptr, nullptr, num_folds);
}

int hmcx_temper_swap(float* q_cur, int32_t C, int32_t ld, int32_t num_temps, const double* betas, const double* ll,
                     int32_t round, const hmcx_rng_t* rng, const double* log_uniforms, int8_t* accepted, void* stream) {
    return hmcx::temper_swap(q_cur, C, ld, num_temps, betas, ll, round, rng, log_uniforms, accepted,
                             (cudaStream_t)stream);
}

int hmcx_hyper_gamma_draws(uint64_t seed, uint64_t chain_offset, int32_t C, int32_t iter_begin, int32_t iter_end,
                           int32_t K, const double* shapes, double* out, void* stream) {
    return hmcx::hyper_gamma_draws(seed, chain_offset, C, iter_begin, iter_end, K, shapes, out, (cudaStream_t)stream);
}

int hmcx_split_leapfrog(const hmcx_target_t* target, const hmcx_mass_t* mass, const hmcx_rng_t* rng, int32_t scheme,
                        double step_size, const float* q_in, const float* p_in, float* eps, int32_t C, int32_t ld, int32_t L,
                        float* q_traj, float* p_traj, void* stream) {
    if (!target || !rng) return HMCX_ERR_INVALID_ARG;
    if (target->kind != HMCX_TARGET_MLP) return HMCX_ERR_UNSUPPORTED;
    return hmcx::mlp_leapfrog(target, mass, rng, scheme, step_size, q_in, p_in, eps, C, ld, L, q_traj, p_traj,
                              (cudaStream_t)stream);
}

int hmcx_rmhmc_run(const hmcx_target_t* target, const hmcx_rmhmc_t* cfg, const hmcx_rng_t* rng, const float* q_init,
                   float* q_cur, const float* eps, int32_t C, int32_t ld, int32_t L, int32_t num_samples,
                   int32_t burn, int32_t iter_begin, int32_t iter_end, float* samples_out, uint8_t* accept_out,
                   uint8_t* diverged_out, float* ham_out, int32_t* num_rejected, void* stream) {
    // metric / eigenvectors in shared memory, one CTA per chain (hmcx_rmhmc_cta.cu); HMCX_RMHMC_FORCE_CTA=1 sends the small
    // problems there too (tests run every golden chain through both kernels)
    const char* force = getenv("HMCX_RMHMC_FORCE_CTA");
    if (target && (target->dim > 16 || (force && force[0] == '1')))
        return hmcx::rmhmc_cta_run(target, cfg, rng, q_init, q_cur, eps, C, ld, L, num_samples, burn, iter_begin, iter_end,
                                   samples_out, accept_out, diverged_out, ham_out, num_rejected, nullptr, nullptr, nullptr,
                                   nullptr, nullptr, 0, nullptr, (cudaStream_t)stream);
    return hmcx::rmhmc_run(target, cfg, rng, q_init, q_cur, eps, C, ld, L, num_samples, burn, iter_begin, iter_end,
                           samples_out, accept_out, diverged_out, ham_out, num_rejected, (cudaStream_t)stream);
}

int hmcx_rmhmc_leapfrog(const hmcx_target_t* target, const hmcx_rmhmc_t* cfg, const hmcx_rng_t* rng, const float* q_in,
                        const float* p_in, const float* eps, int32_t C, int32_t ld, int32_t L, float* q_traj,
                        float* p_traj, float* q_copy_out, float* p_copy_out, uint8_t* flags_out, void* stream) {
    if (!q_in || !p_in || !q_traj || !p_traj) return HMCX_ERR_INVALID_ARG;
    // one "iteration" with the momentum given and no MH
    return hmcx::rmhmc_cta_run(target, cfg, rng, q_in, nullptr, eps, C, ld, L, 1, 0, 0, 1, nullptr, nullptr, flags_out,
                               nullptr, nullptr, p_in, q_traj, p_traj, q_copy_out, p_copy_out, 0, nullptr,
                               (cudaStream_t)stream);
}

int hmcx_rmhmc_hamiltonian(const hmcx_target_t* target, const hmcx_rmhmc_t* cfg, const hmcx_rng_t* rng, const float* q,
                           const float* p, int32_t C, int32_t ld, float* H_out, uint8_t* flags_out, void* stream) {
    if (!q || !p || !H_out) return HMCX_ERR_INVALID_ARG;
    return hmcx::rmhmc_cta_run(target, cfg, rng, q, nullptr, nullptr, C, ld, 1, 1, 0, 0, 1, nullptr, nullptr, flags_out,
                               nullptr, nullptr, p, nullptr, nullptr, nullptr, nullptr, 1, H_out, (cudaStream_t)stream);
}

size_t hmcx_rmhmc_dense_workspace_bytes(int32_t C, int32_t D) {
    return hmcx::dense_rmhmc_workspace_floats(C, D) * sizeof(float);
}

int hmcx_rmhmc_dense_run(const hmcx_target_t* target, const hmcx_rmhmc_t* cfg, const hmcx_const_metric_t* metric,
                         const hmcx_rng_t* rng, const float* q_init, float* q_cur, const float* eps, int32_t C,
                         int32_t ld, int32_t L, int32_t num_samples, int32_t burn, int32_t iter_begin, int32_t iter_end,
                         float* samples_out, uint8_t* accept_out, uint8_t* diverged_out, float* ham_out,
                         int32_t* num_rejected, float* workspace, void* stream) {
    return hmcx::dense_rmhmc_run(target, cfg, metric, rng, q_init, q_cur, eps, C, ld, L, num_samples, burn, iter_begin,
                                 iter_end, samples_out, accept_out, diverged_out, ham_out, num_rejected, workspace,
                                 (cudaStream_t)stream);
}

int hmcx_gemm_nt_tf32x3(const float* A, const float* B, float* D, int32_t M, int32_t N, int32_t K, void* stream) {
    return hmcx::gemm_nt_tf32x3(A, B, D, M, N, K, (cudaStream_t)stream);
}

int hmcx_grad_log_prob(const hmcx_target_t* target, const float* q, int32_t C, int32_t ld, int32_t split,
                       float* grad_out, float* log_prob_out, void* stream) {
    if (!target) return HMCX_ERR_INVALID_ARG;
    if (target->kind == HMCX_TARGET_MLP)
        return hmcx::mlp_grad_log_prob(target, q, C, ld, split, grad_out, log_prob_out, (cudaStream_t)stream);
    return HMCX_ERR_UNSUPPORTED;
}

int hmcx_mlp_predict(const hmcx_target_t* target, const float* samples, int32_t S, int32_t ld, float* pred_out,
                     float* log_prob_out, void* stream) {
    if (!target) return HMCX_ERR_INVALID_ARG;
    if (target->kind != HMCX_TARGET_MLP) return HMCX_ERR_UNSUPPORTED;
    return hmcx::mlp_predict(target, samples, S, ld, pred_out, log_prob_out, (cudaStream_t)stream);
}

size_t hmcx_mlp_packed_x_bytes(const hmcx_target_t* target) {
    if (!target || target->kind != HMCX_TARGET_MLP) return 0;
    return hmcx::mlp_packed_x_floats(target) * sizeof(float);
}

int hmcx_mlp_pack_x(const hmcx_target_t* target, float* packed_out, void* stream) {
    if (!target) return HMCX_ERR_INVALID_ARG;
    if (target->kind != HMCX_TARGET_MLP) return HMCX_ERR_UNSUPPORTED;
    return hmcx::mlp_pack_x(target, packed_out, (cudaStream_t)stream);
}

int hmcx_copy_rows_async(void* dst, size_t dpitch, const void* src, size_t spitch, size_t width, size_t height,
                         void* stream) {
    if (!dst || !src || width > dpitch || width > spitch) return HMCX_ERR_INVALID_ARG;
    if (width == 0 || height == 0) return HMCX_OK;
    return cudaMemcpy2DAsync(dst, dpitch, src, spitch, width, height, cudaMemcpyDefault, (cudaStream_t)stream) == cudaSuccess
               ? HMCX_OK : HMCX_ERR_CUDA;
}

static inline bool diag_args_ok(const float* x, int64_t cs, int64_t ds, int32_t C, int32_t n, int32_t D) {
    return x && cs >= 0 && ds >= 0 && C >= 1 && n >= 4 && D >= 1;
}

int hmcx_diag_means(const float* x, int64_t chain_stride, int64_t draw_stride, int32_t C, int32_t n, int32_t D,
                    double* mu_out, double* mu_sum_out, void* stream) {
    if (!diag_args_ok(x, chain_stride, draw_stride, C, n, D) || !mu_out || !mu_sum_out) return HMCX_ERR_INVALID_ARG;
    return hmcx::diag_means(x, chain_stride, draw_stride, C, n, D, mu_out, mu_sum_out, (cudaStream_t)stream);
}

int hmcx_diag_acov(const float* x, int64_t chain_stride, int64_t draw_stride, int32_t C, int32_t n, int32_t D,
                   const double* mu, const double* mu_bar, int32_t lag_begin, double* acov_out, double* between_out,
                   void* stream) {
    if (!diag_args_ok(x, chain_stride, draw_stride, C, n, D) || !mu || !acov_out || lag_begin < 0 ||
        (mu_bar && !between_out))
        return HMCX_ERR_INVALID_ARG;
    return hmcx::diag_acov(x, chain_stride, draw_stride, C, n, D, mu, mu_bar, lag_begin, acov_out, between_out,
                           (cudaStream_t)stream);
}

static inline bool rank_shape_ok(int32_t C, int32_t n) {
    return C >= 1 && n >= 4 && (int64_t)C * n <= HMCX_RANK_MAX_DRAWS;
}

static inline bool rank_slab_ok(int32_t k) {
    return k >= 1 && k <= HMCX_RANK_MAX_SLAB;
}

size_t hmcx_rank_workspace_bytes(int32_t C, int32_t n, int32_t k) {
    if (!rank_shape_ok(C, n) || !rank_slab_ok(k)) return 0;
    return hmcx::rank_workspace_bytes(C, n, k);
}

int hmcx_rank_pass(const float* x, int64_t chain_stride, int64_t draw_stride, int32_t C, int32_t n, int32_t D,
                   int32_t d0, int32_t k, float* bulk_z, int64_t bulk_chain_stride, int64_t bulk_draw_stride,
                   float* fold_z, int64_t fold_chain_stride, int64_t fold_draw_stride, double* quantiles,
                   int32_t* nonfinite, void* workspace, size_t workspace_bytes, void* stream) {
    if (!diag_args_ok(x, chain_stride, draw_stride, C, n, D) || !rank_shape_ok(C, n) || !bulk_z || !fold_z ||
        !quantiles || !nonfinite || !workspace || bulk_chain_stride < 0 || bulk_draw_stride < 0 ||
        fold_chain_stride < 0 || fold_draw_stride < 0 || d0 < 0 || !rank_slab_ok(k) || (int64_t)d0 + k > D ||
        workspace_bytes < hmcx::rank_workspace_bytes(C, n, k))
        return HMCX_ERR_INVALID_ARG;
    return hmcx::rank_pass(x, chain_stride, draw_stride, C, n, D, d0, k, bulk_z, bulk_chain_stride, bulk_draw_stride,
                           fold_z, fold_chain_stride, fold_draw_stride, quantiles, nonfinite, workspace,
                           (cudaStream_t)stream);
}

int hmcx_rank_indicator(const float* x, int64_t chain_stride, int64_t draw_stride, int32_t C, int32_t n, int32_t D,
                        const double* thr, float* out, int64_t out_chain_stride, int64_t out_draw_stride, void* stream) {
    if (!diag_args_ok(x, chain_stride, draw_stride, C, n, D) || !thr || !out || out_chain_stride < 0 ||
        out_draw_stride < 0)
        return HMCX_ERR_INVALID_ARG;
    return hmcx::rank_indicator(x, chain_stride, draw_stride, C, n, D, thr, out, out_chain_stride, out_draw_stride,
                                (cudaStream_t)stream);
}

int hmcx_mlp_pointwise_ll(const hmcx_target_t* target, const float* samples, int64_t chain_stride, int64_t draw_stride,
                          int32_t C, int32_t n, int32_t row_begin, int32_t row_end, float* ll_out,
                          int64_t ll_chain_stride, int64_t ll_draw_stride, void* stream) {
    if (!target) return HMCX_ERR_INVALID_ARG;
    if (target->kind != HMCX_TARGET_MLP) return HMCX_ERR_UNSUPPORTED;
    return hmcx::mlp_pointwise_ll(target, samples, chain_stride, draw_stride, C, n, row_begin, row_end, ll_out,
                                  ll_chain_stride, ll_draw_stride, (cudaStream_t)stream, nullptr, 0, 0);
}

int hmcx_mlp_pointwise_ll_tau(const hmcx_target_t* target, const float* samples, int64_t chain_stride,
                              int64_t draw_stride, int32_t C, int32_t n, int32_t row_begin, int32_t row_end,
                              const float* tau_out, int64_t tau_chain_stride, int64_t tau_draw_stride, float* ll_out,
                              int64_t ll_chain_stride, int64_t ll_draw_stride, void* stream) {
    if (!target) return HMCX_ERR_INVALID_ARG;
    if (target->kind != HMCX_TARGET_MLP) return HMCX_ERR_UNSUPPORTED;
    return hmcx::mlp_pointwise_ll(target, samples, chain_stride, draw_stride, C, n, row_begin, row_end, ll_out,
                                  ll_chain_stride, ll_draw_stride, (cudaStream_t)stream, tau_out, tau_chain_stride,
                                  tau_draw_stride);
}

static inline bool loo_shape_ok(int32_t C, int32_t n) {
    return C >= 1 && n >= 1 && (int64_t)C * n >= 2 && (int64_t)C * n <= HMCX_RANK_MAX_DRAWS;
}

size_t hmcx_loo_workspace_bytes(int32_t C, int32_t n, int32_t k) {
    if (!loo_shape_ok(C, n) || !rank_slab_ok(k)) return 0;
    return hmcx::loo_workspace_bytes(C, n, k);
}

int hmcx_loo_pass(const float* ll, int64_t chain_stride, int64_t draw_stride, int32_t C, int32_t n, int32_t N,
                  int32_t i0, int32_t k, double r_eff, double* pointwise, int32_t* tail_size, int32_t* nonfinite,
                  void* workspace, size_t workspace_bytes, void* stream) {
    if (!ll || !pointwise || !tail_size || !nonfinite || !workspace || chain_stride < 0 || draw_stride < 0 ||
        !loo_shape_ok(C, n) || N < 1 || i0 < 0 || !rank_slab_ok(k) || (int64_t)i0 + k > N || !(r_eff > 0.0) ||
        !(r_eff <= DBL_MAX) || workspace_bytes < hmcx::loo_workspace_bytes(C, n, k))
        return HMCX_ERR_INVALID_ARG;
    return hmcx::loo_pass(ll, chain_stride, draw_stride, C, n, N, i0, k, r_eff, pointwise, tail_size, nonfinite,
                          workspace, (cudaStream_t)stream);
}

int hmcx_mlp_pointwise_out(const hmcx_target_t* target, const float* samples, int64_t chain_stride,
                           int64_t draw_stride, int32_t C, int32_t n, int32_t row_begin, int32_t row_end, float* out,
                           int64_t out_chain_stride, int64_t out_draw_stride, void* stream) {
    if (!target) return HMCX_ERR_INVALID_ARG;
    if (target->kind != HMCX_TARGET_MLP) return HMCX_ERR_UNSUPPORTED;
    return hmcx::mlp_pointwise_out(target, samples, chain_stride, draw_stride, C, n, row_begin, row_end, out,
                                   out_chain_stride, out_draw_stride, (cudaStream_t)stream);
}

static inline bool pred_shape_ok(int32_t C, int32_t n, int32_t k) {
    return C >= 1 && n >= 1 && (int64_t)C * n <= 0x7fffffffLL && k >= 1 && n <= (0x7fffffff - 64) / 2;
}

static inline int pred_form(int32_t loss) {
    return loss == HMCX_LOSS_MULTICLASS_LOGSOFTMAX ? HMCX_LOSS_MULTICLASS : loss;
}

static inline bool pred_loss_ok(int32_t loss) {
    return loss >= HMCX_LOSS_REGRESSION && loss <= HMCX_LOSS_MULTICLASS_LOGSOFTMAX;
}

size_t hmcx_pred_workspace_bytes(int32_t C, int32_t n, int32_t O, int32_t loss, int32_t k) {
    if (!pred_shape_ok(C, n, k) || O < 1 || O > 0xffffff || !pred_loss_ok(loss)) return 0;
    return hmcx::pred_workspace_bytes(n, O, pred_form(loss), k);
}

int hmcx_pred_pass(const float* f, int64_t chain_stride, int64_t draw_stride, int32_t C, int32_t n, int32_t O,
                   int32_t loss, const float* y, const float* tau_out, int64_t tau_chain_stride, int64_t tau_draw_stride,
                   int32_t N, int32_t i0, int32_t k, double* pointwise, double* per_output, int32_t* nonfinite,
                   double* partials, void* workspace, size_t workspace_bytes, void* stream) {
    if (!f || !y || !pointwise || !per_output || !nonfinite || !partials || !workspace || chain_stride < 0 ||
        draw_stride < 0 || !pred_shape_ok(C, n, k) || O < 1 || O > 0xffffff || N < 1 || i0 < 0 ||
        (int64_t)i0 + k > N || !pred_loss_ok(loss) ||
        (loss == HMCX_LOSS_REGRESSION && (!tau_out || tau_chain_stride < 0 || tau_draw_stride < 0)) ||
        workspace_bytes < hmcx::pred_workspace_bytes(n, O, pred_form(loss), k))
        return HMCX_ERR_INVALID_ARG;
    if (hmcx::pred_scan_smem(pred_form(loss), O) > 227 * 1024) return HMCX_ERR_UNSUPPORTED;
    return hmcx::pred_pass(f, chain_stride, draw_stride, C, n, O, pred_form(loss), y, tau_out, tau_chain_stride,
                           tau_draw_stride, N, i0, k, pointwise, per_output, nonfinite, partials, workspace,
                           (cudaStream_t)stream, nullptr);
}

int hmcx_pred_pass_weighted(const float* f, int64_t chain_stride, int64_t draw_stride, int32_t C, int32_t n, int32_t O,
                            int32_t loss, const float* y, const float* tau_out, int64_t tau_chain_stride,
                            int64_t tau_draw_stride, int32_t N, int32_t i0, int32_t k, double* pointwise,
                            double* per_output, int32_t* nonfinite, double* partials, void* workspace,
                            size_t workspace_bytes, const double* chain_weights, void* stream) {
    if (!chain_weights) return HMCX_ERR_INVALID_ARG;
    if (!f || !y || !pointwise || !per_output || !nonfinite || !partials || !workspace || chain_stride < 0 ||
        draw_stride < 0 || !pred_shape_ok(C, n, k) || O < 1 || O > 0xffffff || N < 1 || i0 < 0 ||
        (int64_t)i0 + k > N || !pred_loss_ok(loss) ||
        (loss == HMCX_LOSS_REGRESSION && (!tau_out || tau_chain_stride < 0 || tau_draw_stride < 0)) ||
        workspace_bytes < hmcx::pred_workspace_bytes(n, O, pred_form(loss), k))
        return HMCX_ERR_INVALID_ARG;
    if (hmcx::pred_scan_smem(pred_form(loss), O) > 227 * 1024) return HMCX_ERR_UNSUPPORTED;
    return hmcx::pred_pass(f, chain_stride, draw_stride, C, n, O, pred_form(loss), y, tau_out, tau_chain_stride,
                           tau_draw_stride, N, i0, k, pointwise, per_output, nonfinite, partials, workspace,
                           (cudaStream_t)stream, chain_weights);
}

int hmcx_pred_totals(const double* partials, int32_t n, int32_t N, double* totals, void* stream) {
    if (!partials || !totals || n < 1 || n > (0x7fffffff - 64) / 2 || N < 1) return HMCX_ERR_INVALID_ARG;
    return hmcx::pred_totals(partials, n, N, totals, (cudaStream_t)stream);
}

int hmcx_adapt_diag_mass(float* sum, float* sumsq, float* sum_lo, float* sumsq_lo, int32_t C, int32_t ld, int32_t D,
                         int32_t n, const float* eps, int32_t C_chains, float* inv_mass, float* mass_factor,
                         double* mu_chain, double* h_bar, double* eps_bar, void* stream) {
    if (!sum || !sumsq || !sum_lo || !sumsq_lo || !eps || !inv_mass || !mass_factor || !mu_chain || !h_bar || !eps_bar ||
        C < 1 || C_chains < 1 || n < 2 || D < 1 || ld < D || (ld & 3))
        return HMCX_ERR_INVALID_ARG;
    return hmcx::adapt_diag_mass(sum, sumsq, sum_lo, sumsq_lo, C, ld, D, n, eps, C_chains, inv_mass, mass_factor, mu_chain,
                                 h_bar, eps_bar, (cudaStream_t)stream);
}

// The SBC entry points take an MLP target with data: 1 on success, 0 for invalid arguments, -1 for other target kinds.
static inline int sbc_target_ok(const hmcx_target_t* target) {
    if (!target) return 0;
    if (target->kind != HMCX_TARGET_MLP) return -1;
    const hmcx_mlp_t* m = target->mlp;
    return m && m->x && m->y && m->num_rows >= 1 && m->num_layers >= 1 && m->num_layers <= HMCX_MLP_MAX_LAYERS ? 1 : 0;
}

static inline int mlp_dim(const hmcx_mlp_t* m) {
    int D = 0;
    for (int l = 0; l < m->num_layers; ++l) D += m->widths[l] * m->widths[l + 1] + m->widths[l + 1];
    return D;
}

int hmcx_sbc_prior(const hmcx_target_t* target, uint64_t seed, int64_t sim_begin, int32_t M, int32_t R, int32_t ld,
                   float* out, void* stream) {
    const int ok = sbc_target_ok(target);
    if (ok < 0) return HMCX_ERR_UNSUPPORTED;
    if (!ok || !out || sim_begin < 0 || M < 1 || R < 0 || ld < mlp_dim(target->mlp) || (ld & 3))
        return HMCX_ERR_INVALID_ARG;
    return hmcx::sbc_prior(target, seed, sim_begin, M, R, ld, out, (cudaStream_t)stream);
}

int hmcx_sbc_simulate(const hmcx_target_t* target, const float* f, uint64_t seed, int64_t sim_begin, int32_t M,
                      float* y_out, void* stream) {
    const int ok = sbc_target_ok(target);
    if (ok < 0) return HMCX_ERR_UNSUPPORTED;
    if (!ok || !f || !y_out || sim_begin < 0 || M < 1) return HMCX_ERR_INVALID_ARG;
    const hmcx_mlp_t* m = target->mlp;
    if (m->loss == HMCX_LOSS_MULTICLASS_LOGSOFTMAX || (m->loss != HMCX_LOSS_REGRESSION && m->tau_out != 1.0f) ||
        m->loss < HMCX_LOSS_REGRESSION || m->loss > HMCX_LOSS_MULTICLASS_LOGSOFTMAX || !(m->tau_out > 0.0f))
        return HMCX_ERR_UNSUPPORTED;
    return hmcx::sbc_simulate(target, f, seed, sim_begin, M, y_out, (cudaStream_t)stream);
}

int hmcx_sbc_rank(const float* samples, int64_t chain_stride, int64_t draw_stride, int32_t C, int32_t keep, int32_t K,
                  int32_t D, const float* truth, int64_t truth_stride, int32_t* ranks_out, void* stream) {
    if (!samples || !truth || !ranks_out || chain_stride < 0 || draw_stride < 0 || truth_stride < 0 || C < 1 || K < 1 ||
        K > 65535 || C % K || keep < 2 || D < 1 || (int64_t)(C / K) * (keep - 1) > 0x7fffffffLL)
        return HMCX_ERR_INVALID_ARG;
    return hmcx::sbc_rank(samples, chain_stride, draw_stride, C, keep, K, D, truth, truth_stride, ranks_out,
                          (cudaStream_t)stream);
}

int hmcx_ppc_pass(const hmcx_target_t* target, const float* f, int32_t k, const int64_t* draws, uint64_t seed,
                  const float* tau_out, float* y_rep, double* stats, double* dev_obs, int32_t* nonfinite, void* stream) {
    const int ok = sbc_target_ok(target);
    if (ok < 0) return HMCX_ERR_UNSUPPORTED;
    if (!ok || !f || !draws || !y_rep || !stats || !dev_obs || !nonfinite || k < 1) return HMCX_ERR_INVALID_ARG;
    const hmcx_mlp_t* m = target->mlp;
    if (m->loss < HMCX_LOSS_REGRESSION || m->loss > HMCX_LOSS_MULTICLASS_LOGSOFTMAX) return HMCX_ERR_INVALID_ARG;
    if (m->loss == HMCX_LOSS_REGRESSION && !tau_out && !(m->tau_out > 0.0f)) return HMCX_ERR_INVALID_ARG;
    return hmcx::ppc_pass(target, f, k, (const long long*)draws, seed, tau_out, y_rep, stats, dev_obs, nonfinite,
                          (cudaStream_t)stream);
}

int hmcx_loo_pit_pass(const float* ll, int64_t chain_stride, int64_t draw_stride, const float* f, int64_t f_chain_stride,
                      int64_t f_draw_stride, int32_t C, int32_t n, int32_t O, int32_t N, int32_t i0, int32_t k,
                      double r_eff, const float* y, const float* tau_out, int64_t tau_chain_stride,
                      int64_t tau_draw_stride, double* pit, double* pareto_k, int32_t* nonfinite, void* workspace,
                      size_t workspace_bytes, void* stream) {
    if (!ll || !f || !y || !tau_out || !pit || !pareto_k || !nonfinite || !workspace || chain_stride < 0 ||
        draw_stride < 0 || f_chain_stride < 0 || f_draw_stride < 0 || tau_chain_stride < 0 || tau_draw_stride < 0 ||
        O < 1 || !loo_shape_ok(C, n) || N < 1 || i0 < 0 || !rank_slab_ok(k) || (int64_t)i0 + k > N ||
        !(r_eff > 0.0) || !(r_eff <= DBL_MAX) || workspace_bytes < hmcx::loo_workspace_bytes(C, n, k))
        return HMCX_ERR_INVALID_ARG;
    return hmcx::loo_pit_pass(ll, chain_stride, draw_stride, f, f_chain_stride, f_draw_stride, C, n, O, i0, k, r_eff, y,
                              tau_out, tau_chain_stride, tau_draw_stride, pit, pareto_k, nonfinite, workspace,
                              (cudaStream_t)stream);
}

int hmcx_loo_chain_pass(const float* ll, int64_t chain_stride, int64_t draw_stride, int32_t C, int32_t n, int32_t N,
                        int32_t i0, int32_t k, double r_eff, double* out, int32_t* tail_size, int32_t* nonfinite,
                        void* stream) {
    if (!ll || !out || !tail_size || !nonfinite || chain_stride < 0 || draw_stride < 0 || C < 1 || C > 65535 ||
        n < 2 || n > HMCX_LOO_CHAIN_MAX_DRAWS || N < 1 || i0 < 0 || !rank_slab_ok(k) || (int64_t)i0 + k > N ||
        !(r_eff > 0.0) || !(r_eff <= DBL_MAX))
        return HMCX_ERR_INVALID_ARG;
    return hmcx::loo_chain_pass(ll, chain_stride, draw_stride, C, n, N, i0, k, r_eff, out, tail_size, nonfinite,
                                (cudaStream_t)stream);
}

static inline bool stack_shape_ok(int32_t K, int32_t N) {
    return K >= 1 && K <= 65535 && N >= 1 && (int64_t)K * N <= 0x7fffffffLL;
}

size_t hmcx_stack_workspace_bytes(int32_t K, int32_t N) {
    if (!stack_shape_ok(K, N)) return 0;
    return hmcx::stack_workspace_bytes(K, N);
}

int hmcx_stack_eval(const double* E, int32_t K, int32_t N, const double* w, double* objective, double* grad,
                    double* pointwise, void* workspace, size_t workspace_bytes, void* stream) {
    if (!E || !w || !objective || !grad || !pointwise || !workspace || !stack_shape_ok(K, N) ||
        workspace_bytes < hmcx::stack_workspace_bytes(K, N))
        return HMCX_ERR_INVALID_ARG;
    return hmcx::stack_eval(E, K, N, w, objective, grad, pointwise, workspace, (cudaStream_t)stream);
}

int hmcx_stack_em(const double* E, int32_t K, int32_t N, double tol, int32_t iterations, double* w, double* objective,
                  double* grad, double* pointwise, int32_t* state, void* workspace, size_t workspace_bytes,
                  void* stream) {
    if (!E || !w || !objective || !grad || !pointwise || !state || !workspace || !stack_shape_ok(K, N) ||
        iterations < 1 || !(tol >= 0.0) || !(tol <= DBL_MAX) || workspace_bytes < hmcx::stack_workspace_bytes(K, N))
        return HMCX_ERR_INVALID_ARG;
    return hmcx::stack_em(E, K, N, tol, iterations, w, objective, grad, pointwise, state, workspace,
                          (cudaStream_t)stream);
}

int hmcx_mlp_log_prior(const float* samples, int64_t chain_stride, int64_t draw_stride, int32_t C, int32_t n,
                       int32_t num_tensors, const int32_t* sizes, const double* tau, double* out, void* stream) {
    if (!samples || !sizes || !tau || !out || chain_stride < 0 || draw_stride < 0 || C < 1 || n < 1 ||
        (int64_t)C * n > 0x7fffffffLL || num_tensors < 1 || num_tensors > 2 * HMCX_MLP_MAX_LAYERS)
        return HMCX_ERR_INVALID_ARG;
    int64_t total = 0;
    for (int t = 0; t < num_tensors; ++t) {
        if (sizes[t] < 1 || !(tau[t] >= 0.0) || !(tau[t] <= DBL_MAX)) return HMCX_ERR_INVALID_ARG;
        total += sizes[t];
    }
    if (total > 0x7fffffffLL) return HMCX_ERR_INVALID_ARG;
    return hmcx::mlp_log_prior(samples, chain_stride, draw_stride, C, n, num_tensors, sizes, tau, out,
                               (cudaStream_t)stream);
}

int hmcx_psens_ll_totals(const float* ll, int64_t chain_stride, int64_t draw_stride, int32_t C, int32_t n, int32_t r0,
                         int32_t k, const double* coef, double* totals, void* stream) {
    if (!ll || !totals || chain_stride < 0 || draw_stride < 0 || !loo_shape_ok(C, n) || r0 < 0 || r0 % 128 || k < 1 ||
        (int64_t)r0 + k > 0x7fffffffLL)
        return HMCX_ERR_INVALID_ARG;
    return hmcx::psens_ll_totals(ll, chain_stride, draw_stride, C, n, r0, k, coef, totals, (cudaStream_t)stream);
}

size_t hmcx_psens_workspace_bytes(int32_t C, int32_t n, int32_t k) {
    if (!loo_shape_ok(C, n) || !rank_slab_ok(k)) return 0;
    return hmcx::psens_workspace_bytes(C, n, k);
}

int hmcx_psens_weights(const float* neg_log_ratio, int64_t chain_stride, int64_t draw_stride, int32_t C, int32_t n,
                       int32_t K, double r_eff, double* weights, double* pareto_k, int32_t* tail_size,
                       int32_t* nonfinite, void* workspace, size_t workspace_bytes, void* stream) {
    if (!neg_log_ratio || !weights || !pareto_k || !tail_size || !nonfinite || !workspace || chain_stride < 0 ||
        draw_stride < 0 || !loo_shape_ok(C, n) || !rank_slab_ok(K) || !(r_eff > 0.0) || !(r_eff <= DBL_MAX) ||
        workspace_bytes < hmcx::psens_workspace_bytes(C, n, K))
        return HMCX_ERR_INVALID_ARG;
    return hmcx::psens_weights(neg_log_ratio, chain_stride, draw_stride, C, n, K, r_eff, weights, pareto_k, tail_size,
                               nonfinite, workspace, (cudaStream_t)stream);
}

int hmcx_psens_pass(const float* x, int64_t chain_stride, int64_t draw_stride, int32_t C, int32_t n, int32_t D,
                    int32_t d0, int32_t k, const double* weights, double* out, int32_t* nonfinite, void* workspace,
                    size_t workspace_bytes, void* stream) {
    if (!x || !weights || !out || !nonfinite || !workspace || chain_stride < 0 || draw_stride < 0 ||
        !loo_shape_ok(C, n) || D < 1 || d0 < 0 || !rank_slab_ok(k) || (int64_t)d0 + k > D ||
        workspace_bytes < hmcx::psens_workspace_bytes(C, n, k))
        return HMCX_ERR_INVALID_ARG;
    return hmcx::psens_pass(x, chain_stride, draw_stride, C, n, D, d0, k, weights, out, nonfinite, workspace,
                            (cudaStream_t)stream);
}

}  // extern "C"
