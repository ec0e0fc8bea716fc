/*
 * hmcx.h -- C ABI of libhmcx.so, the H100 (sm_90a) batched-chain Hamiltonian Monte Carlo engine.
 *
 * Drop-in boundary for the hot path of AdamCobb/hamiltorch (reference, pure Python): the reference has no
 * FFI of its own, its boundary is the Python function surface (SURVEY.md section 8b).  Each entry point below
 * names the reference function (hamiltorch/samplers.py, file:line) whose arithmetic it replaces for a whole
 * batch of C independent chains; hamiltorch_b200/_native.py binds them with ctypes (INTEGRATION.md shows the
 * stub a reference maintainer would add).
 *
 * Conventions
 *   - plain C types only: raw DEVICE pointers + sizes + an opaque cudaStream_t (void*); the library never
 *     allocates, never synchronises, keeps no global state; calls are re-entrant given distinct buffers.
 *   - state arrays are fp32 row-major (C, ld): row c = chain c, ld >= D, ld % 4 == 0, 16-byte aligned,
 *     pad elements are ignored on input and written as 0.
 *   - return value: HMCX_OK or a negative HMCX_ERR_* code (hmcx_status_string()).  Numerical divergence is
 *     NOT an error: like the reference's LogProbError -> reject (samplers.py:1045) it is reported per chain
 *     and iteration in `diverged_out`.
 *   - fp32 arithmetic follows the reference's operation order with fused multiply-add contraction disabled,
 *     so that elementwise state is bit-identical to the reference's PyTorch-CPU path; reductions (the
 *     Hamiltonian sums) differ from torch.dot only in summation order.
 */
#ifndef HMCX_H
#define HMCX_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HMCX_ABI_VERSION 12

#define HMCX_MLP_TC_AUTO 0
#define HMCX_MLP_TC_OFF  1

/* status codes */
#define HMCX_OK                0
#define HMCX_ERR_INVALID_ARG  -1
#define HMCX_ERR_UNSUPPORTED  -2
#define HMCX_ERR_CUDA         -3

/* hmcx_target_t.kind -- the log-densities the kernels can differentiate (hamiltorch_b200/targets.py) */
#define HMCX_TARGET_GAUSS_ISO   0   /* log p = -0.5*sum(x*x) + log_norm                               */
#define HMCX_TARGET_GAUSS_DIAG  1   /* log p = -0.5*sum((x-mean)^2*inv_var) + log_norm                 */
#define HMCX_TARGET_GAUSS_FULL  2   /* log p = -0.5*(x-mean).P(x-mean) + log_norm                      */
#define HMCX_TARGET_FUNNEL      3   /* Neal's funnel, notebooks/hamiltorch_log_prob_examples.ipynb c22 */
#define HMCX_TARGET_MLP         4   /* define_model_log_prob, samplers.py:1093-1201 (regression, MLP)   */

/* hmcx_mass_t.kind -- the inv_mass argument of sample()/leapfrog() (samplers.py:283-296) */
#define HMCX_MASS_NONE  0
#define HMCX_MASS_DIAG  1           /* inv_mass 1-D, samplers.py:296, :814, gibbs :201                 */
#define HMCX_MASS_FULL  2           /* inv_mass 2-D, samplers.py:294, :812, gibbs :199                 */

/* hmcx_rng_t.mode */
#define HMCX_RNG_INJECTED 0         /* host supplies the reference's own random stream (parity mode)   */
#define HMCX_RNG_PHILOX   1         /* in-kernel Philox4x32-10 keyed by (seed, chain, iteration)       */

/* Dense-stack Bayesian NN target == the closure define_model_log_prob builds (samplers.py:1093-1201) for a
 * Linear/activation stack with model_loss='regression', plus its data-split form (define_split_model_log_prob,
 * :1203-1258): split m owns data rows [split_begin[m], split_begin[m+1]) and divides the prior by prior_scale.
 * Flat parameter layout = util.flatten (util.py:121-136): per Linear the (out,in) row-major weight, then the bias. */
#define HMCX_MLP_MAX_LAYERS 8
#define HMCX_MLP_MAX_SPLITS 64
#define HMCX_ACT_NONE 0
#define HMCX_ACT_RELU 1
#define HMCX_ACT_TANH 2
#define HMCX_ACT_SIGMOID 3
#define HMCX_LOSS_REGRESSION            0   /* 'regression'                      samplers.py:1182-1184          */
#define HMCX_LOSS_BINARY                1   /* 'binary_class_linear_output'      :1170-1172 (BCE with logits)   */
#define HMCX_LOSS_MULTICLASS            2   /* 'multi_class_linear_output'       :1173-1177 (cross entropy, sum) */
#define HMCX_LOSS_MULTICLASS_LOGSOFTMAX 3   /* 'multi_class_log_softmax_output'  :1179-1180 (log-softmax output +
                                               nll_loss with its default MEAN reduction)                        */

typedef struct hmcx_mlp {
    int32_t num_layers;                            /* number of Linear layers                                  */
    int32_t widths[HMCX_MLP_MAX_LAYERS + 1];       /* n_0 (inputs) ... n_L (outputs)                           */
    int32_t activation[HMCX_MLP_MAX_LAYERS];       /* applied after layer l (last must be NONE)                */
    int32_t loss;
    float   tau_out;                               /* likelihood precision (samplers.py:1184)                  */
    float   prior_scale;                           /* l_prior / prior_scale (:1199); = num_splits when split   */
    /* Gaussian prior per parameter tensor i = (W_0, b_0, W_1, b_1, ...), constants carrying the reference's fp32
     * roundings of torch.distributions.Normal(0, tau_i^-1/2).log_prob (:1143, :1156):                           */
    float   prior_two_var[2 * HMCX_MLP_MAX_LAYERS];    /* 2*scale_i^2                                          */
    float   prior_log_scale[2 * HMCX_MLP_MAX_LAYERS];  /* log(scale_i)                                         */
    float   prior_grad_coef[2 * HMCX_MLP_MAX_LAYERS];  /* (1/prior_scale)/(2*scale_i^2): d prior/dw = -(coef*2w) */
    const float* x;                                /* [num_rows, n_0] device; NULL = sample the prior (:1160)    */
    const float* y;                                /* [num_rows, n_L] device (regression / binary) or [num_rows]
                                                      class indices stored as float (multi-class)              */
    int32_t num_rows;
    int32_t num_splits;                            /* M >= 1                                                    */
    int32_t split_begin[HMCX_MLP_MAX_SPLITS + 1];
    int32_t cluster_size;                          /* CTAs (SMs) cooperating on one chain: 0 = automatic, 1 / 2 / 4 =
                                                      pinned (bit-reproducibility across chain counts)          */
    int32_t tensor_cores;                          /* HMCX_MLP_TC_AUTO: first-layer GEMMs on the tensor cores (3xTF32, fp32-level
                                                      accuracy) when the stack is n0 -> 128 -> nL with n0 in
                                                      {16,32,48,64}, nL <= 4; HMCX_MLP_TC_OFF: fp32 SIMT tiles  */
    const float* x_packed;                         /* device buffer of hmcx_mlp_packed_x_bytes() filled by hmcx_mlp_pack_x():
                                                      x as ready-made tensor-core operands (tf32 hi | lo, both GEMM layouts),
                                                      one bulk TMA copy per tile.  NULL: fp32 SIMT tiles               */
} hmcx_mlp_t;

typedef struct hmcx_target {
    int32_t kind;
    int32_t dim;                    /* D                                                               */
    const float* mean;              /* [D] device, GAUSS_DIAG / GAUSS_FULL (NULL = zeros)              */
    const float* inv_var;           /* [D] device, GAUSS_DIAG                                          */
    const float* prec;              /* [D,D] device row-major symmetric, GAUSS_FULL                    */
    float log_norm;                 /* additive constant of log p                                      */
    float funnel_inv_var_v;         /* FUNNEL: 1/sigma_v^2                                             */
    const hmcx_mlp_t* mlp;          /* MLP: HOST pointer to the network / data description             */
} hmcx_target_t;

typedef struct hmcx_mass {
    int32_t kind;
    const float* inv_mass;          /* DIAG: [D]; FULL: [D,D] row-major                                */
    const float* mass_factor;       /* DIAG: sqrt(1/inv_mass) [D] (gibbs :201);
                                       FULL: lower Cholesky factor of inverse(inv_mass) [D,D] (:199)   */
} hmcx_mass_t;

typedef struct hmcx_rng {
    int32_t mode;
    uint64_t seed;                  /* PHILOX key                                                      */
    uint64_t chain_offset;          /* PHILOX: global id of local chain 0 (multi-GPU sharding)         */
    const float* normals;           /* INJECTED: standard normals [iter_end-iter_begin, C, ld]         */
    const float* log_uniforms;      /* INJECTED: log(U) of the MH test [iter_end-iter_begin, C]        */
    const int32_t* perms;           /* INJECTED, SPLITTING_RAND only: randperm(M) per trajectory (:550)
                                       [iter_end-iter_begin, C, M]                                     */
    const float* uniforms;          /* INJECTED, RMHMC with jitter: the torch.rand(D) draws of fisher()
                                       (:115) in call order [iter_end-iter_begin, C, uniforms_per_iter, ld]   */
    int32_t uniforms_per_iter;      /* explicit integrator: 8*L+3 (gibbs, H, 8 per step, H_new)        */
} hmcx_rng_t;

/* Dual-averaging step-size adaptation ("HMC_NUTS"), samplers.py:629-674, per chain.
 * `table` holds, for t = 1..burn+1, the five Python-double constants the reference evaluates each call:
 *   {1-1/(t+10), 1/(t+10), sqrt(t)/0.05, t^-0.75, 1-t^-0.75}            (row-major [burn+1][5], device) */
typedef struct hmcx_nuts {
    int32_t enabled;
    double  desired_accept_rate;
    double  mu;                     /* float(log(10*eps0)) evaluated in fp32 as samplers.py:664        */
    const double* table;
    double* h_bar;                  /* [C] in/out, running H_t (starts at 0, samplers.py:938)          */
    double* eps_bar;                /* [C] in/out, running eps_bar (starts at 1, samplers.py:939)      */
    const float* eps_schedule;      /* optional [num_samples, C]: use THIS step size in iteration n instead of
                                       the adapted one ("teacher forcing": parity tests replay the reference's
                                       schedule because adaptation amplifies fp32 summation-order noise)       */
    float* eps_trace;               /* optional [C, num_samples]: the step size the kernel's own adaptation
                                       yields after iteration n (i.e. for iteration n+1)                       */
    double step_size_init;          /* the Python-double step size the run starts from (0 = not given; read even when
                                       enabled == 0).  The splitting integrators divide the DOUBLE step size before the
                                       product with the fp32 tensor rounds it (step_size/K_div, samplers.py:513, :558):
                                       while a chain's fp32 step size still equals (float)step_size_init the drift
                                       coefficient is (float)(step_size_init / K); an adapted step size is an fp32
                                       value in the reference too (:668) and is divided as such.                   */
    const double* mu_chain;         /* optional [C] (ABI v11): per-chain mu replacing the scalar `mu`, written by
                                       hmcx_adapt_diag_mass when the dual averaging restarts after a mass update.
                                       Read by the sink forms only (hmcx_hmc_run_sink / hmcx_split_run_sink with a
                                       sink; a thin = 1 sink without sums still selects the sink form when mu_chain is
                                       set); hmcx_hmc_run and hmcx_split_run return HMCX_ERR_UNSUPPORTED for it   */
} hmcx_nuts_t;

int         hmcx_abi_version(void);
const char* hmcx_status_string(int status);

/*
 * hmcx_leapfrog == samplers.leapfrog, plain-HMC branch (samplers.py:269-304) for C chains at once.  Targets GAUSS_ISO /
 * GAUSS_DIAG / GAUSS_FULL / FUNNEL, mass none / diagonal / full, any D (element-wise cases: the streaming HBM-roofline
 * kernel; coupled gradients or a full mass matrix: one CTA per chain with the state in shared memory).
 *   q_in, p_in   [C, ld]   start state (not modified)
 *   eps          [C]       per-chain step size
 *   q_out, p_out [C, ld]   state after L steps, p_out with the half-step correction of :302 applied
 *   q_traj, p_traj          optional (NULL to skip) [L, C, ld]: the L intermediate clones the reference returns
 *                           (ret_params / ret_momenta, :299-300; p_traj[L-1] is the corrected one)
 */
int hmcx_leapfrog(const hmcx_target_t* target, const hmcx_mass_t* mass,
                  const float* q_in, const float* p_in, const float* eps,
                  int32_t C, int32_t ld, int32_t L,
                  float* q_out, float* p_out, float* q_traj, float* p_traj, void* stream);

/*
 * hmcx_hamiltonian == samplers.hamiltonian, sampler=HMC (samplers.py:779-815); same target / mass coverage as
 * hmcx_leapfrog.
 *   H_out [C]; flags_out [C] (optional) = 1 where log p is non-finite (the reference raises LogProbError, :783-785)
 */
int hmcx_hamiltonian(const hmcx_target_t* target, const hmcx_mass_t* mass,
                     const float* q, const float* p, int32_t C, int32_t ld,
                     float* H_out, uint8_t* flags_out, void* stream);

/*
 * hmcx_gibbs == samplers.gibbs, sampler=HMC (samplers.py:185-202), PHILOX mode only: p ~ N(0, M) for C chains
 * and iteration index `iter` (the same stream hmcx_hmc_run consumes for that iteration).
 */
int hmcx_gibbs(const hmcx_mass_t* mass, const hmcx_rng_t* rng, int32_t D, int32_t C, int32_t ld,
               int64_t iter, float* p_out, void* stream);

/*
 * hmcx_hmc_run == the sample() loop (samplers.py:954-1067) for sampler in {HMC, HMC_NUTS}: per iteration
 * gibbs -> hamiltonian -> leapfrog -> hamiltonian -> acceptance/MH -> bookkeeping (-> adaptation), as ONE
 * persistent kernel launch that advances iterations [iter_begin, iter_end) of C chains.
 *   q_init      [C, ld]  params_init (read only; needed again for the reference's first-post-burn-reject quirk)
 *   q_cur       [C, ld]  in/out: current `params`; must equal q_init when iter_begin == 0
 *   eps         [C]      in/out: per-chain step size (changes only when nuts->enabled)
 *   samples_out [C, num_samples-burn, ld]  slot 0 = params_init (:959), slot n-burn = iteration n > burn
 *   accept_out / diverged_out  optional [C, num_samples] (uint8); ham_out optional [C, num_samples, 2] = (H_old, H_new)
 *   num_rejected optional [C] int32 in/out counter (:961, :1016, :1046)
 *   workspace    hmcx_hmc_workspace_bytes() bytes of device scratch (NULL when that is 0).  For element-wise targets with
 *                ld <= 4096 these are C floats that carry log p(q_cur) from one window of iterations to the next: pass the
 *                SAME buffer to the launches [0, a), [a, b), ... of a run and they reproduce the single launch [0, S) bit for
 *                bit; with NULL a window recomputes log p(q_cur) (a reduction that associates differently from the loop's:
 *                H_old of its first iteration may differ in the last bit)
 *   tuning       0 = automatic register geometry (one float4 per thread for D <= 2560, two above); 1 = one float4 per
 *                thread; 2 / 4 = that many float4 groups per thread; 21 / 22 = one / two float2 groups per thread
 *                (tests and tuning sweeps; element-wise state and the random stream never depend on it)
 */
int hmcx_hmc_run(const hmcx_target_t* target, const hmcx_mass_t* mass, const hmcx_rng_t* rng,
                 const hmcx_nuts_t* nuts,
                 const float* q_init, float* q_cur, float* eps,
                 int32_t C, int32_t ld, int32_t L, int32_t num_samples, int32_t burn,
                 int32_t iter_begin, int32_t iter_end,
                 float* samples_out, uint8_t* accept_out, uint8_t* diverged_out, float* ham_out,
                 int32_t* num_rejected, int32_t tuning, float* workspace, void* stream);

/* Scratch hmcx_hmc_run needs in `workspace` (device bytes; 0 = may pass NULL).  Element-wise targets with D > 4096 are
 * advanced by a streamed form of the kernel that parks each proposal in a caller-provided (C, ld) buffer. */
size_t hmcx_hmc_workspace_bytes(const hmcx_target_t* target, const hmcx_mass_t* mass, int32_t C, int32_t ld);

/* sampler=RMHMC configuration (samplers.py:850 arguments that only this sampler reads) */
typedef struct hmcx_rmhmc {
    int32_t integrator;             /* Integrator enum value: 1 EXPLICIT (:389-462), 2 IMPLICIT (:305-387)         */
    int32_t metric;                 /* Metric enum value: 1 HESSIAN, 2 SOFTABS (:116-122), 3 JACOBIAN_DIAG (:100-106,
                                       hmcx_rmhmc_run only: the metric diag((d log p/d theta_i)^2) is never constant)  */
    float   softabs_const;          /* alpha                                                                      */
    float   jitter;                 /* scale of the uniform diagonal jitter (:113-115); < 0 = None                */
    float   pi_term;                /* D*log(2*pi) evaluated in fp32 as :712                                      */
    float   cos_2we, sin_2we;       /* cos/sin(2*explicit_binding_const*step_size) in fp32 as :435-436            */
    float   fixed_point_threshold;  /* implicit: :337, :356                                                       */
    int32_t fixed_point_max_iterations;
    int32_t jitter_max_tries;       /* NaN-gradient retries before LogProbError (:402-410)                        */
} hmcx_rmhmc_t;

/* integrators of the HMC family (samplers.py:269, :494, :548, :575) */
#define HMCX_SCHEME_PLAIN       0   /* plain leapfrog on the whole potential (sample_model)             */
#define HMCX_SCHEME_SPLIT_SYM   1   /* Integrator.SPLITTING       (:494-547)                             */
#define HMCX_SCHEME_SPLIT_RAND  2   /* Integrator.SPLITTING_RAND  (:548-571)                             */
#define HMCX_SCHEME_SPLIT_KMID  3   /* Integrator.SPLITTING_KMID  (:575-601)                             */

/*
 * hmcx_split_run == the sample() loop for a data-split potential U = sum_m U_m (sample_split_model, samplers.py:1364
 * -> sample with integrator in {SPLITTING, SPLITTING_RAND, SPLITTING_KMID}), and with HMCX_SCHEME_PLAIN the same
 * loop for the un-split Bayesian NN (sample_model, :1261).  Target must be HMCX_TARGET_MLP.  Arguments as
 * hmcx_hmc_run; the Hamiltonian sums the split log-probs (:787-796).
 */
int hmcx_split_run(const hmcx_target_t* target, const hmcx_mass_t* mass, const hmcx_rng_t* rng,
                   const hmcx_nuts_t* nuts, int32_t scheme,
                   const float* q_init, float* q_cur, float* eps,
                   int32_t C, int32_t ld, int32_t L, int32_t num_samples, int32_t burn,
                   int32_t iter_begin, int32_t iter_end,
                   float* samples_out, uint8_t* accept_out, uint8_t* diverged_out, float* ham_out,
                   int32_t* num_rejected, void* stream);

/*
 * hmcx_rmhmc_run == the sample() loop for sampler=RMHMC (samplers.py:965-1067 with gibbs :183-184, rm_hamiltonian
 * :677-736, fisher :69-127, explicit :389-462 / implicit :305-387 leapfrog).  Targets: FUNNEL, GAUSS_ISO, GAUSS_DIAG,
 * GAUSS_FULL (closed-form Hessian and third-derivative contraction), any jitter, metrics HESSIAN / SOFTABS /
 * JACOBIAN_DIAG.  dim <= 16: one thread per chain (dim == 2 with the explicit integrator -- BASELINE config 3 -- a
 * pair of warps per 32 chains that evaluates dH/dtheta and dH/dp concurrently); 16 < dim <= 64: one CTA per chain, the
 * metric assembled, eigen-decomposed (parallel-order Jacobi) and solved in shared memory.  Arguments as hmcx_hmc_run
 * (eps is read-only: the reference never adapts the step size of RMHMC).
 */
int hmcx_rmhmc_run(const hmcx_target_t* target, const hmcx_rmhmc_t* cfg, const hmcx_rng_t* rng,
                   const float* q_init, float* q_cur, const float* eps,
                   int32_t C, int32_t ld, int32_t L, int32_t num_samples, int32_t burn,
                   int32_t iter_begin, int32_t iter_end,
                   float* samples_out, uint8_t* accept_out, uint8_t* diverged_out, float* ham_out,
                   int32_t* num_rejected, void* stream);

/*
 * hmcx_rmhmc_leapfrog == samplers.leapfrog with sampler=RMHMC called on its own (explicit :389-462, implicit :305-387):
 * L steps from (q_in, p_in), same targets / metrics as hmcx_rmhmc_run, dim <= 64.
 *   q_traj, p_traj   [L, C, ld]  theta and p after every step (the reference's ret_params / ret_momenta lists)
 *   q_copy_out, p_copy_out  optional [C, ld]: the explicit integrator's params_copy / momentum_copy after the last step
 *                    (second elements of the pairs it returns, :462)
 *   flags_out        [C] (uint8) 1 where the reference raises LogProbError inside the trajectory (outputs of that chain
 *                    from the failing step on are unspecified)
 * rng: jitter draws of the fisher() calls in call order from row 0 (INJECTED: uniforms [1, C, J, ld]) or Philox with
 * iteration index 0; normals / log_uniforms are not read.
 */
int hmcx_rmhmc_leapfrog(const hmcx_target_t* target, const hmcx_rmhmc_t* cfg, const hmcx_rng_t* rng,
                        const float* q_in, const float* p_in, const float* eps, int32_t C, int32_t ld, int32_t L,
                        float* q_traj, float* p_traj, float* q_copy_out, float* p_copy_out, uint8_t* flags_out,
                        void* stream);

/*
 * hmcx_rmhmc_hamiltonian == samplers.hamiltonian with sampler=RMHMC (:817-829) == rm_hamiltonian (:677-736):
 * H_out[c] = -log p + 0.5 D log 2pi + 0.5 log det G + 0.5 p.G^-1 p (the caller doubles it for the explicit integrator's
 * augmented form, :822); flags_out [C] = 1 where the reference raises LogProbError.  One jitter row (row 0).
 */
int hmcx_rmhmc_hamiltonian(const hmcx_target_t* target, const hmcx_rmhmc_t* cfg, const hmcx_rng_t* rng,
                           const float* q, const float* p, int32_t C, int32_t ld, float* H_out, uint8_t* flags_out,
                           void* stream);

/*
 * hmcx_grad_log_prob == collect_gradients(log_prob_func(params), params) (samplers.py:33-66, :270-278) for C
 * parameter vectors: grad_out[c] = d log p_split(q[c]) / dq.  split = -1 sums all splits.  Any target kind.
 * log_prob_out optional [C].
 */
int hmcx_grad_log_prob(const hmcx_target_t* target, const float* q, int32_t C, int32_t ld, int32_t split,
                       float* grad_out, float* log_prob_out, void* stream);

/*
 * hmcx_mlp_predict == predict_model (samplers.py:1468-1562): forward pass of every sample over the target's data.
 *   samples [S, ld];  pred_out [S, num_rows, n_L];  log_prob_out [S] = ll + prior/prior_scale (:1197)
 */
int hmcx_mlp_predict(const hmcx_target_t* target, const float* samples, int32_t S, int32_t ld,
                     float* pred_out, float* log_prob_out, void* stream);

/*
 * hmcx_split_leapfrog == samplers.leapfrog called directly with Integrator.SPLITTING / SPLITTING_RAND / SPLITTING_KMID on the
 * list define_split_model_log_prob returns (samplers.py:494-603): L steps from (q_in, p_in) [C, ld]; q_traj / p_traj
 * [L, C, ld] receive params and momentum after EVERY step (the reference's ret_params / ret_momenta lists).  eps [C] =
 * (float)step_size per chain; step_size is the Python double the drifts divide before rounding (:513, :558).
 * SPLITTING_RAND takes its one randperm(M) per call (:550) from rng->perms [C, M] (INJECTED) or from the Philox PERM stream.
 */
int hmcx_split_leapfrog(const hmcx_target_t* target, const hmcx_mass_t* mass, const hmcx_rng_t* rng, int32_t scheme,
                        double step_size, const float* q_in, const float* p_in, float* eps, int32_t C, int32_t ld,
                        int32_t L, float* q_traj, float* p_traj, void* stream);

/*
 * Packed X operands of the BNN tensor-core path (hmcx_mlp_t.x_packed).  The data matrix of define_model_log_prob
 * (samplers.py:1093-1201) never changes during a run, so its tf32 hi / lo split and the two tensor-core operand layouts
 * (forward: rows x inputs, backward: inputs x rows) are built once per target:
 *   hmcx_mlp_packed_x_bytes   size of the buffer (0: this stack has no tensor-core form -- leave x_packed NULL)
 *   hmcx_mlp_pack_x           fills it from target->mlp->x on `stream` (x_packed itself is not read)
 */
size_t hmcx_mlp_packed_x_bytes(const hmcx_target_t* target);
int hmcx_mlp_pack_x(const hmcx_target_t* target, float* packed_out, void* stream);

/*
 * hmcx_gemm_nt_tf32x3: D[M,N] = A[M,K] . B[N,K]^T on the Hopper tensor cores (wgmma.mma_async tf32 with 3xTF32 split
 * operands => fp32-accurate, fp32 accumulation in registers).  Row-major fp32 device arrays;
 * M, N multiples of 128, K a multiple of 32.  The dense contraction behind full-covariance targets / full mass
 * matrices at large D (grad log p of ALL chains = -(Q - mu) P: M = chains, N = K = D; samplers.py:294, :812).
 */
int hmcx_gemm_nt_tf32x3(const float* A, const float* B, float* D, int32_t M, int32_t N, int32_t K, void* stream);

/*
 * Constant-metric RMHMC on the tensor cores.  For Gaussian targets without jitter the metric of samplers.py:69-127
 * (G = -Hessian, or its softabs map V diag(lambda coth(alpha lambda)) V^T) is one matrix for every chain and every
 * point, so the flows of the explicit (:427-458) and implicit (:363-386) integrators are (chains x D).(D x D)
 * contractions: dH/dp = G^-1 p (the metric solve of cholesky_inverse, :130-149) and dH/dtheta = P (theta - mu).
 * The caller evaluates, once, with the reference's own torch ops:
 *   metric_inv  [D,D]  G^-1        metric_chol [D,D]  lower Cholesky factor of G (gibbs :183-184)
 *   log_det            log det G   (sum log lambda~ for SOFTABS :726, slogdet for HESSIAN :728)
 */
typedef struct hmcx_const_metric {
    const float* metric_inv;
    const float* metric_chol;
    float log_det;
} hmcx_const_metric_t;

size_t hmcx_rmhmc_dense_workspace_bytes(int32_t C, int32_t D);

/*
 * hmcx_rmhmc_dense_run == the sample() loop for sampler=RMHMC (as hmcx_rmhmc_run) for targets GAUSS_ISO / GAUSS_DIAG /
 * GAUSS_FULL of ANY dimension with cfg->jitter < 0 (None): every flow is a tensor-core GEMM over all chains (3xTF32,
 * operands packed for 1-D bulk TMA), 8 per explicit leapfrog step.  workspace: hmcx_rmhmc_dense_workspace_bytes().
 * D <= 128 (and ld <= D rounded up to 32): the whole run is ONE persistent launch instead (hmcx_flow.cu: the matrices in
 * shared memory, a warp owns 1-4 chains, exact fp32 FMAs; the workspace is then unused; environment HMCX_FLOW_SMALL=0
 * keeps the GEMM path).  The same holds for hmcx_hmc_run with a dense precision or a 2-D inv_mass at 16 < D <= 128.
 */
int hmcx_rmhmc_dense_run(const hmcx_target_t* target, const hmcx_rmhmc_t* cfg, const hmcx_const_metric_t* metric,
                         const hmcx_rng_t* rng, const float* q_init, float* q_cur, const float* eps,
                         int32_t C, int32_t ld, int32_t L, int32_t num_samples, int32_t burn,
                         int32_t iter_begin, int32_t iter_end,
                         float* samples_out, uint8_t* accept_out, uint8_t* diverged_out, float* ham_out,
                         int32_t* num_rejected, float* workspace, void* stream);

/*
 * Sample sink -- what consumes the retained samples (the store_on_GPU=False contract of samplers.py:1008-1012 and the
 * step after the path, SURVEY 8f-3), for runs whose C*S*D exceeds what the caller wants to keep:
 *   thin   keep every thin-th post-burn iteration: samples_out is [C, 1 + (num_samples-burn-1)/thin, ld], slot 0 =
 *          params_init, slot j = the chain state after iteration burn + j*thin  (thin = 1: the reference's list)
 *   sum, sumsq   optional [C, ld] in/out accumulators: running sum / sum of squares of the chain state over EVERY
 *          iteration n > burn (= elements 1.. of the reference's returned list), so posterior means and variances
 *          need no sample storage at all (samples_out may then be NULL).  Accumulated with Neumaier compensation (the
 *          rounding of x*x included; element-wise kernel: in registers, Bayesian-NN kernel: in place in these arrays at
 *          every iteration, see hmcx_split_run_sink): relative error ~ n*eps^2 after n iterations (eps = 2^-24)
 *          instead of the ~ n*eps of a plain fp32 running sum:
 *   sum_lo, sumsq_lo   optional [C, ld] in/out: the compensation terms; the sums are hi + lo (combine in fp64: var =
 *          E[x^2] - mean^2 then holds for |mean| >> std; measured 1.6e-7 on a variance of 1 at mean 100, n = 2e4, where
 *          the plain sum is off by percents).  Without them the fp32 rounding of hi + lo is stored in sum / sumsq.
 * samples_out may point to device-mapped pinned HOST memory: the kernel's retained-row stores are coalesced 16-byte
 * streaming stores (st.global.cs), which is how samples leave the GPU while the chains keep running.
 */
typedef struct hmcx_sink {
    int32_t thin;
    float*  sum;
    float*  sumsq;
    float*  sum_lo;
    float*  sumsq_lo;
    int32_t moments_all;            /* ABI v11: non-zero = accumulate sum / sumsq over EVERY iteration of the launch
                                       (warm-up included) instead of n > burn only: the moments of a mass-adaptation
                                       window (hmcx_adapt_diag_mass).  0 (a zero-initialised struct): as before   */
} hmcx_sink_t;

/* hmcx_hmc_run with a sample sink (sink == NULL or {1, NULL, NULL, NULL, NULL} without nuts->mu_chain: identical to
 * hmcx_hmc_run).  Element-wise targets (GAUSS_ISO / GAUSS_DIAG, mass none / diagonal, ld <= 4096); other combinations
 * return HMCX_ERR_UNSUPPORTED when the sink asks for thinning or moments.  The workspace carries log p(q_cur) from one
 * window of iterations to the next as in hmcx_hmc_run (ABI v11; the mass-adaptation windows rely on it). */
int hmcx_hmc_run_sink(const hmcx_target_t* target, const hmcx_mass_t* mass, const hmcx_rng_t* rng,
                      const hmcx_nuts_t* nuts,
                      const float* q_init, float* q_cur, float* eps,
                      int32_t C, int32_t ld, int32_t L, int32_t num_samples, int32_t burn,
                      int32_t iter_begin, int32_t iter_end,
                      float* samples_out, uint8_t* accept_out, uint8_t* diverged_out, float* ham_out,
                      int32_t* num_rejected, int32_t tuning, float* workspace, const hmcx_sink_t* sink, void* stream);

/* hmcx_split_run with a sample sink (sink == NULL: identical to hmcx_split_run, which runs as a thin = 1 sink).  In the
 * Bayesian-NN kernel the CTAs of a chain's cluster divide each retained row and its moment updates between them, and the
 * rows go out as 16-byte streaming stores (what pinned host samples_out wants); samples, flags and step sizes are those of
 * hmcx_split_run.  sum / sumsq are read and updated in place at every post-burn iteration, so without sum_lo / sumsq_lo
 * they are plain fp32 running sums: pass both for the compensated sums.  Windows of iterations chain through the
 * accumulators.  thin < 1, sum_lo without sum or sumsq_lo without sumsq: HMCX_ERR_INVALID_ARG. */
int hmcx_split_run_sink(const hmcx_target_t* target, const hmcx_mass_t* mass, const hmcx_rng_t* rng,
                        const hmcx_nuts_t* nuts, int32_t scheme,
                        const float* q_init, float* q_cur, float* eps,
                        int32_t C, int32_t ld, int32_t L, int32_t num_samples, int32_t burn,
                        int32_t iter_begin, int32_t iter_end,
                        float* samples_out, uint8_t* accept_out, uint8_t* diverged_out, float* ham_out,
                        int32_t* num_rejected, const hmcx_sink_t* sink, void* stream);

/*
 * Gamma hyperpriors on the precisions of a Bayesian NN (hmcx_split_run_hyper).  Group k < 2L is parameter tensor k in
 * tau_list order (each Linear's weight, then its bias): w_k ~ Normal(0, tau_k^-1/2), tau_k ~ Gamma(a[k], b[k]) (shape,
 * rate); group 2L is the regression likelihood's precision tau_out ~ Gamma(a[2L], b[2L]).  Every iteration n, after the MH
 * step gives q_n, each sampled group is drawn from its conditional
 *   tau_k ~ Gamma(a_k + n_k / 2, b_k + |w_k|^2 / 2),   tau_out ~ Gamma(a_o + N O / 2, b_o + SSE(q_n) / 2)
 * (n_k = the tensor's size, N = data rows over all splits, O = outputs; |w_k|^2 a fixed-order fp64 sum, SSE the sum over
 * splits of the MH evaluation's squared errors), and iteration n + 1 uses them.  Draws: PHILOX mode Marsaglia-Tsang in fp64
 * on its own counter stream, keyed by (seed, chain_offset + c, n, k, attempt) as hmcx_hyper_gamma_draws writes them;
 * INJECTED mode the standard-gamma draws `gammas`; tau_k = (float)(g / rate).
 *   sampled[k]     non-zero: group k is Gibbs-updated (a[k], b[k] > 0 and finite); zero: fixed at the target's value
 *   tau, tau_out   [C, 2L] / [C] device in/out: the chains' current precisions (initialise them to the target's tau_list /
 *                  tau_out); windows of iterations chain through them
 *   tau_trace, tau_out_trace   optional [C, keep, 2L] / [C, keep] device: the precisions of every retained sample slot
 *                  (the sink's slots, thinned alike; slot 0 = the initial values)
 *   gammas         INJECTED: [iter_end - iter_begin, C, 2L + 1] fp64 device, entry k of row (n, c) the Gamma(shape_k, 1)
 *                  draw of group k (entries of fixed groups are not read)
 */
#define HMCX_HYPER_GROUPS (2 * HMCX_MLP_MAX_LAYERS + 1)
typedef struct hmcx_hyper {
    int32_t sampled[HMCX_HYPER_GROUPS];
    double  a[HMCX_HYPER_GROUPS];
    double  b[HMCX_HYPER_GROUPS];
    float*  tau;
    float*  tau_out;
    float*  tau_trace;
    float*  tau_out_trace;
    const double* gammas;
} hmcx_hyper_t;

/* hmcx_split_run_sink with Gamma hyperpriors (hyper == NULL: identical to hmcx_split_run_sink; sink == NULL with a hyper:
 * a thin = 1 sink).  Checked before any CUDA work: a sampled group outside [0, 2L], a or b not in (0, inf), NULL tau /
 * tau_out, INJECTED without gammas, a tau_out prior without data: HMCX_ERR_INVALID_ARG; a tau_out prior with a
 * classification loss (tau_out tempers those likelihoods, it is not a noise precision): HMCX_ERR_UNSUPPORTED.  The
 * proposal's log p and any gradient carried into the next trajectory belong to the old precisions: after each update the
 * kernel re-evaluates log p(q_n) (one forward pass) and starts the next trajectory with a fresh gradient. */
int hmcx_split_run_hyper(const hmcx_target_t* target, const hmcx_mass_t* mass, const hmcx_rng_t* rng,
                         const hmcx_nuts_t* nuts, int32_t scheme,
                         const float* q_init, float* q_cur, float* eps,
                         int32_t C, int32_t ld, int32_t L, int32_t num_samples, int32_t burn,
                         int32_t iter_begin, int32_t iter_end,
                         float* samples_out, uint8_t* accept_out, uint8_t* diverged_out, float* ham_out,
                         int32_t* num_rejected, const hmcx_sink_t* sink, const hmcx_hyper_t* hyper, void* stream);

/* The PHILOX-mode standard-gamma draws of hmcx_split_run_hyper, from the same device function: out[n - iter_begin, c, k] =
 * the Gamma(shapes[k], 1) draw of group k, chain chain_offset + c, iteration n.  shapes: HOST array of K <=
 * HMCX_HYPER_GROUPS values in (0, inf); out: [iter_end - iter_begin, C, K] fp64 device.  Other arguments out of range:
 * HMCX_ERR_INVALID_ARG. */
int hmcx_hyper_gamma_draws(uint64_t seed, uint64_t chain_offset, int32_t C, int32_t iter_begin, int32_t iter_end,
                           int32_t K, const double* shapes, double* out, void* stream);

/*
 * Replica exchange (parallel tempering) for Bayesian NNs (additive v12 symbols; DESIGN §3.17).  Callers of an older v12
 * library check for the symbols.  The C rows form R = C / T ladders laid out ladder-major: row r*T + t runs rung t of
 * ladder r, the power posterior p(theta) L(theta)^beta_t, which is the target with tau_out replaced by beta_t * tau_out
 * (every loss is linear in its c_ll).  Rung 0 is beta = 1.
 *   num_temps      T in [1, HMCX_TEMPER_MAX_TEMPS]; C must be a multiple of T
 *   tau_out        HOST values: rung t's tau_out, rounded to fp32 as hmcx_mlp_t.tau_out holds it; finite, >= 0,
 *                  non-increasing in t.  The kernel derives the rung's c_ll from it as it does from hmcx_mlp_t.tau_out.
 *   ll_out         optional [C] fp64 device: when the launch ends, the UNTEMPERED log-likelihood at q_cur, sum over splits
 *                  of c_ll * loss_m (the log-softmax loss: c_ll * loss_m / n_m, its per-split mean), c_ll the target's
 *                  own; the value the kernel's last MH evaluation of q_cur produced (no extra forward pass).
 */
#define HMCX_TEMPER_MAX_TEMPS 32
typedef struct hmcx_temper {
    int32_t num_temps;
    float   tau_out[HMCX_TEMPER_MAX_TEMPS];
    double* ll_out;
} hmcx_temper_t;

/* hmcx_split_run_sink with every row at its rung (the sink form; sink == NULL: a thin = 1 sink).  Samples are stored for
 * rung 0 only: row r*T of the ladders goes to row r of samples_out, [C / T, keep, ld]; accept / diverged / ham / step
 * sizes / num_rejected and the sink moments stay per row ([C, ...]).  Windows of iterations chain through q_cur as in
 * hmcx_split_run_sink (log p(q_cur) is re-evaluated at the start of every launch), so q_cur rows may be exchanged between
 * two launches.  Checked before any CUDA work: NULL target or temper, T out of range, C % T != 0, a tau_out value that is
 * negative, not finite or larger than its predecessor, the sink checks of hmcx_split_run_sink: HMCX_ERR_INVALID_ARG;
 * non-MLP targets: HMCX_ERR_UNSUPPORTED; otherwise the checks of hmcx_split_run_sink. */
int hmcx_split_run_temper(const hmcx_target_t* target, const hmcx_mass_t* mass, const hmcx_rng_t* rng,
                          const hmcx_nuts_t* nuts, int32_t scheme,
                          const float* q_init, float* q_cur, float* eps,
                          int32_t C, int32_t ld, int32_t L, int32_t num_samples, int32_t burn,
                          int32_t iter_begin, int32_t iter_end,
                          float* samples_out, uint8_t* accept_out, uint8_t* diverged_out, float* ham_out,
                          int32_t* num_rejected, const hmcx_sink_t* sink, const hmcx_temper_t* temper, void* stream);

/* Swap round `round` of the ladders: deterministic even-odd pairing, the pairs (t, t + 1) with t = round (mod 2).  Pair t of
 * ladder r swaps when  log u < (beta_t - beta_{t+1}) (ll[r*T + t + 1] - ll[r*T + t])  in fp64; an accepted pair exchanges
 * its two q_cur rows (16-byte copies), nothing else.  accepted[r*(T-1) + t] = 1 / 0, or -1 where the pair is not in this
 * round.  One thread per (ladder, pair) decides, no atomics: the same bytes on every call.
 *   betas          HOST [T] fp64: betas[0] == 1, strictly decreasing, finite, >= 0
 *   ll             [C] fp64 device (hmcx_temper_t.ll_out of the launch before)
 *   rng            PHILOX: log u = log((double)u01(x)), x word 0 of the Philox block with counter (t, round, STREAM_SWAP << 24,
 *                  ladder lo) and key (seed lo, seed hi ^ ladder hi), ladder = chain_offset / T + r, so the decisions do not
 *                  depend on how ladders are sharded (chain_offset must be a multiple of T); INJECTED: log_uniforms
 *                  [R, T - 1] fp64 device (this round's)
 * NULL pointers, C < 1, T < 2 or > HMCX_TEMPER_MAX_TEMPS, C % T != 0, ld < 4 or not a multiple of 4, q_cur not 16-byte
 * aligned, round < 0, bad betas, a PHILOX chain_offset that is not a multiple of T, an unknown rng mode:
 * HMCX_ERR_INVALID_ARG. */
int hmcx_temper_swap(float* q_cur, int32_t C, int32_t ld, int32_t num_temps, const double* betas, const double* ll,
                     int32_t round, const hmcx_rng_t* rng, const double* log_uniforms, int8_t* accepted, void* stream);

/*
 * K-fold refits of a Bayesian NN in one launch (additive v12 symbol; DESIGN §3.18).  Callers of an older v12 library check
 * for the symbol.  hmcx_split_run_sink (sink may be NULL) with the target's K = num_folds splits read as K training sets:
 * split k holds the rows of fold k's fit (every row not in fold k, in data order).  The chain with GLOBAL id
 * g = rng->chain_offset + c evaluates split g mod K as its whole potential -- ll of that split plus the prior once -- in
 * every gradient, both Hamiltonians and the gradient carried between iterations, i.e. it samples what hmcx_split_run_sink
 * with HMCX_SCHEME_PLAIN samples on a target holding split k alone.  The automatic cluster size counts the tiles of the
 * smallest split, a whole training set.  Checked before any CUDA work: NULL target, num_folds < 2 or
 * > HMCX_MLP_MAX_SPLITS, num_splits != num_folds, a target without data, the sink checks of hmcx_split_run_sink:
 * HMCX_ERR_INVALID_ARG; non-MLP targets and a scheme other than HMCX_SCHEME_PLAIN: HMCX_ERR_UNSUPPORTED; otherwise the
 * checks of hmcx_split_run_sink.
 */
int hmcx_split_run_folds(const hmcx_target_t* target, const hmcx_mass_t* mass, const hmcx_rng_t* rng,
                         const hmcx_nuts_t* nuts, int32_t scheme,
                         const float* q_init, float* q_cur, float* eps,
                         int32_t C, int32_t ld, int32_t L, int32_t num_samples, int32_t burn,
                         int32_t iter_begin, int32_t iter_end,
                         float* samples_out, uint8_t* accept_out, uint8_t* diverged_out, float* ham_out,
                         int32_t* num_rejected, const hmcx_sink_t* sink, int32_t num_folds, void* stream);

/*
 * hmcx_adapt_diag_mass (ABI v11): the pooled diagonal mass estimate at the end of a warm-up window (Stan's windowed
 * adaptation, regularised as Stan does) and the restart of the dual averaging that follows it.  One pass, fixed order, no
 * atomics.  Inputs: the per-chain compensated sums of a window of n >= 2 draws, [C, ld] each, as a sink launch with
 * moments_all leaves them (sum, sumsq, sum_lo, sumsq_lo; true sums hi + lo).  Per dimension d < D, in fp64:
 *   m_c = S1_c / n,   v_c = (S2_c - S1_c * m_c) / (n - 1),   W = (sum_{c = 0..C-1} v_c, in that order) / C,   N = C * n,
 *   var = (N / (N + 5)) * W + 1e-3 * (5 / (N + 5))
 * inv_mass[d] = (float)var and mass_factor[d] = sqrtf(1 / inv_mass[d]) in IEEE fp32 (the hmcx_mass_t DIAG pair: bit-equal
 * to what the Python binding builds from the same inv_mass on the device); lanes D..ld-1 of both are written as 0.  The four sums are
 * zeroed (all ld lanes) for the next window.  For the C_chains chains whose step size adapts on this device:
 *   mu_chain[c] = log(10 * eps[c]) (10 * eps in fp32, then the correctly rounded fp32 log), h_bar[c] = 0, eps_bar[c] = 1.
 * C and C_chains differ when the sums were gathered from several devices (all chains, global order) and this device
 * restarts its own chains only.  NULL pointers, C < 1, C_chains < 1, n < 2, D < 1, ld < D or ld % 4 != 0:
 * HMCX_ERR_INVALID_ARG.
 */
int hmcx_adapt_diag_mass(float* sum, float* sumsq, float* sum_lo, float* sumsq_lo, int32_t C, int32_t ld, int32_t D,
                         int32_t n, const float* eps, int32_t C_chains, float* inv_mass, float* mass_factor,
                         double* mu_chain, double* h_bar, double* eps_bar, void* stream);

/*
 * hmcx_copy_rows_async: `height` rows of `width` bytes from `src` (row pitch `spitch`) to `dst` (row pitch `dpitch`), either
 * side device or PINNED host memory, enqueued on `stream` (cudaMemcpy2DAsync, cudaMemcpyDefault).  The delivery half of a
 * windowed run: hmcx_hmc_run over iterations [a, b) on one stream, then the window's sample slots -- the same columns of
 * every chain's [num_samples-burn, ld] block -- leave for the host on a second stream through the copy engine while the next
 * window computes (the reference's store_on_GPU=False, samplers.py:1008-1012, without stalling the chains on PCIe).
 */
int hmcx_copy_rows_async(void* dst, size_t dpitch, const void* src, size_t spitch, size_t width, size_t height,
                         void* stream);

/*
 * Convergence diagnostics of a sample block (ABI v9): the two streaming passes behind split-R-hat, effective sample size
 * and Monte-Carlo standard error (Stan reference manual; hamiltorch_b200/diagnostics.py runs the Geyer scan on their
 * output).  The block is fp32 x[c, s, d] = x[c*chain_stride + s*draw_stride + d] (strides in elements, unit stride along
 * D): C chains of n >= 4 draws.  Half-chain 2c is draws [0, m) of chain c and 2c+1 is draws [n-m, n), m = n/2 (an odd n
 * drops the middle draw).  All sums are fp64 and run in a fixed order (no atomics): the same block gives the same bits.
 * The stages are separate calls so that ranks holding different chains can all-reduce between them.
 *   hmcx_diag_means  mu_out [2C, D] fp64: the mean of every half-chain;  mu_sum_out [D] fp64: sum over half-chains of mu
 *   hmcx_diag_acov   acov_out [HMCX_DIAG_LAG_BLOCK, D] fp64: row k = sum_j gamma_j(lag_begin + k),
 *                    gamma_j(t) = (1/m) sum_{s < m-t} (x_s - mu_j)(x_{s+t} - mu_j) over half-chain j (0 for t >= m);
 *                    mu = hmcx_diag_means' mu_out.  With mu_bar [D] (the pooled mean of the half-chain means, may be
 *                    NULL) between_out [D] = sum_j (mu_j - mu_bar)^2.
 * NULL x / outputs, C < 1, n < 4, D < 1, negative strides or lag_begin: HMCX_ERR_INVALID_ARG.
 */
#define HMCX_DIAG_LAG_BLOCK 32

int hmcx_diag_means(const float* x, int64_t chain_stride, int64_t draw_stride, int32_t C, int32_t n, int32_t D,
                    double* mu_out, double* mu_sum_out, void* stream);
int hmcx_diag_acov(const float* x, int64_t chain_stride, int64_t draw_stride, int32_t C, int32_t n, int32_t D,
                   const double* mu, const double* mu_bar, int32_t lag_begin, double* acov_out, double* between_out,
                   void* stream);

/*
 * Rank-normalised diagnostics (ABI v10): the passes behind rank-normalised, folded split-R-hat, bulk-ESS and tail-ESS
 * (Vehtari, Gelman, Simpson, Carpenter & Buerkner 2021; hamiltorch_b200/diagnostics.py::rank_summary feeds their blocks
 * through hmcx_diag_means / hmcx_diag_acov).  Same block layout as the v9 entries; L = C*n must be at most
 * HMCX_RANK_MAX_DRAWS.  The split set is the draws of the half-chains above (Ns = 2*C*(n/2)); the full set is all L.
 *   hmcx_rank_workspace_bytes  bytes of sort workspace a slab of k dimensions needs (0 for invalid arguments).  The
 *                    library never allocates: the caller passes the workspace to every hmcx_rank_pass.
 *   hmcx_rank_pass   for the dimensions d in [d0, d0 + k): per draw of the split set, with r its average rank (ties share
 *                    the mean of their positions; -0.0 ties with +0.0) among the split draws,
 *                    bulk_z[c, s, d] = (float) Phi^-1((r - 3/8) / (Ns + 1/4)), and fold_z the same with the ranks of
 *                    |x - median|; both blocks hold 0 at the dropped middle draw of an odd n.  Each block has its own
 *                    strides (unit stride along D).  quantiles [3, D] fp64: rows q05, median, q95 of the full set
 *                    (np.quantile(method='linear') / np.median arithmetic; NaN for a non-finite dimension);
 *                    nonfinite [D] int32: 1 where the dimension has a non-finite draw, else 0.  Deterministic: the
 *                    outputs depend on the block only, not on the slab.
 *   hmcx_rank_indicator  out[c, s, d] = x[c, s, d] <= thr[d] (fp64 comparison) as fp32 0 / 1, thr [D] fp64.
 * NULL pointers, C < 1, n < 4, D < 1, L too large, negative strides, a slab outside [0, D), k > HMCX_RANK_MAX_SLAB
 * or a workspace smaller than hmcx_rank_workspace_bytes(C, n, k): HMCX_ERR_INVALID_ARG.  The quantiles equal numpy's
 * as values; a zero quantile is always +0.0 (numpy may return -0.0, which compares equal).
 */
#define HMCX_RANK_MAX_DRAWS 2147418112      /* 2^31 - 2^16: draw indices and tile arithmetic stay in int32 */
#define HMCX_RANK_MAX_SLAB 65535            /* dimensions per hmcx_rank_pass: one grid row per dimension */

size_t hmcx_rank_workspace_bytes(int32_t C, int32_t n, int32_t k);
int hmcx_rank_pass(const float* x, int64_t chain_stride, int64_t draw_stride, int32_t C, int32_t n, int32_t D,
                   int32_t d0, int32_t k, float* bulk_z, int64_t bulk_chain_stride, int64_t bulk_draw_stride,
                   float* fold_z, int64_t fold_chain_stride, int64_t fold_draw_stride, double* quantiles,
                   int32_t* nonfinite, void* workspace, size_t workspace_bytes, void* stream);
int hmcx_rank_indicator(const float* x, int64_t chain_stride, int64_t draw_stride, int32_t C, int32_t n, int32_t D,
                        const double* thr, float* out, int64_t out_chain_stride, int64_t out_draw_stride, void* stream);

/*
 * Model comparison for Bayesian NNs (ABI v12): PSIS-LOO and WAIC (Vehtari, Gelman & Gabry 2017; hamiltorch_b200/loo.py).
 *   hmcx_mlp_pointwise_ll  ll_out[c, s, i - row_begin] = log p(y_i | theta_{c,s}) for the data rows [row_begin, row_end)
 *                    of an HMCX_TARGET_MLP target (split targets: rows in split order), draw theta_{c,s} at samples +
 *                    c*chain_stride + s*draw_stride (unit stride along D).  One CTA per draw runs the forward pass of
 *                    hmcx_mlp_predict (SIMT tiles, or the tensor-core form when x_packed is set) over the target's own
 *                    x / y / x_packed in place; the network outputs stay in shared memory.  Per row, f = network output:
 *                      REGRESSION      sum_o -0.5 tau_out (f_o - y_o)^2 + 0.5 O log(tau_out / 2 pi)
 *                      BINARY          sum_o -BCEWithLogits(f_o, y_o)
 *                      MULTICLASS      log_softmax(f)[y]
 *                      .._LOGSOFTMAX   f[y]
 *                    tau_out (a tempering of the classification likelihoods while sampling) is not part of the last three.
 *                    NULL pointers, C < 1, n < 1, C*n > INT32_MAX, negative strides, a target without data or a row range
 *                    outside [0, num_rows) or empty: HMCX_ERR_INVALID_ARG; other target kinds: HMCX_ERR_UNSUPPORTED.
 *   hmcx_loo_workspace_bytes  sort workspace a slab of k points needs (0 for invalid arguments).
 *   hmcx_loo_pass    for the points i in [i0, i0 + k) of an fp32 block ll[c, s, i] (strides as the v9 entries, N points,
 *                    S = C*n >= 2 pooled draws per point): the segmented radix sort of hmcx_rank_pass, then per point in fp64
 *                    r = -ll - max(-ll); M = ceil(min(0.2 S, 3 sqrt(S / r_eff))); cutoff = max(the (M+1)-th largest r,
 *                    log DBL_MIN); tail = {r > cutoff}, M' = its size (tail_size[i]); for M' > 4 the Zhang-Stephens GPD fit
 *                    of the exceedances exp(r) - exp(cutoff) gives k-hat and sigma, and the tail's log-ratios become
 *                    log(q_z + exp(cutoff)), q_z the GPD quantile at (z - 1/2)/M'; M' <= 4: k-hat = +inf, no smoothing.
 *                    Log-ratios capped at 0 and normalised: lw.  pointwise [6, N] fp64, rows:
 *                      0 elpd_loo = logsumexp(lw + ll)       1 p_loo = lppd - elpd_loo      2 pareto_k = k-hat
 *                      3 lppd = logsumexp(ll) - log S        4 p_waic = var(ll) (ddof 1)    5 elpd_waic = lppd - p_waic
 *                    nonfinite [N] int32: 1 where the point has a non-finite draw (its six outputs are NaN).  Fixed-order
 *                    sums, no atomics: the outputs depend on the block only, not on the slab.  NULL pointers, C < 1,
 *                    n < 1, S < 2 or > HMCX_RANK_MAX_DRAWS, negative strides, a slab outside [0, N), k >
 *                    HMCX_RANK_MAX_SLAB, r_eff not in (0, inf) or a workspace smaller than hmcx_loo_workspace_bytes(C, n,
 *                    k): HMCX_ERR_INVALID_ARG.
 */
int hmcx_mlp_pointwise_ll(const hmcx_target_t* target, const float* samples, int64_t chain_stride, int64_t draw_stride,
                          int32_t C, int32_t n, int32_t row_begin, int32_t row_end, float* ll_out,
                          int64_t ll_chain_stride, int64_t ll_draw_stride, void* stream);
/* hmcx_mlp_pointwise_ll with a per-draw tau_out (the draws of a run with a tau_out hyperprior, hmcx_split_run_hyper):
 * draw (c, s) uses tau_out[c*tau_chain_stride + s*tau_draw_stride] (fp32 device) in the regression density, its constant
 * 0.5 O log(tau / 2 pi) evaluated in fp64 and rounded to fp32 as hmcx_mlp_pointwise_ll does for the target's tau_out.
 * tau_out == NULL: identical to hmcx_mlp_pointwise_ll.  Classification losses do not read it.  Negative tau strides:
 * HMCX_ERR_INVALID_ARG; otherwise the checks of hmcx_mlp_pointwise_ll. */
int hmcx_mlp_pointwise_ll_tau(const hmcx_target_t* target, const float* samples, int64_t chain_stride,
                              int64_t draw_stride, int32_t C, int32_t n, int32_t row_begin, int32_t row_end,
                              const float* tau_out, int64_t tau_chain_stride, int64_t tau_draw_stride, float* ll_out,
                              int64_t ll_chain_stride, int64_t ll_draw_stride, void* stream);
size_t hmcx_loo_workspace_bytes(int32_t C, int32_t n, int32_t k);
int hmcx_loo_pass(const float* ll, int64_t chain_stride, int64_t draw_stride, int32_t C, int32_t n, int32_t N,
                  int32_t i0, int32_t k, double r_eff, double* pointwise, int32_t* tail_size, int32_t* nonfinite,
                  void* workspace, size_t workspace_bytes, void* stream);

/*
 * Held-out evaluation of Bayesian NNs (additive v12 symbols; hamiltorch_b200/predictive.py).  Callers of an older v12
 * library check for the symbols.
 *   hmcx_mlp_pointwise_out  out[c*out_chain_stride + s*out_draw_stride + (i - row_begin)*O + o] = output o of the network
 *                    of draw (c, s) at data row i in [row_begin, row_end), O the output width: the values hmcx_mlp_predict
 *                    writes for that row (log-probabilities for HMCX_LOSS_MULTICLASS_LOGSOFTMAX), bit for bit, computed
 *                    with the tile loop of hmcx_mlp_pointwise_ll (SIMT tiles, or the tensor-core form when x_packed is
 *                    set; split targets: rows in split order, read in place).  Argument checks as hmcx_mlp_pointwise_ll:
 *                    NULL pointers, C < 1, n < 1, C*n > INT32_MAX, negative strides, a target without data or a row range
 *                    outside [0, num_rows) or empty: HMCX_ERR_INVALID_ARG; other target kinds: HMCX_ERR_UNSUPPORTED.
 *   hmcx_pred_workspace_bytes  workspace hmcx_pred_pass needs for a slab of k points: 8 (2n + 46 + n R) k bytes with
 *                    R = O + 4 (multi-class), 3 O + 2 (binary) or 3 O + 4 (regression) per-step sums (0 for C < 1, n < 1,
 *                    C*n > INT32_MAX, O < 1, k < 1 or an unknown loss).
 *   hmcx_pred_pass   for the points i in [i0, i0 + k) of an fp32 block f[c, s, i, o] at f + c*chain_stride +
 *                    s*draw_stride + i*O + o (C chains of n draws, N points): the posterior predictive over the S = C*n
 *                    pooled draws, in fp64, and the curves over the first t draws of every chain (St = C*t draws).
 *                    y: fp32 targets, [N, O] (regression, binary) or [N] labels in [0, O) (multi-class, both losses).
 *                    tau_out: fp32 per-draw noise precision at tau_out + c*tau_chain_stride + s*tau_draw_stride
 *                    (regression only; a stride of 0 repeats one value; classification may pass NULL).
 *                      MULTICLASS*   p = softmax(f) per draw, pbar = its mean; label argmax pbar (lowest on ties);
 *                                    nll = -(logsumexp_s log p_s[y] - log S)
 *                      BINARY        each output a Bernoulli, pbar = mean sigmoid(f); predicted pbar > 0.5, correct when
 *                                    it equals y > 0.5; nll, brier, entropies summed over the outputs; log p(y) =
 *                                    y log sigmoid(f) + (1 - y) log sigmoid(-f)
 *                      REGRESSION    mu = mean f, var = mean 1/tau + var f (ddof 0), ll_s = sum_o -0.5 tau (f_o - y_o)^2
 *                                    + 0.5 O log(tau / 2 pi), lppd = logsumexp_s ll_s - log S, pit = mean Phi((y - f)
 *                                    sqrt(tau))
 *                    pointwise [7, N] fp64 rows: 0 nll (regression -lppd), 1 brier (regression sum_o (mu_o - y_o)^2),
 *                      2 entropy H[pbar], 3 mean_s H[p_s], 4 mutual information 2 - 3, 5 correct predictions of the
 *                      point, 6 predicted label (multi-class; rows 2-6 are 0 where they do not apply).
 *                    per_output [1, N, O] fp64 (classification: pbar) or [4, N, O] (regression: mu, var, var f, pit).
 *                    nonfinite [N] int32: 1 where the point has a non-finite output (all its outputs are NaN).
 *                    partials [2n + 46, ceil(N / 128)] fp64, the sums of 128-point groups aligned to the point index,
 *                    each in point order, continued across slabs (so every slab of a call sequence that covers [0, N) in
 *                    order adds to the same array); rows: t - 1 < n: correct predictions with St draws (regression:
 *                    squared error of the St-draw mean); n + t - 1: nll with St draws; 2n: brier; 2n + 1 + 3b .. 3 + 3b:
 *                    count, confidence sum, correct sum of confidence bin b ((b/15, (b + 1)/15], b < 15; top label,
 *                    binary: max(pbar, 1 - pbar) per output); regression 2n .. 2n + 3: the outputs with |pit - 0.5| <=
 *                    level / 2 for levels 0.5, 0.8, 0.9, 0.95.  No atomics: the results depend on the block alone.
 *                    NULL pointers (tau_out for regression), C < 1, n < 1, O < 1, N < 1, k < 1, negative strides, a slab
 *                    outside [0, N), an unknown loss or a workspace smaller than
 *                    hmcx_pred_workspace_bytes(C, n, O, loss, k): HMCX_ERR_INVALID_ARG; running sums beyond one SM's
 *                    shared memory (128 (1, 3 or 4) O doubles): HMCX_ERR_UNSUPPORTED.  The pass sums the C draws of
 *                    every step t per point in parallel (fp64, chain order) into the workspace, then scans t per point.
 *   hmcx_pred_totals totals[r] = sum over groups of partials[r, :] in group order, 2n + 46 rows, once every slab is in.
 *                    NULL pointers, n < 1 or N < 1: HMCX_ERR_INVALID_ARG.
 */
int hmcx_mlp_pointwise_out(const hmcx_target_t* target, const float* samples, int64_t chain_stride,
                           int64_t draw_stride, int32_t C, int32_t n, int32_t row_begin, int32_t row_end, float* out,
                           int64_t out_chain_stride, int64_t out_draw_stride, void* stream);
size_t hmcx_pred_workspace_bytes(int32_t C, int32_t n, int32_t O, int32_t loss, int32_t k);
int hmcx_pred_pass(const float* f, int64_t chain_stride, int64_t draw_stride, int32_t C, int32_t n, int32_t O,
                   int32_t loss, const float* y, const float* tau_out, int64_t tau_chain_stride, int64_t tau_draw_stride,
                   int32_t N, int32_t i0, int32_t k, double* pointwise, double* per_output, int32_t* nonfinite,
                   double* partials, void* workspace, size_t workspace_bytes, void* stream);
int hmcx_pred_totals(const double* partials, int32_t n, int32_t N, double* totals, void* stream);

/*
 * Simulation-based calibration of Bayesian NNs (additive v12 symbols; DESIGN §3.19, hamiltorch_b200/sbc.py).  Callers of
 * an older v12 library check for the symbols.  Sim m (GLOBAL id sim_begin + local index) draws from two Philox streams
 * whose chain word is m, so a sim's values do not depend on how many sims a call holds:
 *   prior  (stream 6) counter (v, j lo, j hi | 6 << 24, m lo), key (seed lo, seed hi ^ m hi)
 *   data   (stream 7) the same counter layout with j = 0
 * Normals are the canonical Box-Muller of the momentum stream: words (x, y) -> elements 4v, 4v + 1, (z, w) -> 4v + 2, 4v + 3;
 * uniforms are u01(word) = fma((float)word, 2^-32, 2^-33) in (0, 1].
 *   hmcx_sbc_prior     out[m, j, :] [M, 1 + R, ld] fp32: row j = 0 is the sim's true parameter vector, row 1 + r the start
 *                      of chain r, element d < D = z_d sqrt(prior_scale / tau_k) (tau_k = 2 / prior_two_var[k], k the
 *                      parameter tensor holding d), lanes D .. ld - 1 written as 0.
 *   hmcx_sbc_simulate  y from the network outputs f [M, num_rows, O] fp32 (hmcx_mlp_pointwise_out of the true parameters):
 *                        REGRESSION  y [M, num_rows, O] = f + z / sqrt(tau_out), z the normals of the flattened (row, o)
 *                        BINARY      y [M, num_rows, O] = 1 if u01(word e mod 4 of vector e / 4) < sigmoid(f_e) (fp64)
 *                                    else 0, e the flattened (row, o)
 *                        MULTICLASS  y [M, num_rows] = the first class c with u sum_c' exp(f_c' - max f) <= the same sum
 *                                    over c' <= c (fp64, class order; O - 1 if none), u = u01(word x of vector = row)
 *                      The log-softmax loss is not a likelihood of independent labels (nll_loss takes the mean), and a
 *                      classification tau_out other than 1 tempers the likelihood: both HMCX_ERR_UNSUPPORTED.
 *   hmcx_sbc_rank      ranks[m, d] [K, D] int32 = #{(r, s) : x[r K + m, s, d] < truth[m, d]}, r < C / K, 1 <= s < keep,
 *                      x[c, s, d] at samples + c chain_stride + s draw_stride + d, truth[m, d] at truth + m truth_stride + d
 *                      (fp32 comparisons: NaN draws and ties count as "not less").  Slot 0 (params_init) is not a draw.
 * NULL pointers, a target without data, M < 1, R < 0, ld < D or not a multiple of 4, C < 1, K < 1, C % K != 0, keep < 2,
 * D < 1, negative strides: HMCX_ERR_INVALID_ARG; non-MLP targets and the two refused likelihoods: HMCX_ERR_UNSUPPORTED.
 */
int hmcx_sbc_prior(const hmcx_target_t* target, uint64_t seed, int64_t sim_begin, int32_t M, int32_t R, int32_t ld,
                   float* out, void* stream);
int hmcx_sbc_simulate(const hmcx_target_t* target, const float* f, uint64_t seed, int64_t sim_begin, int32_t M,
                      float* y_out, void* stream);
int hmcx_sbc_rank(const float* samples, int64_t chain_stride, int64_t draw_stride, int32_t C, int32_t keep, int32_t K,
                  int32_t D, const float* truth, int64_t truth_stride, int32_t* ranks_out, void* stream);

/*
 * Posterior predictive checks of Bayesian NNs (additive v12 symbols; DESIGN §3.20, hamiltorch_b200/ppc.py).  Callers of
 * an older v12 library check for the symbols.
 *   hmcx_ppc_pass    for a slab of k posterior draws, draw j the pooled draw g = draws[j] (int64 device, g = c n + s) with
 *                    network outputs f [k, num_rows, O] fp32 (hmcx_mlp_pointwise_out): one replicated data set per draw
 *                    from Philox stream 8, counter (v, 0, 8 << 24, g lo), key (seed lo, seed hi ^ g hi), with the element
 *                    definitions of hmcx_sbc_simulate (v the vector of 4 flattened outputs e = i O + o for regression
 *                    and binary, v = row for multi-class; both multi-class losses draw from softmax f), written to
 *                    y_rep [k, num_rows, y_cols] (y_cols = O, or 1 for multi-class).  Regression noise sd =
 *                    1 / sqrt(tau), tau = tau_out[j] (fp32 device), or the target's tau_out when tau_out is NULL.
 *                    stats [k, K] fp64, K = 4 O + 1 (regression: mean, sd (ddof 1), min, max of each output column in
 *                    column order), O + 1 (binary: the mean of each column; multi-class: the frequency of each class);
 *                    column K - 1 the deviance -2 sum_i ll_i(y_rep | theta_g), dev_obs [k] = -2 sum_i ll_i(y | theta_g)
 *                    with y the target's data and ll the density of hmcx_mlp_pointwise_ll_tau evaluated in fp64 from the
 *                    fp32 outputs.  nonfinite [k] int32: 1 where the draw has a non-finite output (its statistics and
 *                    deviances are NaN).  One CTA per draw, fixed-order fp64 sums, no atomics: a draw's results depend on
 *                    (seed, g, its outputs) only.  NULL pointers (tau_out excepted), a target without data, k < 1 or a
 *                    non-positive target tau_out with tau_out NULL (regression): HMCX_ERR_INVALID_ARG; non-MLP targets:
 *                    HMCX_ERR_UNSUPPORTED.
 *   hmcx_loo_pit_pass  LOO-PIT of the points [i0, i0 + k) of a regression: the sort and the Pareto smoothing of
 *                    hmcx_loo_pass on the log-likelihood block ll (the same arguments, N points), then per point i and
 *                    output o in fp64 pit[i, o] = sum_p w_p Phi((y[i, o] - f[c_p, s_p, i, o]) sqrt(tau[c_p, s_p])) over the
 *                    sorted draws p, w_p the normalised smoothed weights exp(lw_p) and (c_p, s_p) the draw the stable sort
 *                    put at p; Phi(x) = erfc(-x / sqrt 2) / 2.  f at f + c*f_chain_stride + s*f_draw_stride + i*O + o, y
 *                    [N, O] fp32, tau at tau_out + c*tau_chain_stride + s*tau_draw_stride (a stride of 0 repeats one
 *                    value).  pit [N, O], pareto_k [N] fp64 (k-hat, the bits hmcx_loo_pass writes for the same block and
 *                    r_eff), nonfinite [N] int32 (1: NaN pit and k-hat).  Workspace: hmcx_loo_workspace_bytes(C, n, k).
 *                    The checks of hmcx_loo_pass, and NULL f / y / tau_out, O < 1 or negative strides:
 *                    HMCX_ERR_INVALID_ARG.
 */
int hmcx_ppc_pass(const hmcx_target_t* target, const float* f, int32_t k, const int64_t* draws, uint64_t seed,
                  const float* tau_out, float* y_rep, double* stats, double* dev_obs, int32_t* nonfinite, void* stream);
int hmcx_loo_pit_pass(const float* ll, int64_t chain_stride, int64_t draw_stride, const float* f, int64_t f_chain_stride,
                      int64_t f_draw_stride, int32_t C, int32_t n, int32_t O, int32_t N, int32_t i0, int32_t k,
                      double r_eff, const float* y, const float* tau_out, int64_t tau_chain_stride,
                      int64_t tau_draw_stride, double* pit, double* pareto_k, int32_t* nonfinite, void* workspace,
                      size_t workspace_bytes, void* stream);

/*
 * Stacking of chains and models (additive v12 symbols; DESIGN §3.21, hamiltorch_b200/loo.py).  Callers of an older v12
 * library check for the symbols.
 *   hmcx_loo_chain_pass  per-chain PSIS-LOO of the points [i0, i0 + k) of the block ll (the strides of hmcx_loo_pass, N
 *                    points): for every chain c the PSIS-LOO of hmcx_loo_pass over that chain's n draws alone, M =
 *                    ceil(min(0.2 n, 3 sqrt(n / r_eff))).  One CTA per (point, chain) sorts the chain's n keys in shared
 *                    memory, so n <= HMCX_LOO_CHAIN_MAX_DRAWS; no workspace.  out [3, C, N] fp64, rows: 0 elpd_loo,
 *                    1 lppd, 2 pareto_k -- column c the bits hmcx_loo_pass writes (rows 0, 3, 2) for the one-chain block
 *                    of chain c; tail_size [C, N] int32 (M'); nonfinite [C, N] int32 (1: the chain has a non-finite draw
 *                    at the point, its three outputs NaN).  NULL pointers, C < 1 or > 65535, n < 2 or >
 *                    HMCX_LOO_CHAIN_MAX_DRAWS, negative strides, a slab outside [0, N), k > HMCX_RANK_MAX_SLAB or r_eff
 *                    not in (0, inf): HMCX_ERR_INVALID_ARG.
 *   hmcx_stack_workspace_bytes  workspace of hmcx_stack_eval / hmcx_stack_em: 8 (K N + (K + 1) ceil(N / 128)) bytes (0 for
 *                    K < 1, K > 65535, N < 1 or K N > INT32_MAX).
 *   hmcx_stack_eval  for E [K, N] fp64 and weights w [K] fp64 (device): pointwise [N] = m_i + log sum_k w_k exp(E_ki - m_i),
 *                    m_i = max_k E_ki (rows with w_k = 0 add nothing); objective [1] = sum_i pointwise_i; grad [K] =
 *                    sum_i exp(E_ki - m_i) / s_i, s_i the inner sum.  Sums over points in 128-point groups in point
 *                    order, then the groups in order; no atomics, so the same inputs give the same bits.
 *   hmcx_stack_em    `iterations` rounds of: hmcx_stack_eval at w, then, unless max_k grad_k <= N (1 + tol) (state[0] :=
 *                    1, and every later round of this and later calls does nothing), w_k := w_k grad_k / N and state[1]
 *                    += 1.  state [2] int32 device (0, 0 to start).  Once converged, objective / grad / pointwise hold
 *                    the evaluation at the returned w.
 *                    NULL pointers, bad shapes, iterations < 1, tol not in [0, inf) or a workspace smaller than
 *                    hmcx_stack_workspace_bytes(K, N): HMCX_ERR_INVALID_ARG.
 *   hmcx_pred_pass_weighted  hmcx_pred_pass over the mixture sum_c w_c (chain c's draws, equally weighted), chain_weights
 *                    [C] fp64 device, non-negative and summing to 1: every per-step sum takes chain c's terms scaled by
 *                    C w_c and its log-densities shifted by log(C w_c); chains with w_c = 0 are not read (but the first
 *                    draw of chain 0 is the regression moments' shift).  Curves: the mixture of the first t draws of every
 *                    chain.  The checks of hmcx_pred_pass, and NULL chain_weights: HMCX_ERR_INVALID_ARG.
 */
#define HMCX_LOO_CHAIN_MAX_DRAWS 8192          /* 2 n uint32 keys of a chain in 64 KB of shared memory */
int hmcx_loo_chain_pass(const float* ll, int64_t chain_stride, int64_t draw_stride, int32_t C, int32_t n, int32_t N,
                        int32_t i0, int32_t k, double r_eff, double* out, int32_t* tail_size, int32_t* nonfinite,
                        void* stream);
size_t hmcx_stack_workspace_bytes(int32_t K, int32_t N);
int hmcx_stack_eval(const double* E, int32_t K, int32_t N, const double* w, double* objective, double* grad,
                    double* pointwise, void* workspace, size_t workspace_bytes, void* stream);
int hmcx_stack_em(const double* E, int32_t K, int32_t N, double tol, int32_t iterations, double* w, double* objective,
                  double* grad, double* pointwise, int32_t* state, void* workspace, size_t workspace_bytes,
                  void* stream);
int hmcx_pred_pass_weighted(const float* f, int64_t chain_stride, int64_t draw_stride, int32_t C, int32_t n, int32_t O,
                            int32_t loss, const float* y, const float* tau_out, int64_t tau_chain_stride,
                            int64_t tau_draw_stride, int32_t N, int32_t i0, int32_t k, double* pointwise,
                            double* per_output, int32_t* nonfinite, double* partials, void* workspace,
                            size_t workspace_bytes, const double* chain_weights, void* stream);

/*
 * Power-scaling prior and likelihood sensitivity (additive v12 symbols; DESIGN §3.22, hamiltorch_b200/sensitivity.py).
 * Callers of an older v12 library check for the symbols.  Draws are pooled as g = c n + s, S = C n.
 *   hmcx_mlp_log_prior  out [S] fp64 (device) = sum over the parameter tensors t with tau[t] > 0 of the Normal(0,
 *                    tau_t^-1/2) log density of the tensor's entries, -tau_t / 2 sum_i w_i^2 + n_t / 2 (log tau_t - log
 *                    2 pi), in fp64.  The tensors are consecutive in the draw, sizes [num_tensors] and tau [num_tensors]
 *                    are host arrays (tau 0: the tensor is left out).  One CTA per draw reads the draw once; the sums
 *                    are in a fixed order.  NULL pointers, a bad shape, num_tensors not in [1, 2 HMCX_MLP_MAX_LAYERS],
 *                    a size < 1 or a tau that is negative or not finite: HMCX_ERR_INVALID_ARG.
 *   hmcx_psens_ll_totals  totals [S] fp64 (device) += sum_i coef[r0 + i] ll[c, s, i] over the slab's rows i in [0, k)
 *                    (ll[c, s, i] at ll + c chain_stride + s draw_stride + i; coef NULL: 1), in 128-row groups in row
 *                    order, each group a fixed-order sum.  With r0 a multiple of 128 and totals zeroed before the first
 *                    slab, the totals are the same bits for every split of the rows into slabs.  r0 not a multiple of
 *                    128 or the checks below: HMCX_ERR_INVALID_ARG.
 *   hmcx_psens_workspace_bytes  workspace of hmcx_psens_weights (k = K) and hmcx_psens_pass for a slab of k columns.
 *   hmcx_psens_weights  the Pareto-smoothed importance weights of K log-ratio columns: neg_log_ratio [C, n, K] fp32 holds
 *                    -r (unit stride along K), each column smoothed as hmcx_loo_pass smooths a point's ll (M =
 *                    ceil(min(0.2 S, 3 sqrt(S / r_eff)))).  weights [K, S] fp64 the normalised weights in flat-draw
 *                    order, pareto_k [K], tail_size [K] (M'), nonfinite [K] (1: a non-finite -r, NaN weights and k-hat).
 *   hmcx_psens_pass  for the columns [d0, d0 + k) of x (the strides of hmcx_rank_pass, D columns) and the weights
 *                    [HMCX_PSENS_SETS, S] of hmcx_psens_weights: out [HMCX_PSENS_ROWS, D] fp64, rows 0..3 the cumulative
 *                    Jensen-Shannon distance max(cjs+, cjs-) of each weight set against equal weights, 4 the mean, 5..8
 *                    the weighted means, 9 the sd, 10..13 the weighted sds; nonfinite [D] (1: a non-finite draw, NaN in
 *                    every row).  Fixed-order sums, no atomics: the outputs depend on the inputs alone.
 *   For the three workspace users: NULL pointers, negative strides, C n < 2 or > HMCX_RANK_MAX_DRAWS, n < 1, a slab
 *   outside [0, D), k (or K) not in [1, HMCX_RANK_MAX_SLAB], r_eff not in (0, inf) or a workspace smaller than
 *   hmcx_psens_workspace_bytes: HMCX_ERR_INVALID_ARG.
 */
#define HMCX_PSENS_SETS 4
#define HMCX_PSENS_ROWS 14
int hmcx_mlp_log_prior(const float* samples, int64_t chain_stride, int64_t draw_stride, int32_t C, int32_t n,
                       int32_t num_tensors, const int32_t* sizes, const double* tau, double* out, void* stream);
int hmcx_psens_ll_totals(const float* ll, int64_t chain_stride, int64_t draw_stride, int32_t C, int32_t n, int32_t r0,
                         int32_t k, const double* coef, double* totals, void* stream);
size_t hmcx_psens_workspace_bytes(int32_t C, int32_t n, int32_t k);
int hmcx_psens_weights(const float* neg_log_ratio, int64_t chain_stride, int64_t draw_stride, int32_t C, int32_t n,
                       int32_t K, double r_eff, double* weights, double* pareto_k, int32_t* tail_size,
                       int32_t* nonfinite, void* workspace, size_t workspace_bytes, void* stream);
int hmcx_psens_pass(const float* x, int64_t chain_stride, int64_t draw_stride, int32_t C, int32_t n, int32_t D,
                    int32_t d0, int32_t k, const double* weights, double* out, int32_t* nonfinite, void* workspace,
                    size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* HMCX_H */
