"""ctypes binding of libhmcx.so (include/hmcx.h).  No torch types cross the boundary: tensors are passed as raw
device pointers (``Tensor.data_ptr()``) plus sizes, the CUDA stream as an opaque ``void*``.

The product path FAILS LOUDLY when the library is missing or no CUDA device is present -- there is no CPU
fallback (the CPU restatement lives in oracle/ and is test infrastructure only).
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'lib', 'libhmcx.so')

OK, ERR_INVALID_ARG, ERR_UNSUPPORTED, ERR_CUDA = 0, -1, -2, -3
MASS_NONE, MASS_DIAG, MASS_FULL = 0, 1, 2
RNG_INJECTED, RNG_PHILOX = 0, 1
ABI_VERSION = 12


class NativeError(RuntimeError):
    pass


MLP_MAX_LAYERS, MLP_MAX_SPLITS = 8, 64
SCHEME_PLAIN, SCHEME_SPLIT_SYM, SCHEME_SPLIT_RAND, SCHEME_SPLIT_KMID = 0, 1, 2, 3


class MlpStruct(C.Structure):
    _fields_ = [('num_layers', C.c_int32), ('widths', C.c_int32 * (MLP_MAX_LAYERS + 1)),
                ('activation', C.c_int32 * MLP_MAX_LAYERS), ('loss', C.c_int32), ('tau_out', C.c_float),
                ('prior_scale', C.c_float), ('prior_two_var', C.c_float * (2 * MLP_MAX_LAYERS)),
                ('prior_log_scale', C.c_float * (2 * MLP_MAX_LAYERS)),
                ('prior_grad_coef', C.c_float * (2 * MLP_MAX_LAYERS)), ('x', C.c_void_p), ('y', C.c_void_p),
                ('num_rows', C.c_int32), ('num_splits', C.c_int32), ('split_begin', C.c_int32 * (MLP_MAX_SPLITS + 1)),
                ('cluster_size', C.c_int32), ('tensor_cores', C.c_int32), ('x_packed', C.c_void_p)]


class TargetStruct(C.Structure):
    _fields_ = [('kind', C.c_int32), ('dim', C.c_int32), ('mean', C.c_void_p), ('inv_var', C.c_void_p),
                ('prec', C.c_void_p), ('log_norm', C.c_float), ('funnel_inv_var_v', C.c_float),
                ('mlp', C.POINTER(MlpStruct))]


class MassStruct(C.Structure):
    _fields_ = [('kind', C.c_int32), ('inv_mass', C.c_void_p), ('mass_factor', C.c_void_p)]


class RngStruct(C.Structure):
    _fields_ = [('mode', C.c_int32), ('seed', C.c_uint64), ('chain_offset', C.c_uint64),
                ('normals', C.c_void_p), ('log_uniforms', C.c_void_p), ('perms', C.c_void_p),
                ('uniforms', C.c_void_p), ('uniforms_per_iter', C.c_int32)]


class RmhmcStruct(C.Structure):
    _fields_ = [('integrator', C.c_int32), ('metric', C.c_int32), ('softabs_const', C.c_float), ('jitter', C.c_float),
                ('pi_term', C.c_float), ('cos_2we', C.c_float), ('sin_2we', C.c_float),
                ('fixed_point_threshold', C.c_float), ('fixed_point_max_iterations', C.c_int32),
                ('jitter_max_tries', C.c_int32)]


class ConstMetricStruct(C.Structure):
    _fields_ = [('metric_inv', C.c_void_p), ('metric_chol', C.c_void_p), ('log_det', C.c_float)]


class SinkStruct(C.Structure):
    _fields_ = [('thin', C.c_int32), ('sum', C.c_void_p), ('sumsq', C.c_void_p), ('sum_lo', C.c_void_p),
                ('sumsq_lo', C.c_void_p), ('moments_all', C.c_int32)]


HYPER_GROUPS = 2 * MLP_MAX_LAYERS + 1


class HyperStruct(C.Structure):
    _fields_ = [('sampled', C.c_int32 * HYPER_GROUPS), ('a', C.c_double * HYPER_GROUPS), ('b', C.c_double * HYPER_GROUPS),
                ('tau', C.c_void_p), ('tau_out', C.c_void_p), ('tau_trace', C.c_void_p), ('tau_out_trace', C.c_void_p),
                ('gammas', C.c_void_p)]


TEMPER_MAX_TEMPS = 32


class TemperStruct(C.Structure):
    _fields_ = [('num_temps', C.c_int32), ('tau_out', C.c_float * TEMPER_MAX_TEMPS), ('ll_out', C.c_void_p)]


class NutsStruct(C.Structure):
    _fields_ = [('enabled', C.c_int32), ('desired_accept_rate', C.c_double), ('mu', C.c_double),
                ('table', C.c_void_p), ('h_bar', C.c_void_p), ('eps_bar', C.c_void_p),
                ('eps_schedule', C.c_void_p), ('eps_trace', C.c_void_p), ('step_size_init', C.c_double),
                ('mu_chain', C.c_void_p)]


_PROTOS = {
    'hmcx_abi_version': (C.c_int, []),
    'hmcx_status_string': (C.c_char_p, [C.c_int]),
    'hmcx_leapfrog': (C.c_int, [C.POINTER(TargetStruct), C.POINTER(MassStruct), C.c_void_p, C.c_void_p, C.c_void_p,
                                C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                C.c_void_p]),
    'hmcx_hamiltonian': (C.c_int, [C.POINTER(TargetStruct), C.POINTER(MassStruct), C.c_void_p, C.c_void_p,
                                   C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    'hmcx_gibbs': (C.c_int, [C.POINTER(MassStruct), C.POINTER(RngStruct), C.c_int32, C.c_int32, C.c_int32,
                             C.c_int64, C.c_void_p, C.c_void_p]),
    'hmcx_hmc_run': (C.c_int, [C.POINTER(TargetStruct), C.POINTER(MassStruct), C.POINTER(RngStruct),
                               C.POINTER(NutsStruct), C.c_void_p, C.c_void_p, C.c_void_p,
                               C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                               C.c_void_p]),
    'hmcx_hmc_workspace_bytes': (C.c_size_t, [C.POINTER(TargetStruct), C.POINTER(MassStruct), C.c_int32, C.c_int32]),
    'hmcx_split_run': (C.c_int, [C.POINTER(TargetStruct), C.POINTER(MassStruct), C.POINTER(RngStruct),
                                 C.POINTER(NutsStruct), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                 C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'hmcx_rmhmc_run': (C.c_int, [C.POINTER(TargetStruct), C.POINTER(RmhmcStruct), C.POINTER(RngStruct), C.c_void_p,
                                 C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                 C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_void_p]),
    'hmcx_rmhmc_leapfrog': (C.c_int, [C.POINTER(TargetStruct), C.POINTER(RmhmcStruct), C.POINTER(RngStruct), C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'hmcx_rmhmc_hamiltonian': (C.c_int, [C.POINTER(TargetStruct), C.POINTER(RmhmcStruct), C.POINTER(RngStruct),
                                         C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                         C.c_void_p]),
    'hmcx_rmhmc_dense_workspace_bytes': (C.c_size_t, [C.c_int32, C.c_int32]),
    'hmcx_rmhmc_dense_run': (C.c_int, [C.POINTER(TargetStruct), C.POINTER(RmhmcStruct), C.POINTER(ConstMetricStruct),
                                       C.POINTER(RngStruct), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                       C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'hmcx_hmc_run_sink': (C.c_int, [C.POINTER(TargetStruct), C.POINTER(MassStruct), C.POINTER(RngStruct),
                                    C.POINTER(NutsStruct), C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                    C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                                    C.POINTER(SinkStruct), C.c_void_p]),
    'hmcx_split_run_sink': (C.c_int, [C.POINTER(TargetStruct), C.POINTER(MassStruct), C.POINTER(RngStruct),
                                      C.POINTER(NutsStruct), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.POINTER(SinkStruct), C.c_void_p]),
    'hmcx_split_run_hyper': (C.c_int, [C.POINTER(TargetStruct), C.POINTER(MassStruct), C.POINTER(RngStruct),
                                       C.POINTER(NutsStruct), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.POINTER(SinkStruct), C.POINTER(HyperStruct), C.c_void_p]),
    'hmcx_split_run_temper': (C.c_int, [C.POINTER(TargetStruct), C.POINTER(MassStruct), C.POINTER(RngStruct),
                                        C.POINTER(NutsStruct), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.POINTER(SinkStruct), C.POINTER(TemperStruct), C.c_void_p]),
    'hmcx_split_run_folds': (C.c_int, [C.POINTER(TargetStruct), C.POINTER(MassStruct), C.POINTER(RngStruct),
                                       C.POINTER(NutsStruct), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.POINTER(SinkStruct), C.c_int32, C.c_void_p]),
    'hmcx_temper_swap': (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_double), C.c_void_p,
                                   C.c_int32, C.POINTER(RngStruct), C.c_void_p, C.c_void_p, C.c_void_p]),
    'hmcx_hyper_gamma_draws': (C.c_int, [C.c_uint64, C.c_uint64, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                         C.POINTER(C.c_double), C.c_void_p, C.c_void_p]),
    'hmcx_gemm_nt_tf32x3': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    'hmcx_copy_rows_async': (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p]),
    'hmcx_grad_log_prob': (C.c_int, [C.POINTER(TargetStruct), C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                     C.c_void_p, C.c_void_p, C.c_void_p]),
    'hmcx_mlp_predict': (C.c_int, [C.POINTER(TargetStruct), C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                                   C.c_void_p, C.c_void_p]),
    'hmcx_split_leapfrog': (C.c_int, [C.POINTER(TargetStruct), C.POINTER(MassStruct), C.POINTER(RngStruct), C.c_int32,
                                      C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                      C.c_void_p, C.c_void_p, C.c_void_p]),
    'hmcx_mlp_packed_x_bytes': (C.c_size_t, [C.POINTER(TargetStruct)]),
    'hmcx_mlp_pack_x': (C.c_int, [C.POINTER(TargetStruct), C.c_void_p, C.c_void_p]),
    'hmcx_diag_means': (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                  C.c_void_p, C.c_void_p]),
    'hmcx_diag_acov': (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                 C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    'hmcx_rank_workspace_bytes': (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32]),
    'hmcx_rank_pass': (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                 C.c_int32, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_int64,
                                 C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    'hmcx_adapt_diag_mass': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                       C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p]),
    'hmcx_rank_indicator': (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                      C.c_void_p, C.c_int64, C.c_int64, C.c_void_p]),
    'hmcx_mlp_pointwise_ll': (C.c_int, [C.POINTER(TargetStruct), C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32,
                                        C.c_int32, C.c_int32, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p]),
    'hmcx_mlp_pointwise_ll_tau': (C.c_int, [C.POINTER(TargetStruct), C.c_void_p, C.c_int64, C.c_int64, C.c_int32,
                                            C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int64, C.c_int64,
                                            C.c_void_p, C.c_int64, C.c_int64, C.c_void_p]),
    'hmcx_loo_workspace_bytes': (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32]),
    'hmcx_loo_pass': (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    'hmcx_mlp_pointwise_out': (C.c_int, [C.POINTER(TargetStruct), C.c_void_p, C.c_int64, C.c_int64, C.c_int32,
                                         C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int64, C.c_int64,
                                         C.c_void_p]),
    'hmcx_pred_workspace_bytes': (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    'hmcx_pred_pass': (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                 C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32,
                                 C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    'hmcx_pred_totals': (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    'hmcx_sbc_prior': (C.c_int, [C.POINTER(TargetStruct), C.c_uint64, C.c_int64, C.c_int32, C.c_int32, C.c_int32,
                                 C.c_void_p, C.c_void_p]),
    'hmcx_sbc_simulate': (C.c_int, [C.POINTER(TargetStruct), C.c_void_p, C.c_uint64, C.c_int64, C.c_int32, C.c_void_p,
                                    C.c_void_p]),
    'hmcx_sbc_rank': (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                C.c_int64, C.c_void_p, C.c_void_p]),
    'hmcx_ppc_pass': (C.c_int, [C.POINTER(TargetStruct), C.c_void_p, C.c_int32, C.c_void_p, C.c_uint64, C.c_void_p,
                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'hmcx_loo_pit_pass': (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int32,
                                    C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_void_p,
                                    C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_size_t, C.c_void_p]),
    'hmcx_loo_chain_pass': (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                      C.c_int32, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'hmcx_stack_workspace_bytes': (C.c_size_t, [C.c_int32, C.c_int32]),
    'hmcx_stack_eval': (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_size_t, C.c_void_p]),
    'hmcx_stack_em': (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_double, C.c_int32, C.c_void_p, C.c_void_p,
                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    'hmcx_pred_pass_weighted': (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32,
                                          C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int32,
                                          C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    'hmcx_mlp_log_prior': (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32,
                                     C.POINTER(C.c_int32), C.POINTER(C.c_double), C.c_void_p, C.c_void_p]),
    'hmcx_psens_ll_totals': (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                       C.c_void_p, C.c_void_p, C.c_void_p]),
    'hmcx_psens_workspace_bytes': (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32]),
    'hmcx_psens_weights': (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_double,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                     C.c_void_p]),
    'hmcx_psens_pass': (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                  C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
}

DIAG_LAG_BLOCK = 32                     # HMCX_DIAG_LAG_BLOCK: lags per hmcx_diag_acov pass
RANK_MAX_DRAWS = 2147418112             # HMCX_RANK_MAX_DRAWS: largest C*n hmcx_rank_pass takes
RANK_MAX_SLAB = 65535                   # HMCX_RANK_MAX_SLAB: most dimensions per hmcx_rank_pass
LOO_CHAIN_MAX_DRAWS = 8192              # HMCX_LOO_CHAIN_MAX_DRAWS: most draws per chain hmcx_loo_chain_pass sorts
PSENS_SETS, PSENS_ROWS = 4, 14          # HMCX_PSENS_SETS / HMCX_PSENS_ROWS: weight sets and output rows of hmcx_psens_pass

EXPORTED_SYMBOLS = tuple(_PROTOS)

_lib = None


def load_library():
    """dlopen libhmcx.so and attach prototypes.  Raises NativeError if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NativeError(
            'hamiltorch_b200: %s not found.  Build it with `python -m hamiltorch_b200.build` (needs nvcc, '
            'cross-compiles sm_90a without a GPU).  There is no CPU fallback.' % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in _PROTOS.items():
        fn = getattr(lib, name)          # AttributeError here = header/library mismatch
        fn.restype = res
        fn.argtypes = args
    if lib.hmcx_abi_version() != ABI_VERSION:
        raise NativeError('libhmcx.so ABI %d != binding ABI %d: rebuild' % (lib.hmcx_abi_version(), ABI_VERSION))
    _lib = lib
    return lib


def require_cuda():
    if not torch.cuda.is_available():
        raise NativeError('hamiltorch_b200 needs a CUDA device (sm_90a); there is no CPU fallback. '
                          'The CPU restatement under oracle/ is test infrastructure only.')


def check(status, what):
    if status != OK:
        msg = load_library().hmcx_status_string(status).decode()
        raise NativeError('%s failed: %s (%d)' % (what, msg, status))


def ptr(t):
    """Raw device pointer of a tensor (None -> NULL)."""
    if t is None:
        return None
    return C.c_void_p(t.data_ptr())


def stream_ptr(device):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def padded_ld(dim):
    return (int(dim) + 3) // 4 * 4


def pad_rows(x, ld):
    """(C, D) fp32 -> contiguous (C, ld) with zero pad columns."""
    if x.shape[-1] == ld and x.is_contiguous():
        return x
    out = x.new_zeros(x.shape[:-1] + (ld,))
    out[..., :x.shape[-1]] = x
    return out
