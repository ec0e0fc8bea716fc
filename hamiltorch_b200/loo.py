"""Model comparison for Bayesian NNs on the GPU: Pareto-smoothed importance-sampling leave-one-out cross-validation
(PSIS-LOO; Vehtari, Gelman & Gabry 2017, Vehtari, Simpson, Gelman, Yao & Gabry 2024) and WAIC -- what Stan's ``loo``,
ArviZ's ``az.loo`` / ``az.waic`` and PyMC report, restated in numpy fp64 by tests/loo_oracle.py.

    ll = hamiltorch_b200.loo.pointwise_log_lik(res, target)     # (C, n, N) fp32: log p(y_i | theta_{c,s})
    lo = hamiltorch_b200.loo.psis_loo(res, target)              # or psis_loo(ll)
    lo.elpd_loo, lo.se, lo.pareto_k.max(), lo.num_bad_k
    hamiltorch_b200.loo.compare(lo_a, lo_b)                     # elpd differences to the best model
    lo = hamiltorch_b200.loo.reloo(lo, target, params_init, num_samples=..., ...)   # exact refits where k-hat is high
    f = hamiltorch_b200.loo.kfold_split(N, K)                   # K-fold CV: one launch fits every fold
    kf = hamiltorch_b200.loo.kfold(sample_chains(target, params_init, folds=f, ...), target)
    st = hamiltorch_b200.loo.chain_stacking(res, target)        # chain weights of a non-mixing run (psis_loo_chains)
    hamiltorch_b200.loo.stacking_weights(lo_a, lo_b)            # model stacking weights

``target`` is the ``MLPTarget`` of ``define_model_log_prob`` or the list ``define_split_model_log_prob`` returns (data
points in split order).  Two CUDA passes:
  * hmcx_mlp_pointwise_ll: one CTA per draw runs the network over the target's own device data (the SIMT tiles, or the
    3xTF32 tensor-core forward of n0 -> 128 -> nL stacks) and writes one log-likelihood per data row; the network outputs
    never reach device memory.  Regression: the normalised Gaussian density with noise precision ``tau_out``.
    Classification: the categorical / Bernoulli density of the network's logits -- ``tau_out`` tempers these
    likelihoods while sampling but is NOT part of the predictive density LOO and WAIC score.
  * hmcx_loo_pass: per data point, the segmented radix sort of rank_summary over the S = C*n pooled draws, then one fp64
    pass: tail cut, Zhang & Stephens generalised-Pareto fit, smoothed importance weights, LOO and WAIC terms.
Samples plus a target are processed in slabs of data points, so the (S, N) log-likelihood block is never held whole:
each slab's block and sort workspace fit in ``diagnostics.RANK_WORKSPACE_BUDGET`` bytes (at least one point per slab).
"""
import copy
import ctypes as C
import math

import torch

from . import _native as N
from . import diagnostics as _diag
from . import targets as T

_slab_points_override = None            # tests: force this many data points per slab
_ROW_TILE = 128                         # slab boundaries of the likelihood pass: whole tiles of the packed data operand
_ROWS = ('elpd_loo', 'p_loo', 'pareto_k', 'lppd', 'p_waic', 'elpd_waic')


class LooResult:
    """``psis_loo``: per point (N,) fp64 on the block's device -- ``pointwise`` (elpd_loo_i), ``p_loo_i``,
    ``pareto_k``, ``lppd``, ``tail_size`` (int32, M'); totals (Python floats) ``elpd_loo``, ``se``, ``p_loo``,
    ``p_loo_se``, ``looic`` = -2 elpd_loo, ``looic_se``; ``k_threshold`` = min(1 - 1/log10 S, 0.7), ``num_bad_k``
    (points with pareto_k above it), ``num_nonfinite`` (points with a non-finite draw: NaN outputs, and NaN totals),
    ``num_points``, ``num_draws``, ``r_eff``."""

    kind = 'loo'

    def __repr__(self):
        return ('LooResult(elpd_loo=%.3f, se=%.3f, p_loo=%.3f, N=%d, S=%d, bad k-hat=%d, nonfinite=%d)'
                % (self.elpd_loo, self.se, self.p_loo, self.num_points, self.num_draws, self.num_bad_k,
                   self.num_nonfinite))


class WaicResult:
    """``waic``: per point (N,) fp64 -- ``pointwise`` (elpd_waic_i), ``p_waic``, ``lppd``; totals ``elpd_waic``,
    ``se``, ``p_waic_total``, ``p_waic_se``, ``waic`` = -2 elpd_waic, ``waic_se``; ``num_p_waic_warn`` (points with
    p_waic_i > 0.4), ``num_nonfinite``, ``num_points``, ``num_draws``."""

    kind = 'waic'

    def __repr__(self):
        return ('WaicResult(elpd_waic=%.3f, se=%.3f, p_waic=%.3f, N=%d, S=%d, p_waic > 0.4: %d, nonfinite=%d)'
                % (self.elpd_waic, self.se, self.p_waic_total, self.num_points, self.num_draws, self.num_p_waic_warn,
                   self.num_nonfinite))


class Comparison:
    """``compare``: ``elpd`` per model (input order), ``elpd_diff`` = elpd - elpd of the best model (<= 0, 0 for the
    best), ``se_diff`` = sqrt(N) sd(pointwise difference to the best, ddof 1) (0 for the best), ``order`` = model
    indices from best to worst."""

    def __init__(self, elpd, elpd_diff, se_diff, order):
        self.elpd, self.elpd_diff, self.se_diff, self.order = elpd, elpd_diff, se_diff, order

    def __repr__(self):
        rows = ['  model %d: elpd %.3f, elpd_diff %.3f, se_diff %.3f' % (i, self.elpd[i], self.elpd_diff[i],
                                                                         self.se_diff[i]) for i in self.order]
        return 'Comparison(\n%s)' % '\n'.join(rows)


# ------------------------------------------------------------------------------------------------------------------
# Inputs
# ------------------------------------------------------------------------------------------------------------------
def _mlp_targets(target, prefix, use):
    """The MLPTargets of an MLPTarget or a split list, each with data; errors read '<prefix>: ...' and name what the
    points are for (``use``: 'leave out', 'evaluate')."""
    items = target if isinstance(target, list) else [target]
    if not items or not all(isinstance(t, T.MLPTarget) for t in items):
        raise TypeError('%s: the target must be an MLPTarget (define_model_log_prob) or the list '
                        'define_split_model_log_prob returns, got %s' % (prefix, type(target).__name__))
    if any(t.x is None for t in items):
        raise RuntimeError('%s: the target has no data (x is None): there are no points to %s' % (prefix, use))
    return items


def _check_r_eff(r_eff):
    r = float(r_eff)
    if not (r > 0.0 and math.isfinite(r)):
        raise ValueError('loo: r_eff must be a finite positive number, got %r' % (r_eff,))
    return r


def _samples_block(samples, target):
    first = _mlp_targets(target, 'loo', 'leave out')[0]
    if torch.is_tensor(samples) and samples.dim() in (2, 3) and samples.shape[-1] != first.dim:
        raise RuntimeError('loo: the samples have %d parameters per draw, the target has %d'
                           % (samples.shape[-1], first.dim))
    x = _diag.as_block(samples)
    if x.shape[2] != first.dim:
        raise RuntimeError('loo: the samples have %d parameters per draw, the target has %d'
                           % (x.shape[2], first.dim))
    return x


def _tau_block(samples, x, tau_out):
    """The per-draw tau_out of the (C, n, D) block x as a (C, n) fp32 tensor on its device, or None (the target's).
    Explicit ``tau_out``: (C, n), or (n,) for an (n, D) block / a single chain; otherwise an ``HMCResult`` of a run with
    tau_out_prior brings its ``tau_out_trace`` (the same slots as its samples)."""
    if tau_out is None:
        tau_out = getattr(samples, 'tau_out_trace', None)
        if tau_out is None:
            return None
    t = torch.as_tensor(tau_out).detach().to(device=x.device, dtype=torch.float32)
    if t.dim() == 1 and x.shape[0] == 1:
        t = t[None]
    if tuple(t.shape) != (x.shape[0], x.shape[1]):
        raise RuntimeError('loo: tau_out must hold one value per draw, (C, n) = (%d, %d), got %s'
                           % (x.shape[0], x.shape[1], tuple(t.shape)))
    if not bool((t > 0).all()) or not bool(torch.isfinite(t).all()):
        raise ValueError('loo: tau_out must be positive and finite')
    return t


def _native_target(target, device):
    from .engine import native_target
    return native_target(target, device)


# ------------------------------------------------------------------------------------------------------------------
# Pointwise log-likelihood
# ------------------------------------------------------------------------------------------------------------------
def _ll_rows(lib, nt, x, r0, r1, out, tau=None):
    """out[c, s, :] = ll of rows [r0, r1) (out a (C, n, r1 - r0) view with unit stride along its last dimension);
    tau: the (C, n) per-draw tau_out, or None for the target's."""
    tcs, tds = (0, 0) if tau is None else (tau.stride(0), tau.stride(1))
    rc = lib.hmcx_mlp_pointwise_ll_tau(nt.ref(), N.ptr(x), x.stride(0), x.stride(1), int(x.shape[0]), int(x.shape[1]),
                                       r0, r1, N.ptr(tau), tcs, tds, N.ptr(out), out.stride(0), out.stride(1),
                                       N.stream_ptr(x.device))
    N.check(rc, 'hmcx_mlp_pointwise_ll_tau')


def pointwise_log_lik(samples, target, tau_out=None):
    """The (C, n, N) fp32 CUDA tensor ll[c, s, i] = log p(y_i | theta_{c,s}) of every draw and data point.

    ``samples``: what ``diagnostics.summary`` accepts (an ``HMCResult``, a (C, n, D) / (n, D) CUDA fp32 tensor, the list
    ``sample`` returns), refused in the same cases.  ``target``: an ``MLPTarget`` with data, or the list of split
    descriptors (points in split order).  Per point, with f the network output (O values) and tau = tau_out:
    regression sum_o -0.5 tau (f_o - y_o)^2 + 0.5 O log(tau / 2 pi); binary sum_o -BCEWithLogits(f_o, y_o);
    multi-class log_softmax(f)[y]; LogSoftmax output f[y].  tau_out does not enter the classification densities.
    ``tau_out``: one noise precision per draw, (C, n) (or (n,) for one chain), for draws of a run with a tau_out
    hyperprior; an ``HMCResult`` of such a run brings its ``tau_out_trace`` without it.  None: the target's tau_out."""
    x = _samples_block(samples, target)
    tau = _tau_block(samples, x, tau_out)
    N.require_cuda()
    lib = N.load_library()
    nt = _native_target(target, x.device)
    Np = int(nt.mlp_struct.num_rows)
    out = torch.empty((x.shape[0], x.shape[1], Np), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        _ll_rows(lib, nt, x, 0, Np, out, tau)
    return out


# ------------------------------------------------------------------------------------------------------------------
# PSIS / WAIC pass
# ------------------------------------------------------------------------------------------------------------------
def _slab_points(lib, C_, n, Np, extra_per_point=0):
    """Points per slab: the sort workspace (and, from samples, the slab's fp32 likelihood block) within the budget."""
    if _slab_points_override is not None:
        return max(1, min(Np, N.RANK_MAX_SLAB, int(_slab_points_override)))
    budget = _diag.RANK_WORKSPACE_BUDGET
    cost = lambda k: lib.hmcx_loo_workspace_bytes(C_, n, k) + k * extra_per_point
    k = max(1, min(Np, N.RANK_MAX_SLAB, budget // cost(1)))
    while k > 1 and cost(k) > budget:
        k -= 1
    if extra_per_point and _ROW_TILE <= k < Np:
        k -= k % _ROW_TILE
    return k


def _pointwise_pass(x, target, r_eff, tau=None, nt=None, rows=None):
    """(C, n, N) draws -> (pw (6, N) fp64, tail (N,) int32, flag (N,) int32, S, N).  ``nt`` / ``rows``: the native
    form of ``target`` when the caller built it, and the data rows [r0, r1) of it to score (default: all of them)."""
    N.require_cuda()
    lib = N.load_library()
    dev = x.device
    C_, n = int(x.shape[0]), int(x.shape[1])
    S = C_ * n
    if S > N.RANK_MAX_DRAWS:
        raise RuntimeError('loo: %d chains x %d draws exceed the %d draws per point the sort indexes'
                           % (C_, n, N.RANK_MAX_DRAWS))
    if target is None:
        Np = int(x.shape[2])
        k = _slab_points(lib, C_, n, Np)
        nt = None
    else:
        nt = _native_target(target, dev) if nt is None else nt
        r0, r1 = (0, int(nt.mlp_struct.num_rows)) if rows is None else rows
        Np = r1 - r0
        k = _slab_points(lib, C_, n, Np, extra_per_point=4 * S)
    pw = torch.empty((6, Np), dtype=torch.float64, device=dev)
    tail = torch.empty(Np, dtype=torch.int32, device=dev)
    flag = torch.empty(Np, dtype=torch.int32, device=dev)
    ws_bytes = lib.hmcx_loo_workspace_bytes(C_, n, k)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        st = N.stream_ptr(dev)
        blk = None if nt is None else torch.empty((C_, n, k), dtype=torch.float32, device=dev)
        for i0 in range(0, Np, k):
            kk = min(k, Np - i0)
            if nt is None:
                src, base = x, N.ptr(x)
            else:
                _ll_rows(lib, nt, x, r0 + i0, r0 + i0 + kk, blk, tau)
                # the pass reads point i at column i of the block: the slab's block holds columns [i0, i0 + kk)
                src, base = blk, C.c_void_p(blk.data_ptr() - 4 * i0)
            rc = lib.hmcx_loo_pass(base, src.stride(0), src.stride(1), C_, n, Np, i0, kk, float(r_eff), N.ptr(pw),
                                   N.ptr(tail), N.ptr(flag), N.ptr(ws), ws_bytes, st)
            N.check(rc, 'hmcx_loo_pass')
        del ws
    return pw, tail, flag, S, Np


def _total(v):
    """(sum, sqrt(N) * sd(v, ddof 1)) of a per-point fp64 tensor, as Python floats."""
    n = v.numel()
    s = float(v.sum())
    se = float(math.sqrt(n) * v.std(unbiased=True)) if n > 1 else float('nan')
    return s, se


def _prepare(x, target, r_eff=None, tau_out=None):
    if r_eff is not None:
        r_eff = _check_r_eff(r_eff)
    if target is None:
        if tau_out is not None:
            raise RuntimeError('loo: tau_out applies to samples with a target, not to a log-likelihood block')
        return _diag.as_block(x), r_eff, None
    blk = _samples_block(x, target)
    return blk, r_eff, _tau_block(x, blk, tau_out)


def psis_loo(x, target=None, r_eff=1.0, tau_out=None):
    """PSIS-LOO of a Bayesian NN on the GPU.

    ``x``: a log-likelihood block ll[c, s, i] -- a (C, n, N) or (n, N) CUDA fp32 tensor, e.g. ``pointwise_log_lik``'s
    -- or, with ``target``, the samples (read like ``diagnostics.summary`` reads them) whose likelihood is computed slab
    by slab.  ``r_eff``: the relative efficiency of the draws' importance ratios (1 for independent draws), which sets
    the tail length M = ceil(min(0.2 S, 3 sqrt(S / r_eff))).  Per point i over its S = C*n pooled draws (fp64):
    r = -ll shifted to max 0; the tail is the draws with r above the (M+1)-th largest r (ties at the cutoff stay out);
    with more than 4 tail draws a generalised Pareto distribution is fitted to their exceedances (Zhang & Stephens 2009,
    with Vehtari et al.'s prior: pareto_k = (M' xi + 5)/(M' + 10)) and their log-ratios replaced by its quantiles,
    otherwise pareto_k = inf; the log-ratios are capped at 0 and normalised (lw); elpd_loo_i = logsumexp(lw + ll),
    p_loo_i = lppd_i - elpd_loo_i.  Totals are sums over points, se = sqrt(N) sd(pointwise).  A point with a non-finite
    draw gets NaN outputs (so the totals are NaN) and is counted in ``num_nonfinite``.  The same block gives the same
    bits on every call, whatever the slab size.  ``tau_out``: per-draw noise precisions of samples from a run with a
    tau_out hyperprior, as ``pointwise_log_lik`` takes them (an ``HMCResult`` brings its own trace).
    Returns a ``LooResult``."""
    blk, r_eff, tau = _prepare(x, target, r_eff, tau_out)
    pw, tail, flag, S, Np = _pointwise_pass(blk, target, r_eff, tau)
    r = LooResult()
    r.pointwise, r.p_loo_i, r.pareto_k, r.lppd, r.tail_size = pw[0], pw[1], pw[2], pw[3], tail
    r.elpd_loo, r.se = _total(pw[0])
    r.p_loo, r.p_loo_se = _total(pw[1])
    r.looic, r.looic_se = -2.0 * r.elpd_loo, 2.0 * r.se
    r.k_threshold = min(1.0 - 1.0 / math.log10(S), 0.7)
    r.num_bad_k = int((pw[2] > r.k_threshold).sum())
    r.num_nonfinite = int((flag != 0).sum())
    r.num_points, r.num_draws, r.r_eff = Np, S, r_eff
    return r


def waic(x, target=None, tau_out=None):
    """WAIC of a Bayesian NN on the GPU (Watanabe 2010, in the elpd scale of Vehtari et al. 2017): per point
    lppd_i = logsumexp(ll) - log S, p_waic_i = var(ll) over the S pooled draws (ddof 1), elpd_waic_i = lppd_i - p_waic_i;
    totals are sums, se = sqrt(N) sd(pointwise), waic = -2 elpd_waic.  ``x`` / ``target`` as ``psis_loo``.
    ``num_p_waic_warn`` counts points with p_waic_i > 0.4, where WAIC is known to be unreliable (prefer PSIS-LOO).
    ``tau_out`` as ``psis_loo``.  Returns a ``WaicResult``."""
    blk, _, tau = _prepare(x, target, tau_out=tau_out)
    pw, _, flag, S, Np = _pointwise_pass(blk, target, 1.0, tau)
    r = WaicResult()
    r.pointwise, r.p_waic, r.lppd = pw[5], pw[4], pw[3]
    r.elpd_waic, r.se = _total(pw[5])
    r.p_waic_total, r.p_waic_se = _total(pw[4])
    r.waic, r.waic_se = -2.0 * r.elpd_waic, 2.0 * r.se
    r.num_p_waic_warn = int((pw[4] > 0.4).sum())
    r.num_nonfinite = int((flag != 0).sum())
    r.num_points, r.num_draws = Np, S
    return r


def compare(*results):
    """Compare models fitted to the same N data points by their ``psis_loo`` (``reloo`` results included), ``waic``
    or ``kfold`` results: the elpd differences to the best model and se_diff = sqrt(N) sd(diff_i) of the pointwise
    differences (ddof 1).  Refuses results of different kinds or different N.  Returns a ``Comparison``."""
    if len(results) == 1 and isinstance(results[0], (list, tuple)):
        results = tuple(results[0])
    if len(results) < 2:
        raise ValueError('compare: need at least two results')
    kinds = {getattr(r, 'kind', None) for r in results}
    if len(kinds) != 1 or kinds.pop() not in _ELPD:
        raise TypeError('compare: pass psis_loo results only, waic results only or kfold results only')
    n0 = results[0].num_points
    if any(r.num_points != n0 for r in results):
        raise RuntimeError('compare: the results score different numbers of data points (%s); models are compared '
                           'on the same data' % ', '.join(str(r.num_points) for r in results))
    elpd = [getattr(r, _ELPD[r.kind]) for r in results]
    order = sorted(range(len(results)), key=lambda i: -elpd[i])
    best = results[order[0]].pointwise
    diff, se = [], []
    for i, r in enumerate(results):
        d = r.pointwise - best.to(r.pointwise.device)
        diff.append(elpd[i] - elpd[order[0]])
        se.append(0.0 if i == order[0] else _total(d)[1])
    return Comparison(elpd, diff, se, order)


# ------------------------------------------------------------------------------------------------------------------
# K-fold cross-validation and exact refits (reloo)
# ------------------------------------------------------------------------------------------------------------------
_ELPD = {'loo': 'elpd_loo', 'waic': 'elpd_waic', 'kfold': 'elpd_kfold'}
RELOO_MAX_POINTS = N.MLP_MAX_SPLITS     # refitted points per sample_chains call: one fold each


class KfoldResult:
    """``kfold``: ``pointwise`` (N,) fp64 elpd_i in the original data order; totals (Python floats) ``elpd_kfold``,
    ``se`` = sqrt(N) sd(pointwise) (ddof 1), ``kfoldic`` = -2 elpd_kfold, ``kfoldic_se``; ``folds`` (N,) (the run's
    assignment), ``num_folds``, ``num_points``, ``num_draws`` (per fold: R chains x n draws), ``num_nonfinite`` (points
    with a non-finite draw: NaN elpd_i and NaN totals)."""

    kind = 'kfold'

    def __repr__(self):
        return ('KfoldResult(elpd_kfold=%.3f, se=%.3f, K=%d, N=%d, S per fold=%d, nonfinite=%d)'
                % (self.elpd_kfold, self.se, self.num_folds, self.num_points, self.num_draws, self.num_nonfinite))


def kfold_split(N_, K, seed=0):
    """A balanced random assignment of N_ data rows to K folds, as Stan's ``loo::kfold_split_random``: a random
    permutation from a CPU ``torch.Generator`` seeded with ``seed``, dealt round-robin, so fold sizes differ by at most
    one and the same seed gives the same (N_,) int64 CPU tensor on every machine.  2 <= K <= min(N_, 64)."""
    N_, K = int(N_), int(K)
    if not 2 <= K <= min(N_, N.MLP_MAX_SPLITS):
        raise ValueError('kfold_split: need 2 <= K <= min(N, %d), got N=%d, K=%d' % (N.MLP_MAX_SPLITS, N_, K))
    perm = torch.randperm(N_, generator=torch.Generator().manual_seed(int(seed)))
    f = torch.empty(N_, dtype=torch.int64)
    f[perm] = torch.arange(N_, dtype=torch.int64) % K
    return f


def _fold_elpd(x, target, f, K):
    """elpd_i = logsumexp_s ll_is - log S_k (fp64) of every row i with f[i] = k >= 0 under the draws x[k::K] (the chains
    that fit without fold k), in data order; NaN at rows with f = -1.  The likelihood runs on one fold-ordered copy of
    the scored rows, where fold k is the row range [start_k, start_k + n_k); the logsumexp is hmcx_loo_pass's lppd term
    (sorted draws, fixed order), in slabs within the workspace budget.  Returns (elpd (N,), nonfinite count, S_k)."""
    dev = x.device
    n_rows = f.numel()
    order = torch.sort(f, stable=True).indices
    order = order[f[order] >= 0]
    counts = torch.bincount(f[order], minlength=K).tolist()
    ft = copy.copy(target)
    ft.x, ft.y = target.x[order.to(target.x.device)], target.y.reshape(n_rows, target.y_cols)[order.to(target.y.device)]
    nt = _native_target(ft, dev)
    scored = torch.empty(order.numel(), dtype=torch.float64, device=dev)
    bad, s_k, r0 = 0, 0, 0
    for k in range(K):
        pw, _, flag, s_k, _ = _pointwise_pass(x[k::K], ft, 1.0, nt=nt, rows=(r0, r0 + counts[k]))
        scored[r0:r0 + counts[k]] = pw[3]
        bad += int((flag != 0).sum())
        r0 += counts[k]
    out = torch.full((n_rows,), float('nan'), dtype=torch.float64, device=dev)
    out[order.to(dev)] = scored
    return out, bad, s_k


def _whole_target(target, prefix):
    t = _mlp_targets(target, prefix, 'leave out')
    if isinstance(target, list):
        raise TypeError('%s: pass the MLPTarget of the whole data set, not a split list' % prefix)
    return t[0]


def kfold(res, target):
    """K-fold cross-validation of a Bayesian NN from one fold run (``sample_chains(..., folds=f)``, every row in a fold):
    for each fold k the likelihood of its held-out rows under the draws of chains k::K, through
    hmcx_mlp_pointwise_ll_tau, and elpd_i = logsumexp_s ll_is - log S_k in fp64 with S_k = R n.  ``target``: the
    full-data ``MLPTarget`` the run was given.  The same run gives the same bits on every call, whatever the slab size.
    Returns a ``KfoldResult``."""
    f = getattr(res, 'folds', None)
    if f is None:
        raise TypeError('kfold: expected the result of sample_chains(..., folds=...)')
    t = _whole_target(target, 'kfold')
    fc = f.detach().cpu().to(torch.int64)
    if bool((fc < 0).any()):
        raise RuntimeError('kfold: the run leaves rows in every fit (fold -1, as reloo assigns them); kfold scores a run '
                           'that assigns every data row to a fold')
    if fc.numel() != t.x.shape[0]:
        raise RuntimeError('kfold: the run assigns %d rows to folds, the target has %d' % (fc.numel(), t.x.shape[0]))
    K = int(res.num_folds)
    x = _samples_block(res, t)
    if x.shape[0] % K:
        raise RuntimeError('kfold: %d chains are not a multiple of K = %d' % (x.shape[0], K))
    pw, bad, s_k = _fold_elpd(x, t, fc, K)
    r = KfoldResult()
    r.pointwise = pw
    r.elpd_kfold, r.se = _total(pw)
    r.kfoldic, r.kfoldic_se = -2.0 * r.elpd_kfold, 2.0 * r.se
    r.folds, r.num_folds = f, K
    r.num_points, r.num_draws, r.num_nonfinite = fc.numel(), s_k, bad
    return r


def _reloo_batches(points):
    """At most RELOO_MAX_POINTS points per batch, in balanced batches (so no batch holds one point unless only one is
    flagged)."""
    nb = -(-len(points) // RELOO_MAX_POINTS)
    out, i = [], 0
    for b in range(nb):
        size = len(points) // nb + (1 if b < len(points) % nb else 0)
        out.append(points[i:i + size])
        i += size
    return out


def reloo(lo, target, params_init, **sample_kwargs):
    """Exact refits of the points PSIS-LOO cannot score (ArviZ's ``reloo``): every point with pareto_k above
    ``lo.k_threshold`` is left out of a fit of its own and scored exactly under it.  The flagged points go in batches of
    at most 64, each one ``sample_chains`` K-fold run in which every flagged point of the batch is a singleton fold and
    every other row is -1 (in every fit); ``params_init`` ((R, D) or (D,)) starts the R chains of every fold, and
    ``sample_kwargs`` (num_samples, step_size, burn, sampler, seed, ...) go to ``sample_chains``.  A lone flagged point
    is refitted by a plain run on the other rows, which samples the same posterior.  ``target``: the full-data
    ``MLPTarget`` ``lo`` scored.

    Returns a NEW ``LooResult`` (``lo`` is not modified): refitted points take their exact elpd_i, p_loo_i = lppd_i -
    elpd_i and pareto_k = 0 (as ArviZ reports them) and are listed in ``refit_points`` (int64); the totals and
    ``num_bad_k`` are recomputed.  With no flagged point it returns an equal copy and launches nothing."""
    from . import samplers
    from .engine import fold_targets
    if getattr(lo, 'kind', None) != 'loo':
        raise TypeError('reloo: expected a psis_loo result')
    t = _whole_target(target, 'reloo')
    if t.x.shape[0] != lo.num_points:
        raise RuntimeError('reloo: the result scores %d points, the target has %d data rows'
                           % (lo.num_points, t.x.shape[0]))
    if 'folds' in sample_kwargs:
        raise ValueError('reloo: the folds are the flagged points; do not pass folds')
    out = LooResult()
    for k, v in lo.__dict__.items():
        setattr(out, k, v.clone() if torch.is_tensor(v) else v)
    bad = torch.nonzero(lo.pareto_k > lo.k_threshold).flatten().cpu()
    out.refit_points = bad
    if bad.numel() == 0:
        return out
    q0 = params_init if params_init.dim() == 2 else params_init.unsqueeze(0)
    n_rows = lo.num_points
    for batch in _reloo_batches(bad.tolist()):
        K = len(batch)
        f = torch.full((n_rows,), -1, dtype=torch.int64)
        f[batch] = torch.arange(K, dtype=torch.int64)
        if K == 1:                                  # fold 0's training set: every row but the flagged one
            res = samplers.sample_chains(fold_targets(t, f)[0], q0, **sample_kwargs)
        else:
            res = samplers.sample_chains(t, q0.repeat_interleave(K, dim=0), folds=f, **sample_kwargs)
        e, _, _ = _fold_elpd(_samples_block(res, t), t, f, K)
        idx = torch.tensor(batch, dtype=torch.int64, device=out.pointwise.device)
        out.pointwise[idx] = e[idx.to(e.device)].to(out.pointwise.device)
    idx = bad.to(out.pointwise.device)
    out.p_loo_i[idx] = out.lppd[idx] - out.pointwise[idx]
    out.pareto_k[idx] = 0.0
    out.elpd_loo, out.se = _total(out.pointwise)
    out.p_loo, out.p_loo_se = _total(out.p_loo_i)
    out.looic, out.looic_se = -2.0 * out.elpd_loo, 2.0 * out.se
    out.num_bad_k = int((out.pareto_k > out.k_threshold).sum())
    return out



# ------------------------------------------------------------------------------------------------------------------
# Per-chain PSIS-LOO and stacking (Yao, Vehtari, Simpson & Gelman 2018; Yao, Vehtari & Gelman 2022)
# ------------------------------------------------------------------------------------------------------------------
class ChainLooResult:
    """``psis_loo_chains``: per chain and point (C, N) fp64 on the block's device -- ``pointwise`` (elpd_loo_ci of chain
    c's draws alone), ``lppd``, ``pareto_k``, ``tail_size`` (int32, M'); per chain (C,) fp64 ``elpd_loo`` and ``se`` =
    sqrt(N) sd(pointwise[c]) (ddof 1), ``num_bad_k`` (C,) int64 (points with pareto_k above ``k_threshold`` = min(1 -
    1/log10 n, 0.7)); ``num_nonfinite`` ((chain, point) pairs with a non-finite draw: NaN outputs), ``num_chains``,
    ``num_draws`` (n, per chain), ``num_points``, ``r_eff``."""

    kind = 'loo_chains'

    def __repr__(self):
        return ('ChainLooResult(C=%d, n=%d, N=%d, elpd_loo per chain in [%.3f, %.3f], bad k-hat=%d, nonfinite=%d)'
                % (self.num_chains, self.num_draws, self.num_points, float(self.elpd_loo.min()),
                   float(self.elpd_loo.max()), int(self.num_bad_k.sum()), self.num_nonfinite))


class StackingResult:
    """``stacking_weights`` / ``chain_stacking``: ``weights`` (K,) fp64 on the simplex (input order: models, or chains);
    ``pointwise`` (N,) = log sum_k w_k exp(E_ki), ``elpd`` = its sum and ``se`` = sqrt(N) sd(pointwise) (ddof 1).
    ``elpd`` is optimistic: the weights were fitted to the same leave-one-out densities they are scored on, so it is not
    an estimate of the stacked predictive's out-of-sample elpd (score held-out data with ``predictive.evaluate(...,
    chain_weights=weights)`` for that).  ``objective`` = elpd as fitted, ``kkt_gap`` = max_k g_k / N - 1 (>= 0; the
    stopping rule bounds the shortfall from the optimum by N kkt_gap), ``iterations`` (EM updates), ``converged``
    (kkt_gap <= tol), ``num_rows`` (K), ``num_points`` (N), and for ``chain_stacking`` ``chain_loo`` (the
    ``ChainLooResult``; None for models)."""

    def __repr__(self):
        return ('StackingResult(K=%d, N=%d, elpd=%.3f (optimistic), se=%.3f, kkt_gap=%.2e, iterations=%d, converged=%s)'
                % (self.num_rows, self.num_points, self.elpd, self.se, self.kkt_gap, self.iterations, self.converged))


def _draws_per_chain(x):
    """n of what ``diagnostics.as_block`` reads, without touching the device (None when it cannot tell)."""
    from .engine import HMCResult
    if isinstance(x, HMCResult):
        x = x.samples_padded
    if isinstance(x, (list, tuple)):
        return len(x)
    if torch.is_tensor(x):
        return int(x.shape[1]) if x.dim() == 3 else int(x.shape[0]) if x.dim() == 2 else None
    return None


def _chain_slab_points(Np, S, per_point):
    """Points per slab of the per-chain pass: from samples, the slab's fp32 likelihood block within the budget."""
    if _slab_points_override is not None:
        return max(1, min(Np, N.RANK_MAX_SLAB, int(_slab_points_override)))
    k = max(1, min(Np, N.RANK_MAX_SLAB, _diag.RANK_WORKSPACE_BUDGET // max(1, per_point)))
    if per_point and _ROW_TILE <= k < Np:
        k -= k % _ROW_TILE
    return k


def psis_loo_chains(x, target=None, r_eff=1.0, tau_out=None):
    """PSIS-LOO of every chain on its own: for each chain c and point i, the PSIS-LOO of ``psis_loo`` over chain c's n
    draws only (tail M = ceil(min(0.2 n, 3 sqrt(n / r_eff)))).  Column c is bit for bit ``psis_loo(ll[c:c+1])``.  These
    are the rows ``chain_stacking`` weighs: chains that sit in different modes of a multimodal posterior give different
    leave-one-out predictives, and stacking them uses draws that pooled estimators weigh equally.

    ``x`` / ``target`` / ``r_eff`` / ``tau_out`` as ``psis_loo`` (a tempered run's result brings its cold rows).  Each
    chain's draws are sorted in one CTA's shared memory, so n <= 8192 draws per chain (``thin`` a longer run).  K-fold
    runs are refused: their chains are fits of different data.  Returns a ``ChainLooResult``."""
    if getattr(x, 'folds', None) is not None:
        raise TypeError('psis_loo_chains: this is a K-fold run (sample_chains(..., folds=...)): its chains are fits of '
                        'different data, so their leave-one-out densities are not comparable; use kfold')
    n = _draws_per_chain(x)
    if n is not None and n > N.LOO_CHAIN_MAX_DRAWS:
        raise RuntimeError('psis_loo_chains: %d draws per chain exceed the %d a chain\'s shared-memory sort holds; thin '
                           'the run (sample_chains(..., thin=...), or x[:, ::t])' % (n, N.LOO_CHAIN_MAX_DRAWS))
    blk, r_eff, tau = _prepare(x, target, r_eff, tau_out)
    C_, n = int(blk.shape[0]), int(blk.shape[1])
    if C_ > 65535:
        raise RuntimeError('psis_loo_chains: at most 65535 chains, got %d' % C_)
    N.require_cuda()
    lib = N.load_library()
    dev = blk.device
    if target is None:
        Np = int(blk.shape[2])
        k = _chain_slab_points(Np, C_ * n, 0)
        nt = None
    else:
        nt = _native_target(target, dev)
        Np = int(nt.mlp_struct.num_rows)
        k = _chain_slab_points(Np, C_ * n, 4 * C_ * n)
    out = torch.empty((3, C_, Np), dtype=torch.float64, device=dev)
    tail = torch.empty((C_, Np), dtype=torch.int32, device=dev)
    flag = torch.empty((C_, Np), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        st = N.stream_ptr(dev)
        lb = None if nt is None else torch.empty((C_, n, k), dtype=torch.float32, device=dev)
        for i0 in range(0, Np, k):
            kk = min(k, Np - i0)
            if nt is None:
                src, base = blk, N.ptr(blk)
            else:
                _ll_rows(lib, nt, blk, i0, i0 + kk, lb, tau)
                src, base = lb, C.c_void_p(lb.data_ptr() - 4 * i0)   # point i at column i - i0 of the slab's block
            rc = lib.hmcx_loo_chain_pass(base, src.stride(0), src.stride(1), C_, n, Np, i0, kk, float(r_eff),
                                         N.ptr(out), N.ptr(tail), N.ptr(flag), st)
            N.check(rc, 'hmcx_loo_chain_pass')
    r = ChainLooResult()
    r.pointwise, r.lppd, r.pareto_k, r.tail_size = out[0], out[1], out[2], tail
    r.elpd_loo = out[0].sum(1)
    r.se = math.sqrt(Np) * out[0].std(1, unbiased=True) if Np > 1 else torch.full_like(r.elpd_loo, float('nan'))
    r.k_threshold = min(1.0 - 1.0 / math.log10(n), 0.7)
    r.num_bad_k = (out[2] > r.k_threshold).sum(1)
    r.num_nonfinite = int((flag != 0).sum())
    r.num_chains, r.num_draws, r.num_points, r.r_eff = C_, n, Np, r_eff
    return r


def _stack_args(tol, max_iter, prefix):
    t = float(tol)
    if not (t > 0.0 and math.isfinite(t)):
        raise ValueError('%s: tol must be a finite positive number, got %r' % (prefix, tol))
    if isinstance(max_iter, bool) or int(max_iter) != max_iter or int(max_iter) < 1:
        raise ValueError('%s: max_iter must be a positive integer, got %r' % (prefix, max_iter))
    return t, int(max_iter)


def _stack(E, tol, max_iter, prefix):
    """Stacking weights of the rows of E (K, N) fp64 CUDA: the EM update on the device from uniform weights, the
    converged flag read back once per batch of iterations (batches of 16, doubling up to 1024)."""
    K, Np = int(E.shape[0]), int(E.shape[1])
    bad = int((~torch.isfinite(E)).sum())
    if bad:
        raise ValueError('%s: %d of the %d x %d pointwise log densities are not finite; every point must be scored by '
                         'every row (a non-finite draw makes its point NaN)' % (prefix, bad, K, Np))
    N.require_cuda()
    lib = N.load_library()
    dev = E.device
    E = E.contiguous()
    w = torch.full((K,), 1.0 / K, dtype=torch.float64, device=dev)
    obj = torch.empty(1, dtype=torch.float64, device=dev)
    grad = torch.empty(K, dtype=torch.float64, device=dev)
    pw = torch.empty(Np, dtype=torch.float64, device=dev)
    state = torch.zeros(2, dtype=torch.int32, device=dev)
    ws_bytes = lib.hmcx_stack_workspace_bytes(K, Np)
    if ws_bytes == 0:
        raise RuntimeError('%s: %d rows x %d points are beyond the stacking pass' % (prefix, K, Np))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        st = N.stream_ptr(dev)
        done, batch = 0, 16
        while done < max_iter:
            it = min(batch, max_iter - done)
            rc = lib.hmcx_stack_em(N.ptr(E), K, Np, tol, it, N.ptr(w), N.ptr(obj), N.ptr(grad), N.ptr(pw),
                                   N.ptr(state), N.ptr(ws), ws_bytes, st)
            N.check(rc, 'hmcx_stack_em')
            done += it
            batch = min(2 * batch, 1024)
            if int(state[0]):
                break
        # the evaluation at the returned weights (after max_iter updates the last one has not been evaluated yet)
        rc = lib.hmcx_stack_eval(N.ptr(E), K, Np, N.ptr(w), N.ptr(obj), N.ptr(grad), N.ptr(pw), N.ptr(ws), ws_bytes, st)
        N.check(rc, 'hmcx_stack_eval')
    s = state.cpu()
    r = StackingResult()
    r.weights, r.pointwise = w, pw
    r.objective = float(obj)
    r.elpd, r.se = _total(pw)
    r.kkt_gap = float(grad.max()) / Np - 1.0
    r.iterations = int(s[1])
    r.converged = bool(s[0]) or r.kkt_gap <= tol
    r.num_rows, r.num_points, r.tol = K, Np, tol
    r.chain_loo = None
    return r


def stacking_weights(*results, tol=1e-6, max_iter=20000):
    """Model stacking weights (Yao, Vehtari, Simpson & Gelman 2018; ArviZ ``compare``'s default, Stan's
    ``loo_model_weights``): the weights w on the simplex that maximise sum_i log sum_k w_k exp(elpd_ki) over the
    models' pointwise leave-one-out densities -- ``psis_loo`` (``reloo`` included), ``waic`` or ``kfold`` results of one
    kind on the same N points, refused otherwise as ``compare`` refuses them.  The multiplicative (EM) update runs on the
    GPU in fp64 from uniform weights until max_k g_k <= N (1 + tol), g the gradient, or ``max_iter`` updates; the
    objective is then within N tol of its maximum.  A model whose predictive is dominated by the others' mixture gets
    weight ~0; duplicates share their weight.  A non-finite pointwise value is refused.  Returns a ``StackingResult``
    (``elpd`` is optimistic: the weights were fitted to the same densities)."""
    tol, max_iter = _stack_args(tol, max_iter, 'stacking_weights')
    if len(results) == 1 and isinstance(results[0], (list, tuple)):
        results = tuple(results[0])
    if len(results) < 2:
        raise ValueError('stacking_weights: need at least two results')
    kinds = {getattr(r, 'kind', None) for r in results}
    if len(kinds) != 1 or kinds.pop() not in _ELPD:
        raise TypeError('stacking_weights: pass psis_loo results only, waic results only or kfold results only')
    n0 = results[0].num_points
    if any(r.num_points != n0 for r in results):
        raise RuntimeError('stacking_weights: the results score different numbers of data points (%s); models are '
                           'compared on the same data' % ', '.join(str(r.num_points) for r in results))
    dev = results[0].pointwise.device
    E = torch.stack([r.pointwise.to(device=dev, dtype=torch.float64) for r in results])
    if not E.is_cuda:
        raise RuntimeError('stacking_weights: the pointwise values are %s tensors; stacking runs on a CUDA device'
                           % E.device.type)
    return _stack(E, tol, max_iter, 'stacking_weights')


def chain_stacking(x, target=None, r_eff=1.0, tau_out=None, tol=1e-6, max_iter=20000):
    """Stacking of the chains of one run (Yao, Vehtari & Gelman 2022, *Stacking for non-mixing Bayesian computations*):
    ``psis_loo_chains`` gives every chain's own leave-one-out predictive, and the chain weights maximise the leave-one-out
    log score of their mixture, as ``stacking_weights`` does for models.  A run where some chains are stuck in a poor mode
    is reweighted towards the chains that predict well, with no new sampling; score the stacked predictive on held-out
    data with ``predictive.evaluate(..., chain_weights=result.weights)``.  Arguments as ``psis_loo_chains`` and
    ``stacking_weights``.  Returns a ``StackingResult`` with ``chain_loo``; its ``elpd`` is optimistic (the weights were
    fitted to the same leave-one-out densities)."""
    tol, max_iter = _stack_args(tol, max_iter, 'chain_stacking')
    cl = psis_loo_chains(x, target, r_eff, tau_out)
    r = _stack(cl.pointwise, tol, max_iter, 'chain_stacking')
    r.chain_loo = cl
    return r
