"""Power-scaling prior and likelihood sensitivity of Bayesian NNs on the GPU (Kallioinen, Paananen, Buerkner & Vehtari
2023, "Detecting and diagnosing prior and likelihood sensitivity with power-scaling"), restated in numpy fp64 by
tests/psens_oracle.py.  Does the fit depend on the prior?  The draws the run already has answer it, with no refit.

    s = hamiltorch_b200.sensitivity.power_scale(res, target)         # res = sample_chains(...) of the target
    s.prior, s.likelihood, s.diagnosis                                # one entry per column (s.names)
    s.by_tensor                                                       # the same, summarised per parameter tensor
    q = hamiltorch_b200.predictive.pointwise_outputs(res, test_target).reshape(C, n, -1)
    s = hamiltorch_b200.sensitivity.power_scale(res, target, quantities=q)   # sensitivity of the test predictions

For each component (the prior, the likelihood) and each alpha in (lower_alpha, upper_alpha), the posterior draws are
importance-weighted to the posterior with that component raised to the power alpha: log-ratio (alpha - 1) component_s,
Pareto-smoothed as ``loo.psis_loo`` smooths one data point.  The cumulative Jensen-Shannon distance (CJS) of every
column's weighted to its unweighted distribution, divided by |log2 alpha| and averaged over the two alphas, is its
sensitivity to that component.  A column sensitive to the prior but not the likelihood points to a strong prior or a weak
likelihood; one sensitive to both to a conflict between the prior and the data.

Four CUDA passes (hmcx_psens.cu): the prior term of every draw (hmcx_mlp_log_prior) and the likelihood totals from the
pointwise log-likelihood of ``loo`` in 128-row groups (hmcx_psens_ll_totals); the smoothed weights of the four weight
sets (hmcx_psens_weights); the sort of every column and the CJS sums, weighted means and sds (hmcx_psens_pass), in slabs
of columns within ``diagnostics.RANK_WORKSPACE_BUDGET`` bytes.  The same draws give the same bits on every call,
whatever the slab sizes.
"""
import ctypes as C
import math

import torch

from . import _native as N
from . import diagnostics as _diag
from . import loo as _loo
from . import targets as T

_slab_cols_override = None              # tests: force this many columns per slab of the sort pass
_slab_rows_override = None              # tests: force this many data rows (a multiple of 128) per likelihood slab
_GROUP = 128                            # rows per fixed-order group of hmcx_psens_ll_totals
CONFLICT = 'potential prior-data conflict'
STRONG_PRIOR = 'potential strong prior / weak likelihood'
NONE = '-'


class SensitivityResult:
    """``power_scale``: per column (the D parameters, then ``log_prior`` and ``log_lik``, then the Q quantities; see
    ``names``) ``prior`` and ``likelihood`` (fp64 sensitivities) and ``diagnosis`` (a list of str: CONFLICT,
    STRONG_PRIOR or '-'); ``cjs`` (4, cols) the CJS distances of the weight sets (prior, lower_alpha), (prior,
    upper_alpha), (lik, lower_alpha), (lik, upper_alpha); ``mean`` and ``sd`` (5, cols), row 0 unweighted, rows 1..4 the
    weight sets.  ``pareto_k`` (4,) and ``tail_size`` (4,) of the weight sets, ``k_threshold`` = min(1 - 1/log10 S, 0.7),
    ``num_bad_k``; ``num_conflict``, ``num_strong_prior``, ``num_nonfinite`` (columns with a non-finite draw: NaN
    outputs); ``by_tensor`` (one dict per parameter tensor: name, size, max_prior, max_likelihood, num_conflict,
    num_strong_prior); ``log_prior`` and ``log_lik`` (C, n) fp64, ``alphas``, ``threshold``, ``r_eff``, ``num_draws``."""

    def __repr__(self):
        return ('SensitivityResult(S=%d, columns=%d, prior-data conflict=%d, strong prior / weak likelihood=%d, '
                'bad k-hat=%d, nonfinite=%d)' % (self.num_draws, len(self.names), self.num_conflict,
                                                 self.num_strong_prior, self.num_bad_k, self.num_nonfinite))


# ------------------------------------------------------------------------------------------------------------------
# Inputs: every check that needs no device comes first
# ------------------------------------------------------------------------------------------------------------------
def _refuse_folds(x, prefix):
    if getattr(x, 'folds', None) is not None:
        raise TypeError('%s: this is a K-fold run (sample_chains(..., folds=...)): its chains are fits of different '
                        'data, so they are not draws of one posterior' % prefix)


def _chains_draws(x):
    """(C, n) of what ``diagnostics.as_block`` reads, from shapes alone (None when it cannot tell)."""
    from .engine import HMCResult
    if isinstance(x, HMCResult):
        x = x.samples_padded
    if isinstance(x, (list, tuple)):
        return 1, len(x)
    if torch.is_tensor(x):
        if x.dim() == 3:
            return int(x.shape[0]), int(x.shape[1])
        if x.dim() == 2:
            return 1, int(x.shape[0])
    return None


def _check_draws(shape, prefix):
    if shape is None:
        return
    S = shape[0] * shape[1]
    if S < 2:
        raise RuntimeError('%s: need at least 2 pooled draws, got %d' % (prefix, S))
    if S > N.RANK_MAX_DRAWS:
        raise RuntimeError('%s: %d chains x %d draws exceed the %d draws per column the sort indexes'
                           % (prefix, shape[0], shape[1], N.RANK_MAX_DRAWS))


def _check_alphas(lo, hi):
    lo, hi = float(lo), float(hi)
    if not (math.isfinite(lo) and math.isfinite(hi)) or lo <= 0.0 or hi <= 0.0:
        raise ValueError('power_scale: the alphas must be finite and positive, got %r and %r' % (lo, hi))
    if lo >= 1.0 or hi <= 1.0:
        raise ValueError('power_scale: need lower_alpha < 1 < upper_alpha, got %r and %r' % (lo, hi))
    return lo, hi


def _component(v, shape, name):
    """A (C, n) per-draw component; (n,) is taken for one chain."""
    t = torch.as_tensor(v)
    if shape is not None:
        if t.dim() == 1 and shape[0] == 1:
            t = t[None]
        if tuple(t.shape) != tuple(shape):
            raise RuntimeError('power_scale: %s must hold one value per draw, (C, n) = (%d, %d), got %s'
                               % (name, shape[0], shape[1], tuple(t.shape)))
    return t


def _check_quantities(q, shape):
    if not torch.is_tensor(q):
        raise TypeError('power_scale: quantities must be a (C, n, Q) CUDA fp32 tensor, got %s' % type(q).__name__)
    if q.dim() == 2 and shape is not None and shape[0] == 1:
        q = q[None]
    if q.dim() != 3 or (shape is not None and tuple(q.shape[:2]) != tuple(shape)) or q.shape[2] < 1:
        raise RuntimeError('power_scale: quantities must be (C, n, Q) with (C, n) = %s, got %s'
                           % (tuple(shape) if shape else '(C, n)', tuple(q.shape)))
    return q


# ------------------------------------------------------------------------------------------------------------------
# The two components
# ------------------------------------------------------------------------------------------------------------------
def _row_slab(S, Np):
    """Data rows per likelihood slab: a multiple of 128 whose fp32 (C, n, rows) block fits the budget."""
    if _slab_rows_override is not None:
        k = int(_slab_rows_override)
        if k < 1 or k % _GROUP:
            raise ValueError('sensitivity: the row slab must be a positive multiple of %d' % _GROUP)
        return min(k, -(-Np // _GROUP) * _GROUP)
    k = max(_GROUP, _diag.RANK_WORKSPACE_BUDGET // (4 * S) // _GROUP * _GROUP)
    return min(k, -(-Np // _GROUP) * _GROUP)


def _gamma_logpdf(t, a, b):
    """log Gamma(t; shape a, rate b) in fp64."""
    t = t.double()
    return a * math.log(b) - math.lgamma(a) + (a - 1.0) * torch.log(t) - b * t


def log_components(x, target, tau_out=None):
    """The power-scaled components of every pooled draw: ``(log_prior, log_lik)``, each a (C, n) fp64 CUDA tensor.

    ``x``: the samples, read as ``loo.psis_loo`` reads them (an ``HMCResult``, a (C, n, D) / (n, D) CUDA fp32 block or
    the list ``sample`` returns); ``target``: the ``MLPTarget`` with data, or the split list, the run sampled.
    ``log_prior``: sum over the targets t of t.log_prior(theta) / t.prior_scale (a split list's prior counted once), in
    fp64: the Normal(0, tau^-1/2) density of every parameter tensor.  For an ``HMCResult`` of a run with hyperpriors only
    the top-level priors: the Normal terms of the tensors whose tau is fixed, plus log Gamma(tau_k; a_k, b_k) of every
    sampled tau_k (tau_out included), read from the result's ``hyper``, ``tau_list_trace`` and ``tau_out_trace``.
    ``log_lik``: from the per-row log-likelihoods of ``loo.pointwise_log_lik``: regression their sum (each draw's own
    tau_out in a hyperprior run), binary and multi-class linear output tau_out times their sum, LogSoftmax output tau_out
    times the sum over splits of the split's mean.  ``tau_out``: per-draw noise precisions as ``loo`` takes them."""
    _refuse_folds(x, 'log_components')
    items = _loo._mlp_targets(target, 'log_components', 'score')
    first = items[0]
    blk = _loo._samples_block(x, target)
    tau = _loo._tau_block(x, blk, tau_out)
    hyper = getattr(x, 'hyper', None)
    if hyper is None and getattr(x, 'tau_list_trace', None) is not None:
        raise RuntimeError('log_components: the result carries tau traces but no hyper list; pass a result of '
                           'sample_chains(..., tau_prior=...)')
    N.require_cuda()
    lib = N.load_library()
    dev = blk.device
    C_, n, D = (int(v) for v in blk.shape)
    S = C_ * n
    K = 2 * first.num_layers
    sampled = [False] * (K + 1) if hyper is None else [ab is not None for ab in hyper]
    with torch.cuda.device(dev):
        st = N.stream_ptr(dev)
        # prior: the Normal terms of the fixed tensors, counted once (M splits of prior_scale M each)
        taus = [0.0 if sampled[k] else float(first.tau_list[k]) for k in range(K)]
        lp = torch.zeros(S, dtype=torch.float64, device=dev)
        if any(t > 0.0 for t in taus):
            sizes = (C.c_int32 * K)(*first.sizes)
            tv = (C.c_double * K)(*taus)
            rc = lib.hmcx_mlp_log_prior(N.ptr(blk), blk.stride(0), blk.stride(1), C_, n, K, sizes, tv, N.ptr(lp), st)
            N.check(rc, 'hmcx_mlp_log_prior')
            lp = lp * (len(items) / float(first.prior_scale))
        lp = lp.view(C_, n)
        if hyper is not None:
            for k in range(K):
                if sampled[k]:
                    a, b = hyper[k]
                    lp = lp + _gamma_logpdf(_trace(x, 'tau_list_trace', (C_, n), dev)[..., k], float(a), float(b))
            if sampled[K]:
                a, b = hyper[K]
                lp = lp + _gamma_logpdf(_trace(x, 'tau_out_trace', (C_, n), dev), float(a), float(b))
        # likelihood: per-row values in slabs of whole 128-row groups, totals in row order
        nt = _loo._native_target(target, dev)
        Np = int(nt.mlp_struct.num_rows)
        coef = None
        if first.loss_id == T.LOSS_MULTICLASS_LOGSOFTMAX:
            coef = torch.cat([torch.full((t.x.shape[0],), 1.0 / t.x.shape[0], dtype=torch.float64) for t in items])
            coef = coef.to(dev)
        kr = _row_slab(S, Np)
        buf = torch.empty((C_, n, kr), dtype=torch.float32, device=dev)
        ll = torch.zeros(S, dtype=torch.float64, device=dev)
        for r0 in range(0, Np, kr):
            kk = min(kr, Np - r0)
            out = buf[:, :, :kk]
            _loo._ll_rows(lib, nt, blk, r0, r0 + kk, out, tau)
            rc = lib.hmcx_psens_ll_totals(N.ptr(out), out.stride(0), out.stride(1), C_, n, r0, kk, N.ptr(coef),
                                          N.ptr(ll), st)
            N.check(rc, 'hmcx_psens_ll_totals')
        ll = ll.view(C_, n)
        if first.loss_id != T.LOSS_REGRESSION:
            ll = ll * (tau.double() if tau is not None else float(first.tau_out))
    return lp, ll


def _trace(x, name, shape, dev):
    t = getattr(x, name, None)
    if t is None or tuple(t.shape[:2]) != tuple(shape):
        raise RuntimeError('log_components: the result\'s %s does not match its (C, n) = %s samples'
                           % (name, tuple(shape)))
    return t.to(dev)


# ------------------------------------------------------------------------------------------------------------------
# Weights, CJS and the result
# ------------------------------------------------------------------------------------------------------------------
def _slab_cols(lib, C_, n, cols):
    if _slab_cols_override is not None:
        return max(1, min(cols, N.RANK_MAX_SLAB, int(_slab_cols_override)))
    budget = _diag.RANK_WORKSPACE_BUDGET
    k = max(1, min(cols, N.RANK_MAX_SLAB, budget // lib.hmcx_psens_workspace_bytes(C_, n, 1)))
    while k > 1 and lib.hmcx_psens_workspace_bytes(C_, n, k) > budget:
        k -= 1
    return k


def _names(target, D, Q):
    if target is None:
        names = ['theta[%d]' % d for d in range(D)]
        tensors = [('theta', D)]
    else:
        t = _loo._mlp_targets(target, 'power_scale', 'score')[0]
        names, tensors = [], []
        for l in range(t.num_layers):
            n_in, n_out = t.widths[l], t.widths[l + 1]
            names += ['w%d[%d,%d]' % (l, i, j) for i in range(n_out) for j in range(n_in)]
            names += ['b%d[%d]' % (l, i) for i in range(n_out)]
            tensors += [('w%d' % l, n_in * n_out), ('b%d' % l, n_out)]
    return names + ['log_prior', 'log_lik'] + ['q[%d]' % j for j in range(Q)], tensors


def diagnose(prior, likelihood, threshold=0.05):
    """The diagnosis of each column from its prior and likelihood sensitivities: CONFLICT when both reach ``threshold``,
    STRONG_PRIOR when only the prior does, '-' otherwise (NaN included)."""
    out = []
    for p, l in zip(prior.tolist(), likelihood.tolist()):
        if p >= threshold:
            out.append(CONFLICT if l >= threshold else STRONG_PRIOR)
        else:
            out.append(NONE)
    return out


def power_scale(x, target=None, *, log_prior=None, log_lik=None, quantities=None, lower_alpha=0.99, upper_alpha=1.01,
                r_eff=1.0, threshold=0.05, tau_out=None):
    """Power-scaling prior and likelihood sensitivity of every parameter (and of ``quantities``) on the GPU.

    ``x``: the samples as ``loo.psis_loo`` reads them.  With ``target`` (the ``MLPTarget`` or split list the run
    sampled) the components come from ``log_components(x, target, tau_out)``; without it pass both ``log_prior`` and
    ``log_lik`` ((C, n) per-draw values of the prior and likelihood terms of the sampled density), the path for any model
    whose two terms the user can compute.  ``quantities``: an optional (C, n, Q) CUDA fp32 block of derived quantities
    of the draws (e.g. ``predictive.pointwise_outputs`` at test inputs, reshaped).

    Per component c and alpha in (``lower_alpha``, ``upper_alpha``): log-ratios (alpha - 1) c_s in fp64, rounded to fp32
    and Pareto-smoothed as ``loo.psis_loo`` smooths one point (``r_eff`` sets the tail length) into normalised weights
    q.  Per column x and weight set the cumulative Jensen-Shannon distance to the equal weights p = 1/S: over the sorted
    draws, widths d_j = x_(j+1) - x_(j) (the last d_S = x_(S) - x_(S-1)) and prefix sums P_j, Q_j, cjs+ = sqrt(sum_j d_j
    [P_j log2(2 P_j / (P_j + Q_j)) + Q_j log2(2 Q_j / (P_j + Q_j))] / sum_j d_j (P_j + Q_j)) (0 log 0 = 0; 0 for a
    constant column), cjs- the same of -x, CJS = max(cjs+, cjs-).  Sensitivity = the mean over the two alphas of CJS /
    |log2 alpha|.  Diagnosis with ``threshold``: see ``diagnose``.  The weighted means sum q x and sds sqrt(sum q (x -
    mean)^2) show the direction of each shift.  Refused: K-fold runs, a target without data, components or quantities
    that do not match (C, n), alpha <= 0, lower_alpha >= 1 or upper_alpha <= 1, fewer than 2 or more than
    ``RANK_MAX_DRAWS`` draws, samples in pinned host memory.  Returns a ``SensitivityResult``."""
    lo, hi = _check_alphas(lower_alpha, upper_alpha)
    r_eff = _loo._check_r_eff(r_eff)
    thr = float(threshold)
    if not (thr > 0.0 and math.isfinite(thr)):
        raise ValueError('power_scale: threshold must be a finite positive number, got %r' % (threshold,))
    _refuse_folds(x, 'power_scale')
    shape = _chains_draws(x)
    _check_draws(shape, 'power_scale')
    if target is None:
        if log_prior is None or log_lik is None:
            raise ValueError('power_scale: without a target pass both log_prior and log_lik')
        if tau_out is not None:
            raise ValueError('power_scale: tau_out applies with a target')
        log_prior = _component(log_prior, shape, 'log_prior')
        log_lik = _component(log_lik, shape, 'log_lik')
    else:
        if log_prior is not None or log_lik is not None:
            raise ValueError('power_scale: pass a target or the two components, not both')
        _loo._mlp_targets(target, 'power_scale', 'score')
    if quantities is not None:
        quantities = _check_quantities(quantities, shape)
    if target is None:
        blk = _diag.as_block(x)
        lp = log_prior.to(device=blk.device, dtype=torch.float64).reshape(blk.shape[0], blk.shape[1])
        ll = log_lik.to(device=blk.device, dtype=torch.float64).reshape(blk.shape[0], blk.shape[1])
    else:
        blk = _loo._samples_block(x, target)
        lp, ll = log_components(x, target, tau_out)
    C_, n, D = (int(v) for v in blk.shape)
    S = C_ * n
    _check_draws((C_, n), 'power_scale')
    qb = None
    if quantities is not None:
        qb = _diag.as_block(quantities)
        if tuple(qb.shape[:2]) != (C_, n):
            raise RuntimeError('power_scale: quantities must be (C, n, Q) with (C, n) = (%d, %d), got %s'
                               % (C_, n, tuple(qb.shape)))
        if qb.device != blk.device:
            raise RuntimeError('power_scale: the quantities live on %s, the samples on %s' % (qb.device, blk.device))
    bad = int((~torch.isfinite(lp)).sum()) + int((~torch.isfinite(ll)).sum())
    if bad:
        raise ValueError('power_scale: %d of the 2 x %d component values are not finite; every draw needs a finite '
                         'prior and likelihood term' % (bad, S))
    N.require_cuda()
    lib = N.load_library()
    dev = blk.device
    Q = 0 if qb is None else int(qb.shape[2])
    cols = D + 2 + Q
    with torch.cuda.device(dev):
        st = N.stream_ptr(dev)
        # the four weight sets: -r = -(alpha - 1) component, formed in fp64 and rounded to fp32
        nr = torch.stack([-(lo - 1.0) * lp, -(hi - 1.0) * lp, -(lo - 1.0) * ll, -(hi - 1.0) * ll], -1)
        nr = nr.to(torch.float32).contiguous()
        w = torch.empty((N.PSENS_SETS, S), dtype=torch.float64, device=dev)
        khat = torch.empty(N.PSENS_SETS, dtype=torch.float64, device=dev)
        tail = torch.empty(N.PSENS_SETS, dtype=torch.int32, device=dev)
        wflag = torch.empty(N.PSENS_SETS, dtype=torch.int32, device=dev)
        ws_bytes = lib.hmcx_psens_workspace_bytes(C_, n, N.PSENS_SETS)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        rc = lib.hmcx_psens_weights(N.ptr(nr), nr.stride(0), nr.stride(1), C_, n, N.PSENS_SETS, float(r_eff), N.ptr(w),
                                    N.ptr(khat), N.ptr(tail), N.ptr(wflag), N.ptr(ws), ws_bytes, st)
        N.check(rc, 'hmcx_psens_weights')
        del ws
        # every column: the samples, then the two components (in fp32, as every column), then the quantities
        comp = torch.stack([lp, ll], -1).to(torch.float32).contiguous()
        out = torch.empty((N.PSENS_ROWS, cols), dtype=torch.float64, device=dev)
        flag = torch.empty(cols, dtype=torch.int32, device=dev)
        k = _slab_cols(lib, C_, n, cols)
        ws_bytes = lib.hmcx_psens_workspace_bytes(C_, n, k)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        blocks = [(blk, 0), (comp, D)] + ([] if qb is None else [(qb, D + 2)])
        for b, off in blocks:
            width = int(b.shape[2])
            base = C.c_void_p(b.data_ptr() - 4 * off)                # column off + j of the pass is column j of b
            for j0 in range(0, width, k):
                kk = min(k, width - j0)
                rc = lib.hmcx_psens_pass(base, b.stride(0), b.stride(1), C_, n, cols, off + j0, kk, N.ptr(w), N.ptr(out),
                                         N.ptr(flag), N.ptr(ws), ws_bytes, st)
                N.check(rc, 'hmcx_psens_pass')
        del ws
    return _result(out, flag, khat, tail, lp, ll, lo, hi, thr, r_eff, S, target, D, Q)


def _result(out, flag, khat, tail, lp, ll, lo, hi, thr, r_eff, S, target, D, Q):
    r = SensitivityResult()
    r.cjs, r.mean, r.sd = out[0:4], out[4:9], out[9:14]
    a, b = abs(math.log2(lo)), abs(math.log2(hi))
    r.prior = (r.cjs[0] / a + r.cjs[1] / b) / 2.0
    r.likelihood = (r.cjs[2] / a + r.cjs[3] / b) / 2.0
    r.diagnosis = diagnose(r.prior.cpu(), r.likelihood.cpu(), thr)
    r.names, tensors = _names(target, D, Q)
    r.pareto_k, r.tail_size = khat, tail
    r.k_threshold = min(1.0 - 1.0 / math.log10(S), 0.7) if S > 1 else float('nan')
    r.num_bad_k = int((khat > r.k_threshold).sum())
    r.num_conflict = r.diagnosis.count(CONFLICT)
    r.num_strong_prior = r.diagnosis.count(STRONG_PRIOR)
    r.num_nonfinite = int((flag != 0).sum())
    rows, i = [], 0
    pc, lc = r.prior.cpu(), r.likelihood.cpu()
    for name, size in tensors:
        d = r.diagnosis[i:i + size]
        rows.append(dict(name=name, size=size, max_prior=float(pc[i:i + size].max()),
                         max_likelihood=float(lc[i:i + size].max()), num_conflict=d.count(CONFLICT),
                         num_strong_prior=d.count(STRONG_PRIOR)))
        i += size
    r.by_tensor = rows
    r.log_prior, r.log_lik = lp, ll
    r.alphas, r.threshold, r.r_eff, r.num_draws = (lo, hi), thr, r_eff, S
    return r
