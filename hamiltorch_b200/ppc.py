"""Posterior predictive checks of Bayesian NNs on the GPU (Gelman, Meng & Stern 1996; Gelman et al., BDA3 ch. 6; Gabry et
al. 2019): can the fitted model reproduce the data it was fitted to?  What ArviZ's ``plot_ppc``, ``plot_bpv`` and
``loo_pit`` compute, restated in numpy fp64 by tests/ppc_oracle.py.

    y_rep = hamiltorch_b200.ppc.replicate(res, target, draws=torch.arange(20))   # (20, N, y_cols) replicated data sets
    r = hamiltorch_b200.ppc.check(res, target)                     # test statistics and posterior predictive p-values
    r.names, r.p_value
    lp = hamiltorch_b200.ppc.loo_pit(res, target)                  # regression: leave-one-out PIT, uniform if calibrated
    lp.pit, lp.p_value

``res`` and ``target`` are read as ``loo.psis_loo`` reads them: an ``HMCResult``, a (C, n, D) / (n, D) CUDA fp32 block or
the list ``sample`` returns, with the ``MLPTarget`` (or split list) the model was fitted to.  The draws are the ones
``psis_loo`` scores, pooled as g = c n + s.  A run with a tau_out hyperprior brings its ``tau_out_trace``; otherwise pass
``tau_out`` ((C, n)) as ``loo`` takes it.

Two CUDA passes, each in slabs within ``diagnostics.RANK_WORKSPACE_BUDGET`` bytes:
  * hmcx_ppc_pass: for a slab of draws whose outputs hmcx_mlp_pointwise_out wrote, one CTA per draw simulates y_rep ~ p(y |
    theta_g) on Philox stream 8 (chain word g, so a draw's replicate depends on (seed, g) only, not on the slab or on which
    draws are asked for), writes it, and computes its statistics and both realised deviances with fixed-order fp64 sums;
  * hmcx_loo_pit_pass: for a slab of points, the sort and Pareto smoothing of ``psis_loo`` (the same bits: pareto_k is
    psis_loo's), then the PSIS-weighted predictive CDF at every observation from the draws' outputs.
y_rep follows the untempered predictive that ``loo`` and ``predictive`` score: regression f + z / sqrt(tau_g), binary
Bernoulli(sigmoid f) per output, multi-class Categorical(softmax f) for both multi-class losses.
"""
import ctypes
import math

import torch

from . import _native as N
from . import diagnostics as _diag
from . import loo as _loo
from . import predictive as _pred
from . import targets as T

_slab_draws_override = None             # tests: force this many draws per slab of check / replicate


class PpcResult:
    """``check``: ``names`` (K statistics, e.g. 'sd[0]', 'freq[2]', 'deviance'), ``t_rep`` (S, K) fp64 (row g: the
    statistics of draw g's replicate; NaN for a draw with a non-finite output), ``t_obs`` (K,) fp64 (the statistics of
    the observed y; for 'deviance' the mean of ``dev_obs`` over the finite draws, its comparison being draw by draw),
    ``dev_obs`` (S,) the realised deviance -2 sum_i ll_i(y | theta_g), ``p_value`` (K,) = P(T_rep > T_obs) + P(T_rep =
    T_obs) / 2 over the finite draws, ``num_draws`` S, ``num_nonfinite``, ``seed``."""

    def __repr__(self):
        rows = ', '.join('%s %.3f' % (n, p) for n, p in zip(self.names, self.p_value.tolist()))
        return 'PpcResult(S=%d, nonfinite=%d; p-values: %s)' % (self.num_draws, self.num_nonfinite, rows)


class LooPitResult:
    """``loo_pit``: ``pit`` (N, O) fp64 LOO-PIT values, ``pareto_k`` (N,) (psis_loo's, bit for bit), ``k_threshold`` and
    ``num_bad_k`` as ``psis_loo``, ``bins`` B, ``hist`` (B,) int64 counts of the N O values over equal-width bins of [0,
    1], ``chi2`` and ``p_value``: the chi^2 uniformity test (expected N O / B per bin, p = gammaincc((B - 1) / 2, chi2 /
    2)) over the finite values, ``num_nonfinite`` (points with a non-finite draw: NaN pit), ``num_points``,
    ``num_draws``, ``r_eff``."""

    def __repr__(self):
        return ('LooPitResult(N=%d, S=%d, chi2=%.2f, p=%.3g, bad k-hat=%d, nonfinite=%d)'
                % (self.num_points, self.num_draws, self.chi2, self.p_value, self.num_bad_k, self.num_nonfinite))


# ------------------------------------------------------------------------------------------------------------------
# Inputs: every check before the device is touched
# ------------------------------------------------------------------------------------------------------------------
def _target(target, prefix):
    """The first MLPTarget of ``target`` (an MLPTarget with data or a split list), refused otherwise."""
    if not isinstance(target, (list, T.MLPTarget)):
        raise TypeError('%s: posterior predictive checks need a Bayesian-NN target with data (an MLPTarget or the list '
                        'define_split_model_log_prob returns); element-wise targets have no data, got %s'
                        % (prefix, type(target).__name__))
    return _loo._mlp_targets(target, prefix, 'replicate')[0]


def stat_names(target):
    """The K statistic names ``check`` reports for ``target``'s likelihood: regression mean, sd, min, max of every output
    column, binary the mean of every column, multi-class the frequency of every class; then 'deviance'."""
    t = _target(target, 'ppc')
    O_ = t.widths[-1]
    if t.loss_id == T.LOSS_REGRESSION:
        names = ['%s[%d]' % (s, o) for o in range(O_) for s in ('mean', 'sd', 'min', 'max')]
    elif t.loss_id == T.LOSS_BINARY:
        names = ['mean[%d]' % o for o in range(O_)]
    else:
        names = ['freq[%d]' % c for c in range(O_)]
    return names + ['deviance']


def _draw_ids(draws):
    """``draws`` as a 1-D int64 CPU tensor (None stays None: every pooled draw)."""
    if draws is None:
        return None
    d = torch.as_tensor(draws).detach().cpu()
    if d.dim() != 1 or d.numel() < 1 or d.dtype.is_floating_point or d.dtype == torch.bool:
        raise ValueError('ppc: draws must be a non-empty 1-D integer tensor of pooled draw ids, got %s %s'
                         % (d.dtype, tuple(d.shape)))
    return d.to(torch.int64)


def _check_bins(bins):
    if isinstance(bins, bool) or int(bins) != bins or int(bins) < 2:
        raise ValueError('ppc.loo_pit: bins must be an integer >= 2, got %r' % (bins,))
    return int(bins)


def _y(target, dev):
    """The target's y as an (N, y_cols) fp32 tensor on ``dev``, points in split order."""
    items = target if isinstance(target, list) else [target]
    return torch.cat([t.y.detach().reshape(-1, t.y_cols).to(device=dev, dtype=torch.float32) for t in items])


# ------------------------------------------------------------------------------------------------------------------
# Replicated data and test statistics
# ------------------------------------------------------------------------------------------------------------------
def _slab_draws(n_rows, O_, y_cols, D):
    """Draws per slab: the slab's fp32 outputs, replicate and gathered parameters within the budget."""
    if _slab_draws_override is not None:
        return max(1, int(_slab_draws_override))
    return max(1, _diag.RANK_WORKSPACE_BUDGET // (4 * (n_rows * (O_ + y_cols) + D)))


def _pass(x, target, seed, tau_out, draws, keep_rep):
    """Run hmcx_ppc_pass over the selected draws in slabs.  Returns (stats (S', K), dev_obs (S',), nonfinite (S',),
    y_rep (S', N, y_cols) or None, the target's first MLPTarget)."""
    first = _target(target, 'ppc')
    seed = int(seed)
    if not 0 <= seed < 2 ** 64:
        raise ValueError('ppc: seed must be in [0, 2^64), got %d' % seed)
    g_cpu = _draw_ids(draws)
    blk = _loo._samples_block(x, target)
    C_, n, D = (int(v) for v in blk.shape)
    if g_cpu is None:
        g_cpu = torch.arange(C_ * n, dtype=torch.int64)
    elif int(g_cpu.min()) < 0 or int(g_cpu.max()) >= C_ * n:
        raise ValueError('ppc: draw ids must lie in [0, %d) (pooled g = c n + s)' % (C_ * n))
    tau = _loo._tau_block(x, blk, tau_out) if first.loss_id == T.LOSS_REGRESSION else None
    N.require_cuda()
    lib = N.load_library()
    dev = blk.device
    nt = _loo._native_target(target, dev)
    n_rows, O_, yc = int(nt.mlp_struct.num_rows), first.widths[-1], first.y_cols
    K = len(stat_names(target))
    S_ = g_cpu.numel()
    k = min(S_, _slab_draws(n_rows, O_, yc, D))
    g_all = g_cpu.to(dev)
    stats = torch.empty((S_, K), dtype=torch.float64, device=dev)
    dev_obs = torch.empty(S_, dtype=torch.float64, device=dev)
    bad = torch.empty(S_, dtype=torch.int32, device=dev)
    y_rep = torch.empty((S_, n_rows, yc), dtype=torch.float32, device=dev) if keep_rep else None
    with torch.cuda.device(dev):
        st = N.stream_ptr(dev)
        f = torch.empty((k, n_rows, O_), dtype=torch.float32, device=dev)
        scratch = None if keep_rep else torch.empty((k, n_rows, yc), dtype=torch.float32, device=dev)
        for j0 in range(0, S_, k):
            kk = min(k, S_ - j0)
            g = g_all[j0:j0 + kk]
            c, s = g // n, g % n
            th = blk[c, s].contiguous()                                          # (kk, D): the slab's draws
            N.check(lib.hmcx_mlp_pointwise_out(nt.ref(), N.ptr(th), 0, D, 1, kk, 0, n_rows, N.ptr(f), 0,
                                               n_rows * O_, st), 'hmcx_mlp_pointwise_out')
            ts = None if tau is None else tau[c, s].contiguous()
            yr = y_rep[j0:j0 + kk] if keep_rep else scratch
            N.check(lib.hmcx_ppc_pass(nt.ref(), N.ptr(f), kk, N.ptr(g), seed, N.ptr(ts), N.ptr(yr), N.ptr(stats[j0:]),
                                      N.ptr(dev_obs[j0:]), N.ptr(bad[j0:]), st), 'hmcx_ppc_pass')
    return stats, dev_obs, bad, y_rep, first


def replicate(x, target, draws=None, seed=0, tau_out=None):
    """Replicated data sets y_rep ~ p(y | theta_g), one per pooled posterior draw g in ``draws`` (a 1-D index tensor,
    None for all C n of them), at the target's inputs: a (len(draws), N, y_cols) fp32 CUDA tensor in the target's ``y``
    format (points in split order).  Regression f + z / sqrt(tau_g), binary one Bernoulli(sigmoid f) per output,
    multi-class one Categorical(softmax f) label per row -- the definitions of ``sbc.simulate`` on Philox stream 8 keyed
    by (seed, g), so a draw's replicate is the same bits in any ``draws`` subset and on every call.  For plots and
    user-defined statistics; ``check`` computes a fixed menu on the GPU.  ``tau_out`` as ``loo.psis_loo``."""
    return _pass(x, target, seed, tau_out, draws, True)[3]


def _observed(y, loss, O_):
    """The statistics of the observed (N, y_cols) y, fp64, in ``stat_names`` order without the deviance.  Means and
    frequencies are sums divided by N in a true fp64 division (a tensor divisor: a scalar one is a multiplication by its
    reciprocal on the GPU), as the kernel divides, so a replicate with the observed count ties exactly."""
    yd = y.double()
    n = torch.full((yd.shape[1],), float(yd.shape[0]), dtype=torch.float64, device=yd.device)
    if loss == T.LOSS_REGRESSION:
        cols = [yd.sum(0) / n, yd.std(0, unbiased=True), yd.min(0).values, yd.max(0).values]
        return torch.stack(cols, 1).reshape(-1)
    if loss == T.LOSS_BINARY:
        return yd.sum(0) / n
    cnt = torch.bincount(y[:, 0].long(), minlength=O_).double()
    return cnt / torch.full_like(cnt, y.shape[0])


def p_values(t_rep, t_obs):
    """P(T_rep > T_obs) + P(T_rep = T_obs) / 2 per column over the rows of ``t_rep`` (S, K); ``t_obs`` (K,) or (S, K).
    Evaluated as (#greater + #equal / 2) / S, so the value is exact given the two tensors."""
    t_obs = t_obs.expand_as(t_rep)
    gt = (t_rep > t_obs).sum(0).double()
    eq = (t_rep == t_obs).sum(0).double()
    return (gt + 0.5 * eq) / torch.full_like(gt, t_rep.shape[0])


def check(x, target, seed=0, tau_out=None):
    """Posterior predictive check of a Bayesian NN: every pooled draw's replicated data set and its test statistics
    (``stat_names``: regression mean, sd (ddof 1), min, max per output column; binary the mean per column; multi-class
    the frequency per class), compared with the observed data's; and the realised deviance D_g(y) = -2 sum_i ll_i(y |
    theta_g), ll the density of ``loo.pointwise_log_lik`` in fp64 (regression with tau_g), compared draw by draw with
    D_g(y_rep_g).  p-values P(T_rep > T_obs) + P(T_rep = T_obs) / 2 over the draws; values near 0 or 1 flag a feature of
    the data the model does not reproduce.  A draw with a non-finite output gets NaN statistics, is left out of the
    p-values and counted.  The same (x, target, seed) give the same bytes on every call, whatever the slab size.
    ``x``, ``target``, ``tau_out`` as ``loo.psis_loo``; y_rep as ``replicate``.  Returns a ``PpcResult``."""
    stats, dev_obs, bad, _, first = _pass(x, target, seed, tau_out, None, False)
    O_ = first.widths[-1]
    y = _y(target, stats.device)
    obs = _observed(y, first.loss_id, O_)
    ok = bad == 0
    r = PpcResult()
    r.names = stat_names(target)
    r.t_rep, r.dev_obs = stats, dev_obs
    r.num_draws, r.num_nonfinite, r.seed = stats.shape[0], int((~ok).sum()), int(seed)
    dev_mean = dev_obs[ok].mean() if bool(ok.any()) else dev_obs.new_tensor(float('nan'))
    r.t_obs = torch.cat([obs, dev_mean.reshape(1)])
    tr = stats[ok]
    per = torch.cat([obs.expand(tr.shape[0], -1), dev_obs[ok][:, None]], 1)
    r.p_value = p_values(tr, per)
    return r


# ------------------------------------------------------------------------------------------------------------------
# LOO-PIT
# ------------------------------------------------------------------------------------------------------------------
def uniformity(u, bins):
    """Equal-width histogram of the finite values of ``u`` in [0, 1] (a value of 1 goes in the last bin) and its chi^2
    test against the uniform distribution: (hist (B,) int64, chi2, p) with expected count M / B, p = gammaincc((B - 1)
    / 2, chi2 / 2) -- ``sbc.rank_histogram``'s test."""
    v = u[torch.isfinite(u)].reshape(-1)
    B = int(bins)
    b = (v * B).floor().clamp(0, B - 1).to(torch.int64)
    hist = torch.bincount(b, minlength=B)
    expected = v.numel() / B
    chi2 = float(((hist.double() - expected) ** 2 / expected).sum()) if v.numel() else float('nan')
    p = float(torch.special.gammaincc(torch.tensor((B - 1) / 2.0, dtype=torch.float64),
                                      torch.tensor(chi2 / 2.0, dtype=torch.float64)))
    return hist, chi2, p


def loo_pit(x, target, r_eff=1.0, tau_out=None, bins=20):
    """LOO-PIT of a Bayesian-NN regression (Gelfand et al. 1992; Gabry et al. 2019): per point i and output o the
    leave-one-out predictive CDF at the observation, pit[i, o] = sum_p w_p Phi((y_io - f_{g_p, i, o}) sqrt(tau_{g_p})),
    w the normalised PSIS weights of ``psis_loo`` (the same sort, tail, generalised-Pareto fit and cap, so ``pareto_k``
    is psis_loo's bit for bit) and g_p the draw at sorted position p.  Uniform when the model is calibrated: a U shape
    says the predictive is too narrow, a hump that it is too wide, a slope that it is biased.  Unlike ``predictive``'s
    PIT on the training data it does not use each point twice.  ``hist`` and the chi^2 test use ``bins`` equal-width
    bins.  ``x``, ``target``, ``r_eff``, ``tau_out`` as ``psis_loo``.  Classification is refused: use
    ``predictive.evaluate``'s reliability table.  Returns a ``LooPitResult``."""
    first = _target(target, 'ppc.loo_pit')
    if first.loss_id != T.LOSS_REGRESSION:
        raise NotImplementedError('ppc.loo_pit: LOO-PIT is defined here for regression; for a classifier check '
                                  'calibration with predictive.evaluate(...).reliability (and .ece)')
    B = _check_bins(bins)
    r_eff = _loo._check_r_eff(r_eff)
    blk = _loo._samples_block(x, target)
    tau_ll = _loo._tau_block(x, blk, tau_out)               # what psis_loo scores with: None is the target's tau_out
    N.require_cuda()
    lib = N.load_library()
    dev = blk.device
    C_, n = int(blk.shape[0]), int(blk.shape[1])
    S = C_ * n
    if S > N.RANK_MAX_DRAWS:
        raise RuntimeError('ppc.loo_pit: %d chains x %d draws exceed the %d draws per point the sort indexes'
                           % (C_, n, N.RANK_MAX_DRAWS))
    nt = _loo._native_target(target, dev)
    Np, O_ = int(nt.mlp_struct.num_rows), first.widths[-1]
    tau = tau_ll if tau_ll is not None else \
        torch.full((1, 1), float(nt.mlp_struct.tau_out), dtype=torch.float32, device=dev).expand(C_, n)
    y = _y(target, dev).contiguous()
    k = _loo._slab_points(lib, C_, n, Np, extra_per_point=4 * S * (1 + O_))
    pit = torch.empty((Np, O_), dtype=torch.float64, device=dev)
    khat = torch.empty(Np, dtype=torch.float64, device=dev)
    flag = torch.empty(Np, dtype=torch.int32, device=dev)
    ws_bytes = lib.hmcx_loo_workspace_bytes(C_, n, k)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        st = N.stream_ptr(dev)
        ll = torch.empty((C_, n, k), dtype=torch.float32, device=dev)
        f = torch.empty((C_, n, k, O_), dtype=torch.float32, device=dev)
        for i0 in range(0, Np, k):
            kk = min(k, Np - i0)
            _loo._ll_rows(lib, nt, blk, i0, i0 + kk, ll, tau_ll)
            _pred._outputs(lib, nt, blk, i0, i0 + kk, f)
            # the pass reads point i at column i of the likelihood block and row i of the outputs block
            rc = lib.hmcx_loo_pit_pass(ctypes.c_void_p(ll.data_ptr() - 4 * i0), ll.stride(0), ll.stride(1),
                                       ctypes.c_void_p(f.data_ptr() - 4 * i0 * O_), f.stride(0), f.stride(1), C_, n, O_,
                                       Np, i0, kk, float(r_eff), N.ptr(y), N.ptr(tau), tau.stride(0), tau.stride(1),
                                       N.ptr(pit), N.ptr(khat), N.ptr(flag), N.ptr(ws), ws_bytes, st)
            N.check(rc, 'hmcx_loo_pit_pass')
        del ws
    r = LooPitResult()
    r.pit, r.pareto_k = pit, khat
    r.k_threshold = min(1.0 - 1.0 / math.log10(S), 0.7)
    r.num_bad_k = int((khat > r.k_threshold).sum())
    r.num_nonfinite = int((flag != 0).sum())
    r.bins = B
    r.hist, r.chi2, r.p_value = uniformity(pit, B)
    r.num_points, r.num_draws, r.r_eff = Np, S, r_eff
    return r
