"""Held-out evaluation of Bayesian NNs on the GPU: the posterior predictive of every test point over the pooled draws --
ensemble accuracy, NLL, Brier score, calibration (ECE and the reliability table), predictive uncertainty, PIT and
coverage -- and the curves of these scores over the draws, restated in numpy fp64 by tests/predictive_oracle.py.

    r = hamiltorch_b200.predictive.evaluate(res, test_target)       # or samples (C, n, D) / (n, D) / a list of (D,)
    r.accuracy, r.nll, r.brier, r.ece, r.accuracy_curve, r.nll_curve          # classification
    r.rmse, r.nll, r.coverage[0.9], r.pit, r.mean, r.var, r.rmse_curve        # regression
    r = hamiltorch_b200.predictive.evaluate(outputs, y=y, model_loss='multi_class_linear_output')   # (C, n, N, O) block

``test_target`` is an ``MLPTarget`` built on the held-out data (``define_model_log_prob`` / ``MLPTarget.from_model``) or
the list ``define_split_model_log_prob`` returns (points in split order).  Two CUDA passes per slab of points:
  * hmcx_mlp_pointwise_out: one CTA per draw runs the network over the slab's rows (the SIMT tiles, or the 3xTF32
    tensor-core forward of n0 -> 128 -> nL stacks) and writes its outputs -- predict_model's values, bit for bit;
  * hmcx_pred_pass: one thread per point scans the draws t = 1 .. n of every chain, adding the C draws of each step to fp64
    running sums (softmax / sigmoid probabilities, entropies, moments, PIT terms, a running logsumexp of the likelihood),
    and writes the point's terms of every curve entry; the terms are summed in fixed 128-point groups aligned to the point
    index, continued across slabs, and the groups in order (hmcx_pred_totals).
So the (S, N, O) output block is never held: a slab's block and workspace fit ``diagnostics.RANK_WORKSPACE_BUDGET``
bytes (at least one point per slab), and the results are the same bytes whatever the slab size and on every call.

Definitions (per point i, S = C*n pooled draws, f_s the fp32 network outputs, everything else in fp64):
  * multi-class (both losses): p_s = softmax(f_s), pbar = mean_s p_s, predicted label argmax pbar (lowest index on ties),
    nll_i = -log pbar[y_i] (a logsumexp of log p_s[y_i]), brier_i = sum_k (pbar_k - 1[k = y_i])^2, predictive entropy
    H[pbar], expected entropy mean_s H[p_s], mutual information = their difference (0 log 0 = 0);
  * binary (``binary_class_linear_output``): every output an independent Bernoulli, pbar = mean_s sigmoid(f_s);
    accuracy over the N*O predictions pbar > 0.5 against y > 0.5; nll_i, brier_i and the entropies summed over outputs;
  * regression, noise precision tau_s per draw: mean mu = mean_s f_s, var = mean_s 1/tau_s + var_s f_s (ddof 0),
    lppd_i = logsumexp_s ll_s,i - log S with the normalised Gaussian density of ``loo.pointwise_log_lik``,
    PIT u = mean_s Phi((y - f_s) sqrt(tau_s)) (the mixture CDF in closed form).
  tau_out only enters regression.  Curves have n entries: entry t - 1 scores the ensemble of the first t draws of every
  chain (C*t draws); their last entry is the total.
"""
import ctypes as C
import math

import torch

from . import _native as N
from . import diagnostics as _diag
from . import loo as _loo
from . import targets as T

_slab_points_override = None            # tests: force this many data points per slab
_GROUP = 128                            # points per fixed-order group; slab boundaries are multiples of it
BINS = 15                               # equal-width confidence bins (Guo et al. 2017)
LEVELS = (0.5, 0.8, 0.9, 0.95)          # central PIT levels of ``coverage``
_TOTAL_ROWS = 1 + 3 * BINS


class PredictiveResult:
    """``evaluate``'s result.  Per point (CUDA fp64): ``nll_i``, and
      classification: ``probs`` (N, O) = pbar, ``pred`` (N,) int64 labels (multi-class; -1 at a non-finite point) or
        (N, O) bool (binary), ``brier_i``, ``entropy``, ``expected_entropy``, ``mutual_info``;
      regression: ``mean``, ``var``, ``epistemic`` (N, O), ``pit`` (N, O), ``lppd`` (N,).
    Totals (Python floats): ``nll`` = mean nll_i and ``nll_se``; classification ``accuracy``, ``brier`` and their
    ``*_se`` (sd / sqrt N, ddof 1, of the per-point values), ``ece`` and ``reliability`` (15, 3) = count, mean confidence,
    accuracy per bin (NaN for an empty bin); regression ``rmse`` and ``coverage`` {level: fraction}.  Curves (n,) fp64:
    ``nll_curve`` and ``accuracy_curve`` or ``rmse_curve``.  ``num_nonfinite`` counts points with a non-finite output
    (NaN outputs, NaN totals); ``num_points``, ``num_draws``, ``model_loss``; ``chain_weights`` ((C,) fp64 CPU, the
    normalised weights of a weighted evaluation, or None for the pooled draws)."""

    def __repr__(self):
        if self.model_loss == 'regression':
            return ('PredictiveResult(rmse=%.4f, nll=%.4f, coverage90=%.3f, N=%d, S=%d, nonfinite=%d)'
                    % (self.rmse, self.nll, self.coverage[0.9], self.num_points, self.num_draws, self.num_nonfinite))
        return ('PredictiveResult(accuracy=%.4f, nll=%.4f, brier=%.4f, ece=%.4f, N=%d, S=%d, nonfinite=%d)'
                % (self.accuracy, self.nll, self.brier, self.ece, self.num_points, self.num_draws, self.num_nonfinite))


# ------------------------------------------------------------------------------------------------------------------
# Inputs
# ------------------------------------------------------------------------------------------------------------------
def _target_data(target):
    """(loss id, O, y (N, O) or (N,) fp32 CPU tensor in split order, tau_out) of an MLPTarget or a split list."""
    items = _loo._mlp_targets(target, 'predictive', 'evaluate')
    first = items[0]
    O_ = first.widths[-1]
    y = torch.cat([t.y.detach().cpu().reshape(-1, t.y_cols) for t in items])
    return first.loss_id, O_, y, first.tau_out


def _loss_id(model_loss):
    if model_loss not in T.LOSS_ID:
        raise ValueError('predictive: model_loss must be one of %s, got %r' % (sorted(T.LOSS_ID), model_loss))
    return T.LOSS_ID[model_loss]


def _check_y(y, loss, O_, Np):
    y = torch.as_tensor(y).detach().to(torch.float32)
    if loss in (T.LOSS_REGRESSION, T.LOSS_BINARY):
        if y.numel() != Np * O_:
            raise RuntimeError('predictive: y must hold %d x %d values (N points x O outputs), got shape %s'
                               % (Np, O_, tuple(y.shape)))
        y = y.reshape(Np, O_)
        if not bool(torch.isfinite(y).all()):
            raise ValueError('predictive: y must be finite')
    else:
        if y.numel() != Np:
            raise RuntimeError('predictive: y must hold one label per point (%d), got shape %s' % (Np, tuple(y.shape)))
        y = y.reshape(Np)
        if not bool(((y == y.round()) & (y >= 0) & (y < O_)).all()):
            raise ValueError('predictive: multi-class labels must be integers in [0, %d)' % O_)
    return y


def _tau(tau_out, samples, C_, n, device):
    """The (C, n) fp32 per-draw noise precision: ``tau_out`` given (a number, (n,) for one chain, or (C, n)), else the
    ``tau_out_trace`` of an HMCResult; None when neither is there."""
    if tau_out is None:
        tau_out = getattr(samples, 'tau_out_trace', None)
        if tau_out is None:
            return None
    t = torch.as_tensor(tau_out).detach().to(device=device, dtype=torch.float32)
    if t.dim() == 0:
        t = t.expand(C_, n)
    elif t.dim() == 1 and C_ == 1:
        t = t[None]
    if tuple(t.shape) != (C_, n):
        raise RuntimeError('predictive: tau_out must be a number or hold one value per draw, (C, n) = (%d, %d), got %s'
                           % (C_, n, tuple(t.shape)))
    if not bool((t > 0).all()) or not bool(torch.isfinite(t).all()):
        raise ValueError('predictive: tau_out must be positive and finite')
    return t


def _outputs_block(x):
    if not torch.is_tensor(x) or x.dtype != torch.float32:
        raise RuntimeError('predictive: an outputs block must be a CUDA float32 tensor')
    if x.dim() == 3:
        x = x.unsqueeze(0)
    if x.dim() != 4 or min(x.shape) < 1:
        raise RuntimeError('predictive: an outputs block is (C, n, N, O) or (n, N, O), got shape %s' % (tuple(x.shape),))
    if x.stride(3) != 1 or x.stride(2) != x.shape[3]:
        x = x.contiguous()                      # the pass reads each draw's (N, O) rows contiguously
    return x


# ------------------------------------------------------------------------------------------------------------------
# Passes
# ------------------------------------------------------------------------------------------------------------------
def _slab_points(lib, C_, n, O_, loss, Np, block_per_point):
    """Points per slab: the workspace (and, from samples, the slab's fp32 outputs block) within the budget; a multiple
    of 128 points once a slab holds that many."""
    if _slab_points_override is not None:
        return max(1, min(Np, int(_slab_points_override)))
    cost = lib.hmcx_pred_workspace_bytes(C_, n, O_, loss, 1) + block_per_point
    k = max(1, min(Np, _diag.RANK_WORKSPACE_BUDGET // cost))
    if _GROUP <= k < Np:
        k -= k % _GROUP
    return k


def _chain_weights(w):
    """``chain_weights`` as a 1-D fp64 CPU tensor, normalised; refused unless finite, non-negative and summing to 1
    within 1e-6."""
    if w is None:
        return None
    t = torch.as_tensor(w).detach().to(device='cpu', dtype=torch.float64)
    if t.dim() != 1 or t.numel() < 1:
        raise ValueError('predictive: chain_weights must be a (C,) vector, got shape %s' % (tuple(t.shape),))
    if not bool(torch.isfinite(t).all()) or bool((t < 0).any()):
        raise ValueError('predictive: chain_weights must be finite and non-negative')
    total = float(t.sum())
    if abs(total - 1.0) > 1e-6:
        raise ValueError('predictive: chain_weights must sum to 1 (within 1e-6), got %.9g' % total)
    return t / total


def _check_chain_weights(w, C_):
    if w is not None and w.numel() != C_:
        raise ValueError('predictive: chain_weights holds %d weights, the draws come from %d chains' % (w.numel(), C_))


def _run(lib, dev, C_, n, O_, Np, loss, y, tau, fill, cw=None):
    """Drive hmcx_pred_pass (hmcx_pred_pass_weighted with chain weights ``cw``) over the slabs; ``fill(i0, kk)`` returns
    (base pointer of point 0, chain / draw strides)."""
    G = (Np + _GROUP - 1) // _GROUP
    rows = 2 * n + _TOTAL_ROWS
    pw = torch.empty((7, Np), dtype=torch.float64, device=dev)
    po = torch.empty((4 if loss == T.LOSS_REGRESSION else 1, Np, O_), dtype=torch.float64, device=dev)
    flag = torch.empty(Np, dtype=torch.int32, device=dev)
    partials = torch.empty((rows, G), dtype=torch.float64, device=dev)
    totals = torch.empty(rows, dtype=torch.float64, device=dev)
    yd = y.to(dev).contiguous()
    k = fill.k
    ws_bytes = lib.hmcx_pred_workspace_bytes(C_, n, O_, loss, k)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    cwd = None if cw is None else cw.to(dev)
    with torch.cuda.device(dev):
        st = N.stream_ptr(dev)
        for i0 in range(0, Np, k):
            kk = min(k, Np - i0)
            base, cs, ds = fill(i0, kk)
            args = (base, cs, ds, C_, n, O_, loss, N.ptr(yd), N.ptr(tau), 0 if tau is None else tau.stride(0),
                    0 if tau is None else tau.stride(1), Np, i0, kk, N.ptr(pw), N.ptr(po), N.ptr(flag), N.ptr(partials),
                    N.ptr(ws), ws_bytes)
            if cwd is None:
                rc = lib.hmcx_pred_pass(*args, st)
                N.check(rc, 'hmcx_pred_pass')
            else:
                rc = lib.hmcx_pred_pass_weighted(*args, N.ptr(cwd), st)
                N.check(rc, 'hmcx_pred_pass_weighted')
        N.check(lib.hmcx_pred_totals(N.ptr(partials), n, Np, N.ptr(totals), st), 'hmcx_pred_totals')
    return pw, po, flag, totals


def _outputs(lib, nt, x, r0, r1, out):
    """out[c, s, :r1 - r0] = the network outputs of draw (c, s) at rows [r0, r1) (out a (C, n, rows, O) block, each
    draw's rows contiguous)."""
    rc = lib.hmcx_mlp_pointwise_out(nt.ref(), N.ptr(x), x.stride(0), x.stride(1), x.shape[0], x.shape[1], r0, r1,
                                    N.ptr(out), out.stride(0), out.stride(1), N.stream_ptr(x.device))
    N.check(rc, 'hmcx_mlp_pointwise_out')


class _FromSamples:
    def __init__(self, lib, nt, x, O_, k):
        self.lib, self.nt, self.x, self.O, self.k, self.device = lib, nt, x, O_, k, x.device
        self.blk = torch.empty((x.shape[0], x.shape[1], k, O_), dtype=torch.float32, device=x.device)

    def __call__(self, i0, kk):
        b = self.blk
        _outputs(self.lib, self.nt, self.x, i0, i0 + kk, b)
        # the pass reads point i at row i of the block: the slab's block holds rows [i0, i0 + kk)
        return C.c_void_p(b.data_ptr() - 4 * i0 * self.O), b.stride(0), b.stride(1)


class _FromBlock:
    def __init__(self, f, k):
        self.f, self.k, self.device = f, k, f.device

    def __call__(self, i0, kk):
        return N.ptr(self.f), self.f.stride(0), self.f.stride(1)


def pointwise_outputs(samples, target, row_begin=0, row_end=None):
    """The (C, n, rows, O) fp32 CUDA tensor of the network outputs of every draw at the target's rows [row_begin,
    row_end) -- what ``predict_model`` returns for those rows (log-probabilities for a LogSoftmax network), bit for bit.
    ``samples`` / ``target`` as ``evaluate``."""
    loss, O_, _, _ = _target_data(target)
    x = _loo._samples_block(samples, target)
    N.require_cuda()
    lib = N.load_library()
    nt = _loo._native_target(target, x.device)
    Np = int(nt.mlp_struct.num_rows)
    row_end = Np if row_end is None else int(row_end)
    out = torch.empty((x.shape[0], x.shape[1], row_end - row_begin, O_), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        _outputs(lib, nt, x, int(row_begin), row_end, out)
    return out


def _sd_se(v):
    n = v.numel()
    return float(v.std(unbiased=True) / math.sqrt(n)) if n > 1 else float('nan')


def evaluate(x, target=None, *, y=None, model_loss=None, tau_out=None, chain_weights=None):
    """Score the posterior predictive of a Bayesian NN on held-out data, on the GPU.

    Two routes:
      * samples with a target: ``x`` is what ``diagnostics.summary`` reads (an ``HMCResult``, a (C, n, D) / (n, D) CUDA
        fp32 tensor, the list ``sample`` returns), refused in the same cases; ``target`` an ``MLPTarget`` with the
        held-out data, or a split list.  The outputs are computed slab by slab; the (S, N, O) block is never held.
      * an outputs block: ``x`` a (C, n, N, O) or (n, N, O) CUDA fp32 tensor (e.g. ``predict_model``'s outputs
        reshaped), with ``y`` and ``model_loss`` -- or with a ``target`` that brings both (its O must match).
    ``tau_out`` (regression only): a number, or one noise precision per draw, (C, n) (or (n,) for one chain); an
    ``HMCResult`` of a run with a tau_out hyperprior brings its ``tau_out_trace``; otherwise the target's value.  An
    outputs block of a regression without a target needs it.  See the module docstring for the definitions.
    ``chain_weights``: (C,) non-negative weights summing to 1 (normalised; refused if off by more than 1e-6), e.g.
    ``loo.chain_stacking(...).weights``.  The predictive is then the mixture sum_c w_c (chain c's draws, equally
    weighted) instead of the pooled draws, and every curve entry t the same mixture of the first t draws of every chain;
    chains with weight 0 are not read.  None: the pooled predictive.
    Returns a ``PredictiveResult`` (its ``chain_weights``: the normalised weights, or None)."""
    cw = _chain_weights(chain_weights)
    if target is not None and not (torch.is_tensor(x) and x.dim() == 4):
        loss, O_, yv, tau_t = _target_data(target)
        if y is not None or model_loss is not None:
            raise RuntimeError('predictive: y and model_loss come from the target; pass them with an outputs block only')
        Np = int(yv.shape[0])
        yv = _check_y(yv, loss, O_, Np)
        blk = _loo._samples_block(x, target)
        C_, n = int(blk.shape[0]), int(blk.shape[1])
        _check_chain_weights(cw, C_)
        tau = _tau(tau_out, x, C_, n, blk.device) if loss == T.LOSS_REGRESSION else None
        if loss == T.LOSS_REGRESSION and tau is None:
            tau = _tau(tau_t, None, C_, n, blk.device)
        N.require_cuda()
        lib = N.load_library()
        nt = _loo._native_target(target, blk.device)
        k = _slab_points(lib, C_, n, O_, loss, Np, 4 * C_ * n * O_)
        fill = _FromSamples(lib, nt, blk, O_, k)
    else:
        if target is not None:
            loss, O_, yv, tau_t = _target_data(target)
            if y is not None or model_loss is not None:
                raise RuntimeError('predictive: y and model_loss come from the target; pass them without one')
        else:
            if y is None or model_loss is None:
                raise RuntimeError('predictive: an outputs block needs y and model_loss (or a target)')
            loss, yv, tau_t, O_ = _loss_id(model_loss), y, None, None
        f = _outputs_block(x)
        C_, n, Np = int(f.shape[0]), int(f.shape[1]), int(f.shape[2])
        _check_chain_weights(cw, C_)
        if O_ is not None and int(f.shape[3]) != O_:
            raise RuntimeError('predictive: the block has %d outputs per point, the target %d' % (f.shape[3], O_))
        O_ = int(f.shape[3])
        yv = _check_y(yv, loss, O_, Np)
        tau = None
        if loss == T.LOSS_REGRESSION:
            tau = _tau(tau_out if tau_out is not None else tau_t, None, C_, n, f.device)
            if tau is None:
                raise RuntimeError('predictive: a regression outputs block needs tau_out')
        if not f.is_cuda:
            raise RuntimeError('predictive: the outputs block is a %s tensor; the evaluation runs on a CUDA device and '
                               'there is no CPU fallback' % f.device.type)
        N.require_cuda()
        lib = N.load_library()
        fill = _FromBlock(f, _slab_points(lib, C_, n, O_, loss, Np, 0))
    pw, po, flag, tot = _run(lib, fill.device, C_, n, O_, Np, loss, yv, tau, fill, cw)
    r = _result(pw, po, flag, tot, loss, C_, n, O_, Np)
    r.chain_weights = cw
    return r


def _result(pw, po, flag, tot, loss, C_, n, O_, Np):
    r = PredictiveResult()
    r.model_loss = {v: k for k, v in T.LOSS_ID.items()}[loss]
    r.num_points, r.num_draws = Np, C_ * n
    r.num_nonfinite = int((flag != 0).sum())
    r.nll_i = pw[0]
    r.nll_curve = tot[n:2 * n] / Np
    r.nll, r.nll_se = float(r.nll_curve[-1]), _sd_se(pw[0])
    if loss == T.LOSS_REGRESSION:
        r.mean, r.var, r.epistemic, r.pit = po[0], po[1], po[2], po[3]
        r.lppd = -pw[0]
        r.rmse_curve = (tot[:n] / (Np * O_)).sqrt()
        r.rmse = float(r.rmse_curve[-1])
        cov = (tot[2 * n:2 * n + len(LEVELS)] / (Np * O_)).tolist()
        r.coverage = dict(zip(LEVELS, cov))
        return r
    binary = loss == T.LOSS_BINARY
    preds = Np * O_ if binary else Np
    r.probs = po[0]
    r.pred = (po[0] > 0.5) if binary else torch.where(flag != 0, -1, pw[6].nan_to_num(-1.0).to(torch.int64))
    r.brier_i, r.entropy, r.expected_entropy, r.mutual_info = pw[1], pw[2], pw[3], pw[4]
    r.accuracy_curve = tot[:n] / preds
    r.accuracy = float(r.accuracy_curve[-1])
    r.accuracy_se = _sd_se(pw[5] / (O_ if binary else 1))
    r.brier, r.brier_se = float(tot[2 * n] / Np), _sd_se(pw[1])
    bins = tot[2 * n + 1:2 * n + 1 + 3 * BINS].reshape(BINS, 3)
    r.ece = float((bins[:, 2] - bins[:, 1]).abs().sum() / preds)
    r.reliability = torch.stack([bins[:, 0], bins[:, 1] / bins[:, 0], bins[:, 2] / bins[:, 0]], 1)
    return r
