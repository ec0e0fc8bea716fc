"""numpy fp64 restatement of hamiltorch_b200.predictive: the posterior predictive scores of an outputs block
f[c, s, i, o] (C chains, n draws, N points, O outputs), the targets y and the per-draw noise precision tau (C, n).
Independent of the kernels' formulation: probabilities are averaged directly (no running logsumexp), and the curves
come from cumulative sums over the draws."""
import math

import numpy as np
from scipy.special import log_softmax, ndtr

BINS = 15
LEVELS = (0.5, 0.8, 0.9, 0.95)


def _bins(conf, correct):
    b = np.clip(np.ceil(conf * BINS).astype(np.int64) - 1, 0, BINS - 1)
    table = np.zeros((BINS, 3))
    for j in range(BINS):
        m = b == j
        table[j] = m.sum(), conf[m].sum(), correct[m].sum()
    return table


def _se(v):
    return float(np.std(v, ddof=1) / math.sqrt(v.size)) if v.size > 1 else float('nan')


def evaluate(f, y, loss, tau=None):
    """dict of everything ``evaluate`` reports; loss in 'regression', 'binary_class_linear_output',
    'multi_class_linear_output', 'multi_class_log_softmax_output'."""
    f = np.asarray(f, np.float32).astype(np.float64)
    if f.ndim == 3:
        f = f[None]
    C, n, N, O = f.shape
    S = C * n
    cnt = C * np.arange(1, n + 1, dtype=np.float64)                # draws in the ensemble of entry t - 1
    bad_t = np.cumsum((~np.isfinite(f)).any(axis=(0, 3)), axis=0) > 0   # (n, N): a non-finite draw among the first t
    bad = bad_t[-1]
    f = np.where(np.isfinite(f), f, 0.0)
    out = {'num_nonfinite': int(bad.sum())}
    if loss == 'regression':
        y = np.asarray(y, np.float64).reshape(N, O)
        tau = np.broadcast_to(np.asarray(tau, np.float32).astype(np.float64), (C, n))
        tt = tau[:, :, None, None]
        mean_t = np.cumsum(f.sum(0), axis=0) / cnt[:, None, None]                  # (n, N, O)
        ll = (-0.5 * tt * (f - y) ** 2).sum(3) + 0.5 * O * np.log(tau / (2 * math.pi))[:, :, None]   # (C, n, N)
        M = ll.max(axis=(0, 1))
        lppd_t = np.log(np.cumsum(np.exp(ll - M).sum(0), axis=0) / cnt[:, None]) + M   # (n, N)
        sq_t = ((mean_t - y) ** 2).sum(2)
        mu = mean_t[-1]
        epi = f.reshape(S, N, O).var(0)
        var = np.mean(1.0 / tau) + epi
        pit = ndtr((y - f) * np.sqrt(tt)).reshape(S, N, O).mean(0)
        sq_t[bad_t], lppd_t[bad_t] = np.nan, np.nan
        for a in (mu, var, epi, pit):
            a[bad] = np.nan
        out.update(mean=mu, var=var, epistemic=epi, pit=pit, lppd=lppd_t[-1], nll_i=-lppd_t[-1], sqerr=sq_t[-1],
                   rmse_curve=np.sqrt(sq_t.sum(1) / (N * O)), nll_curve=-lppd_t.sum(1) / N)
        out['rmse'], out['nll'] = out['rmse_curve'][-1], out['nll_curve'][-1]
        out['nll_se'] = _se(out['nll_i'])
        out['coverage'] = {lv: float((np.abs(pit - 0.5) <= lv / 2).sum() / (N * O)) if not bad.any() else float('nan')
                           for lv in LEVELS}
        return out
    if loss == 'binary_class_linear_output':
        y = np.asarray(y, np.float64).reshape(N, O)
        p = 1.0 / (1.0 + np.exp(-f))
        py = y * p + (1 - y) * (1 - p)                                              # p_s(y), y in {0, 1}
        pbar_t = np.cumsum(p.sum(0), axis=0) / cnt[:, None, None]
        pyt = np.cumsum(py.sum(0), axis=0) / cnt[:, None, None]
        correct_t = ((pbar_t > 0.5) == (y > 0.5)).sum(2).astype(np.float64)
        nll_t = -np.log(pyt).sum(2)
        h = lambda q: -(np.where(q > 0, q * np.log(np.where(q > 0, q, 1)), 0)
                        + np.where(q < 1, (1 - q) * np.log(np.where(q < 1, 1 - q, 1)), 0))
        pbar = pbar_t[-1]
        ent = h(pbar).sum(1)
        eent = h(p).sum(3).reshape(S, N).mean(0)
        brier = ((pbar - y) ** 2).sum(1)
        conf = np.maximum(pbar, 1 - pbar)
        corr = (pbar > 0.5) == (y > 0.5)
        table = _bins(conf[~bad].ravel(), corr[~bad].ravel())
        preds = N * O
        pred = pbar > 0.5
    else:
        y = np.asarray(y).reshape(N).astype(np.int64)
        lp = log_softmax(f, axis=3)
        p = np.exp(lp)
        pbar_t = np.cumsum(p.sum(0), axis=0) / cnt[:, None, None]                 # (n, N, O)
        correct_t = (pbar_t.argmax(2) == y).astype(np.float64)
        nll_t = -np.log(np.take_along_axis(pbar_t, y[None, :, None], 2)[..., 0])
        pbar = pbar_t[-1]
        ent = -np.where(pbar > 0, pbar * np.log(np.where(pbar > 0, pbar, 1)), 0).sum(1)
        eent = -np.where(p > 0, p * lp, 0).sum(3).reshape(S, N).mean(0)
        brier = ((pbar - np.eye(O)[y]) ** 2).sum(1)
        pred = pbar.argmax(1)
        corr = pred == y
        conf = pbar.max(1)
        table = _bins(conf[~bad], corr[~bad].astype(np.float64))
        preds = N
        out['top2_gap'] = np.diff(np.sort(pbar, 1)[:, -2:], axis=1)[:, 0] if O > 1 else np.ones(N)
    correct_t[bad_t], nll_t[bad_t] = np.nan, np.nan
    nll_i = nll_t[-1]
    correct = correct_t[-1]
    mi = ent - eent
    for a in (pbar, ent, eent, mi, brier):
        a[bad] = np.nan
    out.update(probs=pbar, pred=pred, nll_i=nll_i, brier_i=brier, entropy=ent, expected_entropy=eent, mutual_info=mi,
               correct=correct, accuracy_curve=correct_t.sum(1) / preds, nll_curve=nll_t.sum(1) / N)
    out['accuracy'], out['nll'] = out['accuracy_curve'][-1], out['nll_curve'][-1]
    out['brier'] = brier.sum() / N
    out['accuracy_se'] = _se(correct / (O if loss == 'binary_class_linear_output' else 1))
    out['nll_se'], out['brier_se'] = _se(nll_i), _se(brier)
    out['reliability_sums'] = table if not bad.any() else np.full_like(table, np.nan)
    out['ece'] = np.abs(table[:, 2] - table[:, 1]).sum() / preds if not bad.any() else float('nan')
    return out
