"""numpy fp64 restatement of per-chain PSIS-LOO, stacking and the chain-weighted held-out predictive
(hamiltorch_b200.loo.psis_loo_chains / stacking_weights / chain_stacking, predictive.evaluate(..., chain_weights=)).

Per-chain PSIS is tests/loo_oracle.psis_point on each chain's column.  The stacking objective of E (K, N) at w on the
simplex is f(w) = sum_i log sum_k w_k exp(E_ki), its gradient g_k = sum_i exp(E_ki) / sum_j w_j exp(E_ji).  The reference
solver is the multiplicative (EM) update run to a gap max_k g_k / N - 1 of 1e-12, checked against scipy's SLSQP on the
simplex.  The weighted predictive restates tests/predictive_oracle.py's definitions with a per-draw weight w_c / t for
the t first draws of chain c (probabilities and densities mixed directly, no running logsumexp)."""
import math

import numpy as np
from scipy.optimize import minimize
from scipy.special import log_softmax, ndtr

from tests import loo_oracle as LO
from tests import predictive_oracle as PO


# ------------------------------------------------------------------------------------------------------------------
# Per-chain PSIS-LOO
# ------------------------------------------------------------------------------------------------------------------
def psis_loo_chains(ll, r_eff=1.0):
    """(C, n, N) block -> dict of (C, N) arrays elpd_loo, lppd, pareto_k, tail and (C,) elpd_total, se."""
    a = np.asarray(ll, dtype=np.float64)
    C, n, Np = a.shape
    keys = ('elpd_loo', 'lppd', 'pareto_k', 'tail')
    out = {k: np.zeros((C, Np), dtype=np.int64 if k == 'tail' else np.float64) for k in keys}
    for c in range(C):
        for i in range(Np):
            p = LO.psis_point(a[c, :, i], r_eff)
            for k in keys:
                out[k][c, i] = p[k]
    out['elpd_total'] = out['elpd_loo'].sum(1)
    out['se'] = np.array([LO._se(out['elpd_loo'][c]) for c in range(C)])
    out['k_threshold'] = min(1.0 - 1.0 / math.log10(n), 0.7)
    out['num_bad_k'] = (out['pareto_k'] > out['k_threshold']).sum(1)
    return out


# ------------------------------------------------------------------------------------------------------------------
# Stacking
# ------------------------------------------------------------------------------------------------------------------
def objective(E, w):
    """(f, g, pointwise) at w."""
    E = np.asarray(E, np.float64)
    w = np.asarray(w, np.float64)
    m = E.max(0)
    s = (w[:, None] * np.exp(E - m)).sum(0)
    pw = m + np.log(s)
    g = (np.exp(E - m) / s).sum(1)
    return pw.sum(), g, pw


def solve_em(E, gap=1e-12, max_iter=2000000):
    """EM from uniform weights until max_k g_k / N - 1 <= gap; returns (w, f, iterations)."""
    E = np.asarray(E, np.float64)
    K, Np = E.shape
    w = np.full(K, 1.0 / K)
    for it in range(max_iter):
        f, g, _ = objective(E, w)
        if g.max() / Np - 1.0 <= gap:
            return w, f, it
        w = w * g / Np
    raise RuntimeError('solve_em: no convergence to %g in %d iterations' % (gap, max_iter))


def solve_slsqp(E):
    """The same maximisation by scipy's SLSQP over the simplex (w = softmax-free: bounds [0, 1] and sum w = 1)."""
    E = np.asarray(E, np.float64)
    K = E.shape[0]
    m = E.max(0)
    P = np.exp(E - m)

    def neg(w):
        return -(m + np.log(np.maximum(w @ P, 1e-300))).sum()

    def neg_grad(w):
        return -(P / np.maximum(w @ P, 1e-300)).sum(1)

    res = minimize(neg, np.full(K, 1.0 / K), jac=neg_grad, method='SLSQP', bounds=[(0.0, 1.0)] * K,
                   constraints=[{'type': 'eq', 'fun': lambda w: w.sum() - 1.0, 'jac': lambda w: np.ones(K)}],
                   options={'ftol': 1e-15, 'maxiter': 1000})
    w = np.clip(res.x, 0.0, None)
    w = w / w.sum()
    return w, objective(E, w)[0]


# ------------------------------------------------------------------------------------------------------------------
# The chain-weighted held-out predictive
# ------------------------------------------------------------------------------------------------------------------
def evaluate_weighted(f, y, loss, w, tau=None):
    """predictive_oracle.evaluate's dict for the mixture sum_c w_c (chain c's draws, equally weighted); the curve entry
    t - 1 mixes the first t draws of every chain with the same chain weights.  Chains with w_c = 0 are dropped."""
    f = np.asarray(f, np.float32).astype(np.float64)
    if f.ndim == 3:
        f = f[None]
    w = np.asarray(w, np.float64)
    w = w / w.sum()
    keep = w > 0
    if tau is not None:
        tau = np.broadcast_to(np.asarray(tau, np.float32).astype(np.float64), f.shape[:2])[keep]
    f, w = f[keep], w[keep]
    C, n, Np, O = f.shape
    t = np.arange(1, n + 1, dtype=np.float64)
    # v[c, s, t - 1] = the weight of draw (c, s) in the ensemble of entry t - 1: w_c / t for s < t
    v = np.where(np.arange(n)[None, :, None] < t[None, None, :].astype(np.int64), 1.0, 0.0) * w[:, None, None] / t
    vn = w[:, None] / n * np.ones((C, n))                                     # the full ensemble
    bad_t = np.cumsum((~np.isfinite(f)).any(axis=(0, 3)), axis=0) > 0
    bad = bad_t[-1]
    f = np.where(np.isfinite(f), f, 0.0)
    mix_t = lambda a: np.einsum('cst,csi...->ti...', v, a)                    # (n, N, ...) curve mixtures
    mix = lambda a: np.einsum('cs,csi...->i...', vn, a)                       # (N, ...) full mixture
    out = {'num_nonfinite': int(bad.sum())}
    if loss == 'regression':
        y = np.asarray(y, np.float64).reshape(Np, O)
        tt = tau[:, :, None, None]
        mean_t = mix_t(f)
        ll = (-0.5 * tt * (f - y) ** 2).sum(3) + 0.5 * O * np.log(tau / (2 * math.pi))[:, :, None]
        M = ll.max(axis=(0, 1))
        lppd_t = np.log(mix_t(np.exp(ll - M))) + M
        sq_t = ((mean_t - y) ** 2).sum(2)
        mu = mean_t[-1]
        epi = mix((f - mu) ** 2)
        var = (vn * (1.0 / tau)).sum() + epi
        pit = mix(ndtr((y - f) * np.sqrt(tt)))
        sq_t[bad_t], lppd_t[bad_t] = np.nan, np.nan
        for a in (mu, var, epi, pit):
            a[bad] = np.nan
        out.update(mean=mu, var=var, epistemic=epi, pit=pit, lppd=lppd_t[-1], nll_i=-lppd_t[-1], sqerr=sq_t[-1],
                   rmse_curve=np.sqrt(sq_t.sum(1) / (Np * O)), nll_curve=-lppd_t.sum(1) / Np)
        out['rmse'], out['nll'] = out['rmse_curve'][-1], out['nll_curve'][-1]
        out['nll_se'] = PO._se(out['nll_i'])
        out['coverage'] = {lv: float((np.abs(pit - 0.5) <= lv / 2).sum() / (Np * O)) if not bad.any() else float('nan')
                           for lv in PO.LEVELS}
        return out
    if loss == 'binary_class_linear_output':
        y = np.asarray(y, np.float64).reshape(Np, O)
        p = 1.0 / (1.0 + np.exp(-f))
        py = y * p + (1 - y) * (1 - p)
        pbar_t = mix_t(p)
        correct_t = ((pbar_t > 0.5) == (y > 0.5)).sum(2).astype(np.float64)
        nll_t = -np.log(mix_t(py)).sum(2)
        h = lambda q: -(np.where(q > 0, q * np.log(np.where(q > 0, q, 1)), 0)
                        + np.where(q < 1, (1 - q) * np.log(np.where(q < 1, 1 - q, 1)), 0))
        pbar = pbar_t[-1]
        ent = h(pbar).sum(1)
        eent = mix(h(p).sum(3))
        brier = ((pbar - y) ** 2).sum(1)
        conf = np.maximum(pbar, 1 - pbar)
        corr = (pbar > 0.5) == (y > 0.5)
        table = PO._bins(conf[~bad].ravel(), corr[~bad].ravel())
        preds = Np * O
        pred = pbar > 0.5
    else:
        y = np.asarray(y).reshape(Np).astype(np.int64)
        lp = log_softmax(f, axis=3)
        p = np.exp(lp)
        pbar_t = mix_t(p)
        correct_t = (pbar_t.argmax(2) == y).astype(np.float64)
        nll_t = -np.log(np.take_along_axis(pbar_t, y[None, :, None], 2)[..., 0])
        pbar = pbar_t[-1]
        ent = -np.where(pbar > 0, pbar * np.log(np.where(pbar > 0, pbar, 1)), 0).sum(1)
        eent = mix(-np.where(p > 0, p * lp, 0).sum(3))
        brier = ((pbar - np.eye(O)[y]) ** 2).sum(1)
        pred = pbar.argmax(1)
        corr = pred == y
        conf = pbar.max(1)
        table = PO._bins(conf[~bad], corr[~bad].astype(np.float64))
        preds = Np
        out['top2_gap'] = np.diff(np.sort(pbar, 1)[:, -2:], axis=1)[:, 0] if O > 1 else np.ones(Np)
    correct_t[bad_t], nll_t[bad_t] = np.nan, np.nan
    nll_i = nll_t[-1]
    correct = correct_t[-1]
    mi = ent - eent
    for a in (pbar, ent, eent, mi, brier):
        a[bad] = np.nan
    out.update(probs=pbar, pred=pred, nll_i=nll_i, brier_i=brier, entropy=ent, expected_entropy=eent, mutual_info=mi,
               correct=correct, accuracy_curve=correct_t.sum(1) / preds, nll_curve=nll_t.sum(1) / Np)
    out['accuracy'], out['nll'] = out['accuracy_curve'][-1], out['nll_curve'][-1]
    out['brier'] = brier.sum() / Np
    out['accuracy_se'] = PO._se(correct / (O if loss == 'binary_class_linear_output' else 1))
    out['nll_se'], out['brier_se'] = PO._se(nll_i), PO._se(brier)
    out['reliability_sums'] = table if not bad.any() else np.full_like(table, np.nan)
    out['ece'] = np.abs(table[:, 2] - table[:, 1]).sum() / preds if not bad.any() else float('nan')
    return out
