"""numpy / torch fp64 definition of hamiltorch_b200.loo (PSIS-LOO and WAIC of a Bayesian NN), which the CUDA passes
(hmcx_mlp_pointwise_ll, hmcx_loo_pass) are tested against.

Pointwise log-likelihood, f = network output (O values), tau = tau_out:
    regression   sum_o -0.5 tau (f_o - y_o)^2 + 0.5 O log(tau / 2 pi)      (a normalised density; tau = noise precision)
    binary       sum_o -BCEWithLogits(f_o, y_o), torch's stable form
    multi-class  log_softmax(f)[y];  LogSoftmax output: f[y]
tau_out tempers the classification likelihoods while sampling; it does not enter their predictive density.

PSIS / WAIC per data point over its S pooled draws ll_s (Vehtari, Gelman & Gabry 2017; Vehtari et al. 2024):
 1. r_s = -ll_s, then r_s <- r_s - max r.
 2. M = ceil(min(0.2 S, 3 sqrt(S / r_eff))).
 3. cutoff c = the (M+1)-th largest r, floored at log(DBL_MIN).
 4. tail = {s : r_s > c}, size M' <= M (ties at the cutoff stay out).  M' <= 4: no smoothing, k-hat = +inf.
 5. Zhang & Stephens (2009) fit to the ascending exceedances x_t = exp(r_(t)) - exp(c), t = 1..M':
      m = 30 + floor(sqrt(M')),  b_j = 1/x_M' + (1 - sqrt(m/(j - 1/2))) / (3 x_floor(M'/4 + 1/2))   (1-based, j = 1..m)
      k_j = mean_t log1p(-b_j x_t),  L_j = M' (log(-b_j/k_j) - k_j - 1),  w_j = 1 / sum_l exp(L_l - L_j),
      weights below 10 eps dropped, the rest renormalised,  b = sum w_j b_j,  xi = mean_t log1p(-b x_t),
      sigma = -xi / b,  k-hat = (M' xi + 5) / (M' + 10).
 6. (k-hat finite) the tail's log-ratios, ascending z = 1..M', become log(q_z + exp(c)),
      q_z = sigma/k-hat ((1 - p_z)^-k-hat - 1) evaluated as sigma expm1(-k-hat log1p(-p_z)) / k-hat (k-hat = 0: the limit
      -sigma log1p(-p_z)), p_z = (z - 1/2)/M'; every log-ratio is capped at 0; lw = log-ratios - logsumexp(log-ratios).
 7. elpd_loo = logsumexp(lw + ll), lppd = logsumexp(ll) - log S, p_loo = lppd - elpd_loo, p_waic = var(ll, ddof 1),
    elpd_waic = lppd - p_waic.
 8. totals are sums, se = sqrt(N) sd(pointwise, ddof 1), looic = -2 elpd_loo; bad points: k-hat > min(1 - 1/log10 S, 0.7);
    WAIC warnings: p_waic > 0.4.
 9. a point with a non-finite draw: NaN outputs, counted.
"""
import math

import numpy as np
import torch

DBL_MIN = np.finfo(np.float64).tiny
EPS = np.finfo(np.float64).eps


# ------------------------------------------------------------------------------------------------------------------
# pointwise log-likelihood
# ------------------------------------------------------------------------------------------------------------------
def _split_data(target):
    items = target if isinstance(target, list) else [target]
    first = items[0]
    x = torch.cat([t.x for t in items]).double()
    y = torch.cat([t.y.reshape(t.x.shape[0], first.y_cols) for t in items]).double()
    return first, x, y


def pointwise_log_lik(samples, target):
    """samples (S, D) -> (S, N) fp64 numpy: ll[s, i] = log p(y_i | theta_s), the network evaluated in fp64."""
    first, x, y = _split_data(target)
    th = torch.as_tensor(samples).detach().cpu().double().reshape(-1, first.dim)
    O = first.widths[-1]
    out = []
    for s in range(th.shape[0]):
        h = x
        for l, (W, b) in enumerate(first.unflatten(th[s])):
            h = torch.nn.functional.linear(h, W, b)
            if l < first.num_layers - 1:
                h = {1: torch.relu, 2: torch.tanh, 3: torch.sigmoid}.get(first.acts[l], lambda v: v)(h)
        f = h
        if first.loss_id == 0:
            tau = first.tau_out
            ll = (-0.5 * tau * (f - y) ** 2).sum(1) + 0.5 * O * math.log(tau / (2 * math.pi))
        elif first.loss_id == 1:
            ll = -torch.nn.functional.binary_cross_entropy_with_logits(f, y, reduction='none').sum(1)
        else:
            # multi-class: log_softmax of the logits at the label (a LogSoftmax output layer makes f[y] the same value)
            ll = torch.log_softmax(f, 1).gather(1, y[:, 0].long()[:, None])[:, 0]
        out.append(ll.numpy())
    return np.stack(out)


# ------------------------------------------------------------------------------------------------------------------
# PSIS
# ------------------------------------------------------------------------------------------------------------------
def tail_cap(S, r_eff=1.0):
    return int(math.ceil(min(0.2 * S, 3.0 * math.sqrt(S / r_eff))))


def gpd_fit(x):
    """Zhang & Stephens (2009) with the weakly informative prior on the shape; x ascending exceedances (fp64).
    Returns (k-hat, sigma)."""
    x = np.asarray(x, dtype=np.float64)
    Mt = x.size
    m = 30 + math.isqrt(Mt)
    j = np.arange(1, m + 1, dtype=np.float64)
    b = 1.0 / x[-1] + (1.0 - np.sqrt(m / (j - 0.5))) / (3.0 * x[int(math.floor(Mt / 4.0 + 0.5)) - 1])
    k = np.log1p(-b[:, None] * x[None, :]).mean(1)
    L = Mt * (np.log(-b / k) - k - 1.0)
    with np.errstate(over='ignore'):                           # a sum that overflows gives the weight 0
        w = 1.0 / np.exp(L[None, :] - L[:, None]).sum(1)
    keep = w >= 10 * EPS
    w = w[keep] / w[keep].sum()
    bbar = (w * b[keep]).sum()
    xi = np.log1p(-bbar * x).mean()
    sigma = -xi / bbar
    khat = (Mt * xi + 5.0) / (Mt + 10.0)
    return khat, sigma


def _lse(v):
    mx = v.max()
    return mx + math.log(np.exp(v - mx).sum())


def psis_point(ll, r_eff=1.0):
    """One point's S draws (any order) -> dict of elpd_loo, p_loo, pareto_k, lppd, p_waic, elpd_waic, tail."""
    ll = np.asarray(ll, dtype=np.float64).reshape(-1)
    S = ll.size
    nan = float('nan')
    if not np.all(np.isfinite(ll)):
        return dict(elpd_loo=nan, p_loo=nan, pareto_k=nan, lppd=nan, p_waic=nan, elpd_waic=nan, tail=0)
    r = -ll
    r = r - r.max()
    M = tail_cap(S, r_eff)
    c = max(np.sort(r)[::-1][M], math.log(DBL_MIN))
    order = np.argsort(r, kind='stable')
    in_tail = r > c
    Mt = int(in_tail.sum())
    lw = r.copy()
    khat = float('inf')
    if Mt > 4:
        tail_idx = order[S - Mt:]                              # ascending r
        x = np.exp(r[tail_idx]) - math.exp(c)
        khat, sigma = gpd_fit(x)
        if math.isfinite(khat):
            pz = (np.arange(1, Mt + 1) - 0.5) / Mt
            q = -sigma * np.log1p(-pz) if khat == 0 else sigma * np.expm1(-khat * np.log1p(-pz)) / khat
            lw[tail_idx] = np.log(q + math.exp(c))
    lw = np.minimum(lw, 0.0)
    lw = lw - _lse(lw)
    elpd = _lse(lw + ll)
    lppd = _lse(ll) - math.log(S)
    pw = ll.var(ddof=1)
    return dict(elpd_loo=elpd, p_loo=lppd - elpd, pareto_k=khat, lppd=lppd, p_waic=pw, elpd_waic=lppd - pw, tail=Mt)


def _as_draws(ll):
    a = np.asarray(ll, dtype=np.float64)
    if a.ndim == 3:
        a = a.reshape(-1, a.shape[2])
    return a


def _se(v):
    return math.sqrt(v.size) * v.std(ddof=1) if v.size > 1 else float('nan')


def psis_loo(ll, r_eff=1.0):
    """(C, n, N) or (S, N) block -> per-point arrays and totals (numpy fp64)."""
    a = _as_draws(ll)
    S, Np = a.shape
    pts = [psis_point(a[:, i], r_eff) for i in range(Np)]
    out = {k: np.array([p[k] for p in pts], dtype=np.int64 if k == 'tail' else np.float64) for k in pts[0]}
    out['elpd_total'] = out['elpd_loo'].sum()
    out['se'] = _se(out['elpd_loo'])
    out['p_loo_total'] = out['p_loo'].sum()
    out['looic'] = -2.0 * out['elpd_total']
    out['k_threshold'] = min(1.0 - 1.0 / math.log10(S), 0.7)
    out['num_bad_k'] = int((out['pareto_k'] > out['k_threshold']).sum())
    out['num_nonfinite'] = int((~np.isfinite(a)).any(0).sum())
    return out


def waic(ll):
    a = _as_draws(ll)
    S = a.shape[0]
    bad = ~np.isfinite(a).all(0)
    with np.errstate(invalid='ignore'):
        lppd = np.array([_lse(a[:, i]) for i in range(a.shape[1])]) - math.log(S)
        pw = a.var(0, ddof=1)
    lppd[bad], pw[bad] = np.nan, np.nan                        # 9. a point with a non-finite draw: NaN
    e = lppd - pw
    return dict(lppd=lppd, p_waic=pw, elpd_waic=e, elpd_total=e.sum(), se=_se(e), p_waic_total=pw.sum(),
                num_p_waic_warn=int((pw > 0.4).sum()))
