"""fp64 restatement of K-fold cross-validation for the conjugate nn.Linear(d, 1) regression of
tests/test_loo_cpu.py::_conjugate: for each fold the exact Gaussian posterior of the weights from its training rows, and
the exact Gaussian predictive density of each held-out row under it."""
import math

import numpy as np


def conjugate_kfold(x, y, folds, tau_out, tau_w, tau_b):
    """Exact elpd_i = log p(y_i | y_train(k)) for every row i with folds[i] = k >= 0 (NaN at -1 rows), in data order.
    x (N, d), y (N,), folds (N,) integers; prior w ~ N(0, 1/tau_w), b ~ N(0, 1/tau_b); noise precision tau_out."""
    x = np.asarray(x, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64).reshape(-1)
    f = np.asarray(folds).reshape(-1)
    n, d = x.shape
    X1 = np.concatenate([x, np.ones((n, 1))], 1)
    P0 = np.diag([tau_w] * d + [tau_b])
    out = np.full(n, np.nan)
    for k in range(int(f.max()) + 1):
        tr, ho = f != k, f == k
        Sig = np.linalg.inv(P0 + tau_out * X1[tr].T @ X1[tr])
        mu = Sig @ (tau_out * X1[tr].T @ y[tr])
        for i in np.nonzero(ho)[0]:
            m = X1[i] @ mu
            v = 1.0 / tau_out + X1[i] @ Sig @ X1[i]
            out[i] = -0.5 * math.log(2 * math.pi * v) - 0.5 * (y[i] - m) ** 2 / v
    return out


def logmeanexp(ll):
    """(S, N) -> (N,) log mean exp over the S draws, in fp64."""
    ll = np.asarray(ll, dtype=np.float64)
    mx = ll.max(0)
    return mx + np.log(np.exp(ll - mx).sum(0)) - math.log(ll.shape[0])
