"""CPU oracle of the hyperprior Gibbs steps (DESIGN §3.15): oracle/hmc_oracle.py's sample() loop for the Bayesian NN, with
the precisions drawn from their Gamma conditionals after every MH step and the target rebuilt from them.

Per iteration n: momentum -> trajectory -> MH gives q_n; then, for every sampled group k (the parameter tensors in tau_list
order, then tau_out), tau_k = fp32(g / rate) with g the injected standard-gamma draw of shape a_k + n_k / 2 and
rate = b_k + |w_k|^2 / 2 (tau_out: a_o + N O / 2, b_o + SSE(q_n) / 2), all in fp64; iteration n + 1 samples the target
built (targets.MLPTarget) from the new values.  The trace slots follow the retained samples; slot 0 = the initial values.
"""
import numpy as np
import torch

from hamiltorch_b200 import targets as T
from oracle import hmc_oracle as O


def rebuild(tgt, tau_list, tau_out):
    """The descriptor (or split list) with new precisions: MLPTarget's own fp32 constants."""
    def one(d):
        taus = [torch.tensor(float(t), dtype=torch.float32) for t in tau_list]
        return T.MLPTarget(d.widths, d.acts, d.x, d.y, taus, tau_out, d.prior_scale, d.model_loss, d.final_log_softmax)
    return [one(d) for d in tgt] if isinstance(tgt, list) else one(tgt)


def tensor_sizes(tgt):
    return list((tgt[0] if isinstance(tgt, list) else tgt).sizes)


def n_obs(tgt):
    descs = tgt if isinstance(tgt, list) else [tgt]
    return sum(d.x.shape[0] for d in descs) * descs[0].widths[-1]


def sse(tgt, q):
    """Sum of squared errors over every data row (all splits), fp64."""
    total = 0.0
    for d in (tgt if isinstance(tgt, list) else [tgt]):
        out = d.forward(q, d.x).double()
        total += float(((out - d.y.double().view_as(out)) ** 2).sum())
    return total


def posterior_shape_rate(a, b, n, stat):
    """Gamma(a, b) prior, Gaussian likelihood of n values with sum of squares `stat`: the conditional's (shape, rate)."""
    return a + 0.5 * n, b + 0.5 * stat


def gibbs_update(tgt, q, hyper, tau_list, tau_out, g):
    """One Gibbs step of the precisions given q; g: the standard-gamma draws of the 2L + 1 groups."""
    tau_list, sizes = list(tau_list), tensor_sizes(tgt)
    off = 0
    for k, n in enumerate(sizes):
        if hyper[k] is not None:
            w = q[off:off + n].double()
            shape, rate = posterior_shape_rate(hyper[k][0], hyper[k][1], n, float((w * w).sum()))
            tau_list[k] = float(np.float32(float(g[k]) / rate))
        off += n
    if hyper[-1] is not None:
        shape, rate = posterior_shape_rate(hyper[-1][0], hyper[-1][1], n_obs(tgt), sse(tgt, q))
        tau_out = float(np.float32(float(g[-1]) / rate))
    return tau_list, tau_out


def sample_hyper(tgt, params_init, num_samples, L, step_size, burn, hyper, normals, log_uniforms, gammas, perms=None,
                 split_scheme=None, eps_schedule=None):
    """One chain.  normals (S, D), log_uniforms (S,), gammas (S, 2L + 1), perms (S, M) or None; eps_schedule (S,)
    teacher-forces the step size of every iteration (HMC_NUTS parity).  Returns samples, accepted, ham_old / ham_new and
    the traces tau_list (S - burn, 2L), tau_out (S - burn,)."""
    d0 = tgt[0] if isinstance(tgt, list) else tgt
    tau_list, tau_out = [float(t) for t in d0.tau_list], float(d0.tau_out)
    cur = tgt
    q = params_init.clone()
    burn_prev = params_init.clone()
    kept = [params_init.clone()]
    tr_tau, tr_out = [list(tau_list)], [tau_out]
    accepted, ham_old, ham_new = [], [], []
    for n in range(num_samples):
        eps = step_size if eps_schedule is None else float(eps_schedule[n])
        p = O.momentum_from_normals(normals[n])
        H0 = O.hamiltonian_hmc(cur, q, p)
        if split_scheme is None:
            qs, ps = O.leapfrog_hmc(cur, q, p, L, eps)
        else:
            qs, ps = O.leapfrog_split(cur, q, p, L, eps, None, split_scheme, None if perms is None else perms[n])
        q = qs[-1].detach()
        H1 = O.hamiltonian_hmc(cur, q, ps[-1])
        rho = O.log_accept_ratio(H0, H1)
        ok = rho >= log_uniforms[n].reshape(1)
        accepted.append(bool(ok))
        if ok:
            if n > burn:
                kept.append(qs[-1])
            else:
                burn_prev = qs[-1].clone()
        else:
            q = kept[-1] if n > burn else burn_prev.clone()
            if n > burn:
                kept.append(kept[-1])
        ham_old.append(float(H0))
        ham_new.append(float(H1))
        tau_list, tau_out = gibbs_update(cur, q, hyper, tau_list, tau_out, gammas[n])
        cur = rebuild(tgt, tau_list, tau_out)
        if n > burn:
            tr_tau.append(list(tau_list))
            tr_out.append(tau_out)
    return dict(samples=torch.stack([t.detach() for t in kept]), accepted=accepted, ham_old=ham_old, ham_new=ham_new,
                tau_list=np.array(tr_tau, dtype=np.float32), tau_out=np.array(tr_out, dtype=np.float32))


def linear_gibbs(x, y, a_w, b_w, a_b, b_b, a_o, b_o, num_samples, seed, tau_w=1.0, tau_b=1.0, tau_o=1.0):
    """Exact fp64 Gibbs sampler of Bayesian linear regression y = x w + b + noise, w ~ N(0, 1/tau_w), b ~ N(0, 1/tau_b),
    noise ~ N(0, 1/tau_o), Gamma hyperpriors on the three precisions; (w, b) | tau is Gaussian.  Returns (S, d + 3):
    w, b, log tau_w, log tau_b, log tau_o."""
    rng = np.random.default_rng(seed)
    x = np.asarray(x, np.float64)
    y = np.asarray(y, np.float64).reshape(-1)
    n, d = x.shape
    X = np.hstack([x, np.ones((n, 1))])
    XtX, Xty = X.T @ X, X.T @ y
    out = np.empty((num_samples, d + 4))
    for s in range(num_samples):
        prec = tau_o * XtX + np.diag([tau_w] * d + [tau_b])
        cov = np.linalg.inv(prec)
        mean = cov @ (tau_o * Xty)
        theta = rng.multivariate_normal(mean, cov)
        w, b = theta[:d], theta[d]
        tau_w = rng.gamma(a_w + 0.5 * d, 1.0 / (b_w + 0.5 * float(w @ w)))
        tau_b = rng.gamma(a_b + 0.5, 1.0 / (b_b + 0.5 * b * b))
        r = y - X @ theta
        tau_o = rng.gamma(a_o + 0.5 * n, 1.0 / (b_o + 0.5 * float(r @ r)))
        out[s] = np.concatenate([theta, [np.log(tau_w), np.log(tau_b), np.log(tau_o)]])
    return out
