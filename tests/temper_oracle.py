"""CPU oracle of replica exchange for Bayesian NNs (DESIGN §3.17): oracle/hmc_oracle.py's sample() loop for every row of
the ladders, row r T + t on the target with tau_out replaced by the Python-double product beta_t * tau_out, and after every
window of swap_every iterations (but the last) the even-odd swap round, decided in fp64 on the untempered log-likelihood.

Per iteration n and row c: momentum -> trajectory -> MH, a rejection at n == burn + 1 returning to the row's params_init (the
reference's first-stored-iteration quirk, samplers.py:1018, which the kernel keeps per row).  Only the beta = 1 rows keep
samples: slot 0 = params_init, then the state after every iteration n > burn.
"""
import numpy as np
import torch

from hamiltorch_b200 import targets as T
from oracle import hmc_oracle as O


def tempered(tgt, beta):
    """The descriptor (or split list) at likelihood exponent beta: tau_out -> beta * tau_out."""
    def one(d):
        return T.MLPTarget(d.widths, d.acts, d.x, d.y, d.tau_list, beta * d.tau_out, d.prior_scale, d.model_loss,
                           d.final_log_softmax)
    return [one(d) for d in tgt] if isinstance(tgt, list) else one(tgt)


def c_ll(d):
    """The fp32 likelihood coefficient of a descriptor: -0.5 tau_out (regression), -tau_out (classification)."""
    return float(np.float32(-0.5 * float(np.float32(d.tau_out)) if d.loss_id == T.LOSS_REGRESSION
                            else -float(np.float32(d.tau_out))))


def loglik(tgt, q):
    """Untempered log-likelihood sum_m c_ll * loss_m (the log-softmax loss: its per-split mean) in fp64."""
    descs = tgt if isinstance(tgt, list) else [tgt]
    total = 0.0
    with torch.no_grad():
        for d in descs:
            out = d.forward(q, d.x).double()
            y = d.y.double()
            if d.loss_id == T.LOSS_REGRESSION:
                loss = float(((out - y.view_as(out)) ** 2).sum())
            elif d.loss_id == T.LOSS_BINARY:
                loss = float(torch.nn.BCEWithLogitsLoss(reduction='sum')(out, y.view_as(out)))
            elif d.loss_id == T.LOSS_MULTICLASS:
                loss = float(torch.nn.CrossEntropyLoss(reduction='sum')(out, y.long().view(-1)))
            else:
                loss = float(torch.nn.functional.nll_loss(out, y.long().view(-1)))
            total += c_ll(d) * loss
    return total


def swap_pairs(k, T_):
    """The rungs t of the pairs (t, t + 1) of swap round k."""
    return list(range(k % 2, T_ - 1, 2))


def num_rounds(num_samples, swap_every):
    return max(0, -(-num_samples // swap_every) - 1)


def swap_decision(beta_t, beta_u, ll_t, ll_u, logu):
    """Pair (t, t + 1) swaps when log u < (beta_t - beta_{t+1}) (ll_{t+1} - ll_t), in fp64."""
    return bool(logu < (beta_t - beta_u) * (ll_u - ll_t))


def sample_tempered(tgt, betas, params_init, num_samples, L, step_size, burn, swap_every, normals, log_uniforms,
                    swap_log_uniforms, perms=None, split_scheme=None, eps_schedule=None):
    """params_init (C, D), C = R T ladder-major; normals (S, C, D), log_uniforms (S, C), swap_log_uniforms
    (rounds, R, T - 1), perms (S, C, M) or None, eps_schedule (S, C) teacher-forces the step size.  Returns samples
    (R, S - burn, D) of the beta = 1 rows, accepted (C, S) bools, swap_accepted (rounds, R, T - 1) int8 (-1: not paired),
    swap_ll (rounds, C) and the final states (C, D)."""
    betas = [float(b) for b in betas]
    T_ = len(betas)
    C_, D = params_init.shape
    R = C_ // T_
    targets = [tempered(tgt, b) for b in betas]
    q = [params_init[c].clone() for c in range(C_)]
    kept = [[params_init[r * T_].clone()] for r in range(R)]
    accepted = [[False] * num_samples for _ in range(C_)]
    rounds = num_rounds(num_samples, swap_every)
    swap_acc = np.full((rounds, R, max(T_ - 1, 0)), -1, dtype=np.int8)
    swap_ll = np.zeros((rounds, C_))
    for n in range(num_samples):
        for c in range(C_):
            cur = targets[c % T_]
            eps = step_size if eps_schedule is None else float(eps_schedule[n, c])
            p = O.momentum_from_normals(normals[n, c])
            H0 = O.hamiltonian_hmc(cur, q[c], p)
            if split_scheme is None:
                qs, ps = O.leapfrog_hmc(cur, q[c], p, L, eps)
            else:
                qs, ps = O.leapfrog_split(cur, q[c], p, L, eps, None, split_scheme,
                                          None if perms is None else perms[n, c])
            H1 = O.hamiltonian_hmc(cur, qs[-1].detach(), ps[-1])
            ok = O.log_accept_ratio(H0, H1) >= log_uniforms[n, c].reshape(1)
            accepted[c][n] = bool(ok)
            if ok:
                q[c] = qs[-1].detach().clone()
            elif n == burn + 1:
                q[c] = params_init[c].clone()
            if n > burn and c % T_ == 0:
                kept[c // T_].append(q[c].clone())
        k, last = divmod(n + 1, swap_every)
        if last == 0 and k - 1 < rounds:                       # window k - 1 just ended: swap round k - 1
            k -= 1
            lls = [loglik(tgt, q[c]) for c in range(C_)]
            swap_ll[k] = lls
            for r in range(R):
                for t in swap_pairs(k, T_):
                    a = r * T_ + t
                    acc = swap_decision(betas[t], betas[t + 1], lls[a], lls[a + 1], float(swap_log_uniforms[k, r, t]))
                    swap_acc[k, r, t] = 1 if acc else 0
                    if acc:
                        q[a], q[a + 1] = q[a + 1], q[a]
    return dict(samples=torch.stack([torch.stack(s) for s in kept]), accepted=accepted, swap_accepted=swap_acc,
                swap_ll=swap_ll, final=torch.stack(q))
