"""Test-side definition of diagonal-mass adaptation during HMC_NUTS warm-up (sample_chains(adapt_mass=True), DESIGN §3.13).

It reuses oracle/hmc_oracle.py for every piece of one iteration (momentum, Hamiltonian, leapfrog, MH, the reference's
dual-averaging arithmetic) and adds what the adapted run does on top of it:
  * the sink's running sums in fp32 with Neumaier compensation, restated from hmcx_common.cuh's comp_add;
  * the pooled estimator of hmcx_adapt_diag_mass in its fp64 operation order (numpy float64 is IEEE, so the result is the
    kernel's bit for bit);
  * the run itself: all chains advance window by window, the mass changes after each window of engine.mass_windows(burn)
    and the dual averaging restarts from h_bar = 0, eps_bar = 1, mu = log(10 eps).
The momentum factor of an adapted mass is the kernel's IEEE sqrtf(1 / inv_mass); the caller's initial mass keeps the
reference's ``mass ** 0.5`` (samplers.py:201), which torch's vectorised CPU pow does not always round like sqrt.
"""
import numpy as np
import torch

from hamiltorch_b200 import engine
from oracle import hmc_oracle as O


def comp_add(s, c, x):
    """hmcx_common.cuh comp_add on float32 arrays: returns the new (s, c)."""
    s, c, x = np.float32(s), np.float32(c), np.float32(x)
    t = (s + x).astype(np.float32)
    e = np.where(np.abs(s) >= np.abs(x), (s - t) + x, (x - t) + s).astype(np.float32)
    return t, (c + e).astype(np.float32)


class Sums:
    """The four [C, ld]-style accumulators of one chain (1-D float32 arrays): sum, sum of squares and their compensations,
    updated exactly as the sink updates them."""

    def __init__(self, D):
        self.s, self.c, self.q, self.cq = (np.zeros(D, np.float32) for _ in range(4))

    def add(self, x):
        x = np.asarray(x, np.float32)
        self.s, self.c = comp_add(self.s, self.c, x)
        xx = (x * x).astype(np.float32)
        self.q, self.cq = comp_add(self.q, self.cq, xx)
        err = (x.astype(np.float64) * x.astype(np.float64) - xx.astype(np.float64)).astype(np.float32)   # fmaf(x, x, -xx)
        self.cq = (self.cq + err).astype(np.float32)


def pooled_inv_mass(s, sq, s_lo, sq_lo, n):
    """hmcx_adapt_diag_mass on (C, D) float32 sums of n draws per chain -> (inv_mass, mass_factor), float32 (D,)."""
    s1 = s.astype(np.float64) + s_lo.astype(np.float64)
    s2 = sq.astype(np.float64) + sq_lo.astype(np.float64)
    dn = np.float64(n)
    m = s1 / dn
    v = (s2 - s1 * m) / np.float64(n - 1)
    w = np.zeros(s.shape[1], np.float64)
    for c in range(s.shape[0]):                       # sequentially over the global chain index
        w = w + v[c]
    w = w / np.float64(s.shape[0])
    N = np.float64(s.shape[0]) * dn
    var = (N / (N + 5.0)) * w + 1e-3 * (5.0 / (N + 5.0))
    im = var.astype(np.float32)
    return im, np.sqrt(np.float32(1.0) / im).astype(np.float32)


def restart_mu(eps):
    """mu_chain of hmcx_adapt_diag_mass: fp32 10 * eps, then the correctly rounded fp32 log, as a double."""
    e10 = np.float32(10.0) * np.float32(eps)
    return float(np.float32(np.log(np.float64(e10))))


def dual_average(rho, t, mu, H_t, eps_bar, desired_accept_rate=0.8):
    """O.dual_average with mu given instead of derived from step_size_init (the restarted averaging's mu)."""
    t = t + 1
    if O.nonfinite(torch.tensor([rho])):
        alpha = 0
    else:
        alpha = min(1., float(torch.exp(torch.FloatTensor([rho]))))
    H_t = (1 - (1 / (t + 10))) * H_t + (1 / (t + 10)) * (desired_accept_rate - alpha)
    x_new = mu - (t ** 0.5) / 0.05 * H_t
    step_size = float(torch.exp(torch.FloatTensor([x_new])))
    x_new_bar = t ** -0.75 * x_new + (1 - t ** -0.75) * torch.log(torch.FloatTensor([eps_bar]))
    return step_size, float(torch.exp(x_new_bar)), H_t


def sample_adapted(log_prob, params_init, num_samples, num_steps_per_sample, step_size, burn, inv_mass=None,
                   normals=None, log_uniforms=None, split_scheme=None, perms=None, desired_accept_rate=0.8):
    """C chains of O.sample_hmc(nuts=True) with the pooled mass adaptation.  params_init (C, D); normals (S, C, D),
    log_uniforms (S, C), perms (S, C, M) (the injected stream).  Returns a dict of per-chain lists (samples, accepted,
    ham_old, ham_new, rho: the log acceptance ratios, step_sizes: the eps each iteration used) plus inv_mass_trace (K, D)
    float32 and windows."""
    C, D = params_init.shape
    windows = engine.mass_windows(burn)
    ends = {b: k for k, (_, b) in enumerate(windows)}
    im = None if inv_mass is None else inv_mass.detach().float()
    sd = None if im is None else O.invert_mass(im) ** 0.5          # momentum factor (gibbs :201)
    chains = []
    for c in range(C):
        q = params_init[c].clone()
        chains.append(dict(q=q, burn_prev=q.clone(), kept=[q.clone()], accepted=[], ham_old=[], ham_new=[], rho=[],
                           step_sizes=[], eps=float(step_size), H=0., eps_bar=1., mu=engine.nuts_mu(step_size),
                           t0=0, sums=Sums(D)))
    trace = []
    for n in range(num_samples):
        for c, ch in enumerate(chains):
            ch['step_sizes'].append(ch['eps'])
            h0 = h1 = float('nan')
            rho = float('nan')
            try:
                p = normals[n, c].clone() if sd is None else normals[n, c] * sd
                H0 = O.hamiltonian_hmc(log_prob, ch['q'], p, im)
                h0 = float(H0)
                if split_scheme is None:
                    qs, ps = O.leapfrog_hmc(log_prob, ch['q'], p, num_steps_per_sample, ch['eps'], im)
                else:
                    qs, ps = O.leapfrog_split(log_prob, ch['q'], p, num_steps_per_sample, ch['eps'], im, split_scheme,
                                              None if perms is None else perms[n, c])
                H1 = O.hamiltonian_hmc(log_prob, qs[-1].detach(), ps[-1], im)
                h1 = float(H1)
                rho = O.log_accept_ratio(H0, H1)
                acc = rho >= float(log_uniforms[n, c])
            except O.OracleLogProbError:
                acc = False
            ch['accepted'].append(acc)
            if acc:
                ch['q'] = qs[-1].detach()
                if n > burn:
                    ch['kept'].append(ch['q'])
                else:
                    ch['burn_prev'] = ch['q'].clone()
            elif n > burn:
                ch['q'] = ch['kept'][-1]
                ch['kept'].append(ch['kept'][-1])
            else:
                ch['q'] = ch['burn_prev'].clone()
            ch['ham_old'].append(h0)
            ch['ham_new'].append(h1)
            ch['rho'].append(rho)
            if n <= burn:
                if n < burn or not np.isfinite(h0 + h1):
                    ch['eps'], ch['eps_bar'], ch['H'] = dual_average(rho, n - ch['t0'], ch['mu'], ch['H'], ch['eps_bar'],
                                                                     desired_accept_rate)
                if n == burn:
                    ch['eps'] = ch['eps_bar']
            if any(a <= n < b for a, b in windows):
                ch['sums'].add(ch['q'].numpy())
        if n + 1 in ends:
            a, b = windows[ends[n + 1]]
            st = [np.stack([getattr(ch['sums'], f) for ch in chains]) for f in ('s', 'q', 'c', 'cq')]
            new_im, new_sd = pooled_inv_mass(st[0], st[1], st[2], st[3], b - a)
            trace.append(new_im)
            im, sd = torch.from_numpy(new_im.copy()), torch.from_numpy(new_sd.copy())
            for ch in chains:
                ch['H'], ch['eps_bar'], ch['mu'], ch['t0'], ch['sums'] = 0., 1., restart_mu(ch['eps']), n + 1, Sums(D)
    out = {k: [ch[k] for ch in chains] for k in ('accepted', 'ham_old', 'ham_new', 'rho', 'step_sizes', 'eps', 'eps_bar')}
    out['samples'] = [torch.stack(ch['kept']) for ch in chains]
    out['inv_mass_trace'] = np.stack(trace)
    out['windows'] = windows
    return out


def replay_step_sizes(rho, burn, step_size, restart_eps, desired_accept_rate=0.8):
    """One chain's restarted dual averaging driven by the log acceptance ratios ``rho`` (n = 0 .. burn): the step size after
    every iteration.  ``restart_eps(b)`` is the step size the averaging restarts from at window end b -- the kernel's own,
    when the kernel's trace is compared, so that one window's rounding differences do not carry into the next's mu."""
    ends = [b for _, b in engine.mass_windows(burn)]
    H, eps_bar, mu, t0, eps, out = 0., 1., engine.nuts_mu(step_size), 0, float(step_size), []
    for n in range(burn + 1):
        if n in ends:
            H, eps_bar, mu, t0 = 0., 1., restart_mu(restart_eps(n)), n
        if n < burn or not np.isfinite(rho[n]):
            eps, eps_bar, H = dual_average(rho[n], n - t0, mu, H, eps_bar, desired_accept_rate)
        if n == burn:
            eps = eps_bar
        out.append(eps)
    return out
