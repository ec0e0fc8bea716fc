"""fp64 per-iteration replay of the in-kernel-metric RMHMC kernels: rmhmc2_quad_kernel (D = 2, explicit),
rmhmc_run_kernel<DM> (one thread per chain, D <= 16) and rmhmc_cta_kernel (one CTA per chain, D <= 64).

These kernels build G = -Hessian (or diag(g^2) for JACOBIAN_DIAG) plus the jitter term, eigen-decompose it with Jacobi
sweeps and differentiate H in closed form.  The model here is the oracle itself (oracle/rmhmc_oracle.py: autograd through
the Hessian, eigh and the Cholesky solve), evaluated on fp64 tensors, one chain at a time, inside tests/dense_ref.replay.
Like the kernel it keeps the jitter term u * jitter, pi_term and the binding rotation cos/sin(2 omega eps) in fp32.

Every fisher() call of iteration n consumes the next row of that iteration's injected uniforms (S, C, J, D): gibbs,
H(theta, p), the trajectory (8 per explicit step; 2m + 2 per implicit step when the fixed points never exit early) and
H(theta_L, p_L).  ``draws`` records what each chain consumed; a NaN-gradient retry would shift every later row, so the
replay refuses one.
"""
import types

import torch

from hamiltorch_b200 import targets as T
from oracle import rmhmc_oracle as R

F64 = torch.float64
METRICS = {'HESSIAN': R.HESSIAN, 'SOFTABS': R.SOFTABS, 'JACOBIAN_DIAG': R.JACOBIAN_DIAG}


def log_prob64(target):
    """The target's log p on fp64 inputs, from the fp32 parameters the kernel receives (GaussianFull's torch.mv does not
    promote its fp32 precision; the other targets do)."""
    if isinstance(target, T.GaussianFull):
        P, m, ln = target.prec.to(F64), target.mean.to(F64), target.log_norm
        return lambda x: -0.5 * torch.dot(x - m, torch.mv(P, x - m)) + ln
    return target


class InKernelMetric:
    """A dense_ref.replay model of sampler=RMHMC with the metric assembled from the position.  uniforms (S, C, J, D) fp32:
    the injected jitter rows (None without jitter)."""

    def __init__(self, target, metric, jitter=None, softabs_const=None, explicit=True, omega=100.0,
                 threshold=0.0, max_iter=6, uniforms=None):
        self.t = types.SimpleNamespace(device=torch.device('cpu'))     # dense_ref.replay's device: the oracle is CPU torch
        self.lp = log_prob64(target)
        self.jitter, self.alpha, self.metric = jitter, softabs_const, METRICS[metric]
        self.explicit, self.omega = explicit, float(omega)
        self.threshold, self.max_iter = float(threshold), int(max_iter)
        self.uni = None if uniforms is None else uniforms.detach().to('cpu', torch.float32)
        self.draws = []                   # (S, C): jitter rows each chain consumed in iteration n

    def begin(self, n):
        self.n, self.jit = n, {}
        self.draws.append(self.jit)

    def _src(self, c):
        if c not in self.jit:
            self.jit[c] = R.JitterSource(None if self.uni is None else self.uni[self.n, c])
        return self.jit[c]

    def counts(self):
        """(S, C) jitter rows consumed per iteration and chain."""
        return torch.tensor([[row[c].i for c in sorted(row)] for row in self.draws])

    def _args(self, c):
        return self.lp, self.jitter, self.alpha, self.metric, self._src(c)

    def momentum(self, z, q):                                               # gibbs :183-184
        out = torch.empty_like(z)
        for c in range(z.shape[0]):
            G = R.fisher(q[c], *self._args(c))[0]
            out[c] = torch.mv(torch.linalg.cholesky(G.detach()), z[c])
        return out

    def hamiltonian(self, q, p):                                            # :677-736
        return torch.stack([R.rm_hamiltonian(q[c], p[c], *self._args(c)).detach().reshape(())
                            for c in range(q.shape[0])])

    def trajectory(self, q, p, e, L):
        qs, ps = [], []
        for c in range(q.shape[0]):
            if self.explicit:
                tq, tp = R.leapfrog_explicit(q[c], p[c], self._args(c), L, float(e[c]), self.omega)
            else:
                tq, tp = R.leapfrog_implicit(q[c], p[c], self._args(c), L, float(e[c]), self.threshold, self.max_iter)
            assert self._src(c).retries == 0, 'the fp64 replay made a NaN-gradient retry (chain %d)' % c
            qs.append(tq[-1].detach())
            ps.append(tp[-1].detach())
        return torch.stack(qs), torch.stack(ps)



def rows_per_iteration(explicit, L, m):
    """Jitter rows of one iteration: 8L + 3 explicit; 3 + L (2m + 2) implicit when no fixed point exits early."""
    return 8 * L + 3 if explicit else 3 + L * (2 * m + 2)
