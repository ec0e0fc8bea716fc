"""ORACLE -- TEST INFRASTRUCTURE ONLY.  Never imported by the product path.

CPU restatement (torch, fp32, autograd -- double backward through the Hessian, eigh and Cholesky exactly like the
reference) of the Riemannian-manifold HMC rows of AdamCobb/hamiltorch @ 19b627b, ``hamiltorch/samplers.py``:
``fisher`` (:69-127), ``cholesky_inverse`` (:130-149), ``rm_hamiltonian`` (:677-736), the RMHMC branches of
``hamiltonian`` (:817-829), ``gibbs`` (:183-184), explicit (:389-462) and implicit (:305-387) ``leapfrog`` and the
``sample`` loop around them (:965-1067).

Pinned by tests/golden/rmhmc_*.npz (oracle/gen_golden.py asserts bit-identity with the unmodified reference under
the same torch RNG state).  ``uniforms`` lets the tests replace the jitter draws ``torch.rand(D)`` (:115) by an
injected stream -- the same buffer the CUDA kernel consumes.
"""
import math

import torch

from .hmc_oracle import OracleLogProbError, nonfinite, log_accept_ratio

HESSIAN, SOFTABS, JACOBIAN_DIAG = 1, 2, 3
EXPLICIT, IMPLICIT = 1, 2


class JitterSource:
    """torch.rand(D) by default (the reference's draw, :115); or successive rows of an injected (J, D) tensor."""

    def __init__(self, rows=None):
        self.rows, self.i, self.retries = rows, 0, 0        # retries: NaN-gradient re-evaluations (:402-410)

    def __call__(self, d):
        if self.rows is None:
            self.i += 1
            return torch.rand(d)
        # more draws than rows (NaN-retry loop, :402-410): re-use the last row -- the CUDA kernel's convention
        r = self.rows[min(self.i, len(self.rows) - 1)]
        self.i += 1
        return r


def fisher(q, log_prob, jitter, alpha, metric, jit):
    """samplers.py:69-127 (HESSIAN and SOFTABS metrics)."""
    lp = log_prob(q)
    if nonfinite(lp):
        raise OracleLogProbError()
    if metric == JACOBIAN_DIAG:                                     # :100-106 (util.jacobian of the scalar log p)
        # NB the reference needs `params` to require grad here; after a reject at n <= burn it passes
        # param_burn_prev.clone() (no grad) and crashes with a RuntimeError -- the oracle just re-attaches the graph
        x = q if q.requires_grad else q.detach().requires_grad_()
        out = (lp if q.requires_grad else log_prob(x)).view(-1)
        jac = torch.autograd.grad(out, [x], torch.ones_like(out), allow_unused=True, retain_graph=True,
                                  create_graph=True)[0].contiguous().view(-1)
        fish = torch.matmul(jac.view(-1, 1), jac.view(1, -1)).diag().diag()
    else:
        hess = torch.autograd.functional.hessian(log_prob, q, create_graph=True)
        fish = -hess
    if nonfinite(fish):
        raise OracleLogProbError()
    if jitter is not None:
        n = fish.shape[0]
        fish += (torch.eye(n) * jit(n) * jitter).to(fish.device)
    if metric in (HESSIAN, JACOBIAN_DIAG):
        return fish, None
    lam, vec = torch.linalg.eigh(fish, UPLO='L')
    abs_lam = (1. / torch.tanh(alpha * lam)) * lam
    fish = torch.matmul(vec, torch.matmul(abs_lam.diag(), vec.t()))
    return fish, abs_lam


def cholesky_inverse(fish, p):
    """samplers.py:130-149."""
    lower = torch.linalg.cholesky(fish)
    y = torch.linalg.solve_triangular(lower, p.view(-1, 1), upper=False, unitriangular=False)
    return torch.linalg.solve_triangular(lower.t(), y, upper=True, unitriangular=False)


def rm_hamiltonian(q, p, log_prob, jitter, alpha, metric, jit):
    """samplers.py:677-736."""
    lp = log_prob(q)
    pi_term = q.nelement() * torch.log(2. * torch.tensor(math.pi))
    fish, abs_lam = fisher(q, log_prob, jitter, alpha, metric, jit)
    if abs_lam is not None:
        if nonfinite(fish) or nonfinite(abs_lam):
            raise OracleLogProbError()
    elif nonfinite(fish):
        raise OracleLogProbError()
    log_det = abs_lam.log().sum() if metric == SOFTABS else torch.slogdet(fish)[1]
    quad = torch.matmul(p.view(1, -1), cholesky_inverse(fish, p))
    ham = - lp + 0.5 * pi_term + 0.5 * log_det + 0.5 * quad
    if nonfinite(ham):
        raise OracleLogProbError()
    return ham


def _grad_wrt_params(q, p, args, max_tries):
    """hamAB_grad_params (:395-414) / the implicit integrator's dH/dtheta (:317-331): NaN gradients are retried with a
    fresh jitter draw up to jitter_max_tries."""
    def evaluate():
        x = q.detach().requires_grad_()
        return torch.autograd.grad(rm_hamiltonian(x, p.detach(), *args), x)[0]

    g = evaluate()
    tries = 0
    while nonfinite(g):                  # :402-410 verbatim: re-evaluate FIRST, then count -- the evaluation that
        g = evaluate()                   # exhausts the budget still happens (and still draws its jitter)
        args[-1].retries += 1
        tries += 1
        if tries > max_tries:
            raise OracleLogProbError()
    return g


def _grad_wrt_momentum(q, p, args):
    """hamAB_grad_momentum (:415-422)."""
    x = p.detach().requires_grad_()
    return torch.autograd.grad(rm_hamiltonian(q.detach().requires_grad_(), x, *args), x)[0]


def leapfrog_explicit(q, p, args, steps, step_size, omega, max_tries=10, copies=None):
    """samplers.py:389-462: Cobb et al. 2019 augmented integrator A-B-C-B-A with the SEQUENTIAL C update (:447-450).
    ``copies``: a list that receives the final augmented pair (q_copy, p_copy) (:462)."""
    q, p = q.clone(), p.clone()
    qc, pc = q.clone(), p.clone()
    qs, ps = [], []
    for _ in range(steps):
        p = p - 0.5 * step_size * _grad_wrt_params(q, pc, args, max_tries)
        qc = qc + 0.5 * step_size * _grad_wrt_momentum(q, pc, args)
        q = q + 0.5 * step_size * _grad_wrt_momentum(qc, p, args)
        pc = pc - 0.5 * step_size * _grad_wrt_params(qc, p, args, max_tries)
        c = torch.cos(torch.FloatTensor([2 * omega * step_size]))
        s = torch.sin(torch.FloatTensor([2 * omega * step_size]))
        q = 0.5 * ((q + qc) + c * (q - qc) + s * (p - pc))
        p = 0.5 * ((p + pc) - s * (q - qc) + c * (p - pc))
        qc = 0.5 * ((q + qc) - c * (q - qc) - s * (p - pc))
        pc = 0.5 * ((p + pc) + s * (q - qc) - c * (p - pc))
        q = q + 0.5 * step_size * _grad_wrt_momentum(qc, p, args)
        pc = pc - 0.5 * step_size * _grad_wrt_params(qc, p, args, max_tries)
        p = p - 0.5 * step_size * _grad_wrt_params(q, pc, args, max_tries)
        qc = qc + 0.5 * step_size * _grad_wrt_momentum(q, pc, args)
        qs.append(q.clone())
        ps.append(p.clone())
    if copies is not None:
        copies += [qc, pc]
    return qs, ps


def leapfrog_implicit(q, p, args, steps, step_size, threshold, max_iter, max_tries=10):
    """samplers.py:305-387: generalised leapfrog with fixed-point iterations."""
    q, p = q.clone(), p.clone()
    qs, ps = [], []
    for _ in range(steps):
        p_old = p.clone()
        for _i in range(max_iter):                                           # fixed_point_momentum :312-341
            p_prev = p.clone()
            p = p_old - 0.5 * step_size * _grad_wrt_params(q, p, args, max_tries)
            if torch.max((p_prev - p) ** 2) < threshold:
                break
        q_old = q.clone()                                                    # fixed_point_params :343-360
        g_old = _grad_wrt_momentum(q, p, args).clone()
        for _i in range(max_iter):
            q_prev = q.clone()
            g = _grad_wrt_momentum(q, p, args)
            q = q_old + 0.5 * step_size * g + 0.5 * step_size * g_old
            if torch.max((q_prev - q) ** 2) < threshold:
                break
        p = p - 0.5 * step_size * _grad_wrt_params(q, p, args, max_tries)    # :368-383
        qs.append(q.detach())
        ps.append(p)
    return qs, ps


def sample_rmhmc(log_prob, params_init, num_samples=10, num_steps_per_sample=10, step_size=0.1, burn=0, jitter=None,
                 softabs_const=None, explicit_binding_const=100, fixed_point_threshold=1e-5,
                 fixed_point_max_iterations=1000, jitter_max_tries=10, integrator=EXPLICIT, metric=HESSIAN,
                 normals=None, log_uniforms=None, uniforms=None):
    """samplers.py:965-1067 for sampler=RMHMC.  Injected randomness: ``normals`` (S, D), ``log_uniforms`` (S,),
    ``uniforms`` (S, J, D) = the jitter draws of iteration n in the order the reference makes them (gibbs, ham,
    8 per explicit step, new_ham)."""
    if burn >= num_samples:
        raise RuntimeError('burn must be less than num_samples.')
    q = params_init.clone()
    burn_prev = params_init.clone()
    kept = [params_init.clone()]
    accepted, ham_old, ham_new, diverged = [], [], [], []
    state_in, proposal, jitter_draws, nan_retries, gibbs_done = [], [], [], [], []          # diagnostics for the teacher-forced parity tests
    rejected = 0
    for n in range(num_samples):
        jit = JitterSource(None if uniforms is None else uniforms[n])
        args = (log_prob, jitter, softabs_const, metric, jit)
        h0 = h1 = float('nan')
        state_in.append(q.detach().clone())
        prop = torch.full_like(params_init, float('nan'))
        got_p = False
        try:
            G = fisher(q, log_prob, jitter, softabs_const, metric, jit)[0]                    # gibbs :183-184
            if normals is None:
                p = torch.distributions.MultivariateNormal(torch.zeros_like(q), G, validate_args=False).sample()
            else:
                p = torch.mv(torch.linalg.cholesky(G.detach()), normals[n])
            p = p.detach()
            got_p = True
            H0 = rm_hamiltonian(q, p, *args)                                                  # :971 (explicit: 2H, /2)
            if integrator == EXPLICIT:
                H0 = 2 * H0
                qs, ps = leapfrog_explicit(q, p, args, num_steps_per_sample, step_size, explicit_binding_const,
                                           jitter_max_tries)
                H0 = H0 / 2
            else:
                qs, ps = leapfrog_implicit(q, p, args, num_steps_per_sample, step_size, fixed_point_threshold,
                                           fixed_point_max_iterations, jitter_max_tries)
            h0 = float(H0)
            q = qs[-1].detach()
            prop = q.clone()
            H1 = rm_hamiltonian(q, ps[-1].detach(), *args)                                    # :989 / :995
            h1 = float(H1)
            rho = log_accept_ratio(H0, H1)
            logu = torch.log(torch.rand(1)) if log_uniforms is None else log_uniforms[n].reshape(1)
            if rho >= logu:
                accepted.append(True)
                if n > burn:
                    kept.append(qs[-1].detach())
                else:
                    burn_prev = qs[-1].detach().clone()
            else:
                accepted.append(False)
                rejected += 1
                if n > burn:
                    q = kept[-1]
                    kept.append(kept[-1])
                else:
                    q = burn_prev.clone()
            diverged.append(False)
        except OracleLogProbError:
            accepted.append(False)
            diverged.append(True)
            rejected += 1
            if n > burn:
                q = kept[-1]
                kept.append(kept[-1])
            else:
                q = burn_prev.clone()
        ham_old.append(h0)
        ham_new.append(h1)
        proposal.append(prop)
        jitter_draws.append(jit.i)
        nan_retries.append(jit.retries)
        gibbs_done.append(got_p)
    return dict(samples=[t.detach() for t in kept], accepted=accepted, ham_old=ham_old, ham_new=ham_new,
                num_rejected=rejected, diverged=diverged, state_in=state_in, proposal=proposal,
                jitter_draws=jitter_draws, nan_retries=nan_retries, gibbs_done=gibbs_done)
