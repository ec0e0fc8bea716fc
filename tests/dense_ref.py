"""fp64 per-iteration replay of the dense (chains x D).(D x D), the coupled and the element-wise sampling paths.

A plain batched torch restatement, in fp64 and vectorised over chains, of what hmcx_tc.cu computes for
GaussianIso / GaussianDiag / GaussianFull targets, hmc_small_kernel / hmcx_coupled.cu for those and Neal's funnel, and
the element-wise persistent loop of hmcx_hmc.cu (hmc_run_kernel, hmc_run_big_kernel) for GaussianIso / GaussianDiag
with inv_mass None or (D,):
HMC and HMC_NUTS with inv_mass None, 1-D or 2-D (the reference's
gibbs samplers.py:185-202, leapfrog :267-304, hamiltonian :779-815 and rho = min(0, H_old - H_new) :626), and
constant-metric RMHMC (explicit A-B-C-B-A :389-462 with the sequential C rotation, implicit :305-387, whose fixed
points are exact for a constant metric so that it is a leapfrog with G^-1 as the inverse mass).  It runs on whatever
device its inputs live on.

Per-iteration replay, not a free-running chain: iteration n >= burn + 2 restarts from the kernel's own retained row
n - 1 - burn; iterations up to burn + 1 (whose states are not retained) start from the replay's own proposals, chosen
by the kernel's decisions.  So no error accumulates along the chain, a decision flip does not end the comparison, and
every iteration of every chain is checked (``check``).

The element-wise kernels keep the reference's fp32 operation order, so their retained rows are also held bit for bit to
an fp32 replay of the same kind (``replay_rows32``).
"""
import math

import numpy as np
import torch

from hamiltorch_b200 import engine, targets as T
from tests import parity

F64 = torch.float64


def _f32(x):
    return float(np.float32(x))


class _Target64:
    """log p and grad log p of a Gaussian target in fp64, from the fp32 operands the kernel receives."""

    def __init__(self, target, device):
        self.device = torch.device(device)
        self.log_norm = _f32(target.log_norm)            # added to an fp32 tensor by the reference and the kernel
        self.mean = None if isinstance(target, T.GaussianIso) else target.mean.to(device, F64)
        self.prec = target.prec.to(device, F64) if isinstance(target, T.GaussianFull) else None
        self.ivar = target.inv_var.to(device, F64) if isinstance(target, T.GaussianDiag) else None

    def _y(self, q):
        return q if self.mean is None else q - self.mean

    def grad(self, q):
        y = self._y(q)
        if self.prec is not None:
            return -(y @ self.prec.t())
        return -y if self.ivar is None else -(self.ivar * y)

    def log_prob(self, q):
        y = self._y(q)
        if self.prec is not None:
            quad = (y * (y @ self.prec.t())).sum(1)
        else:
            quad = (y * y).sum(1) if self.ivar is None else (y * y * self.ivar).sum(1)
        return -0.5 * quad + self.log_norm


class _Funnel64:
    """log p and grad log p of targets.Funnel in fp64, from the fp32 constants the kernel receives: inv_var_v and
    log_norm rounded to fp32, 0.5 (D - 1) exact."""

    def __init__(self, target, device):
        self.device = torch.device(device)
        self.log_norm = _f32(target.log_norm)
        self.inv_var_v = _f32(target.inv_var_v)
        self.half_n = 0.5 * (target.dim - 1)

    def grad(self, q):
        v, x = q[:, :1], q[:, 1:]
        ev = torch.exp(v)
        gv = -self.inv_var_v * v + self.half_n - 0.5 * ev * (x * x).sum(1, keepdim=True)
        return torch.cat([gv, -ev * x], 1)

    def log_prob(self, q):
        v, x = q[:, 0], q[:, 1:]
        return -0.5 * self.inv_var_v * v * v + self.half_n * v - 0.5 * torch.exp(v) * (x * x).sum(1) + self.log_norm


def target64(target, device):
    return _Funnel64(target, device) if isinstance(target, T.Funnel) else _Target64(target, device)


class HMC:
    """sampler HMC / HMC_NUTS: ``inv_mass`` None, (D,), (D, D) or a block list (= the block-diagonal matrix)."""

    def __init__(self, target, inv_mass=None, device='cpu'):
        self.t = target64(target, device)
        if isinstance(inv_mass, list):
            inv_mass = torch.block_diag(*[b.to(torch.float32) for b in inv_mass])
        self.im = None if inv_mass is None else inv_mass.to(device, F64)
        self.tril = None
        if self.im is not None and self.im.dim() == 2:
            self.tril = torch.linalg.cholesky(torch.inverse(self.im))          # :199 scale_tril of inverse(inv_mass)

    def minv(self, p):
        if self.im is None:
            return p
        return p @ self.im.t() if self.im.dim() == 2 else self.im * p

    def momentum(self, z, q):                                                   # :185-202
        if self.im is None:
            return z
        return z @ self.tril.t() if self.tril is not None else z * torch.sqrt(1.0 / self.im)

    def hamiltonian(self, q, p):                                                # :779-815
        return -self.t.log_prob(q) + 0.5 * (p * self.minv(p)).sum(1)

    def trajectory(self, q, p, e, L, per_step=False):                          # :267-304
        """The state after L steps, or with ``per_step`` the (L, C, D) states after every step as the stand-alone
        leapfrog returns them (:299-300): momenta after the full kick, the half-kick correction (:302) on the last."""
        e = e[:, None]
        p = p + 0.5 * e * self.t.grad(q)
        qs, ps = [], []
        for _ in range(L):
            q = q + e * self.minv(p)
            g = self.t.grad(q)
            p = p + e * g
            qs.append(q), ps.append(p)
        p = p - 0.5 * e * g
        if per_step:
            return torch.stack(qs), torch.stack(ps[:-1] + [p])
        return q, p


class RMHMC:
    """sampler RMHMC on a Gaussian target without jitter: G^-1, chol G and log det G from engine.const_metric (the host
    inputs of the kernel); explicit (omega = explicit_binding_const) or implicit integrator."""

    def __init__(self, target, softabs, softabs_const=None, explicit=True, omega=10.0, device='cpu'):
        self.t = _Target64(target, device)
        ginv, lower, log_det = engine.const_metric(target, softabs, softabs_const)
        self.ginv, self.lower = ginv.to(device, F64), lower.to(device, F64)
        pi_term = float(target.dim * torch.log(2. * torch.tensor(math.pi)))        # fp32, :711-712
        self.const = 0.5 * pi_term + 0.5 * log_det
        self.explicit, self.omega = explicit, float(omega)

    def minv(self, p):
        return p @ self.ginv.t()

    def momentum(self, z, q):                                                   # :183-184
        return z @ self.lower.t()

    def hamiltonian(self, q, p):                                                # :731
        return -self.t.log_prob(q) + self.const + 0.5 * (p * self.minv(p)).sum(1)

    def trajectory(self, q, p, e, L):
        h = 0.5 * e[:, None]
        grad, minv = self.t.grad, self.minv
        if not self.explicit:                                                   # :363-386, exact fixed points
            for _ in range(L):
                p = p + h * grad(q)
                q = q + h * minv(p) + h * minv(p)
                p = p + h * grad(q)
            return q, p
        # c, s rounded to fp32 as torch.cos(torch.FloatTensor([2 * omega * step_size])) (:435-436), per chain
        arg = torch.tensor([2 * self.omega * float(x) for x in e.cpu()], dtype=torch.float32)
        c = torch.cos(arg).to(q.device, F64)[:, None]
        s = torch.sin(arg).to(q.device, F64)[:, None]
        qc, pc = q.clone(), p.clone()
        for _ in range(L):                                                      # :427-458
            p = p + h * grad(q)
            qc = qc + h * minv(pc)
            q = q + h * minv(p)
            pc = pc + h * grad(qc)
            q = 0.5 * ((q + qc) + c * (q - qc) + s * (p - pc))
            p = 0.5 * ((p + pc) - s * (q - qc) + c * (p - pc))
            qc = 0.5 * ((q + qc) - c * (q - qc) - s * (p - pc))
            pc = 0.5 * ((p + pc) + s * (q - qc) - c * (p - pc))
            q = q + h * minv(p)
            pc = pc + h * grad(qc)
            p = p + h * grad(q)
            qc = qc + h * minv(pc)
        return q, p


class Replay:
    """fp64 H_old / H_new (C, S) of every iteration and the proposals (C, S - burn, D) of the retained iterations
    (slot j <-> iteration burn + j; slot 0 unused)."""

    def __init__(self, h_old, h_new, prop):
        self.h_old, self.h_new, self.prop = h_old, h_new, prop

    @property
    def rho(self):
        return torch.clamp(self.h_old - self.h_new, max=0.0)


def replay(model, params_init, accepted, samples, normals, eps, L, burn):
    """params_init (C, D); accepted (C, S) and samples (C, S - burn, >= D) as the kernel returned them; normals (S, C, D)
    the injected stream; eps (C,) or, for a teacher-forced NUTS schedule, (S, C).  The momentum hook gets the start state
    (a position-dependent metric draws p = chol G(q) z); a model with a ``begin`` hook is told each iteration's index
    before its first evaluation (the in-kernel metric's jitter rows are per iteration)."""
    C, D = params_init.shape
    S = accepted.shape[1]
    dev = model.t.device
    acc = accepted.to(dev).bool()
    rows = samples[..., :D].to(dev, F64)
    eps = eps.to(dev, F64)
    start = params_init.to(dev, F64)
    h_old = torch.empty(C, S, dtype=F64, device=dev)
    h_new = torch.empty_like(h_old)
    prop = torch.zeros(C, S - burn, D, dtype=F64, device=dev)
    for n in range(S):
        if n >= burn + 2:
            start = rows[:, n - 1 - burn]
        if hasattr(model, 'begin'):
            model.begin(n)
        p = model.momentum(normals[n].to(dev, F64), start)
        h_old[:, n] = model.hamiltonian(start, p)
        q1, p1 = model.trajectory(start, p, eps[n] if eps.dim() == 2 else eps, L)
        h_new[:, n] = model.hamiltonian(q1, p1)
        if n > burn:
            prop[:, n - burn] = q1
        else:                                 # the state after iteration n <= burn is the replay's own (:1015-1022)
            start = torch.where(acc[:, n, None], q1, start)
    return Replay(h_old, h_new, prop)


def check(tag, rep, params_init, samples, accepted, ham, log_u, burn, ceiling=2e-4, diverged=None):
    """Compare a kernel run with its replay; returns the number of decisions that differ from the fp64 ones (each
    within 4x the kernel's own Hamiltonian error of that iteration, else the check fails).

    ham (C, S, 2) and log_u (S, C) as given to / returned by the kernel.  ``diverged`` (C, S): the iterations the kernel
    flagged (a non-finite log p, the reference's LogProbError :1045-1067).  Each must be rejected; its Hamiltonians are
    not compared (fp32 overflows where fp64 does not), every other iteration of the chain is."""
    C, D = params_init.shape
    dev = rep.h_old.device
    ham = ham.to(dev, F64)
    acc = accepted.to(dev).bool()
    live = torch.ones_like(acc) if diverged is None else ~diverged.to(dev).bool()
    assert not bool((acc & ~live).any()), tag + ': a flagged (diverged) iteration was accepted'
    parity.assert_close(tag + '/ham_old', ham[..., 0][live].cpu().numpy(), rep.h_old[live].cpu().numpy(), ceiling)
    parity.assert_close(tag + '/ham_new', ham[..., 1][live].cpu().numpy(), rep.h_new[live].cpu().numpy(), ceiling)
    lu = log_u.to(dev, F64).t()
    flip = live & (acc != (rep.rho >= lu))
    dh = (ham[..., 0] - rep.h_old).abs() + (ham[..., 1] - rep.h_new).abs()
    bad = flip & ((rep.rho - lu).abs() > 4 * dh)
    assert not bool(bad.any()), '%s: %d decisions differ from fp64 beyond the kernel\'s Hamiltonian error (first %s)' % (
        tag, int(bad.sum()), tuple(int(i) for i in torch.nonzero(bad)[0]))
    # retained rows: slot 0 = params_init; slot j = iteration burn + j: the proposal if accepted, else the previous slot
    # (params_init at j = 1, the :1018 quirk), bit for bit
    rows = samples[..., :D].to(dev)
    init = params_init.to(dev, rows.dtype)
    assert torch.equal(rows[:, 0], init), tag + ': slot 0 is not params_init'
    took = acc[:, burn + 1:]
    prev = torch.cat([init[:, None], rows[:, 1:-1]], 1)
    same = (rows[:, 1:] == prev).all(2)
    assert bool(same[~took].all()), tag + ': a rejected iteration changed the state'
    parity.assert_close(tag + '/samples', rows[:, 1:][took].double().cpu().numpy(),
                        rep.prop[:, 1:][took].cpu().numpy(), ceiling)
    return int(flip.sum())


def dual_averaging(ham, burn, step_size, desired_accept_rate=0.8, diverged=None):
    """The step sizes HMC_NUTS proposes (samplers.py:629-674, :1030-1035) for iterations 0..burn, in fp64, from the
    kernel's own Hamiltonians ham (C, S, 2): (C, burn + 1).  ``diverged`` (C, S): a flagged iteration (a LogProbError,
    :1045-1067) adapts with alpha = 0, and at n == burn it also adapts before eps_bar is taken."""
    ham = ham.double().cpu()
    C = ham.shape[0]
    flag = torch.zeros(C, burn + 1, dtype=torch.bool)
    if diverged is not None:
        flag = diverged[:, :burn + 1].cpu().bool()
    mu = math.log(10 * _f32(step_size))
    h_t, eps_bar = torch.zeros(C, dtype=F64), torch.ones(C, dtype=F64)
    out = torch.empty(C, burn + 1, dtype=F64)
    for n in range(burn + 1):
        t = n + 1
        alpha = torch.exp(torch.clamp(ham[:, n, 0] - ham[:, n, 1], max=0.0))
        alpha = torch.where(flag[:, n], torch.zeros_like(alpha), alpha)
        h_new = (1 - 1 / (t + 10)) * h_t + (1 / (t + 10)) * (desired_accept_rate - alpha)
        x_new = mu - t ** 0.5 / 0.05 * h_new
        bar_new = torch.exp(t ** -0.75 * x_new + (1 - t ** -0.75) * torch.log(eps_bar))
        upd = flag[:, n] if n == burn else torch.ones(C, dtype=torch.bool)
        h_t, eps_bar = torch.where(upd, h_new, h_t), torch.where(upd, bar_new, eps_bar)
        if n < burn:
            out[:, n] = torch.exp(x_new)
    out[:, burn] = eps_bar
    return out


def replay_rows32(tag, target, inv_mass, params_init, accepted, samples, normals, eps, L, burn, mass_factor=None):
    """fp32 per-iteration replay of an element-wise run (GaussianIso / GaussianDiag, inv_mass None or (D,)): every
    accepted retained row must equal, bit for bit, the trajectory of oracle/hmc_oracle.leapfrog_hmc restated batched
    over chains in its fp32 operation order (p + (0.5 eps) g, q + (eps inv_mass) p, g = -x or -(inv_var (x - mean)), the
    gradient autograd gives for targets.py).  It restarts from the kernel's own row like ``replay``; the warm-up states
    (not retained) are its own, chosen by the kernel's decisions.  The momentum is z times the mass factor
    ``mass_factor`` (default (1 / inv_mass) ** 0.5, the operand engine.NativeMass passes).  Runs on the device of
    ``samples``; returns the number of rows compared."""
    f32 = torch.float32
    C, D = params_init.shape
    S = accepted.shape[1]
    dev = samples.device
    diag = isinstance(target, T.GaussianDiag)
    mean = target.mean.to(dev, f32) if diag else None
    iv = target.inv_var.to(dev, f32) if diag else None
    im = None if inv_mass is None else inv_mass.to(dev, f32)
    if im is not None and mass_factor is None:
        mass_factor = (1 / inv_mass.detach().to(f32)) ** 0.5
    sd = None if im is None else mass_factor.to(dev, f32)

    def grad(q):
        return -q if iv is None else -(iv * (q - mean))

    acc = accepted.to(dev).bool()
    rows = samples[..., :D].to(dev, f32)
    eps = eps.to(dev, f32)
    start = params_init.to(dev, f32)
    compared = 0
    for n in range(S):
        if n >= burn + 2:
            start = rows[:, n - 1 - burn]
        z = normals[n][..., :D].to(dev, f32)
        p = z if sd is None else z * sd
        e = (eps[n] if eps.dim() == 2 else eps)[:, None]
        p = p + (0.5 * e) * grad(start)                                         # :281
        q = start
        for _ in range(L):
            q = q + e * p if im is None else q + e * im * p                     # :284 / :296
            p = p + e * grad(q)
        if n > burn:
            take = acc[:, n]
            bad = (rows[:, n - burn].view(torch.int32) != q.view(torch.int32)).any(1) & take
            assert not bool(bad.any()), '%s: %d accepted rows of iteration %d differ bit-wise from the fp32 replay ' \
                '(first chain %d)' % (tag, int(bad.sum()), n, int(torch.nonzero(bad)[0]))
            compared += int(take.sum())
        else:
            start = torch.where(acc[:, n, None], q, start)
    return compared
