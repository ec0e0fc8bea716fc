"""Simulation-based calibration (SBC; Talts, Betancourt, Simpson, Vehtari & Gelman 2018; Modrák et al. 2023) of Bayesian
NNs on the GPU: does a network, prior, step size, L and warm-up produce the posterior the model defines?

    sim = hamiltorch_b200.sbc.simulate(target, 200)               # prior predictive: theta~ and y~ of 200 sims
    out = hamiltorch_b200.sbc.run(target, 200, num_samples=600, burn=200, step_size=0.05, thin=10,
                                  sampler=hamiltorch_b200.Sampler.HMC_NUTS)
    out.p_value                                                   # (D + 1,): one chi^2 test per parameter + log-lik

Per sim m: theta~_m is drawn from the prior, y~_m from the likelihood at theta~_m, the model is fitted to y~_m from
independent prior draws, and the rank of theta~_m among the posterior draws is recorded.  When the computation is right
the ranks are uniform.  Besides every parameter, the summed log-likelihood of y~_m is ranked (draws against theta~_m): it
does not change under the sign flips and permutations of hidden units that make per-weight ranks hard to read, and it
catches fits that parameter ranks miss -- chains that have barely left their independent prior starts look like prior
draws to every parameter column.

Three CUDA pieces (csrc/hmcx_sbc.cu) and two existing ones:
  * hmcx_sbc_prior draws theta~ and the chain starts; hmcx_mlp_pointwise_out gives the network outputs at theta~ and
    hmcx_sbc_simulate turns them into y~ (Philox streams 6 and 7, keyed by the global sim id);
  * up to 64 sims are fitted in one hmcx_split_run_folds launch (engine.hmc_run with ``fits``): each fit is bit-identical
    to a plain run of its own data set;
  * hmcx_sbc_rank counts the parameter ranks; the log-likelihood column sums hmcx_mlp_pointwise_ll in fp64.
"""
import copy

import torch

from . import _native as N
from . import diagnostics as _diag
from . import engine
from . import targets as T

MAX_SIMS_PER_LAUNCH = N.MLP_MAX_SPLITS
_FIT_DEFAULTS = dict(num_samples=10, num_steps_per_sample=10, step_size=0.1, burn=0, sampler=None, inv_mass=None,
                     desired_accept_rate=0.8, seed=0, thin=1)
_REFUSED = {
    'integrator': 'split lists and SPLITTING integrators',
    'tau_prior': 'hyperpriors (tau_prior / tau_out_prior)',
    'tau_out_prior': 'hyperpriors (tau_prior / tau_out_prior)',
    'betas': 'replica exchange (betas)',
    'adapt_mass': 'adapt_mass: it would pool one mass across the different posteriors of the sims',
    'folds': 'folds: the sims are the fits',
}


class Simulation:
    """``simulate``: ``theta`` (M, D) fp32 true parameters, ``y`` (M, N, y_cols) fp32 simulated data in the target's
    ``y`` format, ``init`` (M, R, D) fp32 chain starts (independent prior draws), all on the device; ``num_sims`` M,
    ``chains_per_sim`` R, ``seed``."""

    def __init__(self, block, y, dim, seed):
        self.block = block                       # (M, 1 + R, ld): row 0 theta~, rows 1 .. R the chain starts
        self.y = y
        self.dim = dim
        self.seed = seed
        self.num_sims, self.chains_per_sim = block.shape[0], block.shape[1] - 1

    @property
    def theta(self):
        return self.block[:, 0, :self.dim]

    @property
    def init(self):
        return self.block[:, 1:, :self.dim]

    def __repr__(self):
        return 'Simulation(M=%d, R=%d, D=%d, seed=%d)' % (self.num_sims, self.chains_per_sim, self.dim, self.seed)


class SbcResult:
    """``run``: ``theta`` (M, D), ``ranks`` (M, D + 1) int32 (column D: the summed log-likelihood), ``num_draws`` L (ranks
    run over 0 .. L), ``bins`` B, ``hist`` (D + 1, B) int64, ``expected`` (B,) fp64, ``chi2`` and ``p_value`` (D + 1,)
    fp64, ``accept_rate`` and ``step_size`` (M, R) per chain, ``num_launches``; ``simulation`` the ``Simulation``."""

    def __repr__(self):
        return ('SbcResult(M=%d, L=%d, B=%d, min p=%.3g (column %d), launches=%d)'
                % (self.ranks.shape[0], self.num_draws, self.bins, float(self.p_value.min()),
                   int(self.p_value.argmin()), self.num_launches))


# ------------------------------------------------------------------------------------------------------------------
# Argument checks: all before any CUDA work
# ------------------------------------------------------------------------------------------------------------------
def _check_target(target):
    if isinstance(target, list):
        raise NotImplementedError('sbc: not with split lists -- pass the MLPTarget of the whole data set')
    if not isinstance(target, T.MLPTarget):
        raise NotImplementedError('sbc: Bayesian-NN targets only (an MLPTarget)')
    if target.x is None:
        raise ValueError('sbc: the target has no data (x is None): the simulated data sets take its inputs x')
    if target.loss_id == T.LOSS_MULTICLASS_LOGSOFTMAX:
        raise NotImplementedError(
            "sbc: model_loss='multi_class_log_softmax_output' takes the MEAN of nll_loss over the rows, which is not the "
            "likelihood of N independent labels; SBC against a simulator of such labels would report a false "
            "miscalibration.  Use 'multi_class_linear_output' (summed cross entropy) for the same network")
    if target.loss_id != T.LOSS_REGRESSION and target.tau_out != 1.0:
        raise NotImplementedError('sbc: a classification target with tau_out = %g: the tempered likelihood is not a '
                                  'generative model (use tau_out = 1)' % target.tau_out)


def _check_counts(num_sims, chains_per_sim):
    if isinstance(num_sims, bool) or int(num_sims) != num_sims or int(num_sims) < 2:
        raise ValueError('sbc: num_sims must be an integer >= 2, got %r' % (num_sims,))
    if isinstance(chains_per_sim, bool) or int(chains_per_sim) != chains_per_sim or int(chains_per_sim) < 1:
        raise ValueError('sbc: chains_per_sim must be an integer >= 1, got %r' % (chains_per_sim,))


def _fit_args(kw):
    """The sampling keywords ``fit`` takes, with defaults, refused outside what the fold path supports."""
    from .samplers import Sampler, _check_sample_args
    for k, v in kw.items():
        if k in _REFUSED:
            if k == 'adapt_mass' and not v:
                continue
            if k in ('tau_prior', 'tau_out_prior', 'betas', 'folds', 'integrator') and v is None:
                continue
            raise NotImplementedError('sbc: not combined with ' + _REFUSED[k])
        if k not in _FIT_DEFAULTS:
            raise TypeError('sbc: unexpected sampling keyword %r (supported: %s)' % (k, ', '.join(sorted(_FIT_DEFAULTS))))
    a = dict(_FIT_DEFAULTS, **{k: v for k, v in kw.items() if k in _FIT_DEFAULTS})
    if a['sampler'] is None:
        a['sampler'] = Sampler.HMC
    if a['sampler'] not in (Sampler.HMC, Sampler.HMC_NUTS):
        raise NotImplementedError('sbc: sampler HMC or HMC_NUTS (not RMHMC)')
    im = a['inv_mass']
    if isinstance(im, list) or (im is not None and (not torch.is_tensor(im) or im.dim() != 1)):
        raise NotImplementedError('sbc: inv_mass None or 1-D (no 2-D or block inv_mass)')
    _check_sample_args(True, a['num_samples'], a['burn'], a['sampler'])
    if isinstance(a['thin'], bool) or int(a['thin']) != a['thin'] or int(a['thin']) < 1:
        raise ValueError('sbc: thin must be an integer >= 1, got %r' % (a['thin'],))
    if _keep(a) < 2:
        raise ValueError('sbc: num_samples=%d, burn=%d, thin=%d keep no posterior draw after params_init'
                         % (a['num_samples'], a['burn'], a['thin']))
    return a


def _keep(a):
    """Retained sample slots of a run: slot 0 is params_init, the others posterior draws."""
    return 1 + (int(a['num_samples']) - int(a['burn']) - 1) // int(a['thin'])


def _sims_of(sim, sims):
    s = list(range(sim.num_sims)) if sims is None else [int(m) for m in sims]
    if not 2 <= len(s) <= MAX_SIMS_PER_LAUNCH:
        raise ValueError('sbc: a launch fits 2 to %d sims, got %d' % (MAX_SIMS_PER_LAUNCH, len(s)))
    if len(set(s)) != len(s) or min(s) < 0 or max(s) >= sim.num_sims:
        raise ValueError('sbc: sims must be distinct ids in 0 .. %d' % (sim.num_sims - 1))
    return s


def chain_offset(first_sim, num_sims, chains_per_sim):
    """The Philox chain id of row 0 of the launch fitting sims first_sim .. first_sim + num_sims - 1: the smallest multiple
    of num_sims (the fold kernel maps chain g to fit g mod K) at or above first_sim (R + 1).  Consecutive launches of one
    ``run`` therefore draw from disjoint chain ids."""
    K = int(num_sims)
    return K * (-(-int(first_sim) * (int(chains_per_sim) + 1) // K))


def batches(num_sims, sims_per_launch):
    """``run``'s launches as (first sim, count): ceil(M / sims_per_launch) balanced batches, sizes differing by at most
    one.  A launch fits at least two sims, so an odd M with sims_per_launch = 2 puts three sims in one launch."""
    M, P = int(num_sims), int(sims_per_launch)
    nb = max(1, min(-(-M // P), M // 2))
    out, a = [], 0
    for b in range(nb):
        k = M // nb + (1 if b < M % nb else 0)
        out.append((a, k))
        a += k
    return out


def default_bins(num_sims):
    """B = min(20, max(2, M // 5)): about five sims per bin."""
    return min(20, max(2, int(num_sims) // 5))


# ------------------------------------------------------------------------------------------------------------------
# Simulation, fits, ranks
# ------------------------------------------------------------------------------------------------------------------
def _device(target):
    return target.x.device if target.x.is_cuda else torch.device('cuda', torch.cuda.current_device())


def simulate(target, num_sims, chains_per_sim=4, seed=0):
    """Draw the prior predictive of ``target`` (an ``MLPTarget`` with data): for every sim m = 0 .. M-1 the true parameters
    theta~_m from the target's prior -- N(0, prior_scale / tau_k) for every element of parameter tensor k, the density
    ``MLPTarget.__call__`` uses (log_prior / prior_scale) --, a data set y~_m at the target's inputs x from the likelihood
    at theta~_m, and R = ``chains_per_sim`` INDEPENDENT prior draws as chain starts (a chain started at theta~_m is
    correlated with it and piles the ranks up in the middle).  Given the network outputs f of theta~_m:
      regression                    y = f + z / sqrt(tau_out)
      binary_class_linear_output    one Bernoulli(sigmoid f) per output
      multi_class_linear_output     one Categorical(softmax f) label per row

    This is also the prior predictive check to run before fitting: ``sim.y`` shows what data the prior considers
    plausible.  Every draw is keyed by (``seed``, sim id), so ``simulate(t, 5)`` equals the first five sims of
    ``simulate(t, 10)`` and two calls give the same bits.  Refused (before any CUDA work): the log-softmax loss (its
    likelihood is a mean over rows, not a generative model of N labels), classification with tau_out != 1, a target
    without data, split lists, num_sims < 2, chains_per_sim < 1.  Returns a ``Simulation``."""
    _check_target(target)
    _check_counts(num_sims, chains_per_sim)
    M, R = int(num_sims), int(chains_per_sim)
    N.require_cuda()
    lib = N.load_library()
    dev = _device(target)
    nt = engine.native_target(target, dev)
    D, ld = nt.dim, N.padded_ld(nt.dim)
    n_rows, n_out = int(target.x.shape[0]), target.widths[-1]
    blk = torch.empty((M, 1 + R, ld), dtype=torch.float32, device=dev)
    f = torch.empty((M, n_rows, n_out), dtype=torch.float32, device=dev)
    y = torch.empty((M, n_rows, target.y_cols), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        st = N.stream_ptr(dev)
        N.check(lib.hmcx_sbc_prior(nt.ref(), int(seed), 0, M, R, ld, N.ptr(blk), st), 'hmcx_sbc_prior')
        # the network outputs of theta~: row 0 of every sim, read in place as one chain of M draws
        N.check(lib.hmcx_mlp_pointwise_out(nt.ref(), N.ptr(blk), 0, (1 + R) * ld, 1, M, 0, n_rows, N.ptr(f), 0,
                                           n_rows * n_out, st), 'hmcx_mlp_pointwise_out')
        N.check(lib.hmcx_sbc_simulate(nt.ref(), N.ptr(f), int(seed), 0, M, N.ptr(y), st), 'hmcx_sbc_simulate')
    return Simulation(blk, y, D, int(seed))


def _fit_targets(sim, target, sims):
    """One copy of ``target`` per sim, holding that sim's simulated y (the network, prior, x and settings shared)."""
    out = []
    for m in sims:
        t = copy.copy(target)
        t.y = sim.y[m]
        out.append(t)
    return out


def fit(sim, target, sims=None, **kw):
    """Fit the sims ``sims`` (default all; 2 to 64 distinct ids) of ``sim`` in ONE launch: with K = len(sims), row r K + k
    is chain r of sim sims[k], started at ``sim.init[sims[k], r]``, so ``res.samples[k::K]`` is that sim's posterior.  The
    launch's chain ids start at ``chain_offset(sims[0], K, R)``; every row is bit-identical to a one-chain
    ``sample_chains`` on the target with that sim's y, with its chain id as ``chain_offset`` and the same ``seed``.

    ``kw``: ``num_samples``, ``num_steps_per_sample``, ``step_size``, ``burn``, ``sampler`` (HMC / HMC_NUTS),
    ``inv_mass`` (None or 1-D), ``desired_accept_rate``, ``seed``, ``thin``, with ``sample_chains``' meaning and
    defaults (seed 0).  Refused before any CUDA work: RMHMC, SPLITTING integrators, hyperpriors, ``betas``,
    ``adapt_mass``, a 2-D or block inv_mass, and what ``simulate`` refuses.  Returns the ``engine.HMCResult``."""
    _check_target(target)
    a = _fit_args(kw)
    s = _sims_of(sim, sims)
    from .samplers import Sampler
    K, R = len(s), sim.chains_per_sim
    q0 = sim.block[s, 1:, :sim.dim].transpose(0, 1).reshape(R * K, sim.dim)
    return engine.hmc_run(None, q0, a['num_samples'], a['num_steps_per_sample'], a['step_size'], burn=a['burn'],
                          inv_mass=a['inv_mass'], nuts=a['sampler'] == Sampler.HMC_NUTS,
                          desired_accept_rate=a['desired_accept_rate'], seed=int(a['seed']),
                          chain_offset=chain_offset(s[0], K, R), scheme=N.SCHEME_PLAIN, thin=int(a['thin']),
                          fits=_fit_targets(sim, target, s))


def _slab_rows(n_draws, n_rows):
    """Data rows per log-likelihood slab: the (R, keep - 1, rows) fp32 block within diagnostics.RANK_WORKSPACE_BUDGET."""
    return max(1, min(n_rows, _diag.RANK_WORKSPACE_BUDGET // (4 * max(1, n_draws))))


def ranks(res, sim, target, sims=None):
    """The SBC ranks of the fit ``res`` = ``fit(sim, target, sims)``: a (K, D + 1) int32 CUDA tensor, row k for sim
    sims[k].  The posterior draws are every retained slot but slot 0 (params_init, not a draw), pooled over the R chains:
    L = R (keep - 1) draws, ranks in 0 .. L.  Column d < D: #{draws with theta_d < theta~_d} (hmcx_sbc_rank).  Column D:
    the same count for the log-likelihood of y~ summed over the rows in fp64, each draw against theta~ (the likelihood
    of hmcx_mlp_pointwise_ll over the sim's own rows, in slabs within diagnostics.RANK_WORKSPACE_BUDGET).  Ties count as
    "not less"; with continuous fp32 draws they have probability ~0."""
    _check_target(target)
    s = _sims_of(sim, sims)
    K, R, D = len(s), sim.chains_per_sim, sim.dim
    x = res.samples_padded
    if x is None or not x.is_cuda:
        raise RuntimeError('sbc.ranks: the fit must keep its samples on the device')
    C_, keep, ld = x.shape
    if C_ != R * K or ld != sim.block.shape[2]:
        raise RuntimeError('sbc.ranks: the result has %d chains of width %d; the fit of %d sims x %d chains has %d of '
                           'width %d' % (C_, ld, K, R, R * K, sim.block.shape[2]))
    if keep < 2:
        raise RuntimeError('sbc.ranks: the fit kept no posterior draw after params_init')
    N.require_cuda()
    lib = N.load_library()
    dev = x.device
    truth = sim.block[s, 0].contiguous()                                         # (K, ld)
    out = torch.empty((K, D + 1), dtype=torch.int32, device=dev)
    n_rows = int(target.x.shape[0])
    nt = engine.native_target(_fit_targets(sim, target, s), dev)                  # sim k: rows [k N, (k + 1) N)
    n = keep - 1
    rows = _slab_rows(R * n, n_rows)
    with torch.cuda.device(dev):
        st = N.stream_ptr(dev)
        par = torch.empty((K, D), dtype=torch.int32, device=dev)
        N.check(lib.hmcx_sbc_rank(N.ptr(x), keep * ld, ld, C_, keep, K, D, N.ptr(truth), ld, N.ptr(par), st),
                'hmcx_sbc_rank')
        out[:, :D] = par
        blk = torch.empty((R, n, rows), dtype=torch.float32, device=dev)
        tll = torch.empty((1, 1, rows), dtype=torch.float32, device=dev)
        for k in range(K):
            ll = torch.zeros((R, n), dtype=torch.float64, device=dev)
            lt = torch.zeros((), dtype=torch.float64, device=dev)
            for r0 in range(0, n_rows, rows):
                kk = min(rows, n_rows - r0)
                a, b = k * n_rows + r0, k * n_rows + r0 + kk
                # draws m::K from slot 1: chain stride K keep ld, draw stride ld
                N.check(lib.hmcx_mlp_pointwise_ll(nt.ref(), N.ptr(x[k, 1]), K * keep * ld, ld, R, n, a, b,
                                                  N.ptr(blk), blk.stride(0), blk.stride(1), st), 'hmcx_mlp_pointwise_ll')
                N.check(lib.hmcx_mlp_pointwise_ll(nt.ref(), N.ptr(truth[k]), 0, 0, 1, 1, a, b, N.ptr(tll), 0, 0, st),
                        'hmcx_mlp_pointwise_ll')
                ll += blk[:, :, :kk].double().sum(2)
                lt += tll[0, 0, :kk].double().sum()
            out[k, D] = (ll < lt).sum().to(torch.int32)
    return out


def rank_histogram(rk, num_draws, bins):
    """Rank histograms and their chi^2 uniformity tests: rank rho of 0 .. L goes in bin floor(rho B / (L + 1)); bin b
    expects M |{rho in 0 .. L : rho in b}| / (L + 1) sims (exact, so L + 1 need not be a multiple of B);
    chi2 = sum_b (count - expected)^2 / expected in fp64 and p = gammaincc((B - 1) / 2, chi2 / 2).  ``rk`` (M, P)
    integer ranks -> (hist (P, B) int64, expected (B,) fp64, chi2 (P,) fp64, p (P,) fp64) on rk's device."""
    L, B = int(num_draws), int(bins)
    M, P = rk.shape
    dev = rk.device
    b = (rk.to(torch.int64) * B) // (L + 1)                                      # (M, P)
    hist = torch.zeros((P, B), dtype=torch.int64, device=dev)
    hist.scatter_add_(1, b.t().contiguous(), torch.ones((P, M), dtype=torch.int64, device=dev))
    width = torch.bincount((torch.arange(L + 1, device=dev) * B) // (L + 1), minlength=B).double()
    expected = M * width / (L + 1)
    chi2 = ((hist.double() - expected) ** 2 / expected).sum(1)
    p = torch.special.gammaincc(torch.full_like(chi2, (B - 1) / 2.0), chi2 / 2.0)
    return hist, expected, chi2, p


def run(target, num_sims, chains_per_sim=4, seed=0, bins=None, sims_per_launch=64, **kw):
    """A complete SBC: ``simulate`` -> ``fit`` in balanced launches of at most ``sims_per_launch`` sims (``batches``) ->
    ``ranks`` -> rank histograms with ``bins`` bins (default ``default_bins(num_sims)``, about five sims per bin) and their
    chi^2 p-values (``rank_histogram``).  ``seed`` keys the simulation (streams 6 and 7) and the fits' momentum and
    accept streams (0 and 1); launch b, fitting sims a_b .. a_b + K_b - 1, uses chain ids from ``chain_offset(a_b, K_b,
    R)``, so results depend on (seed, sims_per_launch, the arguments) and chain ids never repeat within a run.

    Memory: a launch holds K_b copies of the target's data (the fold layout of DESIGN §3.18), plus the tensor-core
    operand of x for n0 -> 128 -> nL stacks; ``sims_per_launch`` lowers it.  Refused before any CUDA work: what
    ``simulate`` and ``fit`` refuse, sims_per_launch outside [2, 64], bins outside [2, L + 1].  Returns an ``SbcResult``.
    """
    _check_target(target)
    _check_counts(num_sims, chains_per_sim)
    if 'seed' in kw:
        raise TypeError("sbc.run: one seed keys the simulation and the fits; pass it as run's own `seed`")
    kw = dict(kw, seed=seed)
    a = _fit_args(kw)
    if isinstance(sims_per_launch, bool) or int(sims_per_launch) != sims_per_launch or \
            not 2 <= int(sims_per_launch) <= MAX_SIMS_PER_LAUNCH:
        raise ValueError('sbc: sims_per_launch must be an integer in [2, %d], got %r'
                         % (MAX_SIMS_PER_LAUNCH, sims_per_launch))
    M, R = int(num_sims), int(chains_per_sim)
    L = R * (_keep(a) - 1)
    B = default_bins(M) if bins is None else bins
    if isinstance(B, bool) or int(B) != B or not 2 <= int(B) <= L + 1:
        raise ValueError('sbc: bins must be an integer in [2, L + 1] = [2, %d], got %r' % (L + 1, bins))
    B = int(B)
    sim = simulate(target, M, R, seed)
    dev = sim.block.device
    rk = torch.empty((M, sim.dim + 1), dtype=torch.int32, device=dev)
    acc = torch.empty((M, R), dtype=torch.float64, device=dev)
    eps = torch.empty((M, R), dtype=torch.float32, device=dev)
    parts = batches(M, sims_per_launch)
    for a0, K in parts:
        s = list(range(a0, a0 + K))
        res = fit(sim, target, sims=s, **kw)
        rk[a0:a0 + K] = ranks(res, sim, target, sims=s)
        acc[a0:a0 + K] = res.accept_rate.reshape(R, K).t()
        eps[a0:a0 + K] = res.step_size.reshape(R, K).t()
    out = SbcResult()
    out.simulation, out.theta, out.ranks = sim, sim.theta, rk
    out.num_draws, out.bins, out.num_launches = L, B, len(parts)
    out.hist, out.expected, out.chi2, out.p_value = rank_histogram(rk, L, B)
    out.accept_rate, out.step_size = acc, eps
    return out
