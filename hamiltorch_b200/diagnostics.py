"""On-device convergence diagnostics for batched chains: split-R-hat, effective sample size (ESS) and Monte-Carlo
standard error (MCSE) of the posterior mean, per dimension -- the definitions of the Stan reference manual and of ArviZ's
``rhat(method="split")`` / ``ess(method="mean")`` / ``mcse(method="mean")`` (restated in numpy fp64 by
oracle/diagnostics_oracle.py, which the kernels are tested against).

    d = hamiltorch_b200.diagnostics.summary(res)        # res = sample_chains(...), or a (C, n, D) / (n, D) CUDA tensor
    d.rhat.max(), d.ess.min(), d.mcse                   # (D,) fp64 on the samples' device

Two streaming passes over the sample block run in CUDA (hmcx_diag_means, hmcx_diag_acov, include/hmcx.h): the mean of
every half-chain, then sums over half-chains of the autocovariances 32 lags at a time.  The Geyer scan that turns them
into ESS is O(lags * D) and runs here with torch ops on the device; it asks for the next lag block only while some
dimension's initial positive sequence has not ended.  Every stage returns sums over half-chains, so the chains of several
GPUs pool with one all-reduce per stage (``distributed.pooled_diagnostics``) instead of a gather of their samples.

``rank_summary`` adds the rank-normalised, folded split-R-hat, bulk-ESS and tail-ESS of Vehtari et al. (2021) --
ArviZ's ``rhat(method="rank")`` / ``ess(method="bulk"|"tail")`` -- and the 5 / 50 / 95 % quantiles: a segmented radix
sort per dimension on the GPU (hmcx_rank.cu) turns the draws into normal scores, which then run through the same passes.

Edge cases per dimension: a non-finite draw makes every output NaN (``max_lag`` 0); when all split draws are equal
ESS = N, R-hat = 1, MCSE = 0 (``max_lag`` 0); W = 0 with B > 0 gives R-hat = +inf.  Both are read off the exact fp64
sums: a finite fp32 block cannot overflow them, and equal draws give exactly zero within- and between-chain sums.
"""
import ctypes as C
import math

import torch

from . import _native as N


class Diagnostics:
    """Per-dimension results of ``summary``: ``mean``, ``sd``, ``mcse``, ``ess``, ``rhat`` (D,) fp64 and ``max_lag`` (D,)
    int64 (the largest autocorrelation lag the Geyer scan read), on the samples' device; ``num_chains`` and
    ``num_draws`` (draws per chain) of the block; ``num_lag_blocks`` autocovariance passes it took."""

    def __init__(self, mean, sd, mcse, ess, rhat, max_lag, num_chains, num_draws, num_lag_blocks):
        self.mean, self.sd, self.mcse, self.ess, self.rhat, self.max_lag = mean, sd, mcse, ess, rhat, max_lag
        self.num_chains, self.num_draws, self.num_lag_blocks = num_chains, num_draws, num_lag_blocks

    def __repr__(self):
        return ('Diagnostics(num_chains=%d, num_draws=%d, D=%d, max rhat=%.4f, min ess=%.1f)'
                % (self.num_chains, self.num_draws, self.mean.numel(), float(self.rhat.max()), float(self.ess.min())))


# ------------------------------------------------------------------------------------------------------------------
# Inputs
# ------------------------------------------------------------------------------------------------------------------
def as_block(samples):
    """The (C, n, D) fp32 CUDA view ``summary`` reads: an HMCResult's ``.samples``, a (C, n, D) or (n, D) tensor, or the
    list of (D,) tensors ``hamiltorch_b200.sample`` returns (one chain).  Refuses what the kernels cannot read."""
    from .engine import HMCResult
    if isinstance(samples, HMCResult):
        if samples.samples_padded is None:
            raise RuntimeError('diagnostics: this run kept no samples (keep_samples=False); run with keep_samples=True')
        x = samples.samples
    elif isinstance(samples, (list, tuple)):
        if len(samples) == 0 or not all(torch.is_tensor(s) and s.dim() == 1 for s in samples):
            raise RuntimeError('diagnostics: a list of samples must hold (D,) tensors, as hamiltorch_b200.sample returns')
        if not all(s.device == samples[0].device for s in samples):
            raise RuntimeError('diagnostics: the samples of the list live on different devices')
        _check_device(samples[0])
        x = torch.stack(list(samples))
    elif torch.is_tensor(samples):
        x = samples
    else:
        raise TypeError('diagnostics: expected an HMCResult, a tensor or a list of tensors, got %s' % type(samples))
    _check_device(x)
    if x.dtype != torch.float32:
        raise RuntimeError('diagnostics: samples must be float32, got %s' % x.dtype)
    if x.dim() == 2:
        x = x.unsqueeze(0)
    if x.dim() != 3:
        raise RuntimeError('diagnostics: samples must be (C, n, D) or (n, D), got shape %s' % (tuple(x.shape),))
    if x.shape[0] < 1 or x.shape[2] < 1 or x.shape[1] < 4:
        raise RuntimeError('diagnostics: need at least one chain, one dimension and 4 draws per chain, got shape %s'
                           % (tuple(x.shape),))
    if x.stride(2) != 1 and x.shape[2] > 1:
        x = x.contiguous()                      # the passes read unit stride along D
    return x


def _check_device(t):
    if t.is_cuda:
        return
    if t.device.type == 'cpu' and t.is_pinned():
        raise RuntimeError('diagnostics: the samples live in pinned host memory (store_on_GPU=False); the diagnostics '
                           'run on the GPU -- keep the samples on the GPU or move them there first')
    raise RuntimeError('diagnostics: the samples are a %s tensor; the diagnostics run on a CUDA device and there is no '
                       'CPU fallback' % t.device.type)


# ------------------------------------------------------------------------------------------------------------------
# Per-rank partial stages.  ``means()`` -> (sum_j mu_j (D,), K); ``acov(mu_bar, t0)`` -> (sum_j gamma_j(t) for t in
# [t0, t0 + lag_block) as (lag_block, D), sum_j (mu_j - mu_bar)^2 (D,) or None when mu_bar is None).  Attributes m, D,
# lag_block, device.  The host logic below only sees these sums, so stages of disjoint chain sets add up.
# ------------------------------------------------------------------------------------------------------------------
class NativePartials:
    """The two CUDA passes (hmcx_diag_means / hmcx_diag_acov) over one (C, n, D) fp32 block on its device."""

    def __init__(self, x):
        self.x = as_block(x)
        N.require_cuda()
        self.lib = N.load_library()
        self.C, self.n, self.D = (int(s) for s in self.x.shape)
        self.m, self.device, self.lag_block = self.n // 2, self.x.device, N.DIAG_LAG_BLOCK
        self.mu = None

    def _args(self):
        return (C.c_void_p(self.x.data_ptr()), self.x.stride(0), self.x.stride(1), self.C, self.n, self.D)

    def means(self):
        self.mu = torch.empty((2 * self.C, self.D), dtype=torch.float64, device=self.device)
        mu_sum = torch.empty(self.D, dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            rc = self.lib.hmcx_diag_means(*self._args(), N.ptr(self.mu), N.ptr(mu_sum), N.stream_ptr(self.device))
        N.check(rc, 'hmcx_diag_means')
        return mu_sum, 2 * self.C

    def acov(self, mu_bar, t0):
        out = torch.empty((self.lag_block, self.D), dtype=torch.float64, device=self.device)
        between = None if mu_bar is None else torch.empty(self.D, dtype=torch.float64, device=self.device)
        mb = None if mu_bar is None else mu_bar.to(device=self.device, dtype=torch.float64).contiguous()
        with torch.cuda.device(self.device):
            rc = self.lib.hmcx_diag_acov(*self._args(), N.ptr(self.mu), N.ptr(mb), int(t0), N.ptr(out), N.ptr(between),
                                         N.stream_ptr(self.device))
        N.check(rc, 'hmcx_diag_acov')
        return out, between


class PooledPartials:
    """Several partial stages over disjoint chain sets of the same (n, D), summed in list order: the diagnostics of
    all their chains together."""

    def __init__(self, parts):
        self.parts = list(parts)
        p0 = self.parts[0]
        if any(p.n != p0.n or p.D != p0.D for p in self.parts):
            raise RuntimeError('pooled diagnostics: every block needs the same number of draws and dimensions')
        self.n, self.m, self.D, self.lag_block, self.device = p0.n, p0.m, p0.D, p0.lag_block, p0.device

    def means(self):
        outs = [p.means() for p in self.parts]
        s = outs[0][0]
        for o in outs[1:]:
            s = s + o[0].to(self.device)
        return s, sum(o[1] for o in outs)

    def acov(self, mu_bar, t0):
        outs = [p.acov(mu_bar, t0) for p in self.parts]
        a = outs[0][0]
        b = outs[0][1]
        for o in outs[1:]:
            a = a + o[0].to(self.device)
            b = None if b is None else b + o[1].to(self.device)
        return a, b


# ------------------------------------------------------------------------------------------------------------------
# Host logic: pooled sums -> R-hat, ESS, MCSE.  ``all_reduce(t)`` sums a tensor over ranks (identity on one process).
# ------------------------------------------------------------------------------------------------------------------
def _geyer_state(rho, m):
    """Vectorised Geyer scan over the lags available in ``rho`` (T, D), rho[0] = 1.  Pair k is rho[2k] + rho[2k+1];
    the initial positive sequence reads pairs 1, 2, ... while the previous pair is > 0 and t = 2k-1 < m-3, i.e. it ends
    at I = min(first k with pair_k <= 0, (m-3)//2).  Returns (I, done): done where pair I is available."""
    T, D = rho.shape
    kp = T // 2
    pairs = rho[0:2 * kp:2] + rho[1:2 * kp:2]                              # (kp, D)
    i_max = max(0, (m - 3) // 2)
    k = torch.arange(kp, device=rho.device)[:, None].expand(kp, D)
    big = torch.full_like(k, 1 << 30)
    kstar = torch.where(pairs <= 0, k, big).min(0).values if kp else torch.full((D,), 1 << 30, device=rho.device)
    I = torch.clamp(kstar, max=i_max)
    return I, pairs, I < kp


def _ess_from_rho(rho, pairs, I, N):
    """tau = -1 + 2 * sum_{k < I} (running minimum of the pairs) + rho_last; ESS = N / max(tau, 1/log10 N)."""
    kp, D = pairs.shape
    k = torch.arange(kp, device=rho.device)[:, None]
    mono = torch.cummin(pairs, dim=0).values
    s = torch.where(k < I[None, :], mono, torch.zeros_like(mono)).sum(0)
    idx = I.clamp(max=kp - 1)[None, :]
    pair_I = pairs.gather(0, idx)[0]
    rho_2I = rho.gather(0, (2 * I).clamp(max=rho.shape[0] - 1)[None, :])[0]
    last = torch.where(I == 0, torch.ones_like(rho_2I),
                       torch.where((pair_I >= 0) | (rho_2I > 0), rho_2I, torch.zeros_like(rho_2I)))
    tau = -1.0 + 2.0 * s + last
    return N / torch.clamp(tau, min=1.0 / math.log10(N))


def _first_stage(partials, red):
    """The means stage and the first lag block, reduced: (K, mu_bar, G (lag_block, D) summed autocovariances, between,
    W, varp, nonfinite, constant) -- everything split-R-hat needs, and the start of the ESS scan."""
    m, D, TB = partials.m, partials.D, partials.lag_block
    mu_sum, K_local = partials.means()
    buf = red(torch.cat([mu_sum.double(), torch.tensor([float(K_local)], dtype=torch.float64, device=mu_sum.device)]))
    K = int(round(float(buf[-1])))
    mu_bar = buf[:D] / K
    acov, between = partials.acov(mu_bar, 0)
    buf = red(torch.cat([acov.double(), between.double()[None]]))
    G, between = buf[:TB], buf[TB]
    W = m / (m - 1) * (G[0] / K)
    Bm = between / (K - 1)
    varp = (m - 1) / m * W + Bm
    nonfinite = ~torch.isfinite(mu_bar)
    constant = (G[0] == 0) & (between == 0) & ~nonfinite
    return K, mu_bar, G, between, W, varp, nonfinite, constant


def _rhat_from_partials(partials):
    """Split-R-hat alone of the chains behind ``partials``: the means stage and the first lag block, no Geyer scan.
    Equals ``summary_from_partials(partials).rhat`` bit for bit."""
    _, _, _, _, W, varp, nonfinite, constant = _first_stage(partials, lambda t: t)
    rhat = torch.sqrt(varp / W)
    rhat = torch.where(constant, torch.ones_like(rhat), rhat)
    return torch.where(nonfinite, torch.full_like(rhat, float('nan')), rhat)


def summary_from_partials(partials, all_reduce=None, num_chains=None, num_draws=None):
    """The diagnostics of the chains behind ``partials`` (a NativePartials, a PooledPartials or any object with the same
    ``means`` / ``acov`` stages), with ``all_reduce`` summing each stage's output over ranks: one reduction of the
    half-chain means and count, one of the first lag block together with the between-chain sum, one per further block.
    Every decision is taken on reduced values, so all ranks take the same ones."""
    red = all_reduce or (lambda t: t)
    m = partials.m
    K, mu_bar, G, between, W, varp, nonfinite, constant = _first_stage(partials, red)
    Nd = K * m
    active = ~nonfinite & ~constant
    blocks = 1
    while True:
        rho = 1.0 - (W[None, :] - G / K) / varp[None, :]
        rho[0] = 1.0
        I, pairs, done = _geyer_state(rho, m)
        if bool((done | ~active).all()) or G.shape[0] >= m:
            break
        a, _ = partials.acov(None, G.shape[0])
        G = torch.cat([G, red(a.double())])
        blocks += 1
    ess = _ess_from_rho(rho, pairs, I, Nd)
    sd = torch.sqrt((m * G[0] + m * between) / (Nd - 1))
    rhat = torch.sqrt(varp / W)
    max_lag = torch.clamp(2 * I + 1, min=1).to(torch.int64)
    nan = torch.full_like(sd, float('nan'))
    ess = torch.where(constant, torch.full_like(ess, float(Nd)), ess)
    rhat = torch.where(constant, torch.ones_like(rhat), rhat)
    mcse = torch.where(constant, torch.zeros_like(sd), sd / torch.sqrt(ess))
    max_lag = torch.where(active, max_lag, torch.zeros_like(max_lag))
    mean = torch.where(nonfinite, nan, mu_bar)
    sd, mcse, ess, rhat = (torch.where(nonfinite, nan, t) for t in (sd, mcse, ess, rhat))
    return Diagnostics(mean, sd, mcse, ess, rhat, max_lag, num_chains if num_chains is not None else K // 2,
                       num_draws if num_draws is not None else 2 * m, blocks)


def summary(samples):
    """Split-R-hat, ESS and MCSE of the posterior mean for every dimension of a batched sample block, on its GPU.

    ``samples``: an ``HMCResult`` (its ``.samples``, slot 0 = params_init included; pass ``res.samples[:, 1:]`` to leave
    it out), a CUDA fp32 tensor (C, n, D) -- any chain / draw strides, unit stride along D -- or (n, D), or the list of
    (D,) tensors ``hamiltorch_b200.sample`` returns (one chain).  Needs n >= 4.  Refuses runs with
    ``keep_samples=False``, samples in pinned host memory (``store_on_GPU=False``) and CPU tensors.
    Returns a ``Diagnostics``; the same block gives the same bits on every call."""
    x = as_block(samples)
    return summary_from_partials(NativePartials(x), num_chains=int(x.shape[0]), num_draws=int(x.shape[1]))


# ------------------------------------------------------------------------------------------------------------------
# Rank-normalised diagnostics (Vehtari, Gelman, Simpson, Carpenter & Buerkner 2021)
# ------------------------------------------------------------------------------------------------------------------
class RankDiagnostics:
    """Per-dimension results of ``rank_summary``, (D,) fp64 on the samples' device: ``rhat`` = max(``rhat_bulk``,
    ``rhat_tail``), ``ess_bulk``, ``ess_tail``, ``q05``, ``median``, ``q95``; ``num_chains`` and ``num_draws`` of the
    block; ``max_lag`` (3, D) int64, the largest lag the Geyer scan read on the bulk z, I05 and I95 series, and
    ``num_lag_blocks``, the autocovariance passes each of the three took."""

    def __init__(self, rhat, rhat_bulk, rhat_tail, ess_bulk, ess_tail, q05, median, q95, num_chains, num_draws,
                 max_lag, num_lag_blocks):
        self.rhat, self.rhat_bulk, self.rhat_tail, self.ess_bulk, self.ess_tail = rhat, rhat_bulk, rhat_tail, ess_bulk, ess_tail
        self.q05, self.median, self.q95 = q05, median, q95
        self.num_chains, self.num_draws, self.max_lag, self.num_lag_blocks = num_chains, num_draws, max_lag, num_lag_blocks

    def __repr__(self):
        return ('RankDiagnostics(num_chains=%d, num_draws=%d, D=%d, max rhat=%.4f, min ess_bulk=%.1f, min ess_tail=%.1f)'
                % (self.num_chains, self.num_draws, self.median.numel(), float(self.rhat.max()),
                   float(self.ess_bulk.min()), float(self.ess_tail.min())))


RANK_WORKSPACE_BUDGET = 256 << 20       # bytes of sort workspace one rank_summary call allocates (at least one dimension)
_slab_dims_override = None              # tests: force this many dimensions per slab


def _slab_dims(lib, C, n, D):
    if _slab_dims_override is not None:
        return max(1, min(D, N.RANK_MAX_SLAB, int(_slab_dims_override)))
    k = max(1, min(D, N.RANK_MAX_SLAB, RANK_WORKSPACE_BUDGET // lib.hmcx_rank_workspace_bytes(C, n, 1)))
    while k > 1 and lib.hmcx_rank_workspace_bytes(C, n, k) > RANK_WORKSPACE_BUDGET:
        k -= 1
    return k


def _strides(t):
    return t.stride(0), t.stride(1)


def rank_summary(samples):
    """Rank-normalised, folded split-R-hat, bulk-ESS, tail-ESS and the 5 / 50 / 95 % quantiles of every dimension of a
    batched sample block, on its GPU: the defaults of current Stan, ArviZ (``rhat(method="rank")``,
    ``ess(method="bulk")`` / ``ess(method="tail")``) and PyMC.  Unlike ``summary``'s split-R-hat they flag chains that
    agree in location but not in scale, and they are defined for heavy-tailed posteriors.

    ``samples``: what ``summary`` accepts (an ``HMCResult``, a strided (C, n, D) or (n, D) CUDA fp32 tensor, the list
    ``hamiltorch_b200.sample`` returns), refused in the same cases with the same messages.  Per dimension, with the
    split set = the draws of the half-chains ``summary`` uses (an odd n drops the middle draw) and the full set = all
    draws: the ranks of the split draws (ties share their mean rank; -0.0 ties with +0.0) become normal scores
    z = Phi^-1((r - 3/8) / (Ns + 1/4)) rounded to fp32, for the draws (bulk) and for |x - median| (folded); ``rhat_bulk``
    / ``ess_bulk`` are ``summary``'s split-R-hat / ESS of the bulk scores, ``rhat_tail`` the split-R-hat of the folded
    ones, ``ess_tail`` = min of the ESS of the indicators x <= q05 and x <= q95; the quantiles are numpy's ``median`` /
    ``quantile(method='linear')`` of the full set.  A non-finite draw makes every output of its dimension NaN; a
    constant series has ESS = Ns and R-hat = 1.  The same block gives the same bits on every call.

    Device memory: two (C, n, D) fp32 blocks (the bulk and folded scores; the indicator series reuse them) and one
    sort workspace of at most ``RANK_WORKSPACE_BUDGET`` bytes -- about 20 bytes per draw of a slab of dimensions, the
    slab sized to fit (at least one dimension, so a single dimension of more than about 13 M draws takes more; at most
    65535 dimensions).  The quantiles equal numpy's as values; a zero quantile comes out +0.0 where numpy may give
    -0.0.  The ranks are global over all chains, so the chains of several GPUs
    do not pool by all-reduce: run it where the whole block lives."""
    x = as_block(samples)
    N.require_cuda()
    lib = N.load_library()
    C, n, D = (int(s) for s in x.shape)
    if C * n > N.RANK_MAX_DRAWS:
        raise RuntimeError('rank_summary: %d chains x %d draws exceed the %d draws per dimension the rank pass indexes'
                           % (C, n, N.RANK_MAX_DRAWS))
    dev = x.device
    bulk = torch.empty((C, n, D), dtype=torch.float32, device=dev)
    fold = torch.empty((C, n, D), dtype=torch.float32, device=dev)
    q = torch.empty((3, D), dtype=torch.float64, device=dev)
    flag = torch.empty(D, dtype=torch.int32, device=dev)
    k = _slab_dims(lib, C, n, D)
    ws_bytes = lib.hmcx_rank_workspace_bytes(C, n, k)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        st = N.stream_ptr(dev)
        for d0 in range(0, D, k):
            rc = lib.hmcx_rank_pass(N.ptr(x), *_strides(x), C, n, D, d0, min(k, D - d0), N.ptr(bulk), *_strides(bulk),
                                    N.ptr(fold), *_strides(fold), N.ptr(q), N.ptr(flag), N.ptr(ws), ws_bytes, st)
            N.check(rc, 'hmcx_rank_pass')
        del ws
        b = summary_from_partials(NativePartials(bulk))
        rhat_tail = _rhat_from_partials(NativePartials(fold))
        tails = []
        for row, out in ((0, bulk), (2, fold)):          # I05 over the bulk scores, I95 over the folded ones
            rc = lib.hmcx_rank_indicator(N.ptr(x), *_strides(x), C, n, D, N.ptr(q[row]), N.ptr(out), *_strides(out), st)
            N.check(rc, 'hmcx_rank_indicator')
            tails.append(summary_from_partials(NativePartials(out)))
    bad = flag != 0
    nan = torch.full((D,), float('nan'), dtype=torch.float64, device=dev)
    rhat_bulk = torch.where(bad, nan, b.rhat)
    rhat_tail = torch.where(bad, nan, rhat_tail)
    ess_tail = torch.where(bad, nan, torch.minimum(tails[0].ess, tails[1].ess))
    max_lag = torch.stack([torch.where(bad, torch.zeros_like(t.max_lag), t.max_lag) for t in (b, *tails)])
    return RankDiagnostics(torch.maximum(rhat_bulk, rhat_tail), rhat_bulk, rhat_tail, torch.where(bad, nan, b.ess),
                           ess_tail, q[0], q[1], q[2], C, n, max_lag,
                           tuple(t.num_lag_blocks for t in (b, *tails)))
