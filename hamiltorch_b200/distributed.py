"""Multi-GPU: chains are independent (the reference runs them as separate sample() calls, util.py:386-389), so the
chain batch is sharded by rank -- contiguous blocks, chain c lives on rank floor(c*G/C) -- and every chain's random
stream is keyed by its GLOBAL id (Philox ``chain_offset``) or travels with it (injected mode).  Results therefore do
not depend on the number of GPUs.  There is no collective inside the sampling loop; what is collected afterwards is
a choice: per-chain summaries (tiny) or, with ``gather_samples=True``, every rank's sample block through ONE
``all_gather_into_tensor`` (NCCL over NVLink on GPUs; gloo in the CPU tests of the host logic).

One process per GPU, launched by torchrun; ``torch.distributed`` must be initialised by the caller.
"""
import torch
import torch.distributed as dist


def shard_bounds(num_chains, rank, world):
    """Contiguous block partition: rank r owns chains [lo, hi).  Sizes differ by at most one."""
    lo = (num_chains * rank) // world
    hi = (num_chains * (rank + 1)) // world
    return lo, hi


def _world():
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def all_gather_rows(local, num_chains, group=None):
    """Gather row-sharded tensors (shard r = rows shard_bounds(num_chains, r, world)) into the full (num_chains, ...)
    tensor on every rank with ONE all_gather_into_tensor.  Ragged shards are padded to the largest shard."""
    rank, world = _world()
    if world == 1:
        return local
    sizes = [shard_bounds(num_chains, r, world) for r in range(world)]
    mx = max(hi - lo for lo, hi in sizes)
    pad = local
    if local.shape[0] != mx:
        pad = local.new_zeros((mx,) + tuple(local.shape[1:]))
        pad[:local.shape[0]] = local
    pad = pad.contiguous()
    out = pad.new_empty((world * mx,) + tuple(local.shape[1:]))
    dist.all_gather_into_tensor(out, pad, group=group)
    if all(hi - lo == mx for lo, hi in sizes):
        return out
    return torch.cat([out[r * mx: r * mx + (hi - lo)] for r, (lo, hi) in enumerate(sizes)])


def pooled_moments(moment_sum, moment_sumsq, count_per_chain, group=None):
    """Posterior mean and variance pooled over ALL chains of ALL ranks from the sample sink's per-chain running sums
    (``sample_chains(..., moments=True)``: ``moment_sum`` / ``moment_sumsq`` (C_local, D), ``moment_count`` states per
    chain) with ONE all-reduce of a (2D+1,) fp64 vector -- the multi-GPU consumer that needs no sample gather at all
    (O(D) bytes over NVLink instead of O(C*S*D)).  Returns (mean (D,), var (D,), n) as fp64, identical on every rank;
    var is the population variance of the pooled draws."""
    s = moment_sum.double().sum(0)
    sq = moment_sumsq.double().sum(0)
    n = torch.tensor([float(moment_sum.shape[0]) * float(count_per_chain)], dtype=torch.float64, device=s.device)
    buf = torch.cat([s, sq, n])
    rank, world = _world()
    if world > 1:
        dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=group)
    Dd = s.numel()
    total = float(buf[-1])
    if total <= 0:
        raise RuntimeError('pooled_moments: no post-burn states were accumulated')
    mean = buf[:Dd] / total
    var = buf[Dd:2 * Dd] / total - mean * mean
    return mean, var.clamp_min(0.0), total


def pooled_diagnostics(local_samples, partials=None, group=None):
    """Split-R-hat, ESS and MCSE (``diagnostics.summary``) over the chains of ALL ranks, without moving a sample: each
    rank runs the two streaming passes over its own (C_local, n, D) block and the per-stage sums over half-chains are
    all-reduced -- the half-chain means with the half-chain count (D+1 values), the first lag block with the
    between-chain sum ((32+1)*D), then one (32, D) reduction per further lag block.  Every rank ends with identical
    results.  ``local_samples``: anything ``diagnostics.summary`` accepts (n and D equal on every rank).
    ``partials`` replaces the CUDA stages: a callable local_samples -> an object with ``means`` / ``acov`` stages (used
    by the CPU tests of this host logic).  The rank-normalised diagnostics (``diagnostics.rank_summary``) do not pool
    this way: their ranks are global over all draws of a dimension, so they need the whole block on one GPU."""
    from . import diagnostics
    rank, world = _world()
    part = partials(local_samples) if partials is not None else diagnostics.NativePartials(local_samples)

    def all_reduce(t):
        t = t.contiguous()
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)
        return t

    return diagnostics.summary_from_partials(part, all_reduce, num_draws=part.n)


def sample_chains_sharded(log_prob_func, params_init, gather_samples=False, runner=None, diagnostics=False,
                          diagnostics_partials=None, **kwargs):
    """``sample_chains`` over all ranks.  ``params_init`` is the FULL (C, D) batch on every rank (it is tiny next to
    the samples); each rank advances its block of chains on its own GPU.

    Returns a dict on every rank: ``num_rejected`` (C,), ``step_size`` (C,), ``bounds`` (this rank's [lo, hi)),
    ``local`` (this rank's HMCResult) and, when ``gather_samples``, ``samples`` (C, S-burn, D) collected with one
    all-gather.  With the sample sink's ``moments=True`` the per-chain running sums are pooled over all ranks by one
    O(D) all-reduce: ``posterior_mean`` / ``posterior_var`` (D,) fp64, ``posterior_n`` -- no sample ever leaves its GPU.  Injected-stream arguments ``normals`` (S, C, D) / ``log_uniforms`` (S, C) are sliced per rank.
    With ``diagnostics=True``, ``diagnostics`` holds split-R-hat / ESS / MCSE over all chains of all ranks
    (``pooled_diagnostics`` of each rank's samples; needs the samples on the GPU) -- split-R-hat, not the
    rank-normalised R-hat of ``diagnostics.rank_summary``, whose global ranks need every rank's draws.
    With ``adapt_mass=True`` every warm-up window's per-chain moment sums are gathered in global chain order
    (``all_gather_rows``, one (C, ld) gather per sum) before the pooled estimate, so every rank adapts the same mass from
    all C chains -- with Philox keyed by the global chain id the samples do not depend on the sharding.  ``inv_mass``
    then holds the adapted (D,) mass.
    With hyperpriors (``tau_prior`` / ``tau_out_prior``, passed through) and ``gather_samples``, ``tau_list_trace``
    (C, keep, 2L) and ``tau_out_trace`` (C, keep) are gathered alongside the samples.
    With replica exchange (``betas``, T values) the partition is over the R = C / T ladders, not the chains: rank r owns the
    rows T * shard_bounds(R, r, world), ``swap_log_uniforms`` (rounds, R, T - 1) is sliced by ladder, the per-row vectors are
    gathered with that partition and the gathered ``samples`` are the (R, keep, D) beta = 1 rows.
    With K-fold refits (``folds``, K = max + 1 folds) the partition is over groups of K rows in the same way, so every rank
    holds whole groups and its ``chain_offset`` stays a multiple of K; the injected streams are sliced by row, and the
    gathered ``samples`` are the (C, keep, D) rows in global order (``samples[k::K]`` is fold k).  The folds are different
    posteriors, so sink moments are not pooled across rows: each rank's ``local`` keeps its per-row sums.
    ``runner`` replaces ``samplers.sample_chains`` and ``diagnostics_partials`` the diagnostics' CUDA stages (used by
    the CPU tests of this host logic).
    """
    from . import samplers
    rank, world = _world()
    C = params_init.shape[0]
    kw = dict(kwargs)
    T = 1 if kw.get('betas') is None else len(kw['betas'])
    K = 1 if kw.get('folds') is None else int(kw['folds'].max()) + 1
    G = T if K == 1 else K                         # rows per group: a ladder, or one chain of every fold
    if C % G != 0:
        raise ValueError('sample_chains_sharded: C = %d rows is not a multiple of %s = %d'
                         % (C, 'T' if K == 1 else 'K', G))
    R = C // G                                     # groups (G = 1: every chain is its own)
    llo, lhi = shard_bounds(R, rank, world)
    lo, hi = G * llo, G * lhi
    if hi == lo:
        raise RuntimeError('sample_chains_sharded: rank %d of %d would own no chain (C=%d < world); use fewer ranks'
                           % (rank, world, C))
    for name in ('normals', 'log_uniforms', 'perms', 'uniforms', 'gammas'):     # every injected stream is (S, C, ...)
        if kw.get(name) is not None:
            if kw[name].shape[1] != C:
                raise RuntimeError('%s must be (S, C=%d, ...), got %s' % (name, C, tuple(kw[name].shape)))
            kw[name] = kw[name][:, lo:hi]
    if kw.get('swap_log_uniforms') is not None:
        if kw['swap_log_uniforms'].shape[1] != R:
            raise RuntimeError('swap_log_uniforms must be (rounds, R=%d, T - 1), got %s'
                               % (R, tuple(kw['swap_log_uniforms'].shape)))
        kw['swap_log_uniforms'] = kw['swap_log_uniforms'][:, llo:lhi]
    kw['chain_offset'] = kw.get('chain_offset', 0) + lo
    if kw.get('adapt_mass'):
        kw['mass_pool'] = lambda t: all_gather_rows(t, C)

    def gather_rows(t):                            # per-row vectors, gathered group by group
        if G == 1:
            return all_gather_rows(t, C)
        return all_gather_rows(t.reshape((lhi - llo, G) + tuple(t.shape[1:])), R).reshape((C,) + tuple(t.shape[1:]))
    run = runner if runner is not None else samplers.sample_chains
    local = run(log_prob_func, params_init[lo:hi], **kw)
    out = {'bounds': (lo, hi), 'local': local,
           'num_rejected': gather_rows(local.num_rejected),
           'step_size': gather_rows(local.step_size)}
    if kw.get('adapt_mass'):
        out['inv_mass'] = local.inv_mass
    if gather_samples:
        blk = local.samples_padded
        if not blk.is_cuda and dist.is_initialized() and dist.get_backend() == 'nccl':
            raise RuntimeError('gather_samples with store_on_GPU=False: the samples live in pinned host memory, which '
                               'NCCL cannot gather -- keep them on the GPU or gather on the host')
        out['samples'] = (all_gather_rows(blk, R) if K == 1 else gather_rows(blk))[..., :local.dim]
        if getattr(local, 'tau_list_trace', None) is not None:         # hyperpriors: the precisions of the same slots
            out['tau_list_trace'] = all_gather_rows(local.tau_list_trace, C)
            out['tau_out_trace'] = all_gather_rows(local.tau_out_trace, C)
    if getattr(local, 'moment_sum', None) is not None and K == 1:   # sink moments requested: pool them over all ranks
        out['posterior_mean'], out['posterior_var'], out['posterior_n'] = pooled_moments(   # (the beta = 1 rows)
            local.moment_sum[::T], local.moment_sumsq[::T], local.moment_count)
    if diagnostics:
        from .engine import HMCResult
        src = local if isinstance(local, HMCResult) else local.samples_padded[..., :local.dim]
        out['diagnostics'] = pooled_diagnostics(src, partials=diagnostics_partials)
    return out
