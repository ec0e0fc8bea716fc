"""Host-side mirror of the reference's sampler surface (hamiltorch/samplers.py) on top of the sm_90a kernels.

Same names, argument order, defaults and error behaviour as the reference for the hot path:
``sample`` (samplers.py:850), ``leapfrog`` (:205), ``hamiltonian`` (:738), ``gibbs`` (:152), ``acceptance``
(:609), ``adaptation`` (:629) and the ``Sampler`` / ``Integrator`` / ``Metric`` enums (:11-31).

What differs by design
  * ``log_prob_func`` must be a target descriptor from ``hamiltorch_b200.targets`` (or the list of split
    descriptors ``define_split_model_log_prob`` builds): an opaque Python callable cannot enter a CUDA kernel
    and there is no CPU fallback -> ``TypeError``.
  * the work runs on the current CUDA device whatever ``params_init.device`` is; results are returned on
    ``params_init.device`` so CPU-tensor user code keeps working.
  * extra keyword-only arguments (``rng``, ``seed``) select the random stream; ``sample_chains`` is the batched
    many-chains entry (the engine's native shape), ``sample`` is the one-chain drop-in.
"""
from enum import Enum
import math

import torch

from . import _native as N
from . import engine
from . import targets as T
from . import util


class Sampler(Enum):          # samplers.py:11-14
    HMC = 1
    RMHMC = 2
    HMC_NUTS = 3


class Integrator(Enum):       # samplers.py:19-25
    EXPLICIT = 1
    IMPLICIT = 2
    S3 = 3
    SPLITTING = 4
    SPLITTING_RAND = 5
    SPLITTING_KMID = 6


class Metric(Enum):           # samplers.py:28-31
    HESSIAN = 1
    SOFTABS = 2
    JACOBIAN_DIAG = 3


_SPLIT_INTEGRATORS = (Integrator.SPLITTING, Integrator.SPLITTING_RAND, Integrator.SPLITTING_KMID)


def _require_target(log_prob_func):
    if isinstance(log_prob_func, list):
        if not all(T.is_target(f) for f in log_prob_func):
            raise TypeError('every element of a split log_prob_func list must be a hamiltorch_b200 target')
        return
    if not T.is_target(log_prob_func):
        raise TypeError(
            'hamiltorch_b200 runs the leapfrog loop inside a CUDA kernel and cannot call an opaque Python '
            'log_prob_func.  Pass a descriptor from hamiltorch_b200.targets (GaussianIso, GaussianDiag, '
            'GaussianFull, Funnel) or use sample_model / sample_split_model for Bayesian NNs.  '
            'There is no CPU fallback.')


# ----------------------------------------------------------------------------------------------------------
# small pieces of the reference surface
# ----------------------------------------------------------------------------------------------------------
def acceptance(h_old, h_new):
    """samplers.py:609-626: log acceptance ratio as a Python float."""
    return float(-h_new + h_old)


def adaptation(rho, t, step_size_init, H_t, eps_bar, desired_accept_rate=0.8):
    """samplers.py:629-674, host restatement used only for API completeness (the in-kernel version is what the
    sampler runs).  Same mixed double / fp32 arithmetic."""
    t = t + 1
    if util.has_nan_or_inf(torch.tensor([rho])):
        alpha = 0
    else:
        alpha = min(1., float(torch.exp(torch.FloatTensor([rho]))))
    mu = float(torch.log(10 * torch.FloatTensor([step_size_init])))
    w = 1 / (t + 10)
    H_t = (1 - w) * H_t + w * (desired_accept_rate - alpha)
    x_new = mu - (t ** 0.5) / 0.05 * H_t
    step_size = float(torch.exp(torch.FloatTensor([x_new])))
    x_new_bar = t ** -0.75 * x_new + (1 - t ** -0.75) * torch.log(torch.FloatTensor([eps_bar]))
    eps_bar = float(torch.exp(x_new_bar))
    return step_size, eps_bar, H_t


def gibbs(params, sampler=Sampler.HMC, log_prob_func=None, jitter=None, normalizing_const=1., softabs_const=None,
          mass=None, metric=Metric.HESSIAN):
    """samplers.py:152-202 -- momentum refresh.  Drawn from torch's generator in the reference's way (this is a
    host-side convenience; inside ``sample`` the draw happens in the kernel or is pre-drawn in bulk)."""
    if sampler == Sampler.RMHMC:
        raise NotImplementedError('RMHMC momentum refresh happens inside the RMHMC kernel')
    if mass is None:
        return torch.randn(params.shape, dtype=params.dtype, device=params.device)
    if isinstance(mass, list):                                          # :188-197
        samples = torch.zeros_like(params)
        i = 0
        for block in mass:
            it = block[0].shape[0]
            samples[i:it + i] = torch.distributions.MultivariateNormal(torch.zeros_like(block[0]), block).sample()
            i += it
        return samples
    if mass.dim() == 2:
        return torch.distributions.MultivariateNormal(torch.zeros_like(params), mass).sample()
    return torch.normal(torch.zeros_like(params), mass ** 0.5)


def leapfrog(params, momentum, log_prob_func, steps=10, step_size=0.1, jitter=0.01, normalizing_const=1.,
             softabs_const=1e6, explicit_binding_const=100, fixed_point_threshold=1e-20,
             fixed_point_max_iterations=6, jitter_max_tries=10, inv_mass=None, ham_func=None, sampler=Sampler.HMC,
             integrator=Integrator.IMPLICIT, metric=Metric.HESSIAN, store_on_GPU=True, debug=False, pass_grad=None,
             *, rng_uniforms=None, rng_perms=None):
    """samplers.py:205-606: plain HMC (:269-304), the SPLITTING integrators on a list of data-split closures (:465-603)
    and sampler=RMHMC (:305-462) on the GPU; returns ``(ret_params, ret_momenta)``: two lists of ``steps`` tensors (plain
    HMC: the last momentum carries the half-step correction, :302).  ``params`` may be (D,) as in the reference or (C, D)
    for C chains at once.  ``rng_uniforms`` / ``rng_perms`` inject the jitter draws (RMHMC) / the randperm of
    SPLITTING_RAND instead of consuming torch's generator."""
    _require_target(log_prob_func)
    if sampler == Sampler.HMC and integrator not in _SPLIT_INTEGRATORS:
        if pass_grad is not None:
            raise NotImplementedError('pass_grad: gradients are analytic inside the kernel')
        q_traj, p_traj = engine.leapfrog(log_prob_func, params, momentum, steps, step_size, inv_mass=inv_mass,
                                         return_trajectory=True)
        if params.dim() == 1:
            q_traj, p_traj = q_traj[:, 0], p_traj[:, 0]
        dev = params.device
        return [t.to(dev) for t in q_traj.unbind(0)], [t.to(dev) for t in p_traj.unbind(0)]
    if sampler == Sampler.HMC:
        if type(log_prob_func) is not list:
            raise RuntimeError('For splitting log_prob_func must be list of functions')       # :466-467
        if pass_grad is not None:
            raise RuntimeError('Passing user-determined gradients not implemented for splitting')
        M = len(log_prob_func)
        if M == 1 and integrator in (Integrator.SPLITTING, Integrator.SPLITTING_KMID):
            raise RuntimeError('For symmetric splitting log_prob_func must be list of functions greater than '
                               'length 1')                                                      # :497-498, :577-578
        if integrator not in (Integrator.SPLITTING, Integrator.SPLITTING_RAND, Integrator.SPLITTING_KMID):
            raise NotImplementedError()
        scheme = {Integrator.SPLITTING: N.SCHEME_SPLIT_SYM, Integrator.SPLITTING_RAND: N.SCHEME_SPLIT_RAND,
                  Integrator.SPLITTING_KMID: N.SCHEME_SPLIT_KMID}[integrator]
        perms = None
        if integrator == Integrator.SPLITTING_RAND:
            C_ = 1 if params.dim() == 1 else params.shape[0]
            if rng_perms is not None:                           # (C, M) injected permutations
                perms = rng_perms
            else:                                               # the reference's draw: torch.randperm(M) per call (:550)
                perms = torch.stack([torch.randperm(M) for _ in range(C_)])
        q_traj, p_traj = engine.split_leapfrog(log_prob_func, params, momentum, steps, step_size, scheme,
                                               inv_mass=inv_mass, perms=perms)
        if params.dim() == 1:
            q_traj, p_traj = q_traj[:, 0], p_traj[:, 0]
        dev = params.device
        return [t.to(dev) for t in q_traj.unbind(0)], [t.to(dev) for t in p_traj.unbind(0)]
    if sampler == Sampler.RMHMC:
        if pass_grad is not None:
            raise RuntimeError('Passing user-determined gradients not implemented for RMHMC')  # :310, :390-391
        if integrator not in (Integrator.EXPLICIT, Integrator.IMPLICIT):
            raise NotImplementedError()                                                         # S3: :606
        _check_rmhmc_target(log_prob_func, metric)
        if jitter is not None and rng_uniforms is None and not torch.is_tensor(jitter):
            # the reference draws torch.rand(D) inside every fisher() call (:115): a data-dependent number of draws for
            # the implicit integrator and for NaN retries, so they are drawn on the fly inside the kernel (Philox keyed
            # by a seed taken from torch's generator) unless the caller injects them
            pass
        explicit = integrator == Integrator.EXPLICIT
        seed = int(torch.randint(0, 2 ** 62, (1,)))
        qt, ptj, qcopy, pcopy, failed = engine.rmhmc_leapfrog(
            log_prob_func, params, momentum, steps, step_size, jitter=jitter, softabs_const=softabs_const,
            explicit_binding_const=explicit_binding_const, fixed_point_threshold=fixed_point_threshold,
            fixed_point_max_iterations=fixed_point_max_iterations, jitter_max_tries=jitter_max_tries, explicit=explicit,
            softabs=(metric == Metric.SOFTABS), jacdiag=(metric == Metric.JACOBIAN_DIAG), uniforms=rng_uniforms, seed=seed)
        if int(failed.sum()) > 0:
            raise util.LogProbError()                                                           # :110-112, :717, :733
        dev = params.device
        single = params.dim() == 1
        ret_params = [(t[0] if single else t).to(dev) for t in qt.unbind(0)]
        ret_momenta = [(t[0] if single else t).to(dev) for t in ptj.unbind(0)]
        if explicit:                                                                            # :462
            return [ret_params, (qcopy[0] if single else qcopy).to(dev)], \
                   [ret_momenta, (pcopy[0] if single else pcopy).to(dev)]
        return ret_params, ret_momenta
    raise NotImplementedError()


def _check_rmhmc_target(log_prob_func, metric):
    if isinstance(log_prob_func, list) or not isinstance(log_prob_func, (T.Funnel, T.GaussianIso, T.GaussianDiag,
                                                                         T.GaussianFull)):
        raise NotImplementedError('RMHMC needs closed-form third derivatives: Funnel / Gaussian descriptors')
    if metric not in (Metric.HESSIAN, Metric.SOFTABS, Metric.JACOBIAN_DIAG):
        raise NotImplementedError()
    if log_prob_func.dim > 64:
        raise NotImplementedError('stand-alone RMHMC leapfrog / hamiltonian: D <= 64 (metric in shared memory)')


def hamiltonian(params, momentum, log_prob_func, jitter=0.01, normalizing_const=1., softabs_const=1e6,
                explicit_binding_const=100, inv_mass=None, ham_func=None, sampler=Sampler.HMC,
                integrator=Integrator.EXPLICIT, metric=Metric.HESSIAN, *, rng_uniforms=None):
    """samplers.py:738-846: sampler=HMC (:779-815) and sampler=RMHMC (:817-829 -> rm_hamiltonian).  Raises util.LogProbError on a non-finite log-prob like the
    reference (:783-785).  (D,) -> tensor of shape (); (C, D) -> (C,)."""
    _require_target(log_prob_func)
    if sampler == Sampler.RMHMC:                                                                # :817-829
        _check_rmhmc_target(log_prob_func, metric)
        H, flags = engine.rmhmc_hamiltonian(log_prob_func, params, momentum, jitter=jitter, softabs_const=softabs_const,
                                            softabs=(metric == Metric.SOFTABS), jacdiag=(metric == Metric.JACOBIAN_DIAG),
                                            uniforms=rng_uniforms, seed=int(torch.randint(0, 2 ** 62, (1,))))
        if int(flags.sum()) > 0:
            raise util.LogProbError()
        if integrator == Integrator.EXPLICIT:
            H = 2 * H                                                                           # :822
        H = H.to(params.device)
        return H[0].reshape(1, 1) if params.dim() == 1 else H       # the reference returns a (1, 1) tensor (:731)
    if sampler != Sampler.HMC or isinstance(log_prob_func, list):
        raise NotImplementedError()
    H, flags = engine.hamiltonian(log_prob_func, params, momentum, inv_mass=inv_mass)
    if int(flags.sum()) > 0:
        raise util.LogProbError()
    H = H.to(params.device)
    return H[0] if params.dim() == 1 else H


# ----------------------------------------------------------------------------------------------------------
# sample()
# ----------------------------------------------------------------------------------------------------------
def _sink_supported(log_prob_func, sampler, integrator, inv_mass):
    """The kernels with a sample sink (thin / moments / keep_samples / store_on_GPU=False): plain HMC / HMC_NUTS on an
    element-wise target (GaussianIso, GaussianDiag) and the Bayesian-NN kernel (an MLPRegression, or a list of them with a
    SPLITTING integrator), with inv_mass None or 1-D."""
    if sampler not in (Sampler.HMC, Sampler.HMC_NUTS) or isinstance(inv_mass, list) or \
            (torch.is_tensor(inv_mass) and inv_mass.dim() == 2):
        return False
    if isinstance(log_prob_func, list):
        return integrator in _SPLIT_INTEGRATORS and all(isinstance(f, T.MLPRegression) for f in log_prob_func)
    return integrator not in _SPLIT_INTEGRATORS and isinstance(log_prob_func, (T.GaussianIso, T.GaussianDiag,
                                                                               T.MLPRegression))


def _check_sample_args(params_init_dim_ok, num_samples, burn, sampler):
    if not params_init_dim_ok:
        raise RuntimeError('params_init must be a 1d tensor.')                  # :925-926
    if burn >= num_samples:
        raise RuntimeError('burn must be less than num_samples.')               # :928-929
    if sampler == Sampler.HMC_NUTS and burn == 0:
        raise RuntimeError('burn must be greater than 0 for NUTS.')             # :933-934


def _draw_reference_stream(dim, num_samples, device, num_perm=0, blocks=None, gamma_shapes=None):
    """Pre-draw one chain's randoms from torch's GLOBAL generators in exactly the order the reference consumes
    them (SURVEY.md section 8c fact 3): per iteration the momentum normals -- ``Normal(zeros_like(params),
    ones_like(params)).sample()`` (:186, :202), i.e. the generator of params' device -- then ``torch.rand(1)`` on
    the CPU generator (:1004).  Valid while no LogProbError occurs (that skips the iteration's rand(1)).
    ``gamma_shapes`` (hyperpriors, (K,) fp64 with 0 for a fixed group): after the iteration's rand(1), ONE
    ``torch._standard_gamma`` call on the CPU generator over the sampled groups' posterior shapes in group order; the
    draws come back as the last element, (S, K) fp64 with 0 at the fixed groups."""
    z = torch.empty((num_samples, dim), dtype=torch.float32, device=device)
    logu = torch.empty(num_samples, dtype=torch.float32)
    perms = torch.empty((num_samples, num_perm), dtype=torch.int32) if num_perm else None
    gam = None
    if gamma_shapes is not None:
        gam = torch.zeros((num_samples, gamma_shapes.numel()), dtype=torch.float64)
        live = gamma_shapes > 0
    for n in range(num_samples):
        if blocks:                                          # block-list mass: one draw per block (:188-197)
            z[n] = torch.cat([torch.randn(b, dtype=torch.float32, device=device) for b in blocks])
        else:
            z[n] = torch.randn(dim, dtype=torch.float32, device=device)
        if num_perm:
            perms[n] = torch.randperm(num_perm)             # SPLITTING_RAND: once per trajectory (:550)
        logu[n] = torch.log(torch.rand(1))[0]
        if gam is not None:
            gam[n, live] = torch._standard_gamma(gamma_shapes[live])
    out = (z, logu) + ((perms,) if num_perm else ())
    return out + ((gam,) if gam is not None else ())


def _draw_rmhmc_reference_stream(dim, num_samples, L, jitter, explicit, device):
    """``_draw_reference_stream`` for sampler=RMHMC, as engine.rmhmc_run's ``normals`` / ``log_uniforms`` / ``uniforms``:
    with ``jitter``, the J = 8 L + 3 ``torch.rand(D)`` draws of the explicit integrator's ``fisher`` calls interleave
    with each iteration's momentum normals."""
    if jitter is not None and not explicit:
        raise NotImplementedError(
            "implicit RMHMC with jitter draws a data-dependent number of uniforms per iteration; its "
            "reference stream cannot be pre-drawn -- use rng='philox'")
    J = (8 * L + 3) if jitter is not None else 0
    z = torch.empty((num_samples, dim), dtype=torch.float32, device=device)
    logu = torch.empty(num_samples, dtype=torch.float32)
    uni = torch.zeros((num_samples, max(J, 1), dim), dtype=torch.float32)
    for n in range(num_samples):                     # fisher's rand(D) (:115) is always CPU, gibbs first (:184)
        if J:
            uni[n, 0] = torch.rand(dim)
        z[n] = torch.randn(dim, dtype=torch.float32, device=device)
        for j in range(1, J):
            uni[n, j] = torch.rand(dim)
        logu[n] = torch.log(torch.rand(1))[0]
    return dict(normals=z.unsqueeze(1), log_uniforms=logu.unsqueeze(1), uniforms=uni.unsqueeze(1) if J else None)


def _stream_args(rng, q0, seed, normals, log_uniforms, injected, draw_reference):
    """The random stream of a run as engine.hmc_run / rmhmc_run keyword arguments.  rng='reference': one chain replaying
    torch's global generators, pre-drawn by ``draw_reference()``; 'injected': ``normals`` and ``log_uniforms`` (both
    required) with the sampler family's other streams ``injected``; 'philox': the in-kernel stream keyed by ``seed``
    (None: drawn from torch's RNG)."""
    if rng == 'reference':
        if q0.shape[0] != 1:
            raise RuntimeError("rng='reference' replays torch's global stream and is defined for one chain")
        stream = draw_reference()
    elif rng == 'injected':
        if normals is None or log_uniforms is None:
            raise RuntimeError("rng='injected' needs normals and log_uniforms")
        stream = dict(injected, normals=normals, log_uniforms=log_uniforms)
    elif rng == 'philox':
        if seed is None:
            seed = int(torch.randint(0, 2 ** 62, (1,)))
        stream = dict(normals=None, log_uniforms=None)
    else:
        raise ValueError('unknown rng mode %r' % (rng,))
    return dict(stream, seed=seed or 0)


def sample(log_prob_func, params_init, num_samples=10, num_steps_per_sample=10, step_size=0.1, burn=0, jitter=None,
           inv_mass=None, normalizing_const=1., softabs_const=None, explicit_binding_const=100,
           fixed_point_threshold=1e-5, fixed_point_max_iterations=1000, jitter_max_tries=10, sampler=Sampler.HMC,
           integrator=Integrator.IMPLICIT, metric=Metric.HESSIAN, debug=False, desired_accept_rate=0.8,
           store_on_GPU=True, pass_grad=None, verbose=True, *, rng='reference', seed=None, tau_prior=None,
           tau_out_prior=None):
    """Drop-in for ``hamiltorch.sample`` (samplers.py:850-1091): ONE chain, same arguments, same return value --
    a list of ``num_samples - burn`` detached (D,) tensors whose element 0 is ``params_init`` (:959), plus the
    adapted step size (NUTS) or the acceptance rate when ``debug == 2`` (:1086-1089).

    rng='reference' (default): the chain consumes torch's global random stream exactly like the reference, so
        after ``set_random_seed(s)`` the returned samples equal the reference's (to fp32 summation order in the
        Hamiltonian).  rng='philox': in-kernel counter RNG keyed by ``seed`` (default: drawn from torch's RNG).
    ``tau_prior`` / ``tau_out_prior``: Gamma hyperpriors on the precisions of a Bayesian-NN target (see
    ``sample_chains``).  The call then returns ``(samples, hyper)`` -- ``hyper`` a dict of the retained slots'
    ``'tau_list'`` (S-burn, 2L) and ``'tau_out'`` (S-burn,) -- and ``(samples, hyper, value)`` with ``debug == 2``.
    With rng='reference' the gamma draws come from torch's CPU generator after each iteration's rand(1)
    (``_draw_reference_stream``), so ``set_random_seed`` makes the call reproducible.
    """
    _check_sample_args(params_init.dim() == 1, num_samples, burn, sampler)
    _require_target(log_prob_func)
    if pass_grad is not None:
        if sampler == Sampler.RMHMC:
            raise RuntimeError('Passing user-determined gradients not implemented for RMHMC')     # :310
        if integrator in _SPLIT_INTEGRATORS:
            raise RuntimeError('Passing user-determined gradients not implemented for splitting')  # :468-469
        raise NotImplementedError('pass_grad: gradients are analytic inside the kernel')
    res = _run_chains(log_prob_func, params_init.unsqueeze(0), num_samples, num_steps_per_sample, step_size, burn,
                      jitter, inv_mass, softabs_const, explicit_binding_const, fixed_point_threshold,
                      fixed_point_max_iterations, jitter_max_tries, sampler, integrator, metric,
                      desired_accept_rate, rng=rng, seed=seed, record_ham=(debug == 1),
                      sink=dict(host_samples=True) if (
                          not store_on_GPU and _sink_supported(log_prob_func, sampler, integrator, inv_mass)) else None,
                      hyper=_hyper_groups(log_prob_func, sampler, tau_prior, tau_out_prior))
    if not res.samples_padded.is_cuda:
        torch.cuda.current_stream().synchronize()       # the kernel wrote the samples into pinned host memory
    nuts = sampler == Sampler.HMC_NUTS
    out_dev = params_init.device if store_on_GPU else torch.device('cpu')
    samples = res.samples[0].to(out_dev)
    ret = list(samples.unbind(0))
    num_rejected = int(res.num_rejected[0])
    final_eps = float(res.step_size[0])
    if debug == 1:
        ham = res.ham[0].cpu()
        acc = res.accepted[0].cpu()
        for n in range(num_samples):
            print('Step: {}, Current Hamiltoninian: {}, Proposed Hamiltoninian: {}'.format(n, ham[n, 0], ham[n, 1]))
            print('Accept rho: {}'.format(min(0., float(ham[n, 0] - ham[n, 1]))) if acc[n] else 'REJECT')
    if nuts:
        print('Final Adapted Step Size: ', final_eps)                                              # :1035
    if verbose:
        print('Acceptance Rate {:.2f}'.format(1 - num_rejected / num_samples))                     # :1085
    extra = ()
    if getattr(res, 'tau_list_trace', None) is not None:
        extra = ({'tau_list': res.tau_list_trace[0], 'tau_out': res.tau_out_trace[0]},)
    if nuts and debug == 2:
        return (ret,) + extra + (final_eps,)
    elif debug == 2:
        return (ret,) + extra + (1 - num_rejected / num_samples,)
    return (ret,) + extra if extra else ret


def sample_chains(log_prob_func, params_init, num_samples=10, num_steps_per_sample=10, step_size=0.1, burn=0,
                  jitter=None, inv_mass=None, softabs_const=None, explicit_binding_const=100,
                  fixed_point_threshold=1e-5, fixed_point_max_iterations=1000, jitter_max_tries=10,
                  sampler=Sampler.HMC, integrator=Integrator.IMPLICIT, metric=Metric.HESSIAN,
                  desired_accept_rate=0.8, rng='philox', seed=0, chain_offset=0, normals=None, log_uniforms=None,
                  record_ham=False, out=None, perms=None, uniforms=None, thin=1, moments=False, keep_samples=True,
                  store_on_GPU=True, host_windows=0, adapt_mass=False, mass_pool=None, tau_prior=None,
                  tau_out_prior=None, gammas=None, betas=None, swap_every=10, swap_log_uniforms=None, folds=None):
    """The engine's native entry: C independent chains at once.  ``params_init`` is (C, D); every chain gets the
    reference's ``sample`` semantics.  Returns an ``engine.HMCResult`` whose ``.samples`` is (C, S-burn, D) on the
    GPU (row c = what ``sample`` would have returned for chain c, stacked).

    rng='philox'  in-kernel Philox4x32-10 keyed by (seed, chain_offset + c, iteration) -- results do not depend on
                  how chains are sharded over GPUs.
    rng='injected'  consume ``normals`` (S, C, D) / ``log_uniforms`` (S, C) (parity mode; SPLITTING_RAND also
                  ``perms`` (S, C, M)).
    ``log_prob_func`` may be a Gaussian / funnel descriptor, an ``MLPRegression`` (sample_model) or the list of split
    descriptors ``define_split_model_log_prob`` returns (with a SPLITTING integrator).

    Sample sink (plain HMC / HMC_NUTS on GaussianIso / GaussianDiag, and the Bayesian-NN targets with any of their
    integrators; inv_mass None or 1-D): ``thin`` keeps every thin-th post-burn state;
    ``moments=True`` returns per-chain running sums / sums of squares over all post-burn iterations
    (``.moment_sum``, ``.moment_sumsq``, ``.moment_count``); ``keep_samples=False`` stores no samples;
    ``store_on_GPU=False`` (the reference's flag, samplers.py:1008-1012) streams the retained samples from the kernel
    straight into pinned host memory: ``.samples`` is then a CPU tensor (synchronise the stream before reading).
    ``out=<pinned host block>, host_windows=W`` (W >= 2) delivers into the caller's block through the copy engine instead:
    the run is cut into W windows of iterations and each window's sample slots go to the host on a second stream while the
    next window computes (costs a device staging block).

    ``adapt_mass=True`` adapts one diagonal ``inv_mass`` shared by all chains during warm-up, with Stan's windowed
    schedule (``engine.mass_windows(burn)``): the draws of every chain in a window are pooled into the variance estimate
    of each dimension (regularised as Stan does), and the step-size dual averaging restarts after each update.  Needs
    ``sampler=Sampler.HMC_NUTS`` and ``burn >= 20`` (``RuntimeError``) and a combination with a sample sink: GaussianIso /
    GaussianDiag with D <= 4096, an MLPRegression, or a list of them with a SPLITTING integrator; ``inv_mass`` None or
    1-D (the initial metric); no ``host_windows`` (``NotImplementedError`` otherwise).  ``thin`` / ``moments`` /
    ``keep_samples`` / ``store_on_GPU`` apply to the sampling phase.  The result gains ``.inv_mass`` (D,) fp32 -- the
    mass used after warm-up --, ``.inv_mass_trace`` (K, D), one row per window, and ``.mass_windows``, the K (a, b)
    iteration ranges.  ``mass_pool`` (multi-GPU; ``distributed.sample_chains_sharded`` passes it) maps each (C_local, ld)
    window sum to the sum of all chains in global order, so that every rank adapts the same mass.

    Hyperpriors (an ``MLPRegression`` or a split list of them, HMC / HMC_NUTS; DESIGN §3.15): ``tau_prior`` is ``(a, b)``
    for every parameter tensor or a list of 2L entries in tau_list order, each ``(a, b)`` or ``None`` (fixed at its
    tau_list value); ``tau_out_prior`` is ``(a, b)`` for the regression noise precision.  Gamma(shape a, rate b); every
    iteration, after the MH step, each precision is drawn from its Gamma conditional given the weights (and, for tau_out,
    the sum of squared errors over all data rows) inside the kernel, and the next iteration samples with the new values.
    They start from tau_list / tau_out.  ``rng='injected'`` also takes ``gammas`` (S, C, 2L + 1) fp64: the
    standard-gamma draw of every group (tensors, then tau_out).  The result gains ``.tau_list_trace`` (C, keep, 2L) and
    ``.tau_out_trace`` (C, keep) for the retained sample slots (slot 0 = the initial values; on the device even with
    ``store_on_GPU=False``) and the final state ``.tau_list_final`` / ``.tau_out_final``.

    Replica exchange (an ``MLPTarget`` or a split list of them, HMC / HMC_NUTS; DESIGN §3.17): ``betas`` are T likelihood
    exponents, ``betas[0] == 1.0``, strictly decreasing, all >= 0; rung t samples the power posterior p(theta) L(theta)^beta_t,
    i.e. the target with ``tau_out`` replaced by ``beta_t * tau_out``.  ``params_init`` is (C, D) with C = R T, ladder-major:
    row r T + t is ladder r at beta_t.  The run goes in windows of ``swap_every`` iterations; after window k, if iterations
    remain, swap round k pairs the rungs (t, t + 1) with t = k (mod 2) of every ladder and exchanges their states when
    log u < (beta_t - beta_{t+1}) (ll_{t+1} - ll_t) in fp64, ll the untempered log-likelihood at the row's state.  Step
    sizes, dual averaging, moments and counters stay with the row; swaps run during burn-in too.  ``rng='philox'`` draws u
    from its own stream keyed by the global ladder (``chain_offset`` must be a multiple of T); ``rng='injected'`` reads
    ``swap_log_uniforms`` (rounds, R, T - 1).  Only the beta = 1 rows store samples: ``.samples`` is (R, keep, D) (``thin``,
    ``keep_samples``, ``store_on_GPU`` and ``out`` (R, keep, ld) apply to it); per-row outputs stay (C, ...).  The result
    gains ``.betas``, ``.swap_accepted`` (rounds, R, T - 1) int8 (-1: the pair was not in that round), ``.swap_ll``
    (rounds, C) fp64 and ``.swap_rate`` (T - 1,).  Not combined with RMHMC, non-BNN targets, a 2-D or block ``inv_mass``,
    ``adapt_mass``, hyperpriors or ``rng='reference'``.

    K-fold refits (an ``MLPTarget`` with data, HMC / HMC_NUTS, the plain integrator; DESIGN §3.18): ``folds`` is an (N,)
    integer tensor assigning each data row to a fold 0 .. K-1, or to -1 (never left out); K = max + 1, 2 <= K <= 64, and
    every fold id occurs.  ``params_init`` is (C, D) with C = R K: row r K + k is chain r of the fit WITHOUT fold k, so
    ``.samples[k::K]`` is fold k's posterior.  That row samples exactly what the same call without ``folds`` samples on
    the MLPTarget of the rows {i : folds[i] != k} in their original order (the prior counted once, the log-softmax loss
    a mean over those rows); step size, dual averaging, counters and the sink options stay with the row.  All K fits run
    in one launch.  ``chain_offset`` must be a multiple of K.  The result gains ``.folds`` (on the device) and
    ``.num_folds``; ``loo.kfold`` scores it.  Not combined with split lists, SPLITTING integrators, ``betas``,
    hyperpriors, ``adapt_mass``, RMHMC, a 2-D or block ``inv_mass``, non-BNN targets or ``rng='reference'``.
    """
    if params_init.dim() != 2:
        raise RuntimeError('sample_chains: params_init must be (num_chains, D)')
    _check_sample_args(True, num_samples, burn, sampler)
    _require_target(log_prob_func)
    if adapt_mass:
        _check_adapt_mass(log_prob_func, sampler, integrator, inv_mass, burn, host_windows)
    hyper = _hyper_groups(log_prob_func, sampler, tau_prior, tau_out_prior)
    temper = _temper_args(log_prob_func, params_init, num_samples, sampler, inv_mass, adapt_mass, hyper, rng,
                          chain_offset, betas, swap_every, swap_log_uniforms)
    folds = _fold_args(log_prob_func, params_init, sampler, integrator, inv_mass, adapt_mass, hyper, betas, rng,
                       chain_offset, folds)
    return _run_chains(log_prob_func, params_init, num_samples, num_steps_per_sample, step_size, burn, jitter,
                       inv_mass, softabs_const, explicit_binding_const, fixed_point_threshold,
                       fixed_point_max_iterations, jitter_max_tries, sampler, integrator, metric,
                       desired_accept_rate, rng=rng, seed=seed, chain_offset=chain_offset, normals=normals,
                       log_uniforms=log_uniforms, record_ham=record_ham, out=out, injected_perms=perms,
                       injected_uniforms=uniforms,
                       sink=dict(thin=thin, moments=moments, keep_samples=keep_samples, host_samples=not store_on_GPU,
                                 host_windows=host_windows, **(dict(adapt_mass=True, mass_pool=mass_pool)
                                                               if adapt_mass else {})),
                       hyper=hyper, gammas=gammas, temper=temper, folds=folds)


def _fold_args(log_prob_func, params_init, sampler, integrator, inv_mass, adapt_mass, hyper, betas, rng, chain_offset,
               folds):
    """sample_chains(folds=...) -> the (N,) int64 CPU assignment engine.hmc_run takes (None without folds), checked
    before any CUDA work."""
    if folds is None:
        return None
    if isinstance(log_prob_func, list) or integrator in _SPLIT_INTEGRATORS:
        raise NotImplementedError('K-fold runs: not with split lists or SPLITTING integrators -- pass the MLPTarget of '
                                  'the whole data set with the plain integrator')
    if not isinstance(log_prob_func, T.MLPTarget):
        raise NotImplementedError('K-fold runs: Bayesian-NN targets only (an MLPTarget)')
    if sampler not in (Sampler.HMC, Sampler.HMC_NUTS):
        raise NotImplementedError('K-fold runs: sampler HMC or HMC_NUTS (not RMHMC)')
    if log_prob_func.x is None:
        raise RuntimeError('K-fold runs: the target has no data (x is None): there are no rows to leave out')
    if isinstance(inv_mass, list) or (torch.is_tensor(inv_mass) and inv_mass.dim() != 1):
        raise NotImplementedError('K-fold runs: inv_mass None or 1-D')
    if betas is not None:
        raise NotImplementedError('K-fold runs are not combined with replica exchange (betas)')
    if hyper is not None:
        raise NotImplementedError('K-fold runs are not combined with hyperpriors (tau_prior / tau_out_prior)')
    if adapt_mass:
        raise NotImplementedError('K-fold runs are not combined with adapt_mass: it would pool one mass across the '
                                  'different posteriors of the folds')
    if rng == 'reference':
        raise NotImplementedError("K-fold runs: rng='philox' or 'injected' (the reference stream is one chain)")
    if not torch.is_tensor(folds) or folds.dtype.is_floating_point or folds.dtype.is_complex or \
            folds.dtype == torch.bool:
        raise ValueError('folds must be an integer tensor, got %s' % (folds.dtype if torch.is_tensor(folds)
                                                                      else type(folds).__name__))
    f = folds.detach().to('cpu', torch.int64)
    Nr = log_prob_func.x.shape[0]
    if f.dim() != 1 or f.numel() != Nr:
        raise ValueError('folds must be (N,) = (%d,), one fold per data row, got %s' % (Nr, tuple(folds.shape)))
    K = int(f.max()) + 1
    if int(f.min()) < -1 or not 2 <= K <= N.MLP_MAX_SPLITS:
        raise ValueError('folds must hold values in -1 .. K-1 with 2 <= K <= %d, got min %d, max %d'
                         % (N.MLP_MAX_SPLITS, int(f.min()), K - 1))
    missing = [k for k in range(K) if not bool((f == k).any())]
    if missing:
        raise ValueError('folds: every fold id 0 .. K-1 must occur; missing %s' % missing)
    if params_init.shape[0] % K != 0:
        raise ValueError('K-fold runs: params_init has %d rows, not a multiple of K = %d' % (params_init.shape[0], K))
    if int(chain_offset) % K != 0:
        raise ValueError('K-fold runs: chain_offset %d is not a multiple of K = %d' % (chain_offset, K))
    return f


def _temper_args(log_prob_func, params_init, num_samples, sampler, inv_mass, adapt_mass, hyper, rng, chain_offset,
                 betas, swap_every, swap_log_uniforms):
    """sample_chains(betas=...) -> engine.hmc_run's ``temper`` dict (None without betas), checked before any CUDA work."""
    if betas is None:
        return None
    descs = log_prob_func if isinstance(log_prob_func, list) else [log_prob_func]
    if not descs or not all(isinstance(d, T.MLPRegression) for d in descs):
        raise NotImplementedError('replica exchange: Bayesian-NN targets only (an MLPRegression or a list of them)')
    if sampler not in (Sampler.HMC, Sampler.HMC_NUTS):
        raise NotImplementedError('replica exchange: sampler HMC or HMC_NUTS')
    if isinstance(inv_mass, list) or (torch.is_tensor(inv_mass) and inv_mass.dim() != 1):
        raise NotImplementedError('replica exchange: inv_mass None or 1-D')
    if adapt_mass:
        raise NotImplementedError('replica exchange is not combined with adapt_mass')
    if hyper is not None:
        raise NotImplementedError('replica exchange is not combined with hyperpriors (tau_prior / tau_out_prior)')
    if rng == 'reference':
        raise NotImplementedError("replica exchange: rng='philox' or 'injected' (the reference stream is one chain)")
    try:
        b = [float(v) for v in (betas.tolist() if torch.is_tensor(betas) else betas)]
    except (TypeError, ValueError):
        raise ValueError('betas must be a sequence of floats, got %r' % (betas,))
    if not 1 <= len(b) <= N.TEMPER_MAX_TEMPS:
        raise ValueError('betas needs 1 to %d values, got %d' % (N.TEMPER_MAX_TEMPS, len(b)))
    if b[0] != 1.0 or not all(math.isfinite(v) and v >= 0 for v in b) or any(x <= y for x, y in zip(b, b[1:])):
        raise ValueError('betas must start at 1.0 and decrease strictly to values >= 0, got %r' % (b,))
    Tn, Cn = len(b), params_init.shape[0]
    if Cn % Tn != 0:
        raise ValueError('replica exchange: params_init has %d rows, not a multiple of T = %d' % (Cn, Tn))
    if int(chain_offset) % Tn != 0:
        raise ValueError('replica exchange: chain_offset %d is not a multiple of T = %d' % (chain_offset, Tn))
    if isinstance(swap_every, bool) or int(swap_every) != swap_every or int(swap_every) < 1:
        raise ValueError('swap_every must be an integer >= 1, got %r' % (swap_every,))
    rounds = engine.swap_rounds(num_samples, swap_every)
    if rng == 'injected':
        shape = (rounds, Cn // Tn, Tn - 1)
        if swap_log_uniforms is None or tuple(swap_log_uniforms.shape) != shape:
            raise ValueError("rng='injected' with betas needs swap_log_uniforms of shape (rounds, R, T - 1) = %s, got %s"
                             % (shape, None if swap_log_uniforms is None else tuple(swap_log_uniforms.shape)))
    else:
        swap_log_uniforms = None
    return dict(betas=b, swap_every=int(swap_every), swap_log_uniforms=swap_log_uniforms)


def _check_gamma(ab, what):
    try:
        a, b = (float(v) for v in ab)
    except (TypeError, ValueError):
        raise ValueError('%s must be a pair (a, b), got %r' % (what, ab))
    if not (0 < a < math.inf and 0 < b < math.inf):
        raise ValueError('%s: Gamma(a, b) needs finite a > 0 and b > 0, got (%r, %r)' % (what, a, b))
    return a, b


def _hyper_groups(log_prob_func, sampler, tau_prior, tau_out_prior):
    """tau_prior / tau_out_prior -> the 2L + 1 entries of engine.hmc_run's ``hyper`` (None: no hyperprior), checked
    before any CUDA work."""
    if tau_prior is None and tau_out_prior is None:
        return None
    descs = log_prob_func if isinstance(log_prob_func, list) else [log_prob_func]
    if not descs or not all(isinstance(d, T.MLPRegression) for d in descs):
        raise NotImplementedError('hyperpriors on tau_list / tau_out: Bayesian-NN targets only (an MLPRegression or a '
                                  'list of them)')
    if sampler not in (Sampler.HMC, Sampler.HMC_NUTS):
        raise NotImplementedError('hyperpriors on tau_list / tau_out: sampler HMC or HMC_NUTS')
    K = 2 * descs[0].num_layers
    if tau_prior is None:
        groups = [None] * K
    elif isinstance(tau_prior, list):
        if len(tau_prior) != K:
            raise ValueError('tau_prior needs one entry per parameter tensor (%d), got %d' % (K, len(tau_prior)))
        groups = [None if ab is None else _check_gamma(ab, 'tau_prior[%d]' % k) for k, ab in enumerate(tau_prior)]
    else:
        groups = [_check_gamma(tau_prior, 'tau_prior')] * K
    if tau_out_prior is None:
        groups.append(None)
    else:
        if descs[0].loss_id != T.LOSS_REGRESSION:
            raise NotImplementedError('tau_out_prior: regression only -- the classification losses use tau_out as a '
                                      'tempering factor, not as a noise precision')
        if descs[0].x is None:
            raise RuntimeError('tau_out_prior needs data (x is None samples the prior)')
        groups.append(_check_gamma(tau_out_prior, 'tau_out_prior'))
    return groups


def _reference_gamma_shapes(log_prob_func, hyper):
    """The posterior shapes a_k + n_k / 2 and a_o + N O / 2 of the sampled groups, 0 at the fixed ones (fp64)."""
    descs = log_prob_func if isinstance(log_prob_func, list) else [log_prob_func]
    n_obs = sum(d.x.shape[0] for d in descs if d.x is not None) * descs[0].widths[-1]
    sizes = list(descs[0].sizes) + [n_obs]
    return torch.tensor([0.0 if ab is None else ab[0] + 0.5 * n for ab, n in zip(hyper, sizes)], dtype=torch.float64)


def _check_adapt_mass(log_prob_func, sampler, integrator, inv_mass, burn, host_windows):
    """sample_chains(adapt_mass=True) refusals, raised before any CUDA work."""
    if not _sink_supported(log_prob_func, sampler, integrator, inv_mass) or \
            (isinstance(log_prob_func, (T.GaussianIso, T.GaussianDiag)) and N.padded_ld(log_prob_func.dim) > 4096):
        raise NotImplementedError('adapt_mass: GaussianIso / GaussianDiag with D <= 4096, an MLPRegression or a list of them '
                                  'with a SPLITTING integrator, and inv_mass None or 1-D')
    if sampler != Sampler.HMC_NUTS:
        raise RuntimeError('adapt_mass needs sampler=Sampler.HMC_NUTS: the step size is re-tuned after each mass update')
    if burn < 20:
        raise RuntimeError('adapt_mass needs burn >= 20 (got %d)' % burn)
    if int(host_windows) >= 2:
        raise NotImplementedError('adapt_mass with host_windows: windowed copy-engine delivery is not combined with '
                                  'mass adaptation')


def _run_chains(log_prob_func, q0, num_samples, L, step_size, burn, jitter, inv_mass, softabs_const,
                explicit_binding_const, fixed_point_threshold, fixed_point_max_iterations, jitter_max_tries,
                sampler, integrator, metric, desired_accept_rate, rng='philox', seed=None, chain_offset=0,
                normals=None, log_uniforms=None, record_ham=False, out=None, injected_perms=None,
                injected_uniforms=None, sink=None, hyper=None, gammas=None, temper=None, folds=None):
    nuts = sampler == Sampler.HMC_NUTS
    hyper_kw = {} if hyper is None else dict(hyper=hyper)
    if temper is not None:
        hyper_kw['temper'] = temper
    if folds is not None:
        hyper_kw['folds'] = folds
    gshapes = None if hyper is None else _reference_gamma_shapes(log_prob_func, hyper)
    sink = sink or {}
    if (sink.get('thin', 1) != 1 or sink.get('moments') or not sink.get('keep_samples', True) or
            sink.get('host_samples')) and not _sink_supported(log_prob_func, sampler, integrator, inv_mass):
        raise NotImplementedError('thin / moments / keep_samples / store_on_GPU=False: plain HMC on element-wise targets '
                                  'and the Bayesian-NN targets, with inv_mass None or 1-D')
    if nuts:
        sampler = Sampler.HMC                                                     # :932-936
    if sampler == Sampler.HMC and integrator not in _SPLIT_INTEGRATORS:
        if isinstance(log_prob_func, list):
            raise NotImplementedError('a list log_prob_func needs a SPLITTING integrator')
        scheme = N.SCHEME_PLAIN if isinstance(log_prob_func, T.MLPRegression) else None
        D = log_prob_func.dim
    elif sampler == Sampler.HMC:
        if type(log_prob_func) is not list:
            raise RuntimeError('For splitting log_prob_func must be list of functions')            # :466-467
        if len(log_prob_func) == 1 and integrator in (Integrator.SPLITTING, Integrator.SPLITTING_KMID):
            raise RuntimeError('For symmetric splitting log_prob_func must be list of functions greater than '
                               'length 1')                                                          # :497-498, :577-578
        if isinstance(inv_mass, list):
            raise NotImplementedError('block-list inv_mass with a splitting integrator: the reference ignores the blocks in '
                                      'the drift (samplers.py:514-515); pass the block-diagonal matrix or a 1-D inv_mass')
        scheme = {Integrator.SPLITTING: N.SCHEME_SPLIT_SYM, Integrator.SPLITTING_RAND: N.SCHEME_SPLIT_RAND,
                  Integrator.SPLITTING_KMID: N.SCHEME_SPLIT_KMID}[integrator]
        D = log_prob_func[0].dim
    else:
        if hyper is not None:
            raise NotImplementedError('hyperpriors on tau_list / tau_out: sampler HMC or HMC_NUTS')
        if sampler != Sampler.RMHMC or integrator not in (Integrator.EXPLICIT, Integrator.IMPLICIT):
            raise NotImplementedError()                                                             # :606, :844
        if isinstance(log_prob_func, list) or not isinstance(log_prob_func, (T.Funnel, T.GaussianIso, T.GaussianDiag,
                                                                             T.GaussianFull)):
            raise NotImplementedError('RMHMC needs closed-form third derivatives: Funnel / Gaussian descriptors')
        jacdiag = metric == Metric.JACOBIAN_DIAG
        if metric not in (Metric.HESSIAN, Metric.SOFTABS, Metric.JACOBIAN_DIAG):
            raise NotImplementedError()
        D = log_prob_func.dim
        const_metric = jitter is None and not jacdiag and isinstance(log_prob_func, (T.GaussianIso, T.GaussianDiag,
                                                                                     T.GaussianFull))
        if D > 64 and not const_metric:
            raise NotImplementedError('RMHMC with a position-dependent or jittered metric: D <= 64 (metric, eigenvectors '
                                      'and one work matrix in shared memory); Gaussian targets with jitter=None run on '
                                      'the constant-metric tensor-core path at any D')
        if inv_mass is not None:
            pass                                            # the reference ignores inv_mass for RMHMC (:989 comment)
    if q0.shape[1] != D:
        raise RuntimeError('params_init has %d entries, the target has %d' % (q0.shape[1], D))
    if sampler == Sampler.RMHMC:
        explicit = integrator == Integrator.EXPLICIT
        stream = _stream_args(rng, q0, seed, normals, log_uniforms, dict(uniforms=injected_uniforms),
                              lambda: _draw_rmhmc_reference_stream(D, num_samples, L, jitter, explicit, q0.device))
        return engine.rmhmc_run(log_prob_func, q0, num_samples, L, step_size, burn=burn, jitter=jitter,
                                softabs_const=softabs_const, explicit_binding_const=explicit_binding_const,
                                fixed_point_threshold=fixed_point_threshold,
                                fixed_point_max_iterations=fixed_point_max_iterations,
                                jitter_max_tries=jitter_max_tries, explicit=explicit,
                                softabs=(metric == Metric.SOFTABS), jacdiag=jacdiag, chain_offset=chain_offset,
                                record_ham=record_ham, **stream)

    num_perm = len(log_prob_func) if integrator == Integrator.SPLITTING_RAND else 0

    def draw_reference():
        drawn = _draw_reference_stream(D, num_samples, q0.device, num_perm, gamma_shapes=gshapes,
                                       blocks=[b.shape[0] for b in inv_mass] if isinstance(inv_mass, list) else None)
        return dict(normals=drawn[0].unsqueeze(1), log_uniforms=drawn[1].unsqueeze(1),
                    perms=drawn[2].unsqueeze(1) if num_perm else None,
                    gammas=drawn[-1].unsqueeze(1) if hyper is not None else None)

    stream = _stream_args(rng, q0, seed, normals, log_uniforms,
                          dict(perms=injected_perms if integrator in _SPLIT_INTEGRATORS else None, gammas=gammas),
                          draw_reference)
    return engine.hmc_run(log_prob_func, q0, num_samples, L, step_size, burn=burn, inv_mass=inv_mass, nuts=nuts,
                          desired_accept_rate=desired_accept_rate, chain_offset=chain_offset, record_ham=record_ham,
                          out=out, scheme=scheme, **stream, **hyper_kw, **sink)


# ----------------------------------------------------------------------------------------------------------
# Bayesian neural networks: define_model_log_prob / sample_model / sample_split_model / predict_model
# ----------------------------------------------------------------------------------------------------------
def _check_loss(model_loss):
    if callable(model_loss) or model_loss not in T.LOSS_ID:
        raise NotImplementedError(
            "hamiltorch_b200: model_loss must be one of %s -- a callable loss (samplers.py:1186-1188) cannot enter a "
            "CUDA kernel and there is no CPU fallback; got %r" % (sorted(T.LOSS_ID), model_loss))


def define_model_log_prob(model, model_loss, x, y, params_flattened_list, params_shape_list, tau_list, tau_out,
                          normalizing_const=1., predict=False, prior_scale=1.0, device='cpu'):
    """samplers.py:1093-1201.  Returns the log_prob_func of a dense-stack model as a NATIVE descriptor
    (``targets.MLPRegression``): callable like the reference's closure (same torch ops, same (O,)-shaped value, the
    ``(log_prob, output)`` pair when ``predict``) and understood by the kernels."""
    _check_loss(model_loss)
    desc = T.MLPTarget.from_model(model, x, y, tau_list, tau_out, prior_scale, model_loss)
    if list(params_flattened_list) != desc.sizes:
        raise RuntimeError('params_flattened_list does not match the model')
    desc.predict_mode = bool(predict)
    return desc


def define_split_model_log_prob(model, model_loss, train_loader, num_splits, params_flattened_list, params_shape_list,
                                tau_list, tau_out, normalizing_const=1., predict=False, device='cpu', verbose=True):
    """samplers.py:1203-1258: one descriptor per DataLoader batch (the first ``num_splits`` batches), the prior divided
    by ``num_splits`` (:1254)."""
    log_prob_list = []
    for batch_idx, (data, target) in enumerate(train_loader):
        if batch_idx > num_splits - 1:
            break
        log_prob_list.append(define_model_log_prob(model, model_loss, data.clone().to('cpu'), target.clone().to('cpu'),
                                                   params_flattened_list, params_shape_list, tau_list, tau_out,
                                                   normalizing_const=normalizing_const, prior_scale=num_splits,
                                                   predict=predict, device=device))
    if verbose:
        print('Number of splits: ', len(log_prob_list), ' , each of batch size ', train_loader.batch_size, '\n')
    return log_prob_list


def _model_lists(model, tau_list):
    params_shape_list, params_flattened_list = [], []
    build_tau = tau_list is None
    if build_tau:
        tau_list = []
    for weights in model.parameters():                                                   # :1351-1355
        params_shape_list.append(weights.shape)
        params_flattened_list.append(weights.nelement())
        if build_tau:
            tau_list.append(torch.tensor(1.))
    return params_shape_list, params_flattened_list, tau_list


def sample_model(model, x, y, params_init, model_loss='multi_class_linear_output', num_samples=10,
                 num_steps_per_sample=10, step_size=0.1, burn=0, inv_mass=None, jitter=None, normalizing_const=1.,
                 softabs_const=None, explicit_binding_const=100, fixed_point_threshold=1e-5,
                 fixed_point_max_iterations=1000, jitter_max_tries=10, sampler=Sampler.HMC,
                 integrator=Integrator.IMPLICIT, metric=Metric.HESSIAN, debug=False, tau_out=1., tau_list=None,
                 store_on_GPU=True, desired_accept_rate=0.8, verbose=True, **engine_kwargs):
    """samplers.py:1261-1362: build the model's log_prob_func and delegate to ``sample``."""
    shapes, flat, tau_list = _model_lists(model, tau_list)
    log_prob_func = define_model_log_prob(model, model_loss, x, y, flat, shapes, tau_list, tau_out,
                                          normalizing_const=normalizing_const, device=params_init.device)
    return sample(log_prob_func, params_init, num_samples=num_samples, num_steps_per_sample=num_steps_per_sample,
                  step_size=step_size, burn=burn, jitter=jitter, inv_mass=inv_mass, normalizing_const=normalizing_const,
                  softabs_const=softabs_const, explicit_binding_const=explicit_binding_const,
                  fixed_point_threshold=fixed_point_threshold, fixed_point_max_iterations=fixed_point_max_iterations,
                  jitter_max_tries=jitter_max_tries, sampler=sampler, integrator=integrator, metric=metric, debug=debug,
                  desired_accept_rate=desired_accept_rate, store_on_GPU=store_on_GPU, verbose=verbose, **engine_kwargs)


def sample_split_model(model, train_loader, params_init, num_splits, model_loss='multi_class_linear_output',
                       num_samples=10, num_steps_per_sample=10, step_size=0.1, burn=0, inv_mass=None, jitter=None,
                       normalizing_const=1., softabs_const=None, explicit_binding_const=100,
                       fixed_point_threshold=1e-5, fixed_point_max_iterations=1000, jitter_max_tries=10,
                       sampler=Sampler.HMC, integrator=Integrator.SPLITTING, metric=Metric.HESSIAN, debug=False,
                       tau_out=1., tau_list=None, store_on_GPU=True, desired_accept_rate=0.8, verbose=True,
                       **engine_kwargs):
    """samplers.py:1364-1466: the first ``num_splits`` batches of ``train_loader`` become the data splits."""
    shapes, flat, tau_list = _model_lists(model, tau_list)
    log_prob_func = define_split_model_log_prob(model, model_loss, train_loader, num_splits, flat, shapes, tau_list,
                                                tau_out, normalizing_const=1., predict=False,
                                                device=params_init.device, verbose=verbose)
    return sample(log_prob_func, params_init, num_samples=num_samples, num_steps_per_sample=num_steps_per_sample,
                  step_size=step_size, burn=burn, jitter=jitter, inv_mass=inv_mass, normalizing_const=normalizing_const,
                  softabs_const=softabs_const, explicit_binding_const=explicit_binding_const,
                  fixed_point_threshold=fixed_point_threshold, fixed_point_max_iterations=fixed_point_max_iterations,
                  jitter_max_tries=jitter_max_tries, sampler=sampler, integrator=integrator, metric=metric, debug=debug,
                  desired_accept_rate=desired_accept_rate, store_on_GPU=store_on_GPU, verbose=verbose, **engine_kwargs)


def predict_model(model, samples, x=None, y=None, test_loader=None, model_loss='multi_class_linear_output', tau_out=1.,
                  tau_list=None, verbose=False):
    """samplers.py:1468-1562: network outputs of every sample as a (S, N, O) tensor + the list of S log-probs, from ONE
    launch (one CTA per sample).  With a DataLoader the batches are the splits and, like the reference (:1527), the
    prior is divided by the number of batches."""
    with torch.no_grad():
        shapes, flat, tau_list = _model_lists(model, tau_list)
        if test_loader.__class__ is torch.utils.data.dataloader.DataLoader:
            if len(test_loader.dataset) % test_loader.batch_size == 0.0:
                num_batches = len(test_loader.dataset) / test_loader.batch_size
            else:
                num_batches = int(round(len(test_loader.dataset) / test_loader.batch_size) + 1)
            target = define_split_model_log_prob(model, model_loss, test_loader, num_batches, flat, shapes, tau_list,
                                                 tau_out, normalizing_const=1., predict=True,
                                                 device=samples[0].device, verbose=verbose)
        elif x is not None and y is not None:
            if x.device != samples[0].device:
                raise RuntimeError('x on device: {} and samples on device: {}'.format(x.device, samples[0].device))
            target = define_model_log_prob(model, model_loss, x, y, flat, shapes, tau_list, tau_out, predict=True,
                                           device=samples[0].device)
        else:
            raise RuntimeError('Val data not defined (i.e. arguments x, y, val_loader are all not defined)')
        dev = samples[0].device
        stacked = torch.stack(list(samples))
        cap = N.MLP_MAX_SPLITS
        if isinstance(target, list) and len(target) > cap:
            # a loader with more batches than one launch takes splits (e.g. a 10k test set at batch_size 100): launches of
            # `cap` batches each, predictions concatenated in batch order, log-probs added (the reference's loop :1532-:1537)
            preds, lp = [], None
            for i in range(0, len(target), cap):
                pr, l = engine.mlp_predict(target[i:i + cap], stacked)
                preds.append(pr)
                lp = l if lp is None else lp + l
            pred = torch.cat(preds, dim=1)
        else:
            pred, lp = engine.mlp_predict(target, stacked)
        pred, lp = pred.to(dev), lp.to(dev)
    shape = (1,) if model_loss == 'regression' else ()          # the reference's closure: (O,) vs 0-d (SURVEY 8a)
    return pred, [l.reshape(shape) for l in lp.unbind(0)]
