"""GPU: the coupled-target HMC kernels against the fp64 replay of tests/dense_ref.py.

  hmc_small_kernel<DM>      one thread per chain (hmcx_rmhmc.cu), every coupled run with D <= 16: GaussianFull, Neal's
                            funnel, and any target with a 2-D or block-list inv_mass.  Every width: DM = 2 (D = 2),
                            6 (D = 1, 3, 6), 16 (D = 7, 16); every target x mass combination the kernel serves; C = 300
                            (three 128-thread CTAs, 44 live threads in the last).  Injected streams, per-chain step sizes,
                            burn = 2 and forced rejects (log u > 0), one of them at n = burn + 1 after an accepted
                            warm-up (the :1018 quirk: the state returns to params_init).  NUTS teacher-forced through
                            eps_schedule, a diverging chain inside the batch, and windows of iterations through the C ABI.
  coupled_leapfrog_kernel   the stand-alone leapfrog / hamiltonian for coupled targets (hmcx_coupled.cu, one 256-thread
  coupled_hamiltonian_kernel  CTA per chain, the state in shared memory): per-step q and p and H at D up to 4099 (block
                            sums over several strides), the funnel up to the leapfrog's 200 KiB shared-memory limit
                            D = 12 800, and the refusal one past it.

Hamiltonians, proposals and trajectory states are held to 2e-4 under the measured tolerances of
tests/golden/measured_errors.json (coupled_ref/...).
"""
import ctypes as C

import pytest
import torch

from hamiltorch_b200 import engine, targets as T, _native as N
from tests import dense_ref, parity

pytestmark = pytest.mark.gpu
CEIL = 2e-4
NUTS_EPS0 = 0.2


# ---- problems ----------------------------------------------------------------------------------------------------------
def _spd(D, seed, shift, device='cpu'):
    """A A^T / D + shift I in fp64 (on `device`: the large ones are built on the GPU)."""
    g = torch.Generator(device=device).manual_seed(seed)
    A = torch.randn(D, D, generator=g, dtype=torch.float64, device=device) / D ** 0.5
    return A @ A.t() + shift * torch.eye(D, dtype=torch.float64, device=device)


def _target(kind, D, seed, device='cpu'):
    g = torch.Generator().manual_seed(seed)
    if kind == 'funnel':
        return T.Funnel(D)
    if kind == 'full':
        return T.GaussianFull(0.3 * torch.randn(D, generator=g), prec=_spd(D, seed, 0.5, device))
    if kind == 'diag':
        return T.GaussianDiag(torch.linspace(-1, 1, D), 0.5 + torch.rand(D, generator=g))
    return T.GaussianIso(D)


def _mass(kind, D, seed, device='cpu'):
    if kind == 'diag':
        return 0.5 + torch.rand(D, generator=torch.Generator().manual_seed(seed))
    if kind == 'full':
        return _spd(D, seed, 0.7, device).float()
    if kind == 'blocks':                       # up to three blocks, the last the largest when 3 does not divide D
        sizes = [n for n in (D // 3, D // 3, D - 2 * (D // 3)) if n]
        return [_spd(n, seed + i, 0.7).float() for i, n in enumerate(sizes)]
    return None


def _init(tgt, C, g):
    D = tgt.dim
    if isinstance(tgt, T.Funnel):            # v = O(1): fp32 can follow fp64 through the neck
        return torch.cat([0.3 * torch.randn(C, 1, generator=g), 0.6 * torch.randn(C, D - 1, generator=g)], 1)
    mean = getattr(tgt, 'mean', torch.zeros(D))
    return mean[None] + 0.3 * torch.randn(C, D, generator=g)


def _bits(t):
    t = t.detach().contiguous()
    if t.dtype == torch.float32:
        return t.view(torch.int32)
    return t.view(torch.int64) if t.dtype == torch.float64 else t


OUTPUTS = ('samples_padded', 'accepted', 'diverged', 'ham', 'num_rejected', 'final_state', 'step_size', 'eps_trace',
           'h_bar', 'eps_bar')


def _assert_same_bytes(a, b, what, chains=None):
    for k in OUTPUTS:
        x, y = getattr(a, k, None), getattr(b, k, None)
        assert (x is None) == (y is None), (what, k)
        if x is not None:
            if chains is not None:
                x, y = x[chains], y[chains]
            assert torch.equal(_bits(x), _bits(y)), '%s: %s differs' % (what, k)


# ---- hmc_small_kernel ----------------------------------------------------------------------------------------------------
# target_mass -> step size; every combination hmcx_hmc_run sends to the thread-per-chain kernel
MODES = {
    'full_none': 0.25, 'full_diag': 0.25, 'full_full': 0.2,
    'funnel_none': 0.12, 'funnel_diag': 0.12, 'funnel_full': 0.1,
    'iso_full': 0.25, 'iso_blocks': 0.25, 'diag_full': 0.2, 'diag_blocks': 0.2,
}
DS = (1, 2, 3, 6, 7, 16)                     # DM = 6, 2, 6, 6, 16, 16
C300, BURN = 300, 2


class _Run:
    """A mode at D: inputs of the injected stream with forced rejects, per-chain step sizes (a teacher-forced (S, C)
    schedule for NUTS), the replay model."""

    def __init__(self, mode, D, seed, nuts=False, S=8, L=5):
        tk, mk = mode.split('_')
        self.D, self.C, self.S, self.L, self.burn, self.nuts = D, C300, S, L, BURN, nuts
        self.tgt = _target(tk, D, seed)
        self.im = _mass(mk, D, seed + 1)
        g = torch.Generator().manual_seed(seed + 2)
        self.init = _init(self.tgt, self.C, g)
        self.z = torch.randn(S, self.C, D, generator=g)
        self.logu = torch.log(torch.rand(S, self.C, generator=g))
        self.logu[BURN + 1, ::7] = 1.0        # > 0 >= rho: rejects at n = burn + 1 (:1018), at burn and later on
        self.logu[BURN, 3::11] = 1.0
        self.logu[S - 2:, 5::13] = 1.0
        e0 = MODES[mode] * (0.5 if mk in ('full', 'blocks') and D >= 6 else 1.0)     # acceptance ~ 0.3 .. 0.9
        self.eps = e0 * (0.8 + 0.4 * torch.rand(self.C, generator=g))
        self.sched = None
        if nuts:
            self.sched = e0 * (0.8 + 0.4 * torch.rand(S, self.C, generator=g))
        self.model = dense_ref.HMC(self.tgt, self.im, device='cuda')

    def run(self, eps=None, sched=None):
        eps = self.eps if eps is None else eps
        sched = self.sched if sched is None else sched
        res = engine.hmc_run(self.tgt, self.init, self.S, self.L, NUTS_EPS0 if self.nuts else eps, burn=self.burn,
                             inv_mass=self.im, nuts=self.nuts, normals=self.z, log_uniforms=self.logu, record_ham=True,
                             eps_schedule=sched, record_eps=self.nuts)
        torch.cuda.synchronize()
        return res

    def check(self, tag, res, eps=None, sched=None):
        eps = (self.sched if sched is None else sched) if self.nuts else (self.eps if eps is None else eps)
        rep = dense_ref.replay(self.model, self.init, res.accepted, res.samples, self.z, eps, self.L, self.burn)
        dense_ref.check(tag, rep, self.init, res.samples, res.accepted, res.ham, self.logu, self.burn, ceiling=CEIL,
                        diverged=res.diverged)
        # the pad columns of every retained row (ld = 4 at D = 1, 2, 3; 8 at D = 6, 7) are exactly zero
        assert not bool(res.samples_padded[..., self.D:].any()), tag + ': pad columns written'
        if self.nuts:
            want = dense_ref.dual_averaging(res.ham, self.burn, NUTS_EPS0, diverged=res.diverged)
            got = res.eps_trace[:, :self.burn + 1].double().cpu()
            torch.testing.assert_close(got, want, rtol=2e-4, atol=0)


def _modes_at(D):
    return [(m, D) for m in sorted(MODES) if not (m.startswith('funnel') and D < 2)]


@pytest.mark.parametrize('mode,D', [md for D in DS for md in _modes_at(D)])
def test_small_kernel_vs_fp64_replay(mode, D):
    r = _Run(mode, D, seed=1000 * D + sorted(MODES).index(mode))
    res = r.run()
    assert int(res.diverged.sum()) == 0
    r.check('coupled_ref/%s_d%d' % (mode, D), res)
    acc = res.accepted.bool().cpu()
    assert 0 < int(acc.sum()) < r.C * r.S
    assert bool((res.num_rejected.cpu() == (~acc).sum(1)).all())
    # the :1018 quirk is reached: a forced reject at n = burn + 1 after an accepted warm-up iteration
    forced = torch.zeros(r.C, dtype=torch.bool)
    forced[::7] = True
    assert bool((forced & acc[:, :BURN + 1].any(1)).any())


NUTS_CASES = {'full_full_d6': ('full_full', 6), 'full_full_d2': ('full_full', 2), 'funnel_none_d16': ('funnel_none', 16),
              'funnel_full_d16': ('funnel_full', 16)}


@pytest.mark.parametrize('name', sorted(NUTS_CASES))
def test_small_kernel_nuts_vs_fp64_replay(name):
    """HMC_NUTS with the step size teacher-forced: replay of every iteration, and the kernel's own step-size proposals
    (eps_trace) against the dual averaging of its own Hamiltonians."""
    mode, D = NUTS_CASES[name]
    r = _Run(mode, D, seed=77 * D + len(name), nuts=True, S=10)
    res = r.run()
    assert int(res.diverged.sum()) == 0
    r.check('coupled_ref/nuts_' + name, res)
    assert 0 < int(res.accepted.sum()) < r.C * r.S


@pytest.mark.parametrize('nuts', [False, True])
def test_diverging_chain_stays_in_its_slot(nuts):
    """A funnel chain with a step size of 1e20 inside a C = 300 batch (the middle CTA): every iteration's log p is
    non-finite, flagged and rejected, its rows stay at params_init, and every other chain is byte-identical to the run
    without it.  With NUTS its dual averaging takes alpha = 0 at every warm-up iteration, n = burn included."""
    bad = 200
    r = _Run('funnel_full', 7, seed=4242, nuts=nuts)
    ok = r.run()
    if nuts:
        sched = r.sched.clone()
        sched[:, bad] = 1e20
        res, kw = r.run(sched=sched), dict(sched=sched)
    else:
        eps = r.eps.clone()
        eps[bad] = 1e20
        res, kw = r.run(eps=eps), dict(eps=eps)
    S = r.S
    assert bool(res.diverged[bad].bool().all()) and not bool(res.accepted[bad].bool().any())
    assert int(res.num_rejected[bad]) == S
    init = r.init[bad].cuda()
    assert torch.equal(res.samples[bad], init[None].expand_as(res.samples[bad]))
    assert torch.equal(res.final_state[bad], init)
    others = torch.tensor([c for c in range(r.C) if c != bad], device=res.accepted.device)
    _assert_same_bytes(ok, res, 'chains other than %d' % bad, chains=others)
    assert int(res.diverged[others].sum()) == 0
    r.check('coupled_ref/diverging_%s' % ('nuts' if nuts else 'hmc'), res, **kw)
    if nuts:
        assert float(res.eps_bar[bad].float()) == float(res.eps_trace[bad, r.burn])


# ---- windows of iterations through the C ABI ---------------------------------------------------------------------------
def _abi_windows(r, cuts, philox, nuts):
    """hmcx_hmc_run over the windows [cuts[k], cuts[k + 1]), chaining q_cur, eps and (NUTS) h_bar / eps_bar through their
    in/out buffers: an HMCResult-like namespace of every output."""
    lib = N.load_library()
    dev = torch.device('cuda')
    nt, nm = engine.native_target(r.tgt, dev), engine.native_mass(r.im, r.D, dev)
    D, Cn, S, L, burn = r.D, r.C, r.S, r.L, r.burn
    ld = N.padded_ld(D)
    q_init = N.pad_rows(r.init.cuda().contiguous(), ld)
    q_cur = q_init.clone()
    eps = torch.full((Cn,), NUTS_EPS0, device=dev) if nuts else r.eps.cuda().clone()
    samples = torch.full((Cn, S - burn, ld), float('nan'), device=dev)
    acc = torch.full((Cn, S), 7, dtype=torch.uint8, device=dev)
    div = torch.full_like(acc, 7)
    ham = torch.full((Cn, S, 2), float('nan'), device=dev)
    rej = torch.zeros(Cn, dtype=torch.int32, device=dev)
    z = N.pad_rows(r.z.cuda().contiguous(), ld)
    lu = r.logu.cuda().contiguous()
    ns = N.NutsStruct()
    out = dict(eps_trace=None, h_bar=None, eps_bar=None)
    if nuts:
        table = engine.nuts_table_device(burn, dev)
        out['h_bar'] = torch.zeros(Cn, dtype=torch.float64, device=dev)
        out['eps_bar'] = torch.ones(Cn, dtype=torch.float64, device=dev)
        out['eps_trace'] = torch.zeros((Cn, S), device=dev)
        ns.enabled, ns.desired_accept_rate, ns.mu = 1, 0.8, engine.nuts_mu(NUTS_EPS0)
        ns.table, ns.h_bar, ns.eps_bar = table.data_ptr(), out['h_bar'].data_ptr(), out['eps_bar'].data_ptr()
        ns.eps_trace = out['eps_trace'].data_ptr()
    for it0, it1 in zip(cuts[:-1], cuts[1:]):
        rng = N.RngStruct()
        if philox:
            rng.mode, rng.seed, rng.chain_offset = N.RNG_PHILOX, 0x9E3779B97F4A7C15, 7
        else:                                 # the injected streams are indexed from the window's first iteration
            rng.mode = N.RNG_INJECTED
            rng.normals, rng.log_uniforms = z.data_ptr() + it0 * Cn * ld * 4, lu.data_ptr() + it0 * Cn * 4
        rc = lib.hmcx_hmc_run(nt.ref(), nm.ref(), C.byref(rng), C.byref(ns), N.ptr(q_init), N.ptr(q_cur), N.ptr(eps),
                              Cn, ld, L, S, burn, it0, it1, N.ptr(samples), N.ptr(acc), N.ptr(div), N.ptr(ham),
                              N.ptr(rej), 0, None, N.stream_ptr(dev))
        N.check(rc, 'hmcx_hmc_run')
    torch.cuda.synchronize()

    class _Out:
        pass
    o = _Out()
    o.samples_padded, o.accepted, o.diverged, o.ham, o.num_rejected = samples, acc, div, ham, rej
    o.final_state, o.step_size = q_cur[:, :D], eps
    for k, v in out.items():
        setattr(o, k, v)
    return o


@pytest.mark.parametrize('a', [1, BURN, BURN + 1, BURN + 3])
@pytest.mark.parametrize('rng', ['injected', 'philox'])
@pytest.mark.parametrize('nuts', [False, True])
def test_two_abi_windows_equal_one_launch(a, rng, nuts):
    """[0, a) + [a, S) through hmcx_hmc_run equals one launch in every output, byte for byte: a <= burn splits the
    warm-up (eps, h_bar, eps_bar carried), a = burn + 1 starts the second window at the :1018 iteration."""
    r = _Run('funnel_full', 7, seed=700 + a)
    r.nuts = nuts
    kw = dict(seed=0x9E3779B97F4A7C15, chain_offset=7) if rng == 'philox' else dict(normals=r.z, log_uniforms=r.logu)
    one = engine.hmc_run(r.tgt, r.init, r.S, r.L, NUTS_EPS0 if nuts else r.eps, burn=r.burn, inv_mass=r.im, nuts=nuts,
                         record_ham=True, record_eps=nuts, **kw)
    two = _abi_windows(r, [0, a, r.S], rng == 'philox', nuts)
    _assert_same_bytes(one, two, 'windows [0, %d) + [%d, %d)' % (a, a, r.S))
    assert 0 < int(one.accepted.sum()) < r.C * r.S


# ---- the stand-alone coupled leapfrog and hamiltonian -------------------------------------------------------------------
STANDALONE = [(tm, D) for tm in ('full_none', 'full_diag', 'full_full', 'diag_full') for D in (1, 2, 33, 255, 257, 1000, 4099)]
STANDALONE += [(tm, D) for tm in ('funnel_none', 'funnel_diag', 'funnel_full') for D in (2, 257, 1000)]
STANDALONE += [('funnel_none', 12800)]
SMEM_LIMIT = 200 * 1024                       # bytes of dynamic shared memory hmcx_coupled.cu allows a CTA


def _standalone_problem(mode, D, Cn=3, L=4):
    tk, mk = mode.split('_')
    seed = D + 17 * len(mode)
    tgt = _target(tk, D, seed, device='cuda')
    im = _mass(mk, D, seed + 1, device='cuda')
    g = torch.Generator().manual_seed(seed + 2)
    if tk == 'funnel':                       # sum(x^2) ~ D - 1 balances 0.5 (D - 1) in grad v at v ~ 0: v stays O(1)
        q = torch.cat([0.3 * torch.randn(Cn, 1, generator=g), torch.randn(Cn, D - 1, generator=g)], 1)
    else:
        q = _init(tgt, Cn, g)
    p = torch.randn(Cn, D, generator=g)
    eps = (0.01 if tk == 'funnel' else 0.1) * (0.8 + 0.4 * torch.rand(Cn, generator=g))
    return tgt, im, q.cuda(), p.cuda(), eps.cuda(), L


def _check_hamiltonian(tag, model, tgt, im, q, p):
    H, flags = engine.hamiltonian(tgt, q, p, inv_mass=im)
    torch.cuda.synchronize()
    assert not bool(flags.any())
    want = model.hamiltonian(q.double(), p.double())
    parity.assert_close(tag + '/H', H.double().cpu().numpy(), want.cpu().numpy(), CEIL)


@pytest.mark.parametrize('mode,D', STANDALONE)
def test_standalone_leapfrog_and_hamiltonian_vs_fp64(mode, D):
    """engine.leapfrog(return_trajectory=True): q and p after every step (the full kick, with the half-kick correction
    of :302 on the last step only); its final state equals the last trajectory row; engine.hamiltonian and its flags."""
    tgt, im, q, p, eps, L = _standalone_problem(mode, D)
    assert 16 * D <= SMEM_LIMIT
    model = dense_ref.HMC(tgt, im, device='cuda')
    qs, ps = engine.leapfrog(tgt, q, p, L, eps, inv_mass=im, return_trajectory=True)
    qf, pf = engine.leapfrog(tgt, q, p, L, eps, inv_mass=im)
    torch.cuda.synchronize()
    assert torch.equal(_bits(qf), _bits(qs[-1].contiguous())) and torch.equal(_bits(pf), _bits(ps[-1].contiguous()))
    wq, wp = model.trajectory(q.double(), p.double(), eps.double(), L, per_step=True)
    tag = 'coupled_ref/standalone_%s_d%d' % (mode, D)
    parity.assert_close(tag + '/q', qs.double().cpu().numpy(), wq.cpu().numpy(), CEIL)
    parity.assert_close(tag + '/p', ps.double().cpu().numpy(), wp.cpu().numpy(), CEIL)
    _check_hamiltonian(tag, model, tgt, im, qf, pf)


def test_standalone_leapfrog_refused_past_its_shared_memory_limit():
    """D = 12 801: the leapfrog's 4 D floats exceed 200 KiB, so the call is refused; the hamiltonian (3 D floats, up to
    D = 17 066) still runs and matches fp64."""
    D = 12801
    assert 16 * D > SMEM_LIMIT >= 12 * D
    tgt, im, q, p, eps, L = _standalone_problem('funnel_none', D)
    with pytest.raises(N.NativeError):
        engine.leapfrog(tgt, q, p, L, eps, inv_mass=im)
    with pytest.raises(N.NativeError):
        engine.leapfrog(tgt, q, p, L, eps, inv_mass=im, return_trajectory=True)
    _check_hamiltonian('coupled_ref/standalone_funnel_none_d%d' % D, dense_ref.HMC(tgt, im, device='cuda'), tgt, im,
                       q, p)
