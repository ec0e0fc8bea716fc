"""GPU: the element-wise persistent HMC loop (hmcx_hmc.cu, elem_hmc_run) against the per-iteration replays of
tests/dense_ref.py, in every form the dispatch reaches, for GaussianIso / GaussianDiag targets with inv_mass None or (D,).

  form                                  reached by                                       D
  <4,1,256> injected / Philox NUTS      default, ld <= 1024                              1, 3, 37, 513, 768, 1021
  <4,1,256> Philox, NUTS=false          default, ld <= 768                               1, 3, 37, 513, 768
  <4,2,128> plain paired (PW = 0)       Philox, 768 < ld <= 1024, C = 2 SMs + 1          769, 1000, 1024
  <4,2,128> producer (PW = 2)           the same, C <= 2 SMs (C = 1, P - 1, P)           769, 1000, 1024
  <4,1,1024> injected / Philox          default, 1024 < ld <= 2560 (block_sum3)          1025, 2047, 2560
  <4,2,512> injected / Philox           default, 2560 < ld <= 4096                       2561, 4093, 4096
  hmc_run_big_kernel                    ld > 4096, with the workspace                    4097, 9001
  tuning 2 / 4 / 21 / 22                tuning=                                          near each form's limit
  clusters of 4 / 2 CTAs (41 / 42)      tuning=                                          997, 4093 / 2045
  sink <4,1,256,true> / <4,1,1024,true> thin=1, moments=True (HMC and NUTS)              37, 2047

P = min(256, 2 SMs) is the producer form's largest batch; the chain counts derive from the device.  Every case asserts
the instantiation it ran (tests/launched.py) and checks, for every iteration of every chain:

1. the Hamiltonians against fp64 (dense_ref.check, ceiling 2e-4 under the measured tolerances of
   tests/golden/measured_errors.json, elem_ref/...), every decision that differs from fp64 within 4x the kernel's own
   Hamiltonian error, slot 0 = params_init and rejected rows repeating the previous one;
2. every accepted retained row against the fp32 replay (dense_ref.replay_rows32), bit for bit;
3. num_rejected, final_state = the last retained row, pad columns exactly zero; NUTS: the step sizes the kernel proposes
   during warm-up (eps_trace) against the fp64 dual averaging of its own Hamiltonians, under a teacher-forced schedule.

Injected runs force rejects (log u = +1) at n = burn (after a warm-up), n = burn + 1 (the :1018 restore to params_init)
and late in the run; Philox runs are replayed from the canonical stream (test_philox_stream_gpu._stream) and must reach
the restore in some chain.  After a restore, H_old at n = burn + 2 comes from the recomputed log p of params_init: it
is compared on its own (tag .../restore_h_old).  Beyond the table: runs cut into host windows (H_old at each window's
first iteration comes from the carried log p) and a diverging chain inside a producer-form and a <4,1,1024> batch.
"""
import numpy as np
import pytest
import torch

from hamiltorch_b200 import engine, targets as T, _native as N
from tests import dense_ref, parity
from tests.launched import ran
from tests.test_philox_stream_gpu import OFFSETS, SEEDS, _stream

pytestmark = pytest.mark.gpu
CEIL = 2e-4
NUTS_EPS0 = 0.2
S, L, BURN = 10, 4, 2
TKMK = [('iso', 'none'), ('iso', 'diag'), ('diag', 'none'), ('diag', 'diag')]
KIND = {'iso': 0, 'diag': 1, 'none': 0}          # HMCX_TARGET_GAUSS_ISO / _DIAG, HMCX_MASS_NONE / _DIAG


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _chains(spec):
    """'wide': 2 SMs + 1 (above the producer form's limit); 'P' / 'P-1': the producer form's largest batch and one less;
    or an int"""
    P = min(256, 2 * _sms())
    return {'wide': 2 * _sms() + 1, 'P': P, 'P-1': P - 1}.get(spec, spec)


def _kernel(form, tk, mk):
    """the instantiation name a form runs as: hmc_run_kernel<TK, MK, E, K, MAXT, SINK, PHILOX, CS, NUTS, PW>"""
    if form == 'big':
        return 'hmc_run_big_kernel<%d, %d>' % (KIND[tk], KIND[mk])
    return 'hmc_run_kernel<%d, %d, %s>' % (KIND[tk], KIND[mk], FORMS[form][0])


# form -> (instantiation tail, rng, nuts, extra hmc_run arguments)
FORMS = {
    'k1_256_injected': ('4, 1, 256, false, false, 1, true, 0', 'injected', False, {}),
    'k1_256_philox_nuts': ('4, 1, 256, false, true, 1, true, 0', 'philox', True, {}),
    'k1_256_philox': ('4, 1, 256, false, true, 1, false, 0', 'philox', False, {}),
    'paired': ('4, 2, 128, false, true, 1, false, 0', 'philox', False, {}),
    'producer': ('4, 2, 128, false, true, 1, false, 2', 'philox', False, {}),
    'k1_1024_injected': ('4, 1, 1024, false, false, 1, true, 0', 'injected', False, {}),
    'k1_1024_philox': ('4, 1, 1024, false, true, 1, true, 0', 'philox', False, {}),
    'k2_512_injected': ('4, 2, 512, false, false, 1, true, 0', 'injected', False, {}),
    'k2_512_philox': ('4, 2, 512, false, true, 1, true, 0', 'philox', False, {}),
    'big': (None, 'injected', False, {}),
    'tuning2': ('4, 2, 512, false, false, 1, true, 0', 'injected', False, dict(tuning=2)),
    'tuning4': ('4, 4, 256, false, false, 1, true, 0', 'injected', False, dict(tuning=4)),
    'tuning21': ('2, 1, 1024, false, false, 1, true, 0', 'injected', False, dict(tuning=21)),
    'tuning22': ('2, 2, 1024, false, false, 1, true, 0', 'injected', False, dict(tuning=22)),
    'cluster4': ('4, 1, 256, false, false, 4, true, 0', 'injected', False, dict(tuning=41)),
    'cluster4_philox': ('4, 1, 256, false, true, 4, true, 0', 'philox', False, dict(tuning=41)),
    'cluster2': ('4, 1, 256, false, false, 2, true, 0', 'injected', False, dict(tuning=42)),
    'cluster2_philox': ('4, 1, 256, false, true, 2, true, 0', 'philox', False, dict(tuning=42)),
    'sink_256': ('4, 1, 256, true, false, 1, true, 0', 'injected', False, dict(moments=True)),
    'sink_256_nuts': ('4, 1, 256, true, false, 1, true, 0', 'injected', True, dict(moments=True)),
    'sink_1024': ('4, 1, 1024, true, false, 1, true, 0', 'injected', False, dict(moments=True)),
    'sink_1024_nuts': ('4, 1, 1024, true, false, 1, true, 0', 'injected', True, dict(moments=True)),
}
# form -> [(D, chains)]
SHAPES = {
    'k1_256_injected': [(D, 'wide') for D in (1, 3, 37, 513, 768, 1021)],
    'k1_256_philox_nuts': [(D, 'wide') for D in (1, 3, 37, 513, 768, 1021)],
    'k1_256_philox': [(D, 'wide') for D in (1, 3, 37, 513, 768)],
    'paired': [(D, 'wide') for D in (769, 1000, 1024)],
    'producer': [(769, 1), (1000, 'P-1'), (1024, 'P')],
    'k1_1024_injected': [(D, 'wide') for D in (1025, 2047, 2560)],
    'k1_1024_philox': [(D, 'wide') for D in (1025, 2047, 2560)],
    'k2_512_injected': [(D, 'wide') for D in (2561, 4093, 4096)],
    'k2_512_philox': [(D, 'wide') for D in (2561, 4093, 4096)],
    'big': [(4097, 'wide'), (9001, 'wide')],
    'tuning2': [(4093, 'wide')],
    'tuning4': [(4093, 'wide')],
    'tuning21': [(2045, 'wide')],
    'tuning22': [(4093, 'wide')],
    'cluster4': [(997, 'wide'), (4093, 'wide')],
    'cluster4_philox': [(997, 'wide')],
    'cluster2': [(997, 'wide'), (2045, 'wide')],
    'cluster2_philox': [(997, 'wide')],
    'sink_256': [(37, 'wide')],
    'sink_256_nuts': [(37, 'wide')],
    'sink_1024': [(2047, 'wide')],
    'sink_1024_nuts': [(2047, 'wide')],
}
# forms whose restore (:1018) goes through their own reduction: block_sum1_groups (paired, producer), cluster_sum1
RESTORE_FORMS = ('paired', 'producer', 'cluster4', 'cluster4_philox', 'cluster2', 'cluster2_philox')


def _problem(tk, mk, D, seed):
    g = torch.Generator().manual_seed(seed)
    if tk == 'iso':
        tgt = T.GaussianIso(D)
    else:
        tgt = T.GaussianDiag(torch.linspace(-1, 1, D), 0.5 + torch.rand(D, generator=g))
    im = None if mk == 'none' else 0.5 + torch.rand(D, generator=g)
    return tgt, im, g


class _Run:
    """One case: the problem, its random stream (injected with forced rejects, or the canonical Philox stream), per-chain
    step sizes spread +-20 % around one that accepts ~0.6-0.9 (a teacher-forced (S, C) schedule for NUTS)."""

    def __init__(self, form, tk, mk, D, chains, seed):
        _, self.rng, self.nuts, kw = FORMS[form]
        self.form, self.D, self.C, self.kw = form, D, _chains(chains), dict(kw)
        self.tgt, self.im, g = _problem(tk, mk, D, seed)
        self.kernel = _kernel(form, tk, mk)
        C = self.C
        if tk == 'iso':                        # at the target's stationary distribution
            self.init = torch.randn(C, D, generator=g)
        else:
            self.init = self.tgt.mean + torch.randn(C, D, generator=g) / self.tgt.inv_var.sqrt()
        e0 = min(2.0 * D ** -0.25, 1.1) / (1.0 if (tk, mk) == ('iso', 'none') else 1.2)
        self.eps = e0 * (0.8 + 0.4 * torch.rand(C, generator=g))
        self.sched = e0 * (0.8 + 0.4 * torch.rand(S, C, generator=g)) if self.nuts else None
        if self.rng == 'injected':
            self.z = torch.randn(S, C, D, generator=g)
            self.logu = torch.log(torch.rand(S, C, generator=g))
            self.logu[BURN + 1, ::7] = 1.0     # > 0 >= rho: rejects at n = burn + 1 (:1018), at burn and late on
            self.logu[BURN, 3::11] = 1.0
            self.logu[S - 2:, 5::13] = 1.0
            self.stream = dict(normals=self.z, log_uniforms=self.logu)
        else:
            self.seed, self.offset = SEEDS[seed % 3], OFFSETS[seed % 3]
            s = _stream(self.seed, self.offset, C, S, D)
            self.z, self.logu = s['normals'], s['log_uniforms']
            self.stream = dict(seed=self.seed, chain_offset=self.offset)
        self.model = dense_ref.HMC(self.tgt, self.im, device='cuda')

    def run(self, eps=None, **extra):
        eps = self.eps if eps is None else eps
        kw = dict(self.kw, **extra)
        res = engine.hmc_run(self.tgt, self.init, S, L, NUTS_EPS0 if self.nuts else eps, burn=BURN, inv_mass=self.im,
                             nuts=self.nuts, record_ham=True, eps_schedule=self.sched, record_eps=self.nuts,
                             **self.stream, **kw)
        torch.cuda.synchronize()
        return res

    def check(self, tag, res, eps=None):
        """checks 1-3 of the module docstring; returns the number of chains whose state was restored at n = burn + 1"""
        eps = self.sched if self.nuts else (self.eps if eps is None else eps)
        D, C = self.D, self.C
        samples = res.samples_padded.cuda()
        rep = dense_ref.replay(self.model, self.init, res.accepted, samples[..., :D], self.z, eps, L, BURN)
        dense_ref.check(tag, rep, self.init, samples[..., :D], res.accepted, res.ham, self.logu, BURN, ceiling=CEIL,
                        diverged=res.diverged)
        n = dense_ref.replay_rows32(tag, self.tgt, self.im, self.init, res.accepted, samples, self.z, eps, L, BURN,
                                    mass_factor=None if self.im is None else engine.NativeMass(self.im, D, 'cuda')._keep['sd'])
        acc = res.accepted.bool()
        assert n == int(acc[:, BURN + 1:].sum()) > 0, tag + ': no accepted retained row'
        assert torch.equal(res.num_rejected.long(), (~acc).sum(1)), tag + ': num_rejected'
        assert torch.equal(res.final_state.view(torch.int32), samples[:, -1, :D].view(torch.int32)), tag + ': final_state'
        assert not bool(samples[..., D:].any()), tag + ': pad columns written'
        # the restore: a chain that moved during warm-up and rejects at n = burn + 1 is back at params_init; H_old of
        # n = burn + 2 is then H(params_init, p) from the recomputed log p
        div = res.diverged.bool()
        restored = acc[:, :BURN + 1].any(1) & ~acc[:, BURN + 1] & ~div[:, BURN + 2]
        if bool(restored.any()):
            parity.assert_close(tag + '/restore_h_old', res.ham[restored, BURN + 2, 0].double().cpu().numpy(),
                                rep.h_old[restored, BURN + 2].cpu().numpy(), CEIL)
        if self.nuts:
            want = dense_ref.dual_averaging(res.ham, BURN, NUTS_EPS0, diverged=res.diverged)
            got = res.eps_trace[:, :BURN + 1].double().cpu()
            torch.testing.assert_close(got, want, rtol=2e-4, atol=0)
        return int(restored.sum())


CASES = [(f, D, ch) for f in FORMS for D, ch in SHAPES[f]]


@pytest.mark.parametrize('tk,mk', TKMK)
@pytest.mark.parametrize('form,D,chains', CASES)
def test_elementwise_form_vs_replay(form, D, chains, tk, mk):
    seed = 1000 * CASES.index((form, D, chains)) + TKMK.index((tk, mk))
    r = _Run(form, tk, mk, D, chains, seed)
    res = ran(r.kernel, r.run)
    tag = 'elem_ref/%s_%s_%s_d%d' % (form, tk, mk, D)
    assert int(res.diverged.sum()) == 0
    restored = r.check(tag, res)
    rate = float(res.accepted.float().mean())
    assert 0.3 < rate < 0.99, (tag, rate)
    if r.C > 1:
        assert restored > 0, tag + ': no chain reached the :1018 restore'
    if form.startswith('sink'):           # the running moments of every post-burn iteration against fp64 sums
        rows = res.samples[:, 1:].double()
        parity.assert_close(tag + '/moment_sum', res.moment_sum.cpu().numpy(), rows.sum(1).cpu().numpy(), 1e-6)
        parity.assert_close(tag + '/moment_sumsq', res.moment_sumsq.cpu().numpy(), (rows * rows).sum(1).cpu().numpy(),
                            1e-6)


# ---- host windows: the carried log p at each window's first iteration ------------------------------------------------
WINDOWED = {'producer': (1000, 'P'), 'k1_1024_philox': (2047, 'wide')}


@pytest.mark.parametrize('tk,mk', TKMK)
@pytest.mark.parametrize('form', sorted(WINDOWED))
def test_host_windows_vs_replay(form, tk, mk):
    """host_windows=3 (a pinned `out`): three launches [0, 3), [3, 6), [6, 10) chained through q_cur and the carried
    log p.  The replay checks H_old at 3 (= burn + 1) and 6 like every other iteration."""
    D, chains = WINDOWED[form]
    r = _Run(form, tk, mk, D, chains, 77 + TKMK.index((tk, mk)))
    out = torch.empty((r.C, S - BURN, N.padded_ld(D)), dtype=torch.float32, pin_memory=True)
    res = ran(r.kernel, lambda: r.run(host_windows=3, out=out))
    assert not res.samples_padded.is_cuda
    assert int(res.diverged.sum()) == 0
    r.check('elem_ref/windows_%s_%s_%s_d%d' % (form, tk, mk, D), res)


# ---- a diverging chain inside the batch ---------------------------------------------------------------------------------
def _bits(t):
    return t.detach().contiguous().view(torch.int32) if t.dtype == torch.float32 else t


@pytest.mark.parametrize('form,D,chains', [('producer', 1000, 'P'), ('k1_1024_injected', 2047, 'wide')])
def test_diverging_chain_stays_in_its_slot(form, D, chains):
    """One chain's step size far beyond the leapfrog's stability limit: q overflows, log p is non-finite, and the
    kernel flags (diverged) and rejects every iteration of that chain (the reference's LogProbError).  Every other chain's
    bytes equal the run without it."""
    r = _Run(form, 'diag', 'diag', D, chains, 4242)
    bad = r.C // 2 + 1
    ok = r.run()
    eps = r.eps.clone()
    eps[bad] = 1e20
    res = ran(r.kernel, lambda: r.run(eps=eps))
    assert bool(res.diverged[bad].bool().all()) and not bool(res.accepted[bad].bool().any())
    assert int(res.num_rejected[bad]) == S
    init = r.init[bad].cuda()
    assert torch.equal(res.samples[bad], init[None].expand_as(res.samples[bad]))
    others = torch.tensor([c for c in range(r.C) if c != bad], device=res.accepted.device)
    for k in ('samples_padded', 'accepted', 'diverged', 'ham', 'num_rejected', 'final_state'):
        assert torch.equal(_bits(getattr(ok, k)[others]), _bits(getattr(res, k)[others])), k
    assert int(res.diverged[others].sum()) == 0
    r.check('elem_ref/diverging_%s_d%d' % (form, D), res, eps=eps)
