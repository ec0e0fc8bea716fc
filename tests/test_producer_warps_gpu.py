"""GPU: the producer form of the paired config-2 loop (hmc_run_kernel<..., PW=2>: two producer warps draw every
iteration's momentum, kinetic sums and log-uniform into a shared-memory slot) against one float4 per thread (tuning=1),
bit for bit: accept decisions, Hamiltonians, samples and reject counts.  The cases reach the first and last hand-over
of the slot (S = 1, 2), more than one log-uniform batch (S = 33), odd and even step counts, the :1018 restore (burn-in at
acceptance ~0.5), padding (D = 1000, 800: virtual warps and producer lanes that are all padding), an odd chain count,
runs cut into host windows (the producers start at each window's first iteration) and every target / mass pair against
the injected-stream twin.

elem_hmc_run takes the producer form for at most 2 chains per SM and the plain paired form (PW = 0) above that, so the
chain counts derive from the device's SM count (256 / 255 on a 132-SM H100), and the plain paired form is pinned the
same way at 2 x SM count + 1 chains."""
import pytest
import torch

from hamiltorch_b200 import engine, targets as T, _native as N
from tests.launched import ran as _ran
from tests.test_philox_stream_gpu import OFFSETS, SEEDS, _elem, _init, _philox_vs_injected

pytestmark = pytest.mark.gpu

PRODUCER_KERNEL = ', 4, 2, 128, false, true, 1, false, 2>'
PLAIN_PAIRED_KERNEL = ', 4, 2, 128, false, true, 1, false, 0>'


def _dev():
    return torch.device('cuda', torch.cuda.current_device())


def _sms():
    return torch.cuda.get_device_properties(_dev()).multi_processor_count


def _producer_chains():
    """the largest chain count (at most 256) that runs the producer form"""
    return min(256, 2 * _sms())


def _run_both(tgt, init, S, L, eps, kernel=PRODUCER_KERNEL, **kw):
    """(default run, tuning=1 run); asserts that the default run launched `kernel`"""
    kw = dict(seed=17, record_ham=True, device=_dev(), **kw)
    auto = _ran(kernel, lambda: engine.hmc_run(tgt, init, S, L, eps, **kw))
    one = engine.hmc_run(tgt, init, S, L, eps, tuning=1, **kw)
    torch.cuda.synchronize()
    return auto, one


def _assert_same(auto, one):
    assert torch.equal(auto.accepted, one.accepted)
    assert torch.equal(auto.ham.view(torch.int32), one.ham.view(torch.int32))
    assert torch.equal(auto.samples, one.samples)
    assert torch.equal(auto.num_rejected, one.num_rejected)


@pytest.mark.parametrize('fewer', [0, 1])
@pytest.mark.parametrize('D', [1024, 1000, 800])
@pytest.mark.parametrize('eps,init_scale,burn', [(0.05, 0.1, 1), (0.42, 1.0, 4)])
def test_producer_form_equals_one_group_per_thread(D, fewer, eps, init_scale, burn):
    C = _producer_chains() - fewer
    init = init_scale * torch.randn(C, D, generator=torch.Generator().manual_seed(D + C))
    auto, one = _run_both(T.GaussianIso(D), init, 120, 10, eps, burn=burn)
    rate = float(auto.accepted.float().mean())
    assert (rate > 0.97) if eps < 0.1 else (0.2 < rate < 0.9), rate
    _assert_same(auto, one)


@pytest.mark.parametrize('S', [1, 2, 33])
@pytest.mark.parametrize('L', [1, 4, 10])
def test_producer_form_trip_and_ring_counts(L, S):
    D, C = 1024, _producer_chains()
    init = torch.randn(C, D, generator=torch.Generator().manual_seed(L * 100 + S))
    auto, one = _run_both(T.GaussianIso(D), init, S, L, 0.3)
    _assert_same(auto, one)


def test_producer_form_host_windows_equal_one_launch():
    D, C, S, burn = 1024, _producer_chains(), 33, 2
    init = torch.randn(C, D, generator=torch.Generator().manual_seed(5))
    kw = dict(burn=burn, seed=3, record_ham=True, device=_dev())
    single = _ran(PRODUCER_KERNEL, lambda: engine.hmc_run(T.GaussianIso(D), init, S, 10, 0.4, **kw))
    out = torch.empty((C, S - burn, N.padded_ld(D)), dtype=torch.float32, pin_memory=True)
    win = engine.hmc_run(T.GaussianIso(D), init, S, 10, 0.4, host_windows=3, out=out, **kw)
    torch.cuda.synchronize()
    assert 0.2 < float(single.accepted.float().mean()) < 0.95
    assert torch.equal(win.accepted.cpu(), single.accepted.cpu())
    assert torch.equal(win.ham.cpu().view(torch.int32), single.ham.cpu().view(torch.int32))
    assert torch.equal(win.samples.cpu(), single.samples.cpu())
    assert torch.equal(win.num_rejected.cpu(), single.num_rejected.cpu())


@pytest.mark.parametrize('plain', [False, True])
@pytest.mark.parametrize('tk,mk', [('iso', 'none'), ('iso', 'diag'), ('diag', 'none'), ('diag', 'diag')])
def test_paired_forms_equal_injected_stream(tk, mk, plain):
    D, S, L, burn = 1000, 12, 4, 3
    C = 2 * _sms() + 1 if plain else _producer_chains()
    i = ['none', 'diag'].index(mk) + 2 * ['iso', 'diag'].index(tk)
    tgt, im = _elem(tk, mk, D, 40 + i)
    q0 = _init(C, D, 40 + i, mean=None if tk == 'iso' else tgt.mean)
    eps = 0.9 * D ** -0.25

    def run(**rng):
        fn = lambda: engine.hmc_run(tgt, q0, S, L, eps, burn=burn, inv_mass=im, record_ham=True, **rng)
        return _ran(PLAIN_PAIRED_KERNEL if plain else PRODUCER_KERNEL, fn) if 'seed' in rng else fn()
    _philox_vs_injected(run, SEEDS[i % 3], OFFSETS[(i + 1) % 3], C, S, D)


@pytest.mark.parametrize('D,eps,init_scale,burn', [(1024, 0.05, 0.1, 1), (1024, 0.42, 1.0, 4), (800, 0.45, 1.0, 3)])
def test_plain_paired_form_above_two_chains_per_sm(D, eps, init_scale, burn):
    C = 2 * _sms() + 1
    init = init_scale * torch.randn(C, D, generator=torch.Generator().manual_seed(D + 1))
    auto, one = _run_both(T.GaussianIso(D), init, 120, 10, eps, kernel=PLAIN_PAIRED_KERNEL, burn=burn)
    rate = float(auto.accepted.float().mean())
    assert (rate > 0.97) if eps < 0.1 else (0.2 < rate < 0.9), rate
    _assert_same(auto, one)
