"""GPU: the paired forms of the config-2 loop (producer warps and plain) against one float4 per thread (tuning=1), bit
for bit, at step counts whose last leapfrog step the step loop of trajectory_groups does or does not leave over
(L - 1 even: L = 2 has one peeled step and no trip, L = 3 and 5 end on a full trip; L - 1 odd: L = 6), for the
isotropic and the diagonal target: the final half-kick of both paths."""
import pytest
import torch

from hamiltorch_b200 import engine, targets as T
from tests.test_producer_warps_gpu import (PLAIN_PAIRED_KERNEL, PRODUCER_KERNEL, _assert_same, _producer_chains, _ran,
                                           _sms)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('plain', [False, True])
@pytest.mark.parametrize('diag', [False, True])
@pytest.mark.parametrize('L', [2, 3, 5, 6])
def test_paired_forms_step_counts_equal_one_group_per_thread(L, diag, plain):
    D, S, burn = 1000, 40, 3
    C = 2 * _sms() + 1 if plain else _producer_chains()
    g = torch.Generator().manual_seed(100 * L + 10 * diag + plain)
    if diag:
        tgt = T.GaussianDiag(torch.randn(D, generator=g), 0.5 + torch.rand(D, generator=g))
    else:
        tgt = T.GaussianIso(D)
    init = torch.randn(C, D, generator=g)
    dev = torch.device('cuda', torch.cuda.current_device())
    kw = dict(seed=29, burn=burn, record_ham=True, device=dev)
    auto = _ran(PLAIN_PAIRED_KERNEL if plain else PRODUCER_KERNEL, lambda: engine.hmc_run(tgt, init, S, L, 0.3, **kw))
    one = engine.hmc_run(tgt, init, S, L, 0.3, tuning=1, **kw)
    torch.cuda.synchronize()
    _assert_same(auto, one)
