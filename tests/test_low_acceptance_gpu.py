"""GPU: the plain sample() loop of the persistent HMC kernel against the loop of the sink instantiation, bit for bit, at a
step size where about half of the iterations reject, so that accepts, rejects and the :1018 quirk all occur.  D=300 runs
a CTA of 3 warps (unused reduction slots) and a partial last float4 group (masked normals)."""
import pytest
import torch

import hamiltorch_b200 as hb
from hamiltorch_b200 import targets as T

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('D,C,windows', [(1024, 8, 0), (1024, 8, 5), (300, 6, 0)])
def test_plain_loop_equals_the_sink_loop_at_low_acceptance(D, C, windows):
    g = torch.Generator().manual_seed(11)
    tgt = T.GaussianIso(D)
    init = torch.randn(C, D, generator=g)
    kw = dict(num_samples=120, num_steps_per_sample=10, step_size=0.42 if D == 1024 else 0.5, burn=7, rng='philox',
              seed=5, record_ham=True)
    plain = hb.sample_chains(tgt, init, **kw)
    sink = hb.sample_chains(tgt, init, thin=1, moments=True, **kw)
    torch.cuda.synchronize()
    rate = float(plain.accepted.float().mean())
    assert 0.3 < rate < 0.8, rate
    assert bool((plain.accepted[:, 1:-1] == 0).any()) and bool((plain.accepted[:, 1:-1] == 1).any())
    assert torch.equal(plain.samples, sink.samples)
    assert torch.equal(plain.accepted, sink.accepted) and torch.equal(plain.ham, sink.ham)
    assert torch.equal(plain.num_rejected, sink.num_rejected) and torch.equal(plain.step_size, sink.step_size)
    if windows:
        S, ld = kw['num_samples'], plain.samples_padded.shape[-1]
        host = torch.full((C, S - kw['burn'], ld), float('nan')).pin_memory()
        win = hb.sample_chains(tgt, init, out=host, host_windows=windows, **kw)
        torch.cuda.synchronize()
        assert torch.equal(host, plain.samples_padded.cpu())
        assert torch.equal(win.accepted, plain.accepted) and torch.equal(win.ham, plain.ham)
