"""GPU: the default geometry of the plain Philox sample() loop at BASELINE config-2 sizes (two float4 groups per thread in
CTAs of at most 128 threads) against one float4 per thread (tuning=1), bit for bit.  The paired form reduces every group
in the place it has in the one-group CTA, so accept decisions, Hamiltonians and samples must not change -- at
acceptance ~0.99 (config 2) and ~0.5 (chains started in the typical set, with burn-in so that the :1018 quirk occurs).
D=800 runs 4 warps standing for 8 (the last of them all padding) against a CTA of 7 warps.

The profiler confirms that the default run launched the paired form.  It keeps only the device records it can place
inside its host-side window, and late in a long GPU session a bare window has come back empty for a run that did
launch the kernel; so the check goes through tests/launched.py, which pads the window and retakes an empty trace."""
import pytest
import torch

from hamiltorch_b200 import engine, targets as T
from tests.launched import ran

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('D,eps,init_scale,burn', [(1024, 0.05, 0.1, 0), (1024, 0.42, 1.0, 4), (800, 0.45, 1.0, 3)])
def test_paired_geometry_equals_one_group_per_thread(D, eps, init_scale, burn):
    dev = torch.device('cuda', torch.cuda.current_device())
    C, S = 256, 120
    init = init_scale * torch.randn(C, D, generator=torch.Generator().manual_seed(D))
    kw = dict(burn=burn, seed=17, record_ham=True, device=dev)
    # the paired form (producer warps or not): the profiler window is padded and an empty trace retaken (tests/launched.py)
    auto = ran('hmc_run_kernel<0, 0, 4, 2, 128', lambda: engine.hmc_run(T.GaussianIso(D), init, S, 10, eps, **kw))
    one = engine.hmc_run(T.GaussianIso(D), init, S, 10, eps, tuning=1, **kw)
    torch.cuda.synchronize()
    rate = float(auto.accepted.float().mean())
    assert (rate > 0.97) if eps < 0.1 else (0.3 < rate < 0.8), rate
    assert torch.equal(auto.accepted, one.accepted)
    assert torch.equal(auto.ham, one.ham)
    assert torch.equal(auto.samples, one.samples)
    assert torch.equal(auto.num_rejected, one.num_rejected)
