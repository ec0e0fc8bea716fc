"""Run ONE of BASELINE configs 3 / 4 / 5 (the same inputs as bench.py's other_configs) `reps` times and print the device
time per launch -- the command a profiler wraps for per-config captures.
    python scripts/run_cfg.py 3 [reps] [chains]"""
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import hamiltorch_b200 as hb                                  # noqa: E402
from hamiltorch_b200 import targets as T                      # noqa: E402


def main():
    cfg = int(sys.argv[1])
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    dev = torch.device('cuda', 0)
    g = torch.Generator().manual_seed(0)
    if cfg == 3:
        C = int(sys.argv[3]) if len(sys.argv) > 3 else 512
        S, L = 200, 10
        init = torch.tensor([0., 1.], device=dev).repeat(C, 1)
        run = lambda: hb.sample_chains(T.Funnel(2), init, num_samples=S, num_steps_per_sample=L, step_size=0.05, jitter=1e-3,
                                       softabs_const=1e6, explicit_binding_const=10, sampler=hb.Sampler.RMHMC,
                                       integrator=hb.Integrator.EXPLICIT, metric=hb.Metric.SOFTABS, rng='philox', seed=2)
    elif cfg == 4:
        import torch.nn as nn
        C = int(sys.argv[3]) if len(sys.argv) > 3 else 64
        S, L = int(os.environ.get('CFG4_S', '300')), 10
        X = torch.randn(1024, 64, generator=g)
        w = torch.randn(64, 1, generator=g)
        y = torch.sin(X @ w / 8) + 0.1 * torch.randn(1024, 1, generator=g)
        torch.manual_seed(0)
        model = nn.Sequential(nn.Linear(64, 128), nn.ReLU(), nn.Linear(128, 1))
        descs = [T.MLPRegression.from_model(model, X[m * 256:(m + 1) * 256], y[m * 256:(m + 1) * 256], None, 100.,
                                            prior_scale=4) for m in range(4)]
        D = descs[0].dim
        init = (hb.util.flatten(model).detach()[None] + 0.01 * torch.randn(C, D, generator=g)).to(dev)
        ones = torch.ones(D)
        run = lambda: hb.sample_chains(descs, init, num_samples=S, num_steps_per_sample=L, step_size=5e-4, inv_mass=ones,
                                       integrator=hb.Integrator.SPLITTING, rng='philox', seed=3)
    elif cfg == 5:
        C = int(sys.argv[3]) if len(sys.argv) > 3 else 128
        S, L = 150, 10
        init = (0.1 * torch.randn(C, 4096, generator=g)).to(dev)
        run = lambda: hb.sample_chains(T.GaussianIso(4096), init, num_samples=S, num_steps_per_sample=L, step_size=0.1,
                                       burn=100, sampler=hb.Sampler.HMC_NUTS, rng='philox', seed=1)
    else:
        raise SystemExit('config 3, 4 or 5')
    res = run()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        res = run()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ms = min(ts)
    print('config %d: C=%d S=%d L=%d  %.3f ms per launch (min of %d)  %.4g chain-steps/s  accept %.3f  diverged %.3f'
          % (cfg, C, S, L, ms, reps, C * S * L / (ms * 1e-3), float(res.accepted.float().mean()),
             float(res.diverged.float().mean())))


if __name__ == '__main__':
    main()
