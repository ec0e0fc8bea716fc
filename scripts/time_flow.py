"""Device time of the persistent small-D flow kernel (hmcx_flow.cu) against the step-synchronous tcgen05 path it replaces
at D <= 128 (HMCX_FLOW_SMALL=0), and the chains-per-warp sweep (HMCX_FLOW_R).
    python scripts/time_flow.py > gpurun_out/time_flow.txt"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import hamiltorch_b200 as hb                                  # noqa: E402
from hamiltorch_b200 import targets as T                      # noqa: E402


def timed(f, reps=3):
    f()
    torch.cuda.synchronize()
    best = 1e30
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        r = f()
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1))
    return best, r


def spd(D, seed):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(D, D, generator=g, dtype=torch.float64) / D ** 0.5
    return A @ A.t() + 0.5 * torch.eye(D, dtype=torch.float64)


def run(kind, C, D, S, L):
    tgt = T.GaussianFull(torch.zeros(D), cov=spd(D, 3))
    init = torch.randn(C, D, generator=torch.Generator().manual_seed(5)).cuda() * 0.5
    if kind == 'rmhmc_explicit':
        f = lambda: hb.sample_chains(tgt, init, num_samples=S, num_steps_per_sample=L, step_size=0.1, sampler=hb.Sampler.RMHMC,
                                     integrator=hb.Integrator.EXPLICIT, metric=hb.Metric.HESSIAN, explicit_binding_const=10,
                                     rng='philox', seed=5)
        mv = 6 * L + 4
    elif kind == 'fullmass_hmc':
        im = spd(D, 4).float()
        f = lambda: hb.sample_chains(tgt, init, num_samples=S, num_steps_per_sample=L, step_size=0.1, inv_mass=im, rng='philox', seed=5)
        mv = 2 * L + 6
    else:
        f = lambda: hb.sample_chains(tgt, init, num_samples=S, num_steps_per_sample=L, step_size=0.1, rng='philox', seed=5)
        mv = L + 3
    ms, r = timed(f)
    return ms, r, mv


def main():
    quick = 'quick' in sys.argv
    shapes = [('rmhmc_explicit', 512, 64, 200, 10), ('rmhmc_explicit', 512, 128, 100, 10), ('rmhmc_explicit', 8192, 64, 50, 10),
              ('fullmass_hmc', 512, 64, 200, 10), ('dense_target_hmc', 512, 64, 200, 10), ('fullmass_hmc', 4096, 128, 50, 10)]
    for kind, C, D, S, L in shapes:
        for env in ([('1', None), ('1', '1'), ('1', '2'), ('1', '4'), ('0', None)] if not quick else [('1', None), ('0', None)]):
            os.environ['HMCX_FLOW_SMALL'] = env[0]
            os.environ.pop('HMCX_FLOW_R', None)
            if env[1]:
                os.environ['HMCX_FLOW_R'] = env[1]
            if env[0] == '0' and C * S > 200000:
                S_ = max(4, S // 10)
            else:
                S_ = S
            ms, r, mv = run(kind, C, D, S_, L)
            cs = C * S_ * L / (ms * 1e-3)
            # shared-memory roofline of the flow kernel: every warp-matvec streams D*D*4 bytes; 128 B/clk/SM * #SMs
            print('%-18s C=%5d D=%3d S=%3d L=%d  %-9s R=%-4s %9.3f ms  %.3g chain-steps/s  accept %.2f  matvecs/iter %d'
                  % (kind, C, D, S_, L, 'flow' if env[0] == '1' else 'gemm', env[1] or 'auto', ms, cs,
                     float(r.accepted.float().mean()), mv), flush=True)


if __name__ == '__main__':
    main()
