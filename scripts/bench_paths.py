"""Secondary measurements (not the driver's bench line): BASELINE configs 3, 4, 5 on one GPU, device-timed with CUDA
events, next to the oracle port (the reference's algorithm) on one host core for a bounded sample.
    python scripts/bench_paths.py [base] [dense] [sat] > paths.jsonl
"""
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import hamiltorch_b200 as hb                                    # noqa: E402
from hamiltorch_b200 import targets as T                        # noqa: E402
from oracle import cases, hmc_oracle as O, rmhmc_oracle as R    # noqa: E402


def timed(fn, reps=3):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        r = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps, r


def cfg5():
    C, D, S, L, burn = 128, 4096, 150, 10, 100                  # per-GPU share of the 1024-chain / 8-GPU config
    tgt = T.GaussianIso(D)
    init = 0.1 * torch.randn(C, D, generator=torch.Generator().manual_seed(0))
    ms, res = timed(lambda: hb.sample_chains(tgt, init.cuda(), num_samples=S, num_steps_per_sample=L, step_size=0.1,
                                             burn=burn, sampler=hb.Sampler.HMC_NUTS, rng='philox', seed=1))
    torch.manual_seed(0)
    t0 = time.perf_counter()
    O.sample_hmc(tgt, init[0], num_samples=40, num_steps_per_sample=L, step_size=0.1, burn=30, nuts=True)
    cpu = 40 * L / (time.perf_counter() - t0)
    return dict(config='5: D=4096 iso, HMC_NUTS, 128 chains/GPU, L=10, burn=100, S=150', ms=ms,
                chain_steps_per_s=C * S * L / (ms * 1e-3), cpu_port_1core_chain_steps_per_s=cpu,
                median_adapted_eps=float(res.step_size.median()),
                post_burn_accept=float(res.accepted[:, burn + 1:].float().mean()))


def cfg4(C=64):
    model, x, y = cases.mlp_problem(seed=0, n=1024, n_in=64, hidden=128)
    M, S, L = 4, 30, 10
    descs = [T.MLPRegression.from_model(model, x[m * 256:(m + 1) * 256], y[m * 256:(m + 1) * 256], None, 100.,
                                        prior_scale=M) for m in range(M)]
    D = descs[0].dim
    init = hb.util.flatten(model).detach()[None] + 0.01 * torch.randn(C, D, generator=torch.Generator().manual_seed(0))
    ms, res = timed(lambda: hb.sample_chains(descs, init.cuda(), num_samples=S, num_steps_per_sample=L, step_size=5e-4,
                                             inv_mass=torch.ones(D), integrator=hb.Integrator.SPLITTING,
                                             rng='philox', seed=3), reps=2)
    torch.manual_seed(0)
    t0 = time.perf_counter()
    O.sample_hmc(descs, init[0], num_samples=3, num_steps_per_sample=L, step_size=5e-4, inv_mass=torch.ones(D),
                 split_scheme=O.SPLIT_SYM)
    cpu = 3 * L / (time.perf_counter() - t0)
    flops = 68.7e6 * C * S * L                                   # SURVEY 8d: 68.7 MFLOP per chain-step
    # tensor roofline of the 3xTF32 path: tf32 runs at half the bf16 rate and every product costs three UMMAs
    try:
        peaks = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'MEASURED_PEAKS.json')))
        peak, src = peaks['bf16_tflops_sustained'] / 6.0, 'MEASURED_PEAKS.json bf16_tflops_sustained / 2 (tf32) / 3 (split)'
    except Exception:
        peak, src = 2250.0 / 6.0, 'nominal 2.25 PFLOP/s bf16 / 6'
    tf = flops / (ms * 1e-3) / 1e12
    roof = {'bound': 'tensor', 'achieved': tf, 'peak': peak, 'unit': 'TFLOP/s', 'frac': tf / peak, 'peak_source': src,
            'traffic': None}
    return dict(roofline=roof, config='4: MLP 64-128-1 (D=8449), N=1024, M=4 symmetric split, %d chains on ONE GPU, L=10, S=%d' % (C, S),
                ms=ms, chain_steps_per_s=C * S * L / (ms * 1e-3), achieved_tflops=flops / (ms * 1e-3) / 1e12,
                cpu_port_1core_chain_steps_per_s=cpu, accept=float(res.accepted.float().mean()))


def cfg3():
    C, S, L = 512, 200, 10
    tgt = T.Funnel(2)
    init = torch.tensor([0., 1.]).repeat(C, 1)
    kw = dict(num_samples=S, num_steps_per_sample=L, step_size=0.05, jitter=1e-3, softabs_const=1e6,
              explicit_binding_const=10)
    ms, res = timed(lambda: hb.sample_chains(tgt, init.cuda(), sampler=hb.Sampler.RMHMC,
                                             integrator=hb.Integrator.EXPLICIT, metric=hb.Metric.SOFTABS,
                                             rng='philox', seed=2, **kw))
    torch.distributions.Distribution.set_default_validate_args(False)
    torch.manual_seed(0)
    t0 = time.perf_counter()
    R.sample_rmhmc(tgt, init[0], num_samples=6, num_steps_per_sample=L, step_size=0.05, jitter=1e-3,
                   softabs_const=1e6, explicit_binding_const=10, integrator=R.EXPLICIT, metric=R.SOFTABS)
    cpu = 6 * L / (time.perf_counter() - t0)
    return dict(config='3: explicit RMHMC, 2-D funnel, softabs 1e6, omega=10, 512 chains, L=10, S=200', ms=ms,
                chain_steps_per_s=C * S * L / (ms * 1e-3), cpu_port_1core_chain_steps_per_s=cpu,
                accept=float(res.accepted.float().mean()))


def dense(C=256, D=1024, S=20, L=10):
    """Full-covariance Gaussian on the tcgen05 path: one GEMM (C x D) . (D x D) per leapfrog step."""
    g = torch.Generator().manual_seed(3)
    A = torch.randn(D, D, generator=g, dtype=torch.float64) / D ** 0.5
    cov = A @ A.t() + 0.5 * torch.eye(D, dtype=torch.float64)
    tgt = T.GaussianFull(torch.zeros(D), cov=cov)
    init = torch.randn(C, D, generator=g)
    ms, res = timed(lambda: hb.sample_chains(tgt, init.cuda(), num_samples=S, num_steps_per_sample=L, step_size=0.1,
                                             rng='philox', seed=5), reps=2)
    torch.manual_seed(0)
    t0 = time.perf_counter()
    O.sample_hmc(tgt, init[0], num_samples=5, num_steps_per_sample=L, step_size=0.1)
    cpu = 5 * L / (time.perf_counter() - t0)
    flops = 2.0 * C * D * D * (L + 1) * S                        # algorithmic: one (C x D)(D x D) product per gradient
    return dict(config='dense: GaussianFull D=%d, %d chains, L=%d, S=%d (tcgen05 3xTF32)' % (D, C, L, S), ms=ms,
                chain_steps_per_s=C * S * L / (ms * 1e-3), algorithmic_tflops=flops / (ms * 1e-3) / 1e12,
                cpu_port_1core_chain_steps_per_s=cpu, accept=float(res.accepted.float().mean()))


def _spd(D, seed):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(D, D, generator=g, dtype=torch.float64) / D ** 0.5
    return A @ A.t() + 0.5 * torch.eye(D, dtype=torch.float64)


def fullmass(C=256, D=1024, S=10, L=10, full_target=False):
    """2-D inv_mass at scale (samplers.py:199, :294, :812): momentum refresh, every drift and both kinetic energies as
    tcgen05 GEMMs; a GaussianFull target adds the gradient GEMM."""
    tgt = T.GaussianFull(torch.zeros(D), cov=_spd(D, 3)) if full_target else T.GaussianIso(D)
    im = _spd(D, 4).float()
    init = torch.randn(C, D, generator=torch.Generator().manual_seed(5))
    ms, res = timed(lambda: hb.sample_chains(tgt, init.cuda(), num_samples=S, num_steps_per_sample=L, step_size=0.1,
                                             inv_mass=im, rng='philox', seed=5), reps=2)
    torch.manual_seed(0)
    t0 = time.perf_counter()
    O.sample_hmc(tgt, init[0], num_samples=5, num_steps_per_sample=L, step_size=0.1, inv_mass=im)
    cpu = 5 * L / (time.perf_counter() - t0)
    gemms = (2 * L + 4) if full_target else (L + 3)
    flops = 2.0 * C * D * D * gemms * S
    return dict(config='full inv_mass: %s D=%d, %d chains, L=%d, S=%d (%d tcgen05 GEMMs per iteration)' % (
        type(tgt).__name__, D, C, L, S, gemms), ms=ms, chain_steps_per_s=C * S * L / (ms * 1e-3),
        algorithmic_tflops=flops / (ms * 1e-3) / 1e12, cpu_port_1core_chain_steps_per_s=cpu,
        accept=float(res.accepted.float().mean()))


def rmhmc_dense(C=512, D=64, S=20, L=10, cpu_iters=2):
    """SURVEY 8d: the 'D=64 Gaussian-Hessian variant' of config 3 (and larger D): explicit RMHMC with the constant
    metric G = P; 8 GEMMs per leapfrog step, the metric solve G^-1 p among them."""
    tgt = T.GaussianFull(torch.zeros(D), cov=_spd(D, 3))
    init = torch.randn(C, D, generator=torch.Generator().manual_seed(5))
    kw = dict(num_steps_per_sample=L, step_size=0.1, explicit_binding_const=10)
    ms, res = timed(lambda: hb.sample_chains(tgt, init.cuda(), num_samples=S, sampler=hb.Sampler.RMHMC,
                                             integrator=hb.Integrator.EXPLICIT, metric=hb.Metric.HESSIAN,
                                             rng='philox', seed=2, **kw), reps=2)
    cpu = None
    if cpu_iters:
        torch.manual_seed(0)
        t0 = time.perf_counter()
        R.sample_rmhmc(tgt, init[0], num_samples=cpu_iters, integrator=R.EXPLICIT, metric=R.HESSIAN, **kw)
        cpu = cpu_iters * L / (time.perf_counter() - t0)
    flops = 2.0 * C * D * D * (8 * L + 3) * S
    return dict(config='explicit RMHMC, GaussianFull D=%d (Hessian metric, jitter None), %d chains, L=%d, S=%d' % (D, C, L, S),
                ms=ms, chain_steps_per_s=C * S * L / (ms * 1e-3), algorithmic_tflops=flops / (ms * 1e-3) / 1e12,
                cpu_port_1core_chain_steps_per_s=cpu, accept=float(res.accepted.float().mean()))


def saturation():
    """SURVEY 8d saturation sweep of the persistent plain-HMC kernel: D=1024 isotropic Gaussian, C chains, L in {1, 10};
    S sized so that the retained samples stay below 8 GiB.  Rows with C=256 are BASELINE config 2's shape."""
    D, rows = 1024, []
    for C in (256, 1024, 4096, 16384, 65536):
        for L in (1, 10):
            S = max(8, min(1000, (8 << 30) // (C * D * 4)))
            out = torch.empty((C, S, D), dtype=torch.float32, device='cuda')
            init = torch.zeros(C, D, device='cuda')
            ms, res = timed(lambda: hb.sample_chains(T.GaussianIso(D), init, num_samples=S, num_steps_per_sample=L,
                                                     step_size=0.05, rng='philox', seed=1, out=out), reps=2)
            rows.append(dict(config='saturation: D=1024 iso, C=%d, L=%d, S=%d' % (C, L, S), ms=ms,
                             chain_steps_per_s=C * S * L / (ms * 1e-3),
                             sample_write_gbs=C * S * D * 4 / (ms * 1e-3) / 1e9,
                             streaming_equiv_gbs=C * S * L * 16 * D / (ms * 1e-3) / 1e9))
            del out
    return rows


if __name__ == '__main__':
    torch.set_num_threads(1)
    sel = set(sys.argv[1:]) or {'base'}
    if 'base' in sel:                       # BASELINE configs 5, 4, 3 (+ config 4's per-GPU share on 8 GPUs)
        for f in (cfg5, cfg4, cfg3):
            print(json.dumps(f()), flush=True)
        print(json.dumps(cfg4(C=8)), flush=True)
    if 'dense' in sel:                      # tensor-core paths for dense targets / mass matrices / constant metrics
        print(json.dumps(dense()), flush=True)
        print(json.dumps(fullmass()), flush=True)
        print(json.dumps(fullmass(full_target=True)), flush=True)
        print(json.dumps(rmhmc_dense()), flush=True)
        print(json.dumps(rmhmc_dense(C=1024, D=1024, S=4, cpu_iters=0)), flush=True)
    if 'sat' in sel:
        for r in saturation():
            print(json.dumps(r), flush=True)
