"""Cost of the hyperprior Gibbs steps at BASELINE config 4 (Linear(64,128)-ReLU-Linear(128,1), D = 8449, N = 1024 in
M = 4 splits, symmetric split HMC, 64 chains, L = 10, eps = 5e-4, S = 300).  Every variant keeps moments (moments=True),
so the plain run and the hyperprior runs differ by the hyperprior work and the kernel form only:
  plain       no hyperpriors (mlp_run_kernel<CS, false>)
  (the hyperprior variants run mlp_run_kernel<CS, true>, the chain's model constants in shared memory)
  pinned      hyperpriors so tight (a = 1e8, mean = the initial value) that the precisions stay at tau_list = 1,
              tau_out = 100 to ~1e-4: the same posterior as `plain`, so the difference is the cost of the Gibbs steps
              (2L fp64 reductions, the gamma draws, one forward pass, the lost carried gradient)
  free        tau_prior=(2, 1) on every tensor, tau_out_prior=(2, 0.02): the precisions move (another posterior)
alternated three times each after one warm-up run of each.  Prints the card, its power limit and device-event times per
run as JSON (also written to PATH with --json PATH).

    python scripts/time_hyper.py [--samples 300] [--chains 64] [--json PATH]
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import hamiltorch_b200 as hb                      # noqa: E402
from hamiltorch_b200 import targets as T          # noqa: E402


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in out.split(',')]
        return name, limit
    except Exception as e:                        # the measurement stands without it; say so
        return torch.cuda.get_device_name(0), 'unknown (%s)' % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--samples', type=int, default=300)
    ap.add_argument('--chains', type=int, default=64)
    ap.add_argument('--json', metavar='PATH', default=None, help='also write the result to this file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    dev = torch.device('cuda', 0)
    C, S = args.chains, args.samples
    g = torch.Generator().manual_seed(0)          # the config-4 problem of bench.py
    X = torch.randn(1024, 64, generator=g)
    w = torch.randn(64, 1, generator=g)
    y = torch.sin(X @ w / 8) + 0.1 * torch.randn(1024, 1, generator=g)
    torch.manual_seed(0)
    model = nn.Sequential(nn.Linear(64, 128), nn.ReLU(), nn.Linear(128, 1))
    descs = [T.MLPRegression.from_model(model, X[m * 256:(m + 1) * 256], y[m * 256:(m + 1) * 256], None, 100.,
                                        prior_scale=4) for m in range(4)]
    D = descs[0].dim
    init = (hb.util.flatten(model).detach()[None] + 0.01 * torch.randn(C, D, generator=g)).to(dev)
    kw = dict(num_samples=S, num_steps_per_sample=10, step_size=5e-4, inv_mass=torch.ones(D),
              integrator=hb.Integrator.SPLITTING, rng='philox', seed=3)
    variants = {'plain': dict(moments=True),
                'pinned': dict(moments=True, tau_prior=(1e8, 1e8), tau_out_prior=(1e8, 1e6)),
                'free': dict(moments=True, tau_prior=(2.0, 1.0), tau_out_prior=(2.0, 0.02))}

    def run(name):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        r = hb.sample_chains(descs, init, **kw, **variants[name])
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), r

    times = {k: [] for k in variants}
    results = {}
    for k in variants:                            # warm-up: module load
        _, results[k] = run(k)
    for _ in range(3):
        for k in variants:
            ms, results[k] = run(k)
            times[k].append(ms)
    name, limit = card()
    base = sum(times['plain']) / 3
    out = {'card': name, 'power_limit': limit, 'chains': C, 'num_samples': S, 'D': D, 'ms': times,
           'ratio_to_plain': {k: sum(v) / 3 / base for k, v in times.items()},
           'accept_rate': {k: float(r.accepted.float().mean()) for k, r in results.items()},
           'pinned_tau_out_range': [float(results['pinned'].tau_out_trace.min()),
                                    float(results['pinned'].tau_out_trace.max())],
           'free_tau_out_final_median': float(results['free'].tau_out_final.median())}
    print(json.dumps(out, indent=1))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
