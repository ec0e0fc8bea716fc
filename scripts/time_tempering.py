"""Cost of replica exchange (DESIGN §3.17) and what it buys on a multimodal posterior.

Timing, device events per call, variants alternated three times after one warm-up run of each:
  config 4    Linear(64,128)-ReLU-Linear(128,1), D = 8449, N = 1024 in M = 4 splits, symmetric split HMC, L = 10,
              eps = 5e-4, S = 300: 64 chains as 16 ladders x betas (1, .3, .1, .03) at swap_every 1, 10 and 300, against
              the plain 64-chain run (moments=True everywhere; the plain run is mlp_run_kernel<CS, false>, the tempered
              ones mlp_run_kernel<CS, true>)
  iris        a 4-8-3 tanh classifier on 150 iris-shaped points, 1024 chains (256 ladders x 4 betas), L = 10,
              S = 300: the launch-bound regime
Multimodal report: the sign-symmetric 1-1-1 tanh net of tests/test_tempering_gpu.py, plain chains against tempered cold
chains: the share of draws with w2 > 0, the chains that cross w2 = 0, the swap rates and the rank R-hat of w2.
Prints the card, its power limit and the numbers as JSON (also written to PATH with --json PATH).

    python scripts/time_tempering.py [--json PATH]
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


def timed(fn, variants, reps=3):
    def run(kw):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        r = fn(**kw)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), r
    times = {k: [] for k in variants}
    for k, kw in variants.items():                # warm-up: module load
        run(kw)
    for _ in range(reps):
        for k, kw in variants.items():
            times[k].append(run(kw)[0])
    return times


def config4(dev):
    g = torch.Generator().manual_seed(0)          # the config-4 problem of bench.py
    X = torch.randn(1024, 64, generator=g)
    w = torch.randn(64, 1, generator=g)
    y = torch.sin(X @ w / 8) + 0.1 * torch.randn(1024, 1, generator=g)
    torch.manual_seed(0)
    model = nn.Sequential(nn.Linear(64, 128), nn.ReLU(), nn.Linear(128, 1))
    descs = [T.MLPRegression.from_model(model, X[m * 256:(m + 1) * 256], y[m * 256:(m + 1) * 256], None, 100.,
                                        prior_scale=4) for m in range(4)]
    D = descs[0].dim
    init = (hb.util.flatten(model).detach()[None] + 0.01 * torch.randn(64, D, generator=g)).to(dev)
    kw = dict(num_samples=300, num_steps_per_sample=10, step_size=5e-4, inv_mass=torch.ones(D),
              integrator=hb.Integrator.SPLITTING, rng='philox', seed=3, moments=True)
    betas = [1.0, 0.3, 0.1, 0.03]
    variants = {'plain': {}, 'swap_every_1': dict(betas=betas, swap_every=1),
                'swap_every_10': dict(betas=betas, swap_every=10), 'swap_every_300': dict(betas=betas, swap_every=300)}
    times = timed(lambda **v: hb.sample_chains(descs, init, **kw, **v), variants)
    return {'D': D, 'chains': 64, 'ms': times,
            'ratio_to_plain': {k: sum(v) / sum(times['plain']) for k, v in times.items()}}


def iris(dev):
    g = torch.Generator().manual_seed(1)
    centres = torch.randn(3, 4, generator=g) * 2
    lab = torch.arange(150) % 3
    X = centres[lab] + torch.randn(150, 4, generator=g)
    torch.manual_seed(1)
    model = nn.Sequential(nn.Linear(4, 8), nn.Tanh(), nn.Linear(8, 3))
    tgt = T.MLPTarget.from_model(model, X, lab.float(), None, 1.0, model_loss='multi_class_linear_output')
    D = tgt.dim
    init = (hb.util.flatten(model).detach()[None] + 0.1 * torch.randn(1024, D, generator=g)).to(dev)
    kw = dict(num_samples=300, num_steps_per_sample=10, step_size=0.01, rng='philox', seed=3, moments=True)
    betas = [1.0, 0.3, 0.1, 0.03]
    variants = {'plain': {}, 'swap_every_1': dict(betas=betas, swap_every=1),
                'swap_every_10': dict(betas=betas, swap_every=10), 'swap_every_300': dict(betas=betas, swap_every=300)}
    times = timed(lambda **v: hb.sample_chains(tgt, init, **kw, **v), variants)
    return {'D': D, 'chains': 1024, 'ms': times,
            'ratio_to_plain': {k: sum(v) / sum(times['plain']) for k, v in times.items()}}


def bimodal():
    from tests.test_tempering_gpu import bimodal_runs, BIMODAL_BETAS
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    plain, temp = bimodal_runs()
    e1.record()
    torch.cuda.synchronize()
    out = {'betas': BIMODAL_BETAS, 'ladders': int(temp.samples.shape[0]), 'ms_both_runs': e0.elapsed_time(e1)}
    for name, r in (('plain', plain), ('tempered', temp)):
        w2 = r.samples[:, 1:, 2]
        pos = (w2 > 0).double()
        out[name] = {'share_w2_pos': float(pos.mean()),
                     'per_chain_share_w2_pos': [round(float(v), 4) for v in pos.mean(1)],
                     'chains_crossing': int(((w2[:, 1:] > 0) != (w2[:, :-1] > 0)).any(1).sum()),
                     'rank_rhat_w2': float(hb.diagnostics.rank_summary(w2[..., None].contiguous()).rhat[0])}
    out['tempered']['swap_rate'] = [round(float(v), 4) for v in temp.swap_rate]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--json', metavar='PATH', default=None, help='also write the result to this file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    dev = torch.device('cuda', 0)
    name, limit = card()
    out = {'card': name, 'power_limit': limit, 'config4': config4(dev), 'iris': iris(dev), 'bimodal': bimodal()}
    print(json.dumps(out, indent=1))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
