"""Cost of K-fold refits (DESIGN §3.18) on config 4's network and data.

The Bayesian NN Linear(64,128)-ReLU-Linear(128,1) (D = 8449) of bench.py's config 4 on its N = 1024 rows as one
MLPTarget, plain HMC, L = 10, eps = 5e-4, S = 300, inv_mass = 1, in-kernel Philox:
  fold      one K = 10 x R = 4 fold run (40 chains, each on 921 or 922 training rows), one launch
  plain     the 40-chain plain run on all 1024 rows
  kfold     loo.kfold scoring of the fold run (likelihood of the held-out rows + fp64 logsumexp)
  reloo     loo.reloo of 8 flagged points with R = 4 chains each (one K = 8 fold run, 32 chains, plus its scoring)
Device events per call; fold and plain alternated three times after one warm-up run of each, kfold and reloo timed three
times after a warm-up.  Prints the card, its power limit and the numbers as JSON (also written to PATH with --json PATH).

    python scripts/time_kfold.py [--json PATH]
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
from hamiltorch_b200 import loo as LOO, targets as T    # noqa: E402


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in out.split(',')]
        return name, limit
    except Exception as e:                        # the measurement stands without it; say so
        return torch.cuda.get_device_name(0), 'unknown (%s)' % e


def event_ms(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    r = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--json', metavar='PATH', default=None, help='also write the result to this file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    dev = torch.device('cuda', 0)
    name, limit = card()
    g = torch.Generator().manual_seed(0)          # the config-4 problem of bench.py
    X = torch.randn(1024, 64, generator=g)
    w = torch.randn(64, 1, generator=g)
    y = torch.sin(X @ w / 8) + 0.1 * torch.randn(1024, 1, generator=g)
    torch.manual_seed(0)
    model = nn.Sequential(nn.Linear(64, 128), nn.ReLU(), nn.Linear(128, 1))
    tgt = T.MLPTarget.from_model(model, X, y, None, 100.)
    D = tgt.dim
    K, R = 10, 4
    init = (hb.util.flatten(model).detach()[None] + 0.01 * torch.randn(K * R, D, generator=g)).to(dev)
    kw = dict(num_samples=300, num_steps_per_sample=10, step_size=5e-4, inv_mass=torch.ones(D), rng='philox', seed=3)
    folds = LOO.kfold_split(1024, K, seed=0)
    runs = {'fold': lambda: hb.sample_chains(tgt, init, folds=folds, **kw),
            'plain': lambda: hb.sample_chains(tgt, init, **kw)}
    times = {k: [] for k in runs}
    res = {k: fn() for k, fn in runs.items()}     # warm-up: module load, packed operands
    torch.cuda.synchronize()
    for _ in range(3):
        for k, fn in runs.items():
            ms, res[k] = event_ms(fn)
            times[k].append(ms)
    LOO.kfold(res['fold'], tgt)
    kf_ms = [event_ms(lambda: LOO.kfold(res['fold'], tgt))[0] for _ in range(3)]
    kf = LOO.kfold(res['fold'], tgt)
    lo = LOO.psis_loo(res['plain'], tgt)
    flagged = LOO.LooResult()                     # 8 points marked as flagged, whatever their k-hat
    flagged.__dict__.update({k: (v.clone() if torch.is_tensor(v) else v) for k, v in lo.__dict__.items()})
    pts = torch.randperm(1024, generator=torch.Generator().manual_seed(1))[:8].to(flagged.pareto_k.device)
    flagged.pareto_k[flagged.pareto_k > flagged.k_threshold] = 0.0
    flagged.pareto_k[pts] = 1.0
    rl_kw = dict(kw, num_samples=300)
    LOO.reloo(flagged, tgt, init[:R], **rl_kw)
    rl_ms = [event_ms(lambda: LOO.reloo(flagged, tgt, init[:R], **rl_kw))[0] for _ in range(3)]
    out = {'card': name, 'power_limit': limit, 'D': D, 'N': 1024, 'K': K, 'R': R, 'S': 300, 'L': 10,
           'ms': {'fold_run': times['fold'], 'plain_run_40_chains': times['plain'], 'kfold_scoring': kf_ms,
                  'reloo_8_points': rl_ms},
           'fold_over_plain': sum(times['fold']) / sum(times['plain']),
           'accept_rate': {k: float(r.accepted.float().mean()) for k, r in res.items()},
           'elpd_kfold': kf.elpd_kfold, 'se': kf.se}
    print(json.dumps(out, indent=1))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
