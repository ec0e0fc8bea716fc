"""Device time of power-scaling sensitivity -- ``sensitivity.power_scale(draws, target)`` (the prior and likelihood
components, the four weight sets and the sort / CJS pass over every parameter) -- against ``diagnostics.rank_summary``
and ``loo.psis_loo`` on the same draws, on the BASELINE config-4 network (Linear(64,128)-ReLU-Linear(128,1), N = 1024
rows of oracle/cfg4.py) with 64 chains x 1000 draws.  Medians of ``--reps`` timed calls after a warm-up.  Prints one
JSON line with the card's name and power limit read in the same run.

    python scripts/time_psens.py [--chains 64] [--draws 1000] [--reps 3] [--out FILE]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

from time_loo import card, device_ms          # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--chains', type=int, default=64)
    ap.add_argument('--draws', type=int, default=1000)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('time_psens: needs a CUDA device')
    from hamiltorch_b200 import diagnostics as DG, loo as LOO, sensitivity as SE, targets as T, util
    from oracle import cfg4
    model, X, y = cfg4.problem()
    tgt = T.MLPTarget.from_model(model, X, y, None, cfg4.TAU_OUT)
    flat = util.flatten(model).detach().cuda()
    g = torch.Generator(device='cuda').manual_seed(0)
    draws = flat + 0.01 * torch.randn(a.chains, a.draws, flat.numel(), generator=g, device='cuda')
    out = {'card': card(), 'chains': a.chains, 'draws': a.draws, 'points': int(X.shape[0]), 'params': flat.numel()}
    s = SE.power_scale(draws, tgt)
    out['pareto_k'] = [round(float(k), 4) for k in s.pareto_k.tolist()]
    out['power_scale_ms'] = round(device_ms(lambda: SE.power_scale(draws, tgt), a.reps), 3)
    out['log_components_ms'] = round(device_ms(lambda: SE.log_components(draws, tgt), a.reps), 3)
    out['rank_summary_ms'] = round(device_ms(lambda: DG.rank_summary(draws), a.reps), 3)
    out['psis_loo_ms'] = round(device_ms(lambda: LOO.psis_loo(draws, tgt), a.reps), 3)
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
