"""Device time of hamiltorch_b200.ppc -- ``check`` (hmcx_mlp_pointwise_out + hmcx_ppc_pass per slab of draws) and
``loo_pit`` (hmcx_mlp_pointwise_ll + hmcx_mlp_pointwise_out + hmcx_loo_pit_pass per slab of points) -- against
``loo.psis_loo`` and ``predictive.evaluate`` on the same samples: the BASELINE config-4 network (Linear(64,128)-ReLU-
Linear(128,1), N = 1024 rows of oracle/cfg4.py) with 64 chains x 1000 draws.  Prints one JSON line with the card's name
and power limit read in the same run.

    python scripts/time_ppc.py [--chains 64] [--draws 1000] [--reps 3] [--out FILE]
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
        raise SystemExit('time_ppc: needs a CUDA device')
    from hamiltorch_b200 import loo as LOO, ppc, predictive as PR, targets as T, util
    from oracle import cfg4
    model, X, y = cfg4.problem()
    tgt = T.MLPTarget.from_model(model, X, y, None, cfg4.TAU_OUT)
    flat = util.flatten(model).detach().cuda()
    g = torch.Generator(device='cuda').manual_seed(0)
    draws = flat + 0.01 * torch.randn(a.chains, a.draws, flat.numel(), generator=g, device='cuda')
    out = {'card': card(), 'chains': a.chains, 'draws': a.draws, 'points': int(X.shape[0]), 'params': flat.numel()}
    out['check_ms'] = round(device_ms(lambda: ppc.check(draws, tgt), a.reps), 3)
    out['loo_pit_ms'] = round(device_ms(lambda: ppc.loo_pit(draws, tgt), a.reps), 3)
    out['psis_loo_ms'] = round(device_ms(lambda: LOO.psis_loo(draws, tgt), a.reps), 3)
    out['evaluate_ms'] = round(device_ms(lambda: PR.evaluate(draws, tgt), a.reps), 3)
    sub = torch.arange(0, a.chains * a.draws, 64)
    out['replicate_%d_draws_ms' % sub.numel()] = round(device_ms(lambda: ppc.replicate(draws, tgt, draws=sub), a.reps), 3)
    r, lp = ppc.check(draws, tgt), ppc.loo_pit(draws, tgt)
    out['p_value'] = dict(zip(r.names, [round(v, 4) for v in r.p_value.tolist()]))
    out['loo_pit_chi2_p'] = lp.p_value
    out['pareto_k_equal_psis_loo'] = bool(torch.equal(lp.pareto_k, LOO.psis_loo(draws, tgt).pareto_k))
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
