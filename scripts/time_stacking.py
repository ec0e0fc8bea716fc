"""Device time of chain stacking -- ``loo.psis_loo_chains`` (hmcx_mlp_pointwise_ll + hmcx_loo_chain_pass per slab of
points) against ``loo.psis_loo``, ``loo.chain_stacking`` (the per-chain pass plus the EM solver, hmcx_stack_em) with its
iteration count, and ``predictive.evaluate(..., chain_weights=w)`` (hmcx_pred_pass_weighted) against ``evaluate`` -- on
the BASELINE config-4 network (Linear(64,128)-ReLU-Linear(128,1), N = 1024 rows of oracle/cfg4.py) with 64 chains x
1000 draws.  Prints one JSON line with the card's name and power limit read in the same run.

    python scripts/time_stacking.py [--chains 64] [--draws 1000] [--reps 3] [--out FILE]
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
        raise SystemExit('time_stacking: needs a CUDA device')
    from hamiltorch_b200 import loo as LOO, predictive as PR, targets as T, util
    from oracle import cfg4
    model, X, y = cfg4.problem()
    tgt = T.MLPTarget.from_model(model, X, y, None, cfg4.TAU_OUT)
    flat = util.flatten(model).detach().cuda()
    g = torch.Generator(device='cuda').manual_seed(0)
    # chains around different centres, so the per-chain predictives differ and the weights are not uniform
    centre = 0.02 * torch.randn(a.chains, 1, flat.numel(), generator=g, device='cuda')
    draws = flat + centre + 0.01 * torch.randn(a.chains, a.draws, flat.numel(), generator=g, device='cuda')
    out = {'card': card(), 'chains': a.chains, 'draws': a.draws, 'points': int(X.shape[0]), 'params': flat.numel()}
    out['psis_loo_chains_ms'] = round(device_ms(lambda: LOO.psis_loo_chains(draws, tgt), a.reps), 3)
    out['psis_loo_ms'] = round(device_ms(lambda: LOO.psis_loo(draws, tgt), a.reps), 3)
    st = LOO.chain_stacking(draws, tgt)
    out['chain_stacking_ms'] = round(device_ms(lambda: LOO.chain_stacking(draws, tgt), a.reps), 3)
    cl = st.chain_loo
    out['stacking_solver_ms'] = round(device_ms(lambda: LOO._stack(cl.pointwise, 1e-6, 20000, 'time'), a.reps), 3)
    out['iterations'], out['converged'], out['kkt_gap'] = st.iterations, st.converged, st.kkt_gap
    w = st.weights
    out['weights_above_1e-3'] = int((w > 1e-3).sum())
    out['evaluate_weighted_ms'] = round(device_ms(lambda: PR.evaluate(draws, tgt, chain_weights=w), a.reps), 3)
    out['evaluate_ms'] = round(device_ms(lambda: PR.evaluate(draws, tgt), a.reps), 3)
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
