"""Device time of held-out evaluation (hamiltorch_b200.predictive): the outputs pass (hmcx_mlp_pointwise_out over every
row), the predictive pass (hmcx_pred_pass + hmcx_pred_totals, from the outputs block) and evaluate(samples, target)
end to end, with 64 chains x 1000 draws, on
  * the BASELINE config-4 network (Linear(64,128)-ReLU-Linear(128,1), tensor cores) at N = 1,024 (oracle/cfg4.py) and
    on a 16,384-row synthetic variant;
  * a 10-class Linear(64,128)-Tanh-Linear(128,10) classifier (SIMT tiles) and a 4-class Linear(32,128)-ReLU-Linear(128,4)
    classifier (tensor cores), each on 10,000 synthetic points;
and the path users had before: predict_model on 300 draws of the 10-class classifier plus the notebook's curve loop
(softmax, cumulative ensembles, in torch on the GPU).  Prints one JSON line with the card's name and power limit read in
the same run.

    python scripts/time_predictive.py [--chains 64] [--draws 1000] [--reps 2] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

from time_loo import card, device_ms  # noqa: E402


def case(name, model, x, y, loss, C, n, reps, tau_out=1.0):
    import torch
    from hamiltorch_b200 import _native as N, engine, predictive as P, targets as T, util
    tgt = T.MLPTarget.from_model(model, x, y, None, tau_out, model_loss=loss)
    flat = util.flatten(model).detach().cuda()
    g = torch.Generator(device='cuda').manual_seed(0)
    draws = flat + 0.01 * torch.randn(C, n, flat.numel(), generator=g, device='cuda')
    tc = bool(engine.native_target(tgt, 'cuda').mlp_struct.x_packed)
    row = {'case': name, 'loss': loss, 'chains': C, 'draws': n, 'points': x.shape[0], 'params': flat.numel(),
           'tensor_cores': tc}
    out = P.pointwise_outputs(draws, tgt)
    row['outputs_block_gb'] = round(out.numel() * 4 / 1e9, 3)
    row['pass1_ms'] = round(device_ms(lambda: P.pointwise_outputs(draws, tgt), reps), 2)
    row['pass2_ms'] = round(device_ms(lambda: P.evaluate(out, tgt), reps), 2)
    ref = P.evaluate(out, tgt)
    del out
    torch.cuda.empty_cache()
    row['evaluate_ms'] = round(device_ms(lambda: P.evaluate(draws, tgt), reps), 2)
    r = P.evaluate(draws, tgt)
    row['slab_points'] = P._slab_points(N.load_library(), C, n, tgt.widths[-1], tgt.loss_id, x.shape[0],
                                        4 * C * n * tgt.widths[-1])
    row['same_bytes_as_block_route'] = bool(torch.equal(r.nll_curve, ref.nll_curve))
    row['nll'] = r.nll
    if loss == 'regression':
        row['rmse'], row['coverage90'] = r.rmse, r.coverage[0.9]
    else:
        row['accuracy'], row['ece'] = r.accuracy, r.ece
    return row


def notebook_loop(model, x, y, n):
    """predict_model on n draws, then the notebook's loop over s (probability-averaged ensembles of the first s draws)."""
    import torch
    from hamiltorch_b200 import samplers, util
    flat = util.flatten(model).detach().cuda()
    g = torch.Generator(device='cuda').manual_seed(0)
    samples = list((flat + 0.01 * torch.randn(n, flat.numel(), generator=g, device='cuda')).unbind(0))
    xc, yc = x.cuda(), y.cuda().long()

    def run():
        pred, _ = samplers.predict_model(model, samples, x=xc, y=yc.float(), model_loss='multi_class_linear_output',
                                         tau_out=1.0)
        acc, nll = [], []
        for s in range(1, n + 1):
            ens = torch.softmax(pred[:s], -1).mean(0)
            acc.append((ens.argmax(-1) == yc).float().mean())
            nll.append(-ens.gather(1, yc[:, None]).log().mean())
        return torch.stack(acc), torch.stack(nll)
    return {'case': 'predict_model_plus_notebook_loop', 'draws': n, 'points': x.shape[0],
            'ms': round(device_ms(run, 1), 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--chains', type=int, default=64)
    ap.add_argument('--draws', type=int, default=1000)
    ap.add_argument('--reps', type=int, default=2)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    import torch.nn as nn
    if not torch.cuda.is_available():
        raise SystemExit('time_predictive: needs a CUDA device')
    from oracle import cfg4
    res = {'card': card(), 'cases': []}
    t0 = time.perf_counter()
    model, X, y = cfg4.problem()
    res['cases'].append(case('cfg4_N1024', model, X, y, 'regression', a.chains, a.draws, a.reps, cfg4.TAU_OUT))
    g = torch.Generator().manual_seed(1)
    Xs = torch.randn(16384, cfg4.N_IN, generator=g)
    ys = torch.sin(Xs @ torch.randn(cfg4.N_IN, 1, generator=g) / 8) + 0.1 * torch.randn(16384, 1, generator=g)
    res['cases'].append(case('cfg4_N16384', model, Xs, ys, 'regression', a.chains, a.draws, a.reps, cfg4.TAU_OUT))
    torch.manual_seed(2)
    for name, n0, act, K in (('mc10_simt', 64, nn.Tanh, 10), ('mc4_tc', 32, nn.ReLU, 4)):
        net = nn.Sequential(nn.Linear(n0, 128), act(), nn.Linear(128, K))
        Xc = torch.randn(10000, n0, generator=g)
        yc = net(Xc).detach().argmax(1).float()
        res['cases'].append(case(name, net, Xc, yc, 'multi_class_linear_output', a.chains, a.draws, a.reps))
        if K == 10:
            res['cases'].append(notebook_loop(net, Xc, yc, 300))
    res['wall_s'] = round(time.perf_counter() - t0, 1)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
