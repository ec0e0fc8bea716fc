"""Device time of the two passes behind hamiltorch_b200.loo -- the pointwise log-likelihood (hmcx_mlp_pointwise_ll) and the
PSIS / WAIC pass (hmcx_loo_pass, its sort included) -- on the BASELINE config-4 network (Linear(64,128)-ReLU-Linear(128,1),
N = 1024 rows of oracle/cfg4.py) with 64 chains x 1000 draws, and on a 16,384-row synthetic variant of the same network;
plus the numpy fp64 oracle (tests/loo_oracle.py) on the same block.  Prints one JSON line with the card's name and power
limit read in the same run.

    python scripts/time_loo.py [--chains 64] [--draws 1000] [--reps 3] [--oracle-points 1024] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch
    info = {'device': torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        info['nvidia_smi'] = out[0] if out else None
    except (OSError, subprocess.SubprocessError):
        info['nvidia_smi'] = None
    return info


def device_ms(fn, reps):
    """Median over `reps` timed calls (after one warm-up call) of CUDA-event time, ms."""
    import torch
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


def case(name, model, x, y, C, n, reps, oracle_points):
    import torch
    from hamiltorch_b200 import loo as LOO, targets as T, util
    from oracle import cfg4
    from tests import loo_oracle as O
    tgt = T.MLPTarget.from_model(model, x, y, None, cfg4.TAU_OUT)
    flat = util.flatten(model).detach().cuda()
    g = torch.Generator(device='cuda').manual_seed(0)
    draws = flat + 0.01 * torch.randn(C, n, flat.numel(), generator=g, device='cuda')
    ll = LOO.pointwise_log_lik(draws, tgt)
    t_ll = device_ms(lambda: LOO.pointwise_log_lik(draws, tgt), reps)
    t_psis = device_ms(lambda: LOO.psis_loo(ll), reps)
    t_waic = device_ms(lambda: LOO.waic(ll), reps)
    t_end = device_ms(lambda: LOO.psis_loo(draws, tgt), reps)
    lo = LOO.psis_loo(ll)
    Np = ll.shape[2]
    k = min(Np, oracle_points)
    blk = ll[:, :, :k].cpu().numpy()
    t0 = time.perf_counter()
    ref = O.psis_loo(blk)
    t_oracle = (time.perf_counter() - t0) * 1e3
    diff = float(abs(lo.pointwise[:k].cpu().numpy() - ref['elpd_loo']).max())
    return {'case': name, 'chains': C, 'draws': n, 'points': Np, 'params': flat.numel(),
            'll_pass_ms': round(t_ll, 3), 'psis_pass_ms': round(t_psis, 3), 'waic_ms': round(t_waic, 3),
            'psis_from_samples_ms': round(t_end, 3),
            'oracle_points': k, 'oracle_ms': round(t_oracle, 1), 'oracle_ms_per_point': round(t_oracle / k, 3),
            'max_abs_diff_elpd_vs_oracle': diff, 'elpd_loo': lo.elpd_loo, 'max_pareto_k': float(lo.pareto_k.max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--chains', type=int, default=64)
    ap.add_argument('--draws', type=int, default=1000)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--oracle-points', type=int, default=1024)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('time_loo: needs a CUDA device')
    from oracle import cfg4
    model, X, y = cfg4.problem()
    res = {'card': card(), 'cases': []}
    res['cases'].append(case('cfg4_N1024', model, X, y, a.chains, a.draws, a.reps, a.oracle_points))
    g = torch.Generator().manual_seed(1)
    Xs = torch.randn(16384, cfg4.N_IN, generator=g)
    ys = torch.sin(Xs @ torch.randn(cfg4.N_IN, 1, generator=g) / 8) + 0.1 * torch.randn(16384, 1, generator=g)
    res['cases'].append(case('synthetic_N16384', model, Xs, ys, a.chains, a.draws, a.reps, a.oracle_points))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
