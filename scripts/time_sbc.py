"""Cost of simulation-based calibration (DESIGN §3.19) on config 4's network and data.

The Bayesian NN Linear(64,128)-ReLU-Linear(128,1) (D = 8449) of bench.py's config 4 on its N = 1024 inputs, tau_out = 100,
plain HMC, L = 10, eps = 5e-4, S = 300, in-kernel Philox:
  sbc_run     sbc.run with M = 64 sims x R = 4 chains: simulate, one 256-chain fit launch, ranks, histograms
  plain       a plain 256-chain run of the same target from the same starts
  ranks       sbc.ranks of the fit on its own (parameter ranks + the log-likelihood column)
  rank_kernel hmcx_sbc_rank alone, against the least time to read the (256, 300, 8452) fp32 block at 3.35 TB/s
Device events per call; sbc_run and plain alternated three times after one warm-up run of each, ranks and the rank kernel
timed after a warm-up.  Prints the card, its power limit and the numbers as JSON (also written to PATH with --json PATH).

    python scripts/time_sbc.py [--json PATH]
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
from hamiltorch_b200 import _native as N, sbc, targets as T    # noqa: E402

HBM_BYTES_PER_S = 3.35e12                         # H100 SXM data sheet


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
    tgt = T.MLPTarget.from_model(model, X.to(dev), y.to(dev), None, 100.)
    D = tgt.dim
    M, R, S = 64, 4, 300
    kw = dict(num_samples=S, num_steps_per_sample=10, step_size=5e-4)
    sim = sbc.simulate(tgt, M, R, seed=3)
    init = sim.init.transpose(0, 1).reshape(R * M, D).contiguous()
    runs = {'sbc_run': lambda: sbc.run(tgt, M, R, seed=3, **kw),
            'plain': lambda: hb.sample_chains(tgt, init, rng='philox', seed=3, **kw)}
    times = {k: [] for k in runs}
    res = {k: fn() for k, fn in runs.items()}     # warm-up: module load, packed operands
    torch.cuda.synchronize()
    for _ in range(3):
        for k, fn in runs.items():
            ms, res[k] = event_ms(fn)
            times[k].append(ms)
    fit = sbc.fit(sim, tgt, seed=3, **kw)
    sbc.ranks(fit, sim, tgt)
    rk_ms = [event_ms(lambda: sbc.ranks(fit, sim, tgt))[0] for _ in range(3)]
    lib = N.load_library()
    x = fit.samples_padded
    C_, keep, ld = x.shape
    truth = sim.block[:, 0].contiguous()
    out_rk = torch.empty((M, D), dtype=torch.int32, device=dev)

    def rank_kernel():
        for _ in range(10):
            N.check(lib.hmcx_sbc_rank(N.ptr(x), keep * ld, ld, C_, keep, M, D, N.ptr(truth), ld, N.ptr(out_rk),
                                      N.stream_ptr(dev)), 'hmcx_sbc_rank')
    rank_kernel()
    kern_ms = [event_ms(rank_kernel)[0] / 10 for _ in range(3)]
    block_bytes = C_ * (keep - 1) * D * 4         # the elements the kernel reads
    out = {'card': name, 'power_limit': limit, 'D': D, 'N': 1024, 'M': M, 'R': R, 'S': S, 'L': 10,
           'ms': {'sbc_run': times['sbc_run'], 'plain_run_256_chains': times['plain'], 'ranks': rk_ms,
                  'rank_kernel': kern_ms},
           'sbc_over_plain': sum(times['sbc_run']) / sum(times['plain']),
           'rank_kernel_bytes': block_bytes,
           'rank_kernel_hbm_bound_ms': 1e3 * block_bytes / HBM_BYTES_PER_S,
           'rank_kernel_share_of_hbm_peak': (1e3 * block_bytes / HBM_BYTES_PER_S) / min(kern_ms),
           'accept_rate': {'sbc_run': float(res['sbc_run'].accept_rate.mean()),
                           'plain': float(res['plain'].accept_rate.mean())},
           'min_p_value': float(res['sbc_run'].p_value.min())}
    print(json.dumps(out, indent=1))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
