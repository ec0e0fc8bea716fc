"""Cost of diagonal-mass adaptation during HMC_NUTS warm-up at the config-2 shape (D = 1024 isotropic Gaussian, 256 chains,
L = 10, eps0 = 0.05) with burn = 1000 and S = 2000: the plain HMC_NUTS call against the adapt_mass call of the same length,
alternated after one warm-up call of each.  The difference has two parts, timed apart: every adapt_mass launch runs the
sink form of hmc_run_kernel (runtime Philox branch, moment accumulators), timed as the plain call with moments=True
(`nuts_sink_form`: the same kernel for all S iterations), and the window machinery -- six launches instead of one and
five hmcx_adapt_diag_mass calls, whose device time alone is `reduction_ms` (events over 200 calls at C = 256, D = 1024).
Also reports the minimum bulk-ESS (diagnostics.rank_summary over the post-warm-up block) per second of call, and the card
with its power limit, as JSON (also written to PATH with --json PATH).

    python scripts/time_adapt_mass.py [--repeats 3] [--json PATH]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import hamiltorch_b200 as hb                      # noqa: E402
from hamiltorch_b200 import targets as T, _native as N  # noqa: E402


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
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--json', metavar='PATH', default=None, help='also write the result to this file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    dev = torch.device('cuda', 0)
    D, C, S, L, burn = 1024, 256, 2000, 10, 1000
    tgt = T.GaussianIso(D)
    q0 = (0.1 * torch.randn(C, D, generator=torch.Generator().manual_seed(0))).to(dev)
    kw = dict(num_samples=S, num_steps_per_sample=L, step_size=0.05, burn=burn, sampler=hb.Sampler.HMC_NUTS,
              rng='philox', seed=11)
    variants = {'nuts': {}, 'nuts_sink_form': dict(moments=True), 'nuts_adapt_mass': dict(adapt_mass=True)}

    def run(name):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        res = hb.sample_chains(tgt, q0, **kw, **variants[name])
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), res

    for name in variants:                         # warm-up: module load, tables, allocations
        run(name)
    times = {name: [] for name in variants}
    last = {}
    for _ in range(args.repeats):
        for name in variants:
            ms, last[name] = run(name)
            times[name].append(ms)
    out = {'card': card()[0], 'power_limit': card()[1], 'shape': dict(D=D, chains=C, S=S, burn=burn, L=L, eps0=0.05),
           'ms': times}
    for name, res in last.items():
        ess = float(hb.diagnostics.rank_summary(res.samples[:, 1:]).ess_bulk.min())
        best = min(times[name])
        out[name] = {'best_ms': best, 'min_bulk_ess': ess, 'min_bulk_ess_per_s': ess / (best / 1e3),
                     'accept_rate': float(res.accept_rate.mean()), 'median_step_size': float(res.step_size.median())}
    out['adapt_overhead_ms'] = out['nuts_adapt_mass']['best_ms'] - out['nuts']['best_ms']
    out['adapt_overhead_rel'] = out['adapt_overhead_ms'] / out['nuts']['best_ms']
    out['sink_form_overhead_ms'] = out['nuts_sink_form']['best_ms'] - out['nuts']['best_ms']
    # one hmcx_adapt_diag_mass at this shape (its zeroing makes repeated calls read zeros: same work, same time)
    ld = N.padded_ld(D)
    sums = [torch.zeros((C, ld), device=dev) for _ in range(4)]
    eps = torch.full((C,), 0.1, device=dev)
    im, mf = torch.empty(ld, device=dev), torch.empty(ld, device=dev)
    mu, hb_, eb = (torch.empty(C, dtype=torch.float64, device=dev) for _ in range(3))
    lib = N.load_library()

    def reduce():
        N.check(lib.hmcx_adapt_diag_mass(*(N.ptr(t) for t in sums), C, ld, D, 25, N.ptr(eps), C, N.ptr(im), N.ptr(mf),
                                         N.ptr(mu), N.ptr(hb_), N.ptr(eb), N.stream_ptr(dev)), 'hmcx_adapt_diag_mass')
    reduce()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(200):
        reduce()
    e1.record()
    torch.cuda.synchronize()
    out['reduction_ms'] = e0.elapsed_time(e1) / 200
    print(json.dumps(out))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
