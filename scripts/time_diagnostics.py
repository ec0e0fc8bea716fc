"""Device time of hamiltorch_b200.diagnostics.summary (split-R-hat, ESS, MCSE) and rank_summary (rank-normalised R-hat,
bulk / tail ESS, quantiles) on four workloads, with the bound of each pass and the numpy oracle's host time on the same
block.

    python scripts/time_diagnostics.py [--repeats 10] [--warmup 2] [--no-oracle | --no-summary-oracle] [--out FILE.json]

--no-summary-oracle keeps the rank definition's host time (every 16th dimension) and skips the split-R-hat
definition's, which takes minutes of host time on the whole config-2 block.

Workloads:
  config2  the BASELINE config-2 block from sample_chains: 256 chains x 999 draws (slot 0 = params_init dropped) x D=1024
  config5  one rank's config-5 block: HMC_NUTS, 128 chains, S=150, burn=100 -> 128 x 50 x 4096
  ar1      AR(1) chains with phi = 0.99 (32 x 2000 x 128): many lag blocks
  bnn      a block of the config-4 Bayesian-NN shape, 64 chains x 300 draws x D = 8449 (seeded AR(1) draws with one
           repeated row in four, as rejections leave them; rank_summary only)

rank_summary per workload: device time per call, the kernels of its rank pass from torch.profiler (key build, one
radix pass = histogram + scan + scatter, the rank / z pass with the fold merge) with bytes computed from the shapes and
their share of 3.35 TB/s, the lag blocks of each ESS series, and the host time of tests/rank_oracle.py on every 16th
dimension (the definition is per dimension; the full block takes hours of host time at config 2).

Per workload: device time per summary call (CUDA events around the call, after warm-up), the number of lag blocks, and
for one means pass and one autocovariance pass (timed alone with events): bytes and fp64 FMAs computed from the shapes,
GB/s against 3.35 TB/s HBM3 and the FMA rate against the data sheet's 34 TFLOP/s FP64 (non-tensor, = 17e12 FMA/s), with
the bound (the larger of the two least times) named.  The card name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import hamiltorch_b200 as hb                      # noqa: E402
from hamiltorch_b200 import diagnostics as DG     # noqa: E402
from hamiltorch_b200 import targets as T          # noqa: E402
from oracle import diagnostics_oracle as O        # noqa: E402
from tests import rank_oracle as RO               # noqa: E402

HBM_BYTES_PER_S = 3.35e12                         # H100 SXM data sheet
FP64_FMA_PER_S = 34e12 / 2                        # 34 TFLOP/s FP64 (non-tensor), 2 flops per FMA


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else 'nvidia-smi returned nothing'
    except (OSError, subprocess.SubprocessError) as e:
        return 'nvidia-smi unavailable: %s' % e


def event_ms(fn, repeats, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times)), float(np.min(times))


def roofline(name, ms, nbytes, fmas):
    t_mem, t_fma = nbytes / HBM_BYTES_PER_S, fmas / FP64_FMA_PER_S
    bound = 'HBM bandwidth' if t_mem >= t_fma else 'fp64 FMA throughput'
    return {'pass': name, 'ms': ms, 'bytes': nbytes, 'fp64_fmas': fmas,
            'GB_per_s': nbytes / ms / 1e6, 'share_of_3.35TBps': nbytes / ms / 1e-3 / HBM_BYTES_PER_S,
            'fma_per_s': fmas / ms / 1e-3, 'share_of_fp64_peak': fmas / ms / 1e-3 / FP64_FMA_PER_S,
            'bound': bound, 'share_of_bound': max(t_mem, t_fma) / (ms * 1e-3)}


def workload_blocks(names):
    dev = torch.device('cuda', torch.cuda.current_device())
    if 'config2' in names:
        init = 0.1 * torch.randn(256, 1024, generator=torch.Generator().manual_seed(1234))
        res = hb.sample_chains(T.GaussianIso(1024), init, num_samples=1000, num_steps_per_sample=10, step_size=0.05,
                               rng='philox', seed=0)
        yield 'config2', res.samples[:, 1:]
        del res
    if 'config5' in names:
        init = 0.1 * torch.randn(128, 4096, generator=torch.Generator().manual_seed(5))
        res = hb.sample_chains(T.GaussianIso(4096), init, num_samples=150, num_steps_per_sample=10, step_size=0.1,
                               burn=100, sampler=hb.Sampler.HMC_NUTS, rng='philox', seed=0)
        yield 'config5', res.samples
        del res
    if 'ar1' in names:
        g = torch.Generator(device=dev).manual_seed(7)
        C, n, D, phi = 32, 2000, 128, 0.99
        e = torch.randn(n, C, D, generator=g, device=dev)
        x = torch.empty(n, C, D, device=dev)
        x[0] = e[0]
        for t in range(1, n):                     # test data, not the measured path
            x[t] = phi * x[t - 1] + (1 - phi * phi) ** 0.5 * e[t]
        yield 'ar1', x.transpose(0, 1)            # (C, n, D) view: chain stride D, draw stride C*D
    if 'bnn' in names:
        g = torch.Generator(device=dev).manual_seed(4)
        C, n, D, phi = 64, 300, 8449, 0.9
        x = torch.empty(C, n, D, device=dev)
        x[:, 0] = torch.randn(C, D, generator=g, device=dev)
        for t in range(1, n):                     # test data, not the measured path
            x[:, t] = x[:, t - 1] if t % 4 == 0 else phi * x[:, t - 1] + (1 - phi * phi) ** 0.5 * torch.randn(
                C, D, generator=g, device=dev)
        yield 'bnn', x


RANK_KERNELS = ('rank_keys_kernel', 'radix_hist_kernel', 'seg_scan_kernel', 'radix_scatter_kernel', 'kept_count_kernel',
                'kept_prefix_kernel', 'rank_quantiles_kernel', 'rank_z_kernel', 'rank_indicator_kernel')


def rank_kernel_times(blk):
    """Total device ms per rank kernel over one rank_summary call, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        DG.rank_summary(blk)
        torch.cuda.synchronize()
    out = {k: 0.0 for k in RANK_KERNELS}
    for ev in prof.key_averages():
        for k in RANK_KERNELS:
            if k in ev.key:
                out[k] += ev.device_time_total / 1e3
    return out


def rank_row(blk, args):
    C, n, D = (int(s) for s in blk.shape)
    L = C * n
    r = DG.rank_summary(blk)
    torch.cuda.synchronize()
    ms_med, ms_min = event_ms(lambda: DG.rank_summary(blk), args.repeats, args.warmup)
    kt = rank_kernel_times(blk)
    if not all(kt[k] > 0 for k in ('rank_keys_kernel', 'radix_scatter_kernel', 'rank_z_kernel')):
        kt = rank_kernel_times(blk)             # the profiler occasionally records no device activity: once more
    # bytes from the shapes: key build reads the block and writes key + index; a radix pass reads the keys (histogram)
    # and keys + indices (scatter) and writes keys + indices; the rank / z pass reads keys, indices and the kept prefix
    # and writes the two score blocks.  Searches inside the pass re-read keys from cache and are not counted.
    if not all(kt[k] > 0 for k in ('rank_keys_kernel', 'radix_scatter_kernel', 'rank_z_kernel')):
        raise SystemExit('torch.profiler recorded no rank kernels for %s' % (tuple(blk.shape),))
    passes = [roofline('key build', kt['rank_keys_kernel'], 4 * L * D + 8 * L * D, 0),
              roofline('one radix pass (hist + scan + scatter)',
                       (kt['radix_hist_kernel'] + kt['radix_scatter_kernel']) / 4 + kt['seg_scan_kernel'] / 5,
                       4 * L * D + 16 * L * D, 0),
              roofline('rank / z pass with fold merge', kt['rank_z_kernel'], 12 * L * D + 8 * L * D, 0)]
    row = {'workload': 'rank_summary', 'shape': [C, n, D], 'rank_summary_ms_median': ms_med,
           'rank_summary_ms_min': ms_min, 'kernel_ms': kt, 'lag_blocks_bulk_i05_i95': list(r.num_lag_blocks),
           'max_rhat': float(r.rhat.max()), 'median_ess_bulk': float(r.ess_bulk.median()),
           'median_ess_tail': float(r.ess_tail.median()), 'passes': passes}
    if not args.no_oracle:
        dims = torch.arange(0, D, 16, device=blk.device)
        host = blk[..., dims].cpu().numpy()
        t = time.perf_counter()
        ref = RO.rank_summary(host)
        row['oracle_host_s_every_16th_dim'] = time.perf_counter() - t
        row['oracle_max_rel_err_ess_bulk'] = float(np.max(np.abs(r.ess_bulk[dims].cpu().numpy() - ref['ess_bulk'])
                                                          / ref['ess_bulk']))
        row['oracle_same_quantiles'] = bool(np.array_equal(r.median[dims].cpu().numpy(), ref['median']))
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--no-oracle', action='store_true')
    ap.add_argument('--no-summary-oracle', action='store_true')
    ap.add_argument('--workloads', default='config2,config5,ar1,bnn')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_diagnostics.py measures on a CUDA device; none is present')
    report = {'card': card(), 'torch': torch.__version__, 'host_cores': os.cpu_count(), 'workloads': []}
    print(json.dumps({'card': report['card'], 'host_cores': report['host_cores']}), flush=True)
    for name, blk in workload_blocks(args.workloads.split(',')):
        C, n, D = (int(s) for s in blk.shape)
        K, m = 2 * C, n // 2
        rrow = rank_row(blk, args)
        rrow['workload'] = name + ' rank_summary'
        report['workloads'].append(rrow)
        print(json.dumps(rrow), flush=True)
        if name == 'bnn':
            continue
        d = DG.summary(blk)
        torch.cuda.synchronize()
        ms_med, ms_min = event_ms(lambda: DG.summary(blk), args.repeats, args.warmup)
        part = DG.NativePartials(blk)
        mu_sum, _ = part.means()
        mu_bar = mu_sum / K
        means_ms, _ = event_ms(part.means, args.repeats, args.warmup)
        acov_ms, _ = event_ms(lambda: part.acov(mu_bar, 0), args.repeats, args.warmup)
        passes = [roofline('means', means_ms, 4 * K * m * D, 0),
                  roofline('acov lags [0, 32)', acov_ms, 4 * K * m * D, K * m * D * 32)]
        if d.num_lag_blocks > 1:
            t0 = 32
            later_ms, _ = event_ms(lambda: part.acov(None, t0), args.repeats, args.warmup)
            passes.append(roofline('acov lags [32, 64)', later_ms, 8 * K * max(m - t0, 0) * D,
                                   K * max(m - t0, 0) * D * 32))
        row = {'workload': name, 'shape': [C, n, D], 'summary_ms_median': ms_med, 'summary_ms_min': ms_min,
               'lag_blocks': d.num_lag_blocks, 'max_rhat': float(d.rhat.max()), 'min_ess': float(d.ess.min()),
               'median_ess': float(d.ess.median()), 'passes': passes}
        if not (args.no_oracle or args.no_summary_oracle):
            host = blk.cpu().numpy()
            t = time.perf_counter()
            ref = O.summary(host)
            row['oracle_host_s'] = time.perf_counter() - t
            row['oracle_max_rel_err_ess'] = float(np.max(np.abs(d.ess.cpu().numpy() - ref['ess']) / ref['ess']))
            row['oracle_same_max_lag'] = bool(np.array_equal(d.max_lag.cpu().numpy(), ref['max_lag']))
            del host, ref
        report['workloads'].append(row)
        print(json.dumps(row), flush=True)
        del blk, part
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(report, f, indent=1)


if __name__ == '__main__':
    main()
