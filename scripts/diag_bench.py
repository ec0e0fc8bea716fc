"""Diagnostic: CUDA-event times of the config-2 launch (256 chains, D=1024, L=10, in-kernel Philox), with the card's SM
clock, power limit and name read alongside (nvidia-smi queries only).

Launches of S=1000 and S=2000 iterations alternate; their difference over 1000 is the time of one iteration without
the launch's fixed costs, and times the SM clock gives cycles per iteration.  Set against the
warp-instructions per iteration of the kernel's SASS (4 warps per scheduler at this shape) that gives the issue
efficiency.  --eps 0.42 --init-scale 1 (chains started in the typical set) gives an acceptance of ~0.5 instead of
config 2's ~0.99.  --dump DIR writes a SHA-256 of every output of the last S=1000 launch, so that two builds can be
compared bit for bit."""
import argparse, hashlib, json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from hamiltorch_b200 import engine, targets as T

ap = argparse.ArgumentParser()
ap.add_argument('--eps', type=float, default=0.05)
ap.add_argument('--init-scale', type=float, default=0.1)
ap.add_argument('--reps', type=int, default=10)
ap.add_argument('--dump', default=None)
args = ap.parse_args()

dev = torch.device('cuda', 0)
tgt = engine.NativeTarget(T.GaussianIso(1024), dev)
q0 = (args.init_scale * torch.randn(256, 1024, generator=torch.Generator().manual_seed(0))).to(dev)
outs = {S: torch.empty((256, S, 1024), dtype=torch.float32, device=dev) for S in (1000, 2000)}


def smi(fields):
    return subprocess.run(['nvidia-smi', '--query-gpu=' + fields, '--format=csv,noheader'], capture_output=True,
                          text=True).stdout.strip()


def launch(S, k):
    return engine.hmc_run(tgt, q0, S, 10, args.eps, seed=k, out=outs[S], device=dev)


card = smi('name,power.limit,clocks.max.sm')
for S in (1000, 2000):
    launch(S, 0)
torch.cuda.synchronize()
times = {1000: [], 2000: []}
clocks = []
res = None
for k in range(args.reps):
    for S in (1000, 2000):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        r = launch(S, 1)
        e1.record()
        torch.cuda.synchronize()
        times[S].append(e0.elapsed_time(e1))
        if S == 1000:
            res = r
    clocks.append(float(smi('clocks.sm').split()[0]))
med = {S: sorted(v)[len(v) // 2] for S, v in times.items()}
us_iter = (med[2000] - med[1000]) / 1000 * 1e3
mhz = sorted(clocks)[len(clocks) // 2]
line = {'card': card, 'eps': args.eps, 'init_scale': args.init_scale, 'accept_rate': float(res.accepted.float().mean()),
        'ms_S1000': times[1000], 'ms_S2000': times[2000], 'median_ms': med, 'us_per_iter': us_iter,
        'sm_mhz_median': mhz, 'cycles_per_iter': us_iter * mhz}
print(json.dumps(line))
if args.dump:
    os.makedirs(args.dump, exist_ok=True)
    h = {n: hashlib.sha256(getattr(res, n).contiguous().cpu().numpy().tobytes()).hexdigest()
         for n in ('samples', 'accepted', 'diverged', 'step_size', 'num_rejected')}
    with open(os.path.join(args.dump, 'diag_eps%g.json' % args.eps), 'w') as f:
        json.dump(dict(line, sha256=h), f)
