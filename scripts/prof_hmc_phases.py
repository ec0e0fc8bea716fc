"""Developer tool: where an iteration of the paired config-2 HMC loop goes, from clock64() stamps.

Builds a variant of the library with -DHMCX_HMC_PROF in a temporary directory (hmcx_hmc.cu recompiled, linked with the
other objects of the in-tree build, which must exist: `python -m hamiltorch_b200.build`), runs config 2 (256 chains,
D=1024, L=10, S=1000, in-kernel Philox) and prints one JSON line.  The kernel stamps lane 0 of each of the 4 warps of
every CTA over 64 consecutive iterations (from iteration 256):
  0 the iteration's trajectory starts (gibbs)      1 trajectory and per-thread sums done
  2 slots published                                3 next iteration's normals drawn
  4 the reduction's barrier passed                 5 MH decided, state selected, row stored
  6, 7 (producer form) before and after the wait for the iteration's momentum slot, just before stamp 0
and, in the producer form, when producer warp 0 published each iteration's slot.
Reported per stamp id k: cycles from stamp 0 of the same iteration (mean, std, p10, p90); `iter`: stamp 0 to the next
iteration's stamp 0; `tail`: stamp 1 to the next iteration's stamp 0 (the serial section between two trajectories).
`both_in_tail`: for SMs holding two of the chains, cycles per iteration during which warp 0 of both chains sat in
their tail at once (clock64 is per SM, so the two chains' stamps share a time base).  `slot_wait`: stamp 6 to
stamp 7, how long the compute warps waited for the producer warps (all zero without them).  `published`: the slot's
publication minus stamp 6 of compute warp 0 in the same iteration (negative: the slot was ready before the compute
warps asked for it; null without producer warps)."""
import argparse, ctypes as C, json, os, subprocess, sys, tempfile
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from hamiltorch_b200 import build as B

CTAS, WARPS, ITS, IDS = 256, 4, 64, 8


def build_variant(tmp):
    src = os.path.join(B.CSRC, 'hmcx_hmc.cu')
    obj = os.path.join(tmp, 'hmcx_hmc.o')
    subprocess.check_call([B._nvcc()] + B.NVCC_FLAGS + ['-DHMCX_HMC_PROF', '-c', src, '-o', obj])
    objs = [obj] + [B._obj_of(s) for s in B.sources() if os.path.basename(s) != 'hmcx_hmc.cu']
    missing = [o for o in objs if not os.path.exists(o)]
    if missing:
        raise SystemExit('build the library first (python -m hamiltorch_b200.build): missing %s' % missing)
    lib = os.path.join(tmp, 'libhmcx.so')
    subprocess.check_call([B._nvcc(), '-shared', '-o', lib] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a'])
    return lib


def stats(x):
    x = np.asarray(x, dtype=np.float64)
    return {'mean': round(float(x.mean()), 1), 'std': round(float(x.std()), 1),
            'p10': float(np.percentile(x, 10)), 'p90': float(np.percentile(x, 90))}


def overlap(a, b):
    """total length of the intersection of two sorted lists of disjoint intervals"""
    i = j = 0
    tot = 0
    while i < len(a) and j < len(b):
        lo, hi = max(a[i][0], b[j][0]), min(a[i][1], b[j][1])
        tot += max(0, hi - lo)
        if a[i][1] < b[j][1]:
            i += 1
        else:
            j += 1
    return tot


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--eps', type=float, default=0.05)
    ap.add_argument('--init-scale', type=float, default=0.1)
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    tmp = tempfile.mkdtemp(prefix='hmcx_prof_')
    from hamiltorch_b200 import _native as N
    N.LIB_PATH = build_variant(tmp)
    import torch
    from hamiltorch_b200 import engine, targets as T
    lib = N.load_library()
    lib.hmcx_debug_hmc_prof.restype = C.c_int
    dev = torch.device('cuda', 0)
    tgt = engine.NativeTarget(T.GaussianIso(1024), dev)
    q0 = (args.init_scale * torch.randn(256, 1024, generator=torch.Generator().manual_seed(0))).to(dev)
    out = torch.empty((256, 1000, 1024), dtype=torch.float32, device=dev)
    stamps = (C.c_longlong * (CTAS * WARPS * ITS * IDS))()
    sm = (C.c_int * CTAS)()
    pub = (C.c_longlong * (CTAS * ITS))()
    engine.hmc_run(tgt, q0, 1000, 10, args.eps, seed=0, out=out, device=dev)
    lib.hmcx_debug_hmc_prof(stamps, sm, pub)
    rel = {k: [] for k in range(1, 6)}
    it, tail, both, rate, wait, published = [], [], [], [], [], []
    for rep in range(args.reps):
        r = engine.hmc_run(tgt, q0, 1000, 10, args.eps, seed=1 + rep, out=out, device=dev)
        lib.hmcx_debug_hmc_prof(stamps, sm, pub)
        rate.append(float(r.accepted.float().mean()))
        s = np.frombuffer(stamps, dtype=np.int64).reshape(CTAS, WARPS, ITS, IDS).astype(np.float64)
        for k in rel:
            rel[k].append((s[..., k] - s[..., 0]).ravel())
        it.append((s[:, :, 1:, 0] - s[:, :, :-1, 0]).ravel())
        wait.append((s[..., 7] - s[..., 6]).ravel())
        pb = np.frombuffer(pub, dtype=np.int64).reshape(CTAS, ITS).astype(np.float64)
        if pb.all():
            published.append((pb - s[:, 0, :, 6]).ravel())
        tail.append((s[:, :, 1:, 0] - s[:, :, :-1, 1]).ravel())
        by_sm = {}
        for b in range(CTAS):
            by_sm.setdefault(sm[b], []).append(b)
        for ctas in by_sm.values():
            if len(ctas) != 2:
                continue
            iv = [[(s[b, 0, i, 1], s[b, 0, i + 1, 0]) for i in range(ITS - 1)] for b in ctas]
            lo = max(iv[0][0][0], iv[1][0][0])
            hi = min(iv[0][-1][1], iv[1][-1][1])
            if hi <= lo:
                continue
            clip = [[(max(x, lo), min(y, hi)) for x, y in v if y > lo and x < hi] for v in iv]
            n_it = np.mean([len(v) for v in clip])
            both.append(overlap(*clip) / n_it)
    line = {'eps': args.eps, 'init_scale': args.init_scale, 'accept_rate': rate,
            'since_stamp0': {str(k): stats(np.concatenate(v)) for k, v in rel.items()},
            'iter': stats(np.concatenate(it)), 'slot_wait': stats(np.concatenate(wait)),
            'published': stats(np.concatenate(published)) if published else None, 'tail': stats(np.concatenate(tail)),
            'both_in_tail': stats(both) if both else None, 'sm_pairs': len(both) // args.reps}
    print(json.dumps(line))


if __name__ == '__main__':
    main()
