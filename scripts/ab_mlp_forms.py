"""Every output of the Bayesian-NN kernel (mlp_run_kernel) over a seeded matrix of runs, to one .npz: run it on two builds
and compare the files to show that a change to the kernel leaves every bit of every result as it was.

The matrix: the plain integrator and the three SPLITTING schemes x HMC / HMC_NUTS x a SIMT shape (1-10-10-1, D = 141)
and a tensor-core shape (16-128-1, D = 2305) x pinned cluster sizes 1, 2, 4 x no sink / thin = 3 with moments; then
hyperpriors (Philox and the injected stream, with and without a sink), replica exchange with swaps (regression and
classification, HMC and HMC_NUTS), K-fold runs, and the stand-alone split leapfrog.  Stored per run: samples, accept /
divergence flags, Hamiltonians, step sizes, reject counts, moments, tau traces, swap log-likelihoods -- every tensor the
result carries.  NUTS runs of the first block also carry a diagonal mass.

    python scripts/ab_mlp_forms.py OUT_DIR [--name NAME]        -> OUT_DIR/NAME.npz (NAME defaults to 'mlp_forms')
    python scripts/ab_mlp_forms.py --compare A.npz B.npz        -> lists the arrays that differ; exit 1 if any (CPU only)
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SCHEMES = ('PLAIN', 'SPLITTING', 'SPLITTING_RAND', 'SPLITTING_KMID')


def _arrays(prefix, res, out):
    """Every tensor attribute of a result (or the tensors of a tuple), as raw bytes-comparable numpy arrays."""
    import torch
    items = res.__dict__.items() if hasattr(res, '__dict__') else enumerate(res)
    for k, v in items:
        if torch.is_tensor(v):
            out['%s/%s' % (prefix, k)] = v.detach().cpu().contiguous().numpy()
        elif isinstance(v, (int, float)) and not isinstance(v, bool):
            out['%s/%s' % (prefix, k)] = np.asarray(v)


def collect():
    import torch
    import hamiltorch_b200 as hb
    from hamiltorch_b200 import engine, loo as LOO, samplers, targets as T, _native as N
    from oracle import cases

    integ = {'PLAIN': hb.Integrator.IMPLICIT, 'SPLITTING': hb.Integrator.SPLITTING,
             'SPLITTING_RAND': hb.Integrator.SPLITTING_RAND, 'SPLITTING_KMID': hb.Integrator.SPLITTING_KMID}
    code = {'SPLITTING': N.SCHEME_SPLIT_SYM, 'SPLITTING_RAND': N.SCHEME_SPLIT_RAND, 'SPLITTING_KMID': N.SCHEME_SPLIT_KMID}

    def problem(shape, task='regression'):
        if shape == 'tc':
            return cases.mlp_problem(seed=8, n=512, n_in=16, hidden=128, task=task)
        return cases.mlp_problem(seed=9, n=512, n_in=1, hidden=10, depth=2, task=task)

    loss = {'regression': 'regression', 'binary': 'binary_class_linear_output',
            'multiclass': 'multi_class_linear_output'}

    def targets(model, x, y, splits, cs, task='regression', tau=None, tau_out=20.):
        b = np.linspace(0, x.shape[0], splits + 1).astype(int)
        if splits == 1:
            parts = [T.MLPTarget.from_model(model, x, y, tau, tau_out, model_loss=loss[task])]
        else:
            parts = [T.MLPTarget.from_model(model, x[i:j], y[i:j], tau, tau_out, prior_scale=splits, model_loss=loss[task])
                     for i, j in zip(b[:-1], b[1:])]
        for d in parts:
            d.cluster_size = cs
        return parts[0] if splits == 1 else parts

    def tgt_dim(tgt):
        return (tgt[0] if isinstance(tgt, list) else tgt).dim

    def init(model, C_, seed, scale=0.05):
        q = hb.util.flatten(model).detach()
        return q[None] + scale * torch.randn(C_, q.numel(), generator=torch.Generator().manual_seed(seed))

    out = {}
    # the plain loop and the sink over schemes x samplers x shapes x cluster sizes
    for shape in ('simt', 'tc'):
        model, x, y = problem(shape)
        for scheme in SCHEMES:
            for cs in (1, 2, 4):
                tgt = targets(model, x, y, 1 if scheme == 'PLAIN' else 2, cs)
                for nuts in (False, True):
                    kw = dict(num_samples=12, num_steps_per_sample=3, step_size=0.004, burn=3, integrator=integ[scheme],
                              rng='philox', seed=11 + cs, record_ham=True,
                              sampler=hb.Sampler.HMC_NUTS if nuts else hb.Sampler.HMC)
                    if nuts:                                      # and a diagonal mass
                        kw['inv_mass'] = 0.5 + torch.rand(tgt_dim(tgt), generator=torch.Generator().manual_seed(cs))
                    q0 = init(model, 3, seed=cs)
                    for sink, skw in (('nosink', {}), ('thin3_moments', dict(thin=3, moments=True))):
                        name = 'run/%s/%s/cs%d/%s/%s' % (shape, scheme, cs, 'nuts' if nuts else 'hmc', sink)
                        _arrays(name, hb.sample_chains(tgt, q0, **kw, **skw), out)
    # hyperpriors: Philox and the injected stream (the gamma draws given), with and without a sink
    hyper = [(2.0, 1.0), (1.0, 1.0), (1.5, 0.5), None, (0.5, 2.0), (2.0, 0.05)]
    tau = [torch.tensor(t) for t in (2.0, 1.5, 3.0, 1.0, 1.0, 1.0)]
    for shape in ('simt', 'tc'):
        model, x, y = problem(shape)
        D = hb.util.flatten(model).numel()
        for scheme in ('PLAIN', 'SPLITTING'):
            for cs in (1, 2, 4):
                tgt = targets(model, x, y, 1 if scheme == 'PLAIN' else 2, cs, tau=tau[:2 * (len(model) // 2 + 1)])
                hy = hyper[:2 * (len(model) // 2 + 1)] + [hyper[-1]]
                C_, S = 3, 12
                sch = N.SCHEME_PLAIN if scheme == 'PLAIN' else code[scheme]
                q0 = init(model, C_, seed=20 + cs)
                for nuts in (False, True):
                    kw = dict(burn=3, record_ham=True, scheme=sch, hyper=hy, nuts=nuts)
                    base = 'hyper/%s/%s/cs%d/%s' % (shape, scheme, cs, 'nuts' if nuts else 'hmc')
                    _arrays(base + '/philox', engine.hmc_run(tgt, q0, S, 3, 0.004, seed=5, **kw), out)
                    _arrays(base + '/philox_thin2', engine.hmc_run(tgt, q0, S, 3, 0.004, seed=5, thin=2, moments=True,
                                                                   **kw), out)
                g = torch.Generator().manual_seed(cs)
                shapes = samplers._reference_gamma_shapes(tgt, hy).clamp_min(1.0)
                gam = torch.from_numpy(np.random.default_rng(cs).gamma(shapes.numpy(), size=(S, C_, len(hy))))
                z, lu = torch.randn(S, C_, D, generator=g), torch.log(torch.rand(S, C_, generator=g))
                _arrays('hyper/%s/%s/cs%d/injected' % (shape, scheme, cs),
                        engine.hmc_run(tgt, q0, S, 3, 0.004, burn=3, record_ham=True, scheme=sch, hyper=hy, gammas=gam,
                                       normals=z, log_uniforms=lu), out)
    # replica exchange with swaps
    betas = [1.0, 0.3, 0.1]
    for shape, task in (('simt', 'regression'), ('tc', 'regression'), ('simt', 'binary')):
        model, x, y = problem(shape, task)
        for scheme in ('PLAIN', 'SPLITTING_RAND'):
            for cs in (1, 2, 4):
                tgt = targets(model, x, y, 1 if scheme == 'PLAIN' else 2, cs, task=task,
                              tau_out=20. if task == 'regression' else 1.)
                for nuts in (False, True):
                    r = hb.sample_chains(tgt, init(model, 6, seed=30 + cs), num_samples=12, num_steps_per_sample=3,
                                         step_size=0.004, burn=3, integrator=integ[scheme], rng='philox', seed=7,
                                         record_ham=True, betas=betas, swap_every=2, moments=nuts,
                                         sampler=hb.Sampler.HMC_NUTS if nuts else hb.Sampler.HMC)
                    _arrays('temper/%s/%s/%s/cs%d/%s' % (shape, task, scheme, cs, 'nuts' if nuts else 'hmc'), r, out)
    # K-fold runs
    for shape in ('simt', 'tc'):
        model, x, y = problem(shape)
        for cs in (1, 2, 4):
            K = 4
            tgt = targets(model, x, y, 1, cs)
            f = LOO.kfold_split(x.shape[0], K, seed=cs)
            for nuts in (False, True):
                r = hb.sample_chains(tgt, init(model, 2 * K, seed=40 + cs), num_samples=12, num_steps_per_sample=3,
                                     step_size=0.004, burn=3, rng='philox', seed=9, record_ham=True, folds=f,
                                     thin=2 if nuts else 1, moments=nuts,
                                     sampler=hb.Sampler.HMC_NUTS if nuts else hb.Sampler.HMC)
                _arrays('folds/%s/cs%d/%s' % (shape, cs, 'nuts' if nuts else 'hmc'), r, out)
    # the stand-alone split leapfrog
    for shape in ('simt', 'tc'):
        model, x, y = problem(shape)
        for scheme in ('SPLITTING', 'SPLITTING_RAND', 'SPLITTING_KMID'):
            for cs in (1, 2, 4):
                tgt = targets(model, x, y, 2, cs)
                q0 = init(model, 3, seed=50 + cs)
                p0 = torch.randn(q0.shape, generator=torch.Generator().manual_seed(60 + cs))
                _arrays('leapfrog/%s/%s/cs%d' % (shape, scheme, cs),
                        engine.split_leapfrog(tgt, q0, p0, 4, 0.004, code[scheme], seed=3), out)
    torch.cuda.synchronize()
    return out


def compare(a_path, b_path):
    a, b = np.load(a_path), np.load(b_path)
    bad = sorted(set(a.files) ^ set(b.files))
    for k in sorted(set(a.files) & set(b.files)):
        x, y = a[k], b[k]
        if x.dtype != y.dtype or x.shape != y.shape or x.tobytes() != y.tobytes():
            bad.append(k)
    print('%d arrays, %d differ' % (len(set(a.files) | set(b.files)), len(bad)))
    for k in bad:
        print('  differs:', k)
    return 1 if bad else 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('out_dir', nargs='?')
    ap.add_argument('--name', default='mlp_forms')
    ap.add_argument('--compare', nargs=2, metavar=('A', 'B'))
    args = ap.parse_args()
    if args.compare:
        sys.exit(compare(*args.compare))
    if not args.out_dir:
        ap.error('OUT_DIR or --compare A B')
    out = collect()
    os.makedirs(args.out_dir, exist_ok=True)
    path = os.path.join(args.out_dir, args.name + '.npz')
    np.savez(path, **out)
    print('%d arrays -> %s' % (len(out), path))


if __name__ == '__main__':
    main()
