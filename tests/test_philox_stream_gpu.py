"""GPU: every kernel's in-kernel Philox mode draws the canonical stream (tests/philox_ref.py, DESIGN.md "The canonical
random stream").

(a) engine.gibbs -- the momentum stream -- against the fp64 restatement of its Box-Muller transform, within the error
    bounds of the .approx instructions it is built from.
(b) For each kernel family: a run with ``seed=`` equals, bit for bit, the same run fed the injected stream built from the
    specification: normals = the GPU bits of engine.gibbs for every iteration (Box-Muller is not CPU-reproducible),
    log-uniforms, jitter rows and permutations from philox_ref.  A kernel that drew a wrong counter, reused a stream
    across calls or elements, ignored chain_offset or consumed the normals differently in the two modes fails here even
    when its moments look right.

The injected log-uniforms are correctly rounded; CUDA's logf is within 1 ulp of them.  Every test first checks that no
accept decision of the injected run lies within 4 ulp of its log-uniform, so that difference cannot flip one."""
import numpy as np
import pytest
import torch

import hamiltorch_b200 as hb
from hamiltorch_b200 import engine, targets as T, _native as N
from oracle import cases
from tests import philox_ref as P

pytestmark = pytest.mark.gpu

SEEDS = [0x9E3779B97F4A7C15, 0x0123456789ABCDEF, 0xFFFFFFFF00000001]      # nonzero high words: they enter the key
OFFSETS = [0, 7, 2 ** 32 + 3]                                               # 2^32 + 3: the chain's high word enters the key


# ----------------------------------------------------------------------------------------------------------
# (a) the momentum stream
# ----------------------------------------------------------------------------------------------------------
# Error bounds of the instructions of box_muller (hmcx_common.cuh), from the PTX ISA / CUDA C++ Programming Guide:
LG2_ABS = 2.0 ** -22          # lg2.approx.ftz.f32: absolute error for arguments in [0.5, 2] ...
LG2_REL = 2.0 ** -22          # ... and 2 ulp elsewhere
SQRT_REL = 2.0 ** -22         # sqrt.approx.ftz.f32: relative error (2 ulp)
SINCOS_ABS = 2.0 ** -20.5     # __sincosf (sin / cos.approx.ftz.f32): absolute error on [-pi, pi]
F32 = 2.0 ** -24              # one correctly rounded fp32 operation


@pytest.mark.parametrize('seed,chain_offset,n', [(SEEDS[0], 0, 0), (SEEDS[1], 7, 12345), (SEEDS[2], 2 ** 32 + 3, 2 ** 31 - 5)])
def test_gibbs_matches_the_restated_box_muller(seed, chain_offset, n):
    D, C = 37, 64                                            # D % 4 == 1: the last vector's pair (z, w) is half padding
    z = engine.gibbs(D, C, seed, iteration=n, chain_offset=chain_offset).double().cpu().numpy()
    w = P.momentum_words(seed, chain_offset + np.arange(C, dtype=np.uint64), n, D)          # (C, nv, 4)
    R2, TH = (a.reshape(C, -1) for a in P.box_muller_pairs(w[..., 0::2], w[..., 1::2]))     # per element pair
    L = R2 / (-2.0 * np.log(2.0))                                                           # the exact lg2(u)
    # radius: lg2 error, the fp32 product with -2 ln 2, sqrt.approx (squared), sin^2 + cos^2 - 1 and the two fp32
    # products r*cos, r*sin (squared); factor 2 for the neglected second-order terms
    tol_r2 = 2 * (2 * np.log(2.0) * (LG2_ABS + LG2_REL * np.abs(L)) +
                  R2 * (F32 + 2 * SQRT_REL + 2 * np.sqrt(2.0) * SINCOS_ABS + 4 * F32))
    # angle: (float)b (2^-24 relative on b < 2^32), the fp32 constants and the FFMA rounding (half an ulp at |x| <= pi
    # each), sin / cos absolute errors seen as an angle, and the fp32 products; factor 2 as above
    tol_th = 2 * (2 * np.pi * F32 + 2 * np.pi * F32 + 2 * 2.0 ** -23 + 2 * np.pi * 2.0 ** -32 +
                  np.sqrt(2.0) * SINCOS_ABS + 2 * F32)
    full = D // 2                                            # element pairs that lie inside the chain
    z0, z1 = z[:, 0:2 * full:2], z[:, 1:2 * full:2]
    r2 = z0 * z0 + z1 * z1
    assert np.all(np.abs(r2 - R2[:, :full]) <= tol_r2[:, :full]), np.max(np.abs(r2 - R2[:, :full]) / tol_r2[:, :full])
    big = R2[:, :full] > 1e-6
    dth = np.angle(np.exp(1j * (np.arctan2(z1, z0) - TH[:, :full])))                      # difference modulo 2 pi
    assert np.all(np.abs(dth[big]) <= tol_th), np.max(np.abs(dth[big]))
    # the odd element: z0 of pair D // 2
    last = np.sqrt(R2[:, full]) * np.cos(TH[:, full])
    assert np.all(np.abs(z[:, D - 1] - last) <= np.sqrt(tol_r2[:, full]) + np.sqrt(R2[:, full]) * tol_th)
    # and the whole row against the restated normals
    assert np.allclose(z, P.normals(seed, chain_offset + np.arange(C, dtype=np.uint64), n, D), rtol=0, atol=5e-5)


def test_gibbs_streams_are_distinct_per_chain_iteration_and_seed():
    a = engine.gibbs(8, 4, SEEDS[0], iteration=3, chain_offset=2 ** 32 + 3).cpu()
    assert not torch.equal(a, engine.gibbs(8, 4, SEEDS[0], iteration=4, chain_offset=2 ** 32 + 3).cpu())
    assert not torch.equal(a, engine.gibbs(8, 4, SEEDS[0], iteration=3, chain_offset=3).cpu())     # high word of chain
    assert not torch.equal(a, engine.gibbs(8, 4, SEEDS[0] ^ (1 << 40), iteration=3, chain_offset=2 ** 32 + 3).cpu())
    b = engine.gibbs(8, 6, SEEDS[0], iteration=3, chain_offset=2 ** 32 + 1).cpu()
    assert torch.equal(a, b[2:])                             # chain c = chain_offset + local c


# ----------------------------------------------------------------------------------------------------------
# (b) Philox == injected, per kernel family
# ----------------------------------------------------------------------------------------------------------
def _stream(seed, chain_offset, C, S, D, M=0, J=0):
    """The injected form of the canonical stream of chains chain_offset .. chain_offset + C - 1, iterations 0 .. S-1."""
    chains, its = chain_offset + np.arange(C, dtype=np.uint64), np.arange(S)
    z = torch.stack([engine.gibbs(D, C, seed, iteration=n, chain_offset=chain_offset) for n in range(S)])
    s = dict(normals=z, log_uniforms=torch.from_numpy(P.log_uniforms(seed, chains, its)))
    if M:
        s['perms'] = torch.from_numpy(P.perms(seed, chains, its, M))
    if J:
        s['uniforms'] = torch.from_numpy(P.jitter_rows(seed, chains, its, J, D))
    return s


def _bits(t):
    t = t.detach().cpu().contiguous()
    return t.view(torch.int32) if t.dtype == torch.float32 else t       # NaN Hamiltonians compare too


def _assert_decisions_clear(res, logu):
    """No accept decision of the run lies within 4 ulp of its log-uniform (a tie the 1-ulp logf difference could flip)."""
    ham = res.ham.detach().cpu()
    rho = torch.clamp(ham[..., 0] - ham[..., 1], max=0.0).numpy()                   # min(0, H_old - H_new) in fp32
    lu = logu.t().numpy()
    live = np.isfinite(rho) & ~res.diverged.cpu().numpy().astype(bool) & (lu != 0)
    close = live & (np.abs(rho.astype(np.float64) - lu) <= 4 * np.spacing(np.abs(lu)))
    assert not close.any(), 'an accept decision within 4 ulp of its log-uniform: choose another seed'
    assert live.any()


def _assert_same(a, b):
    for k in ('accepted', 'diverged', 'num_rejected', 'step_size', 'ham', 'eps_trace', 'moment_sum', 'moment_sumsq',
              'final_state'):
        x, y = getattr(a, k, None), getattr(b, k, None)
        assert (x is None) == (y is None), k
        if x is not None:
            assert torch.equal(_bits(x), _bits(y)), k
    if a.samples_padded is not None:
        assert torch.equal(_bits(a.samples), _bits(b.samples)), 'samples'
    # a run that rejects everything, or accepts everything, tests less than it seems
    acc = a.accepted.cpu().bool()
    assert acc.any(), 'no proposal accepted'


def _philox_vs_injected(run, seed, chain_offset, C, S, D, M=0, J=0):
    """run(**rng) -> HMCResult with record_ham; rng = dict(seed=, chain_offset=) or the injected stream."""
    ph = run(seed=seed, chain_offset=chain_offset)
    s = _stream(seed, chain_offset, C, S, D, M, J)
    inj = run(**s)
    torch.cuda.synchronize()
    _assert_decisions_clear(inj, s['log_uniforms'])
    _assert_same(ph, inj)
    return ph


def _init(C, D, seed, scale=0.5, mean=None):
    x = scale * torch.randn(C, D, generator=torch.Generator().manual_seed(seed))
    return x if mean is None else x + mean


def _elem(tk, mk, D, seed):
    g = torch.Generator().manual_seed(seed)
    tgt = T.GaussianIso(D) if tk == 'iso' else T.GaussianDiag(torch.linspace(-1, 1, D), 0.5 + torch.rand(D, generator=g))
    im = None if mk == 'none' else 0.5 + torch.rand(D, generator=g)
    return tgt, im


TKMK = [('iso', 'none'), ('iso', 'diag'), ('diag', 'none'), ('diag', 'diag')]
# name -> (D, engine.hmc_run keyword arguments).  Kernel each one reaches (hmcx_hmc.cu, elem_hmc_run):
ELEM_CASES = {
    'k1_256': (37, {}),                                       # <E=4, K=1, 256>, NUTS=false / injected NUTS=true
    'k1_256_nuts': (37, dict(nuts=True, record_eps=True)),    # the NUTS=true instantiation
    'paired': (999, {}),                                      # the paired K=2 form (768 < ld <= 1024, Philox only)
    'k1_1024': (2000, {}),
    'k2_512': (3000, {}),
    'tuning2': (997, dict(tuning=2)),                         # runtime rng_mode branch
    'tuning4': (997, dict(tuning=4)),
    'tuning21': (997, dict(tuning=21)),
    'tuning22': (997, dict(tuning=22)),
    'cluster4': (997, dict(tuning=41)),
    'cluster2': (997, dict(tuning=42)),
    'sink': (101, dict(thin=3, moments=True)),
    'host_windows': (37, dict(host_windows=3)),
    'big': (4100, {}),                                        # hmc_run_big_kernel (ld > 4096)
}


@pytest.mark.parametrize('tk,mk', TKMK)
@pytest.mark.parametrize('name', sorted(ELEM_CASES))
def test_hmc_run_kernel_families(name, tk, mk):
    D, kw = ELEM_CASES[name]
    i = sorted(ELEM_CASES).index(name) + 5 * TKMK.index((tk, mk))
    seed, chain_offset = SEEDS[i % 3], OFFSETS[(i + 1) % 3]
    C, S, L, burn = 4, 12, 4, 3
    tgt, im = _elem(tk, mk, D, i)
    q0 = _init(C, D, i, mean=None if tk == 'iso' else tgt.mean)
    eps = 0.9 * D ** -0.25

    def run(**rng):
        extra = dict(kw)
        if extra.pop('host_windows', 0):
            keep = S - burn
            extra.update(host_windows=3, out=torch.empty((C, keep, N.padded_ld(D)), dtype=torch.float32, pin_memory=True))
        return engine.hmc_run(tgt, q0, S, L, eps, burn=burn, inv_mass=im, record_ham=True, **rng, **extra)
    _philox_vs_injected(run, seed, chain_offset, C, S, D)


def _spd(D, seed):
    return cases._spd64(D, seed).float()


SMALL_CASES = {            # hmc_small_kernel (D <= 16: coupled gradient or full mass, one thread per chain)
    'full5': lambda: (T.GaussianFull(torch.linspace(-0.5, 0.5, 5), cov=_spd(5, 1)), None, 0.3),
    'full5_nuts': lambda: (T.GaussianFull(torch.linspace(-0.5, 0.5, 5), cov=_spd(5, 1)), None, 0.3),
    'funnel3': lambda: (T.Funnel(3), None, 0.1),
    'blocks6': lambda: (T.GaussianDiag(torch.linspace(-1, 1, 6), 0.5 + torch.arange(6.) / 6),
                        [_spd(2, 2), _spd(4, 3)], 0.3),
    'funnel2_mass': lambda: (T.Funnel(2), _spd(2, 4), 0.1),                        # DM = 2
    'full16_nuts': lambda: (T.GaussianFull(torch.linspace(-0.5, 0.5, 16), cov=_spd(16, 5)), None, 0.2),   # DM = 16
}


@pytest.mark.parametrize('name', sorted(SMALL_CASES))
def test_small_kernel(name):
    tgt, im, eps = SMALL_CASES[name]()
    D, C, S = tgt.dim, 37, 14
    nuts = name.endswith('nuts')
    q0 = _init(C, D, 3, scale=0.3) + (torch.tensor([0.] + [1.] * (D - 1)) if name.startswith('funnel') else 0)

    def run(**rng):
        return engine.hmc_run(tgt, q0, S, 5, eps, burn=3, inv_mass=im, nuts=nuts, record_eps=nuts, record_ham=True, **rng)
    _philox_vs_injected(run, SEEDS[1], OFFSETS[2] if name != 'funnel3' else OFFSETS[1], C, S, D)


DENSE_CASES = {            # (target, inv_mass, C, eps, nuts)
    # flow_small_kernel (hmcx_flow.cu: D <= 128, matrices in shared memory)
    'flow_full96': lambda: (T.GaussianFull(torch.linspace(-0.5, 0.5, 96), cov=_spd(96, 4)), None, 5, 0.15, False),
    'flow_iso48_mass': lambda: (T.GaussianIso(48), _spd(48, 5), 5, 0.2, False),
    'flow_iso48_mass_nuts': lambda: (T.GaussianIso(48), _spd(48, 5), 5, 0.2, True),
    # tensor-core path (hmcx_tc.cu, D > 128): dense_step on a dense precision, dense_lin with a full mass matrix
    'tc_full200': lambda: (T.GaussianFull(torch.linspace(-0.5, 0.5, 200), cov=_spd(200, 6)), None, 130, 0.1, False),
    'tc_diag150_mass': lambda: (T.GaussianDiag(torch.linspace(-1, 1, 150), 0.5 + torch.rand(150, generator=torch.Generator().manual_seed(7))),
                                _spd(150, 8), 130, 0.15, False),
}


@pytest.mark.parametrize('name', sorted(DENSE_CASES))
def test_flow_and_tensor_core_paths(name):
    tgt, im, C, eps, nuts = DENSE_CASES[name]()
    D, S = tgt.dim, 10
    q0 = _init(C, D, 9, scale=0.3)

    def run(**rng):
        return engine.hmc_run(tgt, q0, S, 4, eps, burn=2, inv_mass=im, nuts=nuts, record_eps=nuts, record_ham=True, **rng)
    i = sorted(DENSE_CASES).index(name)
    _philox_vs_injected(run, SEEDS[i % 3], OFFSETS[(i + 2) % 3], C, S, D)


# ---- Bayesian-NN kernel (mlp_run_kernel) ----
SCHEMES = {'PLAIN': None, 'SPLITTING': hb.Integrator.SPLITTING, 'SPLITTING_RAND': hb.Integrator.SPLITTING_RAND,
           'SPLITTING_KMID': hb.Integrator.SPLITTING_KMID}


@pytest.mark.parametrize('cluster', [1, 2, 4])
@pytest.mark.parametrize('shape', ['tc', 'simt'])
@pytest.mark.parametrize('scheme', sorted(SCHEMES))
def test_mlp_run_kernel(scheme, shape, cluster):
    if shape == 'tc':                                        # 16 -> 128 -> 1 on the tensor cores, D = 2305
        model, x, y = cases.mlp_problem(seed=8, n=512, n_in=16, hidden=128)
    else:                                                    # 1 -> 10 -> 10 -> 1, SIMT, D = 141 (D % 4 != 0)
        model, x, y = cases.mlp_problem(seed=9, n=512, n_in=1, hidden=10, depth=2)
    M = 3
    if scheme == 'PLAIN':
        target, integ = T.MLPTarget.from_model(model, x, y, None, 20.), hb.Integrator.IMPLICIT
        target.cluster_size = cluster
    else:
        b = np.linspace(0, x.shape[0], M + 1).astype(int)
        target = [T.MLPTarget.from_model(model, x[i:j], y[i:j], None, 20., prior_scale=M) for i, j in zip(b[:-1], b[1:])]
        target[0].cluster_size = cluster
        integ = SCHEMES[scheme]
    D = hb.util.flatten(model).numel()
    C, S = 3, 10
    q0 = hb.util.flatten(model).detach()[None] + 0.05 * torch.randn(C, D, generator=torch.Generator().manual_seed(cluster))
    i = sorted(SCHEMES).index(scheme) + cluster

    def run(seed=None, chain_offset=0, perms=None, **inj):
        kw = dict(rng='injected', perms=perms, **inj) if inj else dict(rng='philox', seed=seed, chain_offset=chain_offset)
        return hb.sample_chains(target, q0, num_samples=S, num_steps_per_sample=3, step_size=0.004, burn=2,
                                integrator=integ, record_ham=True, **kw)
    _philox_vs_injected(run, SEEDS[i % 3], OFFSETS[i % 3], C, S, D, M=M if scheme == 'SPLITTING_RAND' else 0)


# ---- RMHMC ----
def _rm_run(tgt, q0, S, L, eps, explicit, jitter=1e-3, softabs_const=1e6):
    def run(seed=0, chain_offset=0, **inj):
        return engine.rmhmc_run(tgt, q0, S, L, eps, burn=1, jitter=jitter, softabs_const=softabs_const,
                                explicit_binding_const=10, fixed_point_max_iterations=6, explicit=explicit,
                                softabs=softabs_const is not None, seed=seed, chain_offset=chain_offset,
                                record_ham=True, **inj)
    return run


# The explicit integrator makes 8L+3 fisher() calls per iteration, plus NaN retries; the implicit one at most
# L (2 F + 2) + 3 with F = fixed_point_max_iterations = 6 (plus retries).  Injected mode re-uses its last row once it
# runs out, so J leaves headroom over both.
RM_J = 64


def test_rmhmc2_quad_kernel_config3_settings():
    """BASELINE config 3's kernel (D = 2, explicit): 2-D funnel, softabs 1e6, omega 10, eps .05, L = 10, jitter 1e-3.
    40 chains = one full and one partial CTA of 32."""
    C, S, L = 40, 8, 10
    q0 = torch.tensor([0., 1.]).repeat(C, 1) + _init(C, 2, 11, scale=0.1)
    run = _rm_run(T.Funnel(2), q0, S, L, 0.05, True)
    _philox_vs_injected(run, SEEDS[0], OFFSETS[1], C, S, 2, J=8 * L + 3 + 16)


@pytest.mark.parametrize('explicit', [True, False])
def test_rmhmc_run_kernel_funnel10_jitter(explicit):
    C, S = 5, 10
    q0 = torch.tensor([0.] + [0.5] * 9).repeat(C, 1) + _init(C, 10, 12, scale=0.1)
    run = _rm_run(T.Funnel(10), q0, S, 3, 0.05, explicit)
    _philox_vs_injected(run, SEEDS[2], OFFSETS[2], C, S, 10, J=RM_J)


@pytest.mark.parametrize('explicit', [True, False])
@pytest.mark.parametrize('D', [24, 48])
def test_rmhmc_cta_kernel_jitter(D, explicit):
    """One CTA per chain, 16 < D <= 64.  At D = 48 every fisher() call's jitter row spans 12 counter vectors: the rows
    of consecutive calls must not share counters (they did with a stride of 8 vectors per call)."""
    C, S = 4, 8
    tgt = T.GaussianFull(torch.linspace(-0.5, 0.5, D), cov=cases._spd64(D, 75))
    q0 = _init(C, D, 13, scale=0.2)
    run = _rm_run(tgt, q0, S, 3, 0.3, explicit, softabs_const=1e3)
    _philox_vs_injected(run, SEEDS[D // 24], OFFSETS[1 + explicit], C, S, D, J=RM_J)


@pytest.mark.parametrize('D', [64, 200])
def test_rmhmc_constant_metric_dense_path(D):
    """Gaussian without jitter: hmcx_rmhmc_dense_run (D = 64 persistent flow kernel, D = 200 tensor cores)."""
    C, S = 5, 8
    tgt = T.GaussianFull(torch.linspace(-0.5, 0.5, D), cov=cases._spd64(D, 71))
    q0 = _init(C, D, 14, scale=0.3)
    run = _rm_run(tgt, q0, S, 3, 0.2 if D == 64 else 0.12, True, jitter=None, softabs_const=None)
    _philox_vs_injected(run, SEEDS[1], OFFSETS[D // 100], C, S, D)


# ---- stand-alone calls ----
@pytest.mark.parametrize('explicit', [True, False])
def test_standalone_rmhmc_leapfrog_and_hamiltonian_d48_jitter(explicit):
    """engine.rmhmc_leapfrog / rmhmc_hamiltonian draw their jitter rows at iteration 0 of chains 0 .. C-1."""
    D, C, seed = 48, 3, SEEDS[2]
    tgt = T.GaussianFull(torch.linspace(-0.5, 0.5, D), cov=cases._spd64(D, 75))
    q, p = _init(C, D, 15, scale=0.2), _init(C, D, 16, scale=1.0)
    uni = torch.from_numpy(P.jitter_rows(seed, np.arange(C), [0], RM_J, D)[0])            # (C, J, D)
    kw = dict(jitter=1e-3, softabs_const=1e3, softabs=True)
    lf = dict(kw, explicit_binding_const=10, explicit=explicit)
    a = engine.rmhmc_leapfrog(tgt, q, p, 3, 0.3, seed=seed, **lf)
    b = engine.rmhmc_leapfrog(tgt, q, p, 3, 0.3, uniforms=uni, **lf)
    for x, y, k in zip(a, b, ('q_traj', 'p_traj', 'q_copy', 'p_copy', 'failed')):
        assert torch.equal(_bits(x), _bits(y)), k
    assert not a[4].any()
    Ha, fa = engine.rmhmc_hamiltonian(tgt, q, p, seed=seed, **kw)
    Hb, fb = engine.rmhmc_hamiltonian(tgt, q, p, uniforms=uni, **kw)
    assert torch.equal(_bits(Ha), _bits(Hb)) and torch.equal(fa, fb) and not fa.any()


def test_standalone_split_leapfrog_perms():
    """engine.split_leapfrog(SPLITTING_RAND) draws randperm(M) from the perm stream at iteration 0 of chains 0 .. C-1."""
    model, x, y = cases.mlp_problem(seed=9, n=256, n_in=1, hidden=10, depth=2)
    M, C, seed = 5, 4, SEEDS[0]
    b = np.linspace(0, x.shape[0], M + 1).astype(int)
    descs = [T.MLPTarget.from_model(model, x[i:j], y[i:j], None, 20., prior_scale=M) for i, j in zip(b[:-1], b[1:])]
    D = descs[0].dim
    q = hb.util.flatten(model).detach()[None] + 0.05 * torch.randn(C, D, generator=torch.Generator().manual_seed(1))
    p = torch.randn(C, D, generator=torch.Generator().manual_seed(2))
    pm = torch.from_numpy(P.perms(seed, np.arange(C), [0], M)[0])
    assert len({tuple(r) for r in pm.tolist()}) > 1
    a = engine.split_leapfrog(descs, q, p, 4, 0.004, N.SCHEME_SPLIT_RAND, seed=seed)
    b = engine.split_leapfrog(descs, q, p, 4, 0.004, N.SCHEME_SPLIT_RAND, perms=pm)
    for u, v in zip(a, b):
        assert torch.equal(_bits(u), _bits(v))
