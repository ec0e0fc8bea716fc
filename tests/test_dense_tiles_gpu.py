"""GPU: the step-synchronous dense paths (hmcx_tc.cu) at every column-tile width, checked against the fp64
per-iteration replay of tests/dense_ref.py.

The width BN of dense_step_kernel / dense_lin_kernel (32, 64 or 128 columns; wgmma m64nBNk8, a BN-row packed layout of
every D x D operand, a 3-stage ring at 128) is picked from the batch: the widest that still gives ~100 CTAs, so small
batches always run BN = 32.  HMCX_DENSE_BN forces a width, which makes 64 and 128 reachable at C = 130 (two row tiles,
the second with 2 live rows); the workload-scale cases run C = 1000 under the default rule.  Every chain has its own step
size, so that a row / step-size mix-up across row tiles shows.

All widths accumulate each output element over the same K-chunk sequence; only the per-tile partial sums of the
Hamiltonian (NT = Dp / BN of them) are added in a different grouping.  So the states are bit-identical across widths
(measured on an H100, DESIGN.md section 4) and _assert_widths_agree asserts that; the Hamiltonians differ in the last bits.
"""
import os
import subprocess
import sys

import pytest
import torch

import hamiltorch_b200 as hb
from hamiltorch_b200 import engine, targets as T
from tests import dense_ref

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WIDTHS = (32, 64, 128)
OMEGA, ALPHA = 10.0, 1.0


def _full_target(D, seed):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(D, D, generator=g, dtype=torch.float64) / D ** 0.5
    return T.GaussianFull(torch.randn(D, generator=g), cov=A @ A.t() + 0.5 * torch.eye(D, dtype=torch.float64))


def _diag_target(D, seed):
    g = torch.Generator().manual_seed(seed)
    return T.GaussianDiag(torch.randn(D, generator=g), 0.4 + torch.rand(D, generator=g))


def _spd(D, seed):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(D, D, generator=g, dtype=torch.float64) / D ** 0.5
    return (A @ A.t() + 0.7 * torch.eye(D, dtype=torch.float64)).float()


def _problem(tgt, C, S, seed, eps0):
    """init (C, D) around the mean, injected streams z (S, C, D) / log u (S, C), per-chain step sizes (C,)."""
    D = tgt.dim
    g = torch.Generator().manual_seed(seed)
    mean = getattr(tgt, 'mean', torch.zeros(D))
    init = mean[None] + 0.3 * torch.randn(C, D, generator=g)
    z = torch.randn(S, C, D, generator=g)
    logu = torch.log(torch.rand(S, C, generator=g))
    logu[1::3, ::5] = 1.0               # > 0 >= rho: every fifth chain rejects iterations 1 (the :1018 quirk at burn 0) and 4
    eps = eps0 * (0.8 + 0.4 * torch.rand(C, generator=g))
    return init.cuda(), z.cuda(), logu.cuda(), eps.cuda()


def _run(tgt, init, z, logu, eps, S, L, bn=None, burn=0, inv_mass=None, rm=None, sched=None, monkeypatch=None):
    if bn is None:
        monkeypatch.delenv('HMCX_DENSE_BN', raising=False)
    else:
        monkeypatch.setenv('HMCX_DENSE_BN', str(bn))
    if rm is None:
        nuts = sched is not None
        res = engine.hmc_run(tgt, init, S, L, 0.2 if nuts else eps, burn=burn, inv_mass=inv_mass, nuts=nuts,
                             normals=z, log_uniforms=logu, record_ham=True, eps_schedule=sched, record_eps=nuts)
    else:
        res = engine.rmhmc_run(tgt, init, S, L, eps, burn=burn, softabs_const=ALPHA, explicit_binding_const=OMEGA,
                               explicit=rm['explicit'], softabs=rm['softabs'], normals=z, log_uniforms=logu,
                               record_ham=True)
    torch.cuda.synchronize()
    assert int(res.diverged.sum()) == 0
    return res


def _check(tag, model, init, z, logu, eps, res, L, burn=0):
    rep = dense_ref.replay(model, init, res.accepted, res.samples, z, eps, L, burn)
    return dense_ref.check(tag, rep, init, res.samples, res.accepted, res.ham, logu, burn)


def _assert_widths_agree(runs, burn=0):
    """Against BN = 32: identical decisions, and bit-identical retained states up to a chain's first differing decision
    (only a decision inside the Hamiltonian's summation noise may differ; the replay has bounded those already)."""
    a = runs[32]
    D = a.samples.shape[2]
    for bn, b in runs.items():
        S = a.accepted.shape[1]
        differ = a.accepted != b.accepted
        first = torch.where(differ.any(1), differ.int().argmax(1), torch.full_like(differ[:, 0], S, dtype=torch.long))
        slot = torch.arange(a.samples.shape[1], device=first.device)
        live = slot[None] + burn < first[:, None]
        same = (a.samples[..., :D] == b.samples[..., :D]).all(2)
        assert bool(same[live].all()), 'BN=%d: states differ from BN=32 before any decision does' % bn
        assert int(differ.sum()) <= 1, 'BN=%d: %d decisions differ from BN=32' % (bn, int(differ.sum()))


# ---- dense step (dense_step_kernel): GaussianFull, inv_mass None / 1-D -------------------------------------------------
@pytest.mark.parametrize('D', [250, 383])
@pytest.mark.parametrize('mass', ['none', 'diag'])
def test_dense_step_every_width_vs_fp64_replay(D, mass, monkeypatch):
    C, S, L = 130, 6, 4
    tgt = _full_target(D, 1)
    im = 0.5 + torch.rand(D, generator=torch.Generator().manual_seed(2)) if mass == 'diag' else None
    init, z, logu, eps = _problem(tgt, C, S, 3 + D, 0.25)
    model = dense_ref.HMC(tgt, im, device='cuda')
    runs = {bn: _run(tgt, init, z, logu, eps, S, L, bn=bn, inv_mass=im, monkeypatch=monkeypatch) for bn in WIDTHS}
    for bn, res in runs.items():
        _check('dense_tiles/step_d%d_%s/bn%d' % (D, mass, bn), model, init, z, logu, eps, res, L)
    assert 0 < int(runs[128].accepted.sum()) < C * S
    _assert_widths_agree(runs)


# ---- full inv_mass (dense_lin_kernel): GaussianFull (GEMM kick) and GaussianDiag (element-wise kick) -------------------
@pytest.mark.parametrize('D', [250, 380])
@pytest.mark.parametrize('target', ['full', 'diag'])
def test_full_mass_every_width_vs_fp64_replay(D, target, monkeypatch):
    C, S, L = 130, 6, 4
    tgt = _full_target(D, 11) if target == 'full' else _diag_target(D, 12)
    im = _spd(D, 13)
    init, z, logu, eps = _problem(tgt, C, S, 14 + D, 0.2)
    model = dense_ref.HMC(tgt, im, device='cuda')
    runs = {bn: _run(tgt, init, z, logu, eps, S, L, bn=bn, inv_mass=im, monkeypatch=monkeypatch) for bn in WIDTHS}
    for bn, res in runs.items():
        _check('dense_tiles/fullmass_d%d_%s/bn%d' % (D, target, bn), model, init, z, logu, eps, res, L)
    assert 0 < int(runs[128].accepted.sum()) < C * S
    _assert_widths_agree(runs)


# ---- constant-metric RMHMC above D = 128 (dense_rmhmc_run) -------------------------------------------------------------
RM_CASES = {
    'full_hessian_explicit': dict(target='full', softabs=False, explicit=True, eps=0.3),
    'full_softabs_implicit': dict(target='full', softabs=True, explicit=False, eps=0.3),
    'diag_hessian_explicit': dict(target='diag', softabs=False, explicit=True, eps=0.3),
}


@pytest.mark.parametrize('name', sorted(RM_CASES))
def test_constant_metric_rmhmc_every_width_vs_fp64_replay(name, monkeypatch):
    cs = RM_CASES[name]
    C, S, L, D = 130, 6, 3, 250
    tgt = _full_target(D, 21) if cs['target'] == 'full' else _diag_target(D, 22)
    init, z, logu, eps = _problem(tgt, C, S, 23, cs['eps'])
    if cs['explicit']:
        eps = torch.full_like(eps, cs['eps'])       # one binding rotation per launch: one step size (engine.rmhmc_run)
    model = dense_ref.RMHMC(tgt, cs['softabs'], ALPHA, explicit=cs['explicit'], omega=OMEGA, device='cuda')
    runs = {bn: _run(tgt, init, z, logu, eps, S, L, bn=bn, rm=cs, monkeypatch=monkeypatch) for bn in WIDTHS}
    for bn, res in runs.items():
        _check('dense_tiles/rmhmc_d%d_%s/bn%d' % (D, name, bn), model, init, z, logu, eps, res, L)
    assert 0 < int(runs[128].accepted.sum()) < C * S
    _assert_widths_agree(runs)


def test_explicit_rmhmc_refuses_per_chain_step_sizes():
    """The binding rotation cos/sin(2 omega eps) is one pair per launch: chains with other step sizes would integrate
    with the first chain's rotation, so per-chain step sizes are an error for the explicit integrator."""
    tgt = _full_target(24, 5)
    eps = torch.tensor([0.2, 0.3])
    with pytest.raises(NotImplementedError):
        engine.rmhmc_run(tgt, torch.zeros(2, 24), 3, 2, eps, explicit_binding_const=OMEGA)
    r = engine.rmhmc_run(tgt, torch.zeros(2, 24), 3, 2, torch.tensor([0.2, 0.2]), explicit_binding_const=OMEGA,
                         explicit=True)
    torch.cuda.synchronize()
    assert r.samples.shape == (2, 3, 24)


# ---- HMC_NUTS: teacher-forced step sizes, the kernel's own dual averaging recorded --------------------------------------
@pytest.mark.parametrize('mass', ['none', 'full'])
def test_nuts_wide_tile_vs_fp64_replay(mass, monkeypatch):
    C, S, L, D, burn = 130, 6, 4, 250, 3
    tgt = _full_target(D, 31)
    im = _spd(D, 32) if mass == 'full' else None
    init, z, logu, _ = _problem(tgt, C, S, 33, 0.2)
    sched = 0.2 * (0.8 + 0.4 * torch.rand(S, C, generator=torch.Generator().manual_seed(34))).cuda()
    res = _run(tgt, init, z, logu, None, S, L, bn=128, burn=burn, inv_mass=im, sched=sched, monkeypatch=monkeypatch)
    _check('dense_tiles/nuts_d%d_%s/bn128' % (D, mass), dense_ref.HMC(tgt, im, device='cuda'), init, z, logu, sched,
           res, L, burn)
    want = dense_ref.dual_averaging(res.ham, burn, 0.2)
    got = res.eps_trace[:, :burn + 1].double().cpu()
    torch.testing.assert_close(got, want, rtol=2e-4, atol=0)


# ---- workload scale, default width rule -------------------------------------------------------------------------------
WORKLOADS = {                      # C = 1000 (8 row tiles): what the rule should pick
    'step_d1500': dict(D=1500, kind='step', bn=128, other=64, eps=0.25),
    'step_d700': dict(D=700, kind='step', bn=64, other=128, eps=0.25),
    'fullmass_d1530': dict(D=1530, kind='fullmass', bn=128, other=64, eps=0.1),
    'fullmass_d1470': dict(D=1470, kind='fullmass', bn=64, other=32, eps=0.1),     # Dp 1472: NT = 23
    'rmhmc_d760': dict(D=760, kind='rmhmc', bn=64, other=32, eps=0.25),
}


@pytest.mark.parametrize('name', sorted(WORKLOADS))
def test_workload_scale_default_width_vs_fp64_replay(name, monkeypatch):
    w = WORKLOADS[name]
    C, S, L, D = 1000, 4, 3, w['D']
    tgt = _full_target(D, 41)
    im = _spd(D, 42) if w['kind'] == 'fullmass' else None
    rm = dict(explicit=True, softabs=False) if w['kind'] == 'rmhmc' else None
    init, z, logu, eps = _problem(tgt, C, S, 43, w['eps'])
    if rm:
        eps = torch.full_like(eps, w['eps'])
        model = dense_ref.RMHMC(tgt, False, explicit=True, omega=OMEGA, device='cuda')
    else:
        model = dense_ref.HMC(tgt, im, device='cuda')
    kw = dict(inv_mass=im, rm=rm, monkeypatch=monkeypatch)
    res = _run(tgt, init, z, logu, eps, S, L, **kw)
    _check('dense_tiles/workload_%s' % name, model, init, z, logu, eps, res, L)
    assert 0 < int(res.accepted.sum()) < C * S
    # the rule's choice is observable: the partial-sum grouping of the Hamiltonian is the width's fingerprint
    forced = _run(tgt, init, z, logu, eps, S, L, bn=w['bn'], **kw)
    other = _run(tgt, init, z, logu, eps, S, L, bn=w['other'], **kw)
    assert torch.equal(res.ham, forced.ham) and torch.equal(res.samples, forced.samples)
    assert not torch.equal(res.ham, other.ham)


def test_forced_width_must_fit(monkeypatch):
    """HMCX_DENSE_BN never runs a width it did not ask for: a value that is not 32 / 64 / 128 dividing the padded
    dimension is an error, not a fall-back."""
    tgt = _full_target(1470, 41)                    # full mass: Dp = 1472, not a multiple of 128
    init = tgt.mean[None].repeat(2, 1)
    for bad in ('128', '96', '16', 'x'):
        monkeypatch.setenv('HMCX_DENSE_BN', bad)
        with pytest.raises(RuntimeError):
            engine.hmc_run(tgt, init, 2, 2, 0.1, inv_mass=_spd(1470, 42))
    monkeypatch.setenv('HMCX_DENSE_BN', '64')
    engine.hmc_run(tgt, init, 2, 2, 0.1, inv_mass=_spd(1470, 42))
    torch.cuda.synchronize()


# ---- programmatic dependent launch off: the same bytes ----------------------------------------------------------------
def _pdl_case(path=None):
    """One wide-tile run of each GEMM kernel (dense step, full mass) at BN = 128; saved to `path` if given."""
    os.environ['HMCX_DENSE_BN'] = '128'
    out = []
    for im in (None, _spd(250, 52)):
        tgt = _full_target(250, 51)
        init, z, logu, eps = _problem(tgt, 130, 5, 53, 0.25)
        r = engine.hmc_run(tgt, init, 5, 4, eps, inv_mass=im, normals=z, log_uniforms=logu, record_ham=True)
        torch.cuda.synchronize()
        out += [r.samples.cpu(), r.accepted.cpu(), r.ham.cpu()]
    if path:
        torch.save(out, path)
    return out


def test_wide_tiles_without_pdl_give_the_same_bytes(tmp_path, monkeypatch):
    """HMCX_PDL is read once per process: the plain-stream-order run goes in a subprocess.  Equal bytes mean no kernel
    reads its predecessor's output before griddepcontrol.wait."""
    monkeypatch.setenv('HMCX_DENSE_BN', '128')
    pdl = _pdl_case()
    path = str(tmp_path / 'nopdl.pt')
    env = dict(os.environ, HMCX_PDL='0')
    subprocess.run([sys.executable, '-c', 'import sys; sys.path.insert(0, %r); from tests import test_dense_tiles_gpu '
                    'as m; m._pdl_case(%r)' % (ROOT, path)], cwd=ROOT, env=env, check=True, timeout=600)
    nopdl = torch.load(path)
    assert len(pdl) == len(nopdl) and all(torch.equal(a, b) for a, b in zip(pdl, nopdl))


# ---- Philox statistics at the workload scale (BN = 128 under the default rule) ------------------------------------------
def test_dense_gaussian_full_philox_statistics_c1000_d1500():
    D, C, S, L = 1500, 1000, 30, 8
    tgt = _full_target(D, 3)
    cov = torch.linalg.inv(tgt.prec.double())
    Lc = torch.linalg.cholesky(cov)
    init = tgt.mean[None] + (torch.randn(C, D, dtype=torch.float64, generator=torch.Generator().manual_seed(4)) @ Lc.t()).float()
    res = hb.sample_chains(tgt, init, num_samples=S, num_steps_per_sample=L, step_size=0.12, rng='philox', seed=5,
                           record_ham=True)
    torch.cuda.synchronize()
    assert int(res.diverged.sum()) == 0
    acc = res.accepted.float().mean().item()
    assert 0.6 < acc <= 1.0, acc
    u = torch.randn(D, dtype=torch.float64, generator=torch.Generator().manual_seed(6))
    u /= u.norm()
    proj = ((res.samples[:, S // 2:].cpu().double() - tgt.mean.double()) @ u)
    assert abs(proj.var().item() / float(u @ cov @ u) - 1.0) < 0.1
