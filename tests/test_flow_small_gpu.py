"""GPU: the persistent small-D flow kernel (hmcx_flow.cu, flow_small_kernel<NJ, R>, 16 < D <= 128) at every chains-per-warp
count R, every register-slot count NJ = ceil(D / 32) and the CTA shapes of workload batches, checked against the fp64
per-iteration replay of tests/dense_ref.py.

The launch picks R from the batch (C <= 4 SMs -> 1, <= 12 SMs -> 2, else 4) and w warps per CTA from the warp count, so
small test batches only ever run R = 1 in single-warp CTAs.  HMCX_FLOW_R and HMCX_FLOW_W force both.  At C = 131 the
last warp carries dead slots at R = 2 (1 live, 1 dead) and R = 4 (3 live, 1 dead): a dead slot shadows chain C - 1,
computes alongside it and must never store.  Every chain has its own step size (one per launch for explicit RMHMC, whose
binding rotation is shared), so a slot / step-size mix-up shows.

The number of partial sums per output element is a function of D only and every chain's arithmetic stays in its own
registers and staging row, so R and w never change a chain's bits; the tests assert byte equality with R = 1 for every
output.  _flow_geometry restates the host launch rule (tests/test_flow_geometry_cpu.py checks it against the C++); the
workload cases confirm with the profiler which instantiation the rule launched, since R leaves no trace in the bits.
"""
import time

import numpy as np
import pytest
import torch

from hamiltorch_b200 import engine, targets as T
from tests import dense_ref
from tests.test_dense_tiles_gpu import _diag_target, _full_target, _problem, _spd
from tests.test_philox_stream_gpu import OFFSETS, SEEDS, _philox_vs_injected

pytestmark = pytest.mark.gpu

OMEGA, ALPHA = 10.0, 1.0
NUTS_EPS0 = 0.2                         # step_size of a NUTS run: mu = log(10 eps0) of its dual averaging
SMEM_OPTIN_H100 = 232448                # cudaDevAttrMaxSharedMemoryPerBlockOptin of sm_90


def _flow_geometry(C, D, nmat, sms, R=None, wmax=None):
    """The launch rule of flow_geometry (hmcx_flow.cu) -> (R, w, grid, smem_bytes): R chains per warp, w warps per CTA,
    grid CTAs.  nmat: the D x D matrices held in shared memory (1 for a GaussianFull target, + 2 for a full mass or a
    constant metric).  R / wmax: HMCX_FLOW_R / HMCX_FLOW_W.  C may be an integer array (then so are the results)."""
    NJ = (D + 31) // 32
    DP, K4 = 32 * NJ, (D + 3) // 4 * 4
    if R is None:
        R = np.where(C <= 4 * sms, 1, np.where(C <= 12 * sms, 2, 4))
    warps = -(-C // R)
    matrix_bytes = nmat * K4 * DP * 4
    if wmax is None:
        wmax = 4 if matrix_bytes <= 100 * 1024 else 8
    w = np.clip(-(-warps // sms), 1, wmax)
    grid = -(-warps // w)
    smem = matrix_bytes + w * 2 * R * DP * 4
    if np.ndim(C) == 0:
        return int(R), int(w), int(grid), int(smem)
    return R, w, grid, smem


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _kernel(D, R):
    return 'flow_small_kernel<%d, %d>' % ((D + 31) // 32, R)


def _knobs(monkeypatch, R=None, W=None):
    monkeypatch.setenv('HMCX_FLOW_SMALL', '1')
    for k, v in (('HMCX_FLOW_R', R), ('HMCX_FLOW_W', W)):
        if v is None:
            monkeypatch.delenv(k, raising=False)
        else:
            monkeypatch.setenv(k, str(v))


def _ran(kernel, fn, attempts=3):
    """fn() under the profiler; asserts that it launched `kernel` (a flow_small_kernel<NJ, R> name).  The profiler keeps
    only the device records it can place inside its host-side window, so the window is padded on both sides and a trace
    holding no flow_small_kernel record is taken again (fn is deterministic); a trace that records another form fails."""
    for _ in range(attempts):
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA], acc_events=True) as prof:
            time.sleep(0.05)
            res = fn()
            torch.cuda.synchronize()
            time.sleep(0.05)
        names = sorted({e.name for e in prof.events() if 'flow_small_kernel<' in e.name})
        if names:
            break
    assert any(kernel in n for n in names), ('expected ' + kernel, names)
    return res


# ---- problems ----------------------------------------------------------------------------------------------------------
def _target(kind, D, seed):
    if kind == 'full':
        return _full_target(D, seed)
    return _diag_target(D, seed) if kind == 'diag' else T.GaussianIso(D)


def _mass(kind, D, seed):
    if kind == 'diag':
        return 0.5 + torch.rand(D, generator=torch.Generator().manual_seed(seed))
    if kind == 'full':
        return _spd(D, seed)
    if kind == 'blocks':                                   # three blocks, the last one the largest when 3 does not divide D
        sizes = [D // 3, D // 3, D - 2 * (D // 3)]
        return [_spd(n, seed + i) for i, n in enumerate(sizes)]
    return None


def _nmat(cs):
    return (cs['target'] == 'full') + 2 * (cs.get('mass') in ('full', 'blocks') or 'rm' in cs)


MODES = {
    'full_none': dict(target='full', mass=None, eps=0.25),
    'full_diag': dict(target='full', mass='diag', eps=0.25),
    'full_full': dict(target='full', mass='full', eps=0.2),
    'diag_full': dict(target='diag', mass='full', eps=0.2),
    'iso_blocks': dict(target='iso', mass='blocks', eps=0.2),
    'nuts_full_full': dict(target='full', mass='full', eps=NUTS_EPS0, nuts=True),
    'rm_explicit_full': dict(target='full', rm=dict(explicit=True, softabs=False), eps=0.3),   # paired grad_vel at R <= 2
    'rm_explicit_diag': dict(target='diag', rm=dict(explicit=True, softabs=False), eps=0.3),
    'rm_implicit_softabs_full': dict(target='full', rm=dict(explicit=False, softabs=True), eps=0.3),
}
# NJ = 1: the smallest dense D and a full slot; 2: one live lane in the last slot, D % 4 = 3; 3; 4 (D = 128: 3 x 64 KiB)
DS = (17, 32, 33, 63, 65, 96, 97, 126, 128)


class _Case:
    """A mode at (C, D): target, mass, inputs of the injected stream, per-chain step sizes (a teacher-forced (S, C)
    schedule for NUTS), the replay model."""

    def __init__(self, mode, D, C, seed, S=None, L=None):
        cs = self.cs = MODES[mode]
        self.nuts, self.rm = cs.get('nuts', False), cs.get('rm')
        self.D, self.C = D, C
        self.S = S or (8 if self.nuts else 6)
        self.L = L or (3 if self.rm else 4)
        self.burn = 3 if self.nuts else 0
        self.tgt = _target(cs['target'], D, seed)
        self.im = _mass(cs.get('mass'), D, seed + 1)
        self.init, self.z, self.logu, self.eps = _problem(self.tgt, C, self.S, seed + 2, cs['eps'])
        if self.rm and self.rm['explicit']:
            self.eps = torch.full_like(self.eps, cs['eps'])        # one binding rotation per launch: one step size
        self.sched = None
        if self.nuts:
            g = torch.Generator().manual_seed(seed + 3)
            self.sched = (cs['eps'] * (0.8 + 0.4 * torch.rand(self.S, C, generator=g))).cuda()
        if self.rm:
            self.model = dense_ref.RMHMC(self.tgt, self.rm['softabs'], ALPHA, explicit=self.rm['explicit'], omega=OMEGA,
                                         device='cuda')
        else:
            self.model = dense_ref.HMC(self.tgt, self.im, device='cuda')

    def run(self, eps=None, sched=None):
        eps = self.eps if eps is None else eps
        sched = self.sched if sched is None else sched
        if self.rm:
            res = engine.rmhmc_run(self.tgt, self.init, self.S, self.L, eps, burn=self.burn, softabs_const=ALPHA,
                                   explicit_binding_const=OMEGA, explicit=self.rm['explicit'], softabs=self.rm['softabs'],
                                   normals=self.z, log_uniforms=self.logu, record_ham=True)
        else:
            res = engine.hmc_run(self.tgt, self.init, self.S, self.L, NUTS_EPS0 if self.nuts else eps, burn=self.burn,
                                 inv_mass=self.im, nuts=self.nuts, normals=self.z, log_uniforms=self.logu,
                                 record_ham=True, eps_schedule=sched, record_eps=self.nuts)
        torch.cuda.synchronize()
        return res

    def check(self, tag, res, keep=None):
        """dense_ref.check of the chains `keep` (default all); for NUTS also the recorded dual averaging."""
        k = slice(None) if keep is None else keep
        eps = self.sched[:, k] if self.nuts else self.eps[k]
        rep = dense_ref.replay(self.model, self.init[k], res.accepted[k], res.samples[k], self.z[:, k], eps, self.L,
                               self.burn)
        dense_ref.check(tag, rep, self.init[k], res.samples[k], res.accepted[k], res.ham[k], self.logu[:, k], self.burn)
        if self.nuts:
            want = dense_ref.dual_averaging(res.ham[k], self.burn, NUTS_EPS0)
            got = res.eps_trace[k][:, :self.burn + 1].double().cpu()
            torch.testing.assert_close(got, want, rtol=2e-4, atol=0)


def _bits(t):
    t = t.detach().contiguous()
    if t.dtype == torch.float32:
        return t.view(torch.int32)
    return t.view(torch.int64) if t.dtype == torch.float64 else t


OUTPUTS = ('samples_padded', 'accepted', 'diverged', 'ham', 'num_rejected', 'final_state', 'step_size', 'eps_trace',
           'h_bar', 'eps_bar')


def _assert_same_bytes(a, b, what, chains=None):
    """Every output of two runs (or of the chains `chains` of both) byte for byte."""
    for k in OUTPUTS:
        x, y = getattr(a, k, None), getattr(b, k, None)
        assert (x is None) == (y is None), (what, k)
        if x is not None:
            if chains is not None:
                x, y = x[chains], y[chains]
            assert torch.equal(_bits(x), _bits(y)), '%s: %s differs' % (what, k)


# ---- (a) every R at every register-slot count, C = 131 -------------------------------------------------------------------
@pytest.mark.parametrize('D', DS)
@pytest.mark.parametrize('mode', sorted(MODES))
def test_every_r_vs_fp64_replay(mode, D, monkeypatch):
    """R = 1, 2, 4 forced at C = 131 (dead slots in the last warp at R = 2 and 4): each run against the replay, and R = 2 / 4
    byte-identical to R = 1 in every output."""
    case = _Case(mode, D, 131, seed=100 * D + sorted(MODES).index(mode))
    runs = {}
    for R in (1, 2, 4):
        _knobs(monkeypatch, R=R)
        runs[R] = case.run()
    for R, res in runs.items():
        assert int(res.diverged.sum()) == 0, R
        case.check('flow_small/%s_d%d' % (mode, D), res)
    assert 0 < int(runs[1].accepted.sum()) < case.C * case.S
    for R in (2, 4):
        _assert_same_bytes(runs[1], runs[R], '%s D=%d: R=%d vs R=1' % (mode, D, R))


# ---- (b) workload batch sizes under the default rule --------------------------------------------------------------------
WORKLOADS = {               # chain count = k * SMs + extra; the shape each one covers
    'r1_last': dict(k=4, extra=0, mode='full_full', D=48),              # the last batch before R changes
    'r2_surplus': dict(k=4, extra=1, mode='diag_full', D=72),           # R = 2; the last CTA has surplus warps
    'r4_three_live': dict(k=12, extra=3, mode='rm_explicit_full', D=100),   # R = 4: the last warp has 3 live slots
    'r4_w8_d128': dict(k=28, extra=5, mode='full_full', D=128),         # w = 8 with three 64 KiB matrices: 224 KiB
}
WORKLOAD_R = {'r1_last': 1, 'r2_surplus': 2, 'r4_three_live': 4, 'r4_w8_d128': 4}


@pytest.mark.parametrize('name', sorted(WORKLOADS))
def test_workload_batches_default_rule_vs_fp64_replay(name, monkeypatch):
    wl = WORKLOADS[name]
    sms = _sms()
    C, D = wl['k'] * sms + wl['extra'], wl['D']
    case = _Case(wl['mode'], D, C, seed=7000 + D, S=4, L=3)
    R, w, grid, smem = _flow_geometry(C, D, _nmat(case.cs), sms)
    assert R == WORKLOAD_R[name]
    warps = -(-C // R)
    if name == 'r1_last':
        assert w == 4 and warps == grid * w
    elif name == 'r2_surplus':
        assert grid * w - warps >= 1 and w > 1                   # surplus warps return before the loop
    elif name == 'r4_three_live':
        assert C % 4 == 3
    else:
        assert w == 8 and smem == 229376 <= SMEM_OPTIN_H100
    _knobs(monkeypatch)
    res = _ran(_kernel(D, R), case.run)
    assert int(res.diverged.sum()) == 0
    case.check('flow_small/workload_%s' % name, res)
    assert 0 < int(res.accepted.sum()) < C * case.S
    _knobs(monkeypatch, R=1)
    one = _ran(_kernel(D, 1), case.run)
    _assert_same_bytes(one, res, '%s: default rule (R=%d) vs R=1' % (name, R))


# ---- (c) the CTA width never changes bits ---------------------------------------------------------------------------------
def test_cta_width_never_changes_bits(monkeypatch):
    """C = 28 SMs + 5 at D = 128, GaussianFull + full mass: w = 1, 2, 4, 8 warps per CTA (the staging row of each warp at
    warp * 2 R DP, surplus warps in the last CTA) give the bytes of the default geometry."""
    sms = _sms()
    C, D = 28 * sms + 5, 128
    case = _Case('full_full', D, C, seed=8128, S=4, L=3)
    _knobs(monkeypatch)
    ref = case.run()
    assert 0 < int(ref.accepted.sum()) < C * case.S
    for W in (1, 2, 4, 8):
        assert _flow_geometry(C, D, 3, sms, wmax=W)[3] <= SMEM_OPTIN_H100
        _knobs(monkeypatch, W=W)
        _assert_same_bytes(ref, case.run(), 'HMCX_FLOW_W=%d vs default' % W)


def test_forced_flow_geometry_must_fit(monkeypatch):
    """HMCX_FLOW_R / HMCX_FLOW_W never run a geometry they did not ask for: R outside {1, 2, 4}, W outside 1..8 or
    anything that is not a number is an error before any launch, not a fall-back to the batch rule."""
    case = _Case('full_full', 40, 5, seed=9)
    for R in ('3', 'x', '0', '8', ''):
        _knobs(monkeypatch, R=R)
        with pytest.raises(RuntimeError):
            case.run()
    for W in ('16', '9', '0', '-1', '2x'):
        _knobs(monkeypatch, W=W)
        with pytest.raises(RuntimeError):
            case.run()
    _knobs(monkeypatch, R=4, W=8)
    ok = case.run()
    _knobs(monkeypatch)
    _assert_same_bytes(case.run(), ok, 'HMCX_FLOW_R=4 HMCX_FLOW_W=8 vs default')


# ---- (d) Philox at R = 2 / 4 ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', ['r4_full_full', 'r2_nuts'])
def test_philox_equals_injected_at_r2_r4(name, monkeypatch):
    """In Philox mode every slot stages its momentum draws through its own row xs + r DP: the run equals its
    injected-stream twin at R = 4 (C = 12 SMs + 3) and, for NUTS, at R = 2 (C = 4 SMs + 1)."""
    sms = _sms()
    D, S, L, burn = 97, 10, 4, 2
    nuts = name == 'r2_nuts'
    C = 4 * sms + 1 if nuts else 12 * sms + 3
    assert _flow_geometry(C, D, 3, sms)[0] == (2 if nuts else 4)
    tgt, im = _full_target(D, 61), _spd(D, 62)
    q0 = tgt.mean[None] + 0.3 * torch.randn(C, D, generator=torch.Generator().manual_seed(63))
    _knobs(monkeypatch)

    def run(**rng):
        fn = lambda: engine.hmc_run(tgt, q0, S, L, 0.2, burn=burn, inv_mass=im, nuts=nuts, record_eps=nuts,
                                    record_ham=True, **rng)
        return _ran(_kernel(D, 2 if nuts else 4), fn) if 'seed' in rng else fn()
    _philox_vs_injected(run, SEEDS[1 + nuts], OFFSETS[2] if not nuts else OFFSETS[1], C, S, D)


# ---- (e) a diverging chain does not leak into its warp-mates --------------------------------------------------------------
@pytest.mark.parametrize('nuts', [False, True])
def test_diverging_chain_stays_in_its_slot(nuts, monkeypatch):
    """C = 131 at R = 4: the last warp holds chains 128, 129, 130 and a dead slot shadowing 130.  Chain 129 gets a step
    size of 1e20, which overflows fp32 within its first drift: every iteration diverges and is rejected, its rows stay at
    params_init, and every other chain is byte-identical to a run where chain 129 has an ordinary step size.  With NUTS
    (the step size teacher-forced) its dual averaging takes alpha = 0 at every warm-up iteration, n = burn included."""
    bad, C, D = 129, 131, 65
    case = _Case('nuts_full_full' if nuts else 'full_full', D, C, seed=6565)
    _knobs(monkeypatch, R=4)
    ok = case.run()
    if nuts:
        sched = case.sched.clone()
        sched[:, bad] = 1e20
        res = case.run(sched=sched)
    else:
        eps = case.eps.clone()
        eps[bad] = 1e20
        res = case.run(eps=eps)
    S, burn = case.S, case.burn
    assert bool(res.diverged[bad].bool().all()) and not bool(res.accepted[bad].bool().any())
    assert int(res.num_rejected[bad]) == S
    init = case.init[bad].to(res.samples.dtype)
    assert torch.equal(res.samples[bad], init[None].expand_as(res.samples[bad]))
    assert torch.equal(res.final_state[bad], init)
    others = torch.tensor([c for c in range(C) if c != bad], device=res.accepted.device)
    _assert_same_bytes(ok, res, 'chains other than %d' % bad, chains=others)
    assert int(res.diverged[others].sum()) == 0
    # the diverging chain's fp64 Hamiltonian is finite where the kernel's is not: the replay checks the others only
    case.check('flow_small/diverging_%s' % ('nuts' if nuts else 'hmc'), res, keep=others)
    if nuts:
        # alpha = 0 at n = 0 .. burn: the proposals of n < burn, then eps_bar after the update of n = burn as well
        # (samplers.py:1060-1067 adapts on a LogProbError at n <= burn)
        want = dense_ref.dual_averaging(res.ham[bad:bad + 1], burn, NUTS_EPS0, diverged=res.diverged[bad:bad + 1])[0]
        got = res.eps_trace[bad, :burn + 1].double().cpu()
        torch.testing.assert_close(got, want, rtol=2e-4, atol=0)
        assert float(res.eps_bar[bad].float()) == float(res.eps_trace[bad, burn])
