"""CPU: the held-out evaluation definition of tests/predictive_oracle.py against hand computations, the notebook's curve
loop (cleaned up as the curves define it), degenerate ensembles and the exact predictive of a conjugate linear
regression; the host-side refusals of hamiltorch_b200.predictive and the argument checks of its C-ABI entry points."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
from scipy.stats import norm

from hamiltorch_b200 import predictive as P
from hamiltorch_b200 import targets as T
from tests import predictive_oracle as O
from tests.test_loo_cpu import _conjugate, _loss_target, _posterior_draws

# ------------------------------------------------------------------------------------------------------------------
# the oracle
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('loss', ['multi_class_linear_output', 'multi_class_log_softmax_output'])
def test_two_draws_three_points_multi_class(loss):
    p1 = np.array([[0.8, 0.2], [0.5, 0.5], [0.1, 0.9]])
    p2 = np.array([[0.6, 0.4], [0.35, 0.65], [0.1, 0.9]])
    f = np.log(np.stack([p1, p2]))[None] + (0.0 if loss.endswith('log_softmax_output') else 1.5)   # logits up to a shift
    r = O.evaluate(f, [0, 1, 1], loss)
    pbar = (p1 + p2) / 2
    assert np.allclose(r['probs'], pbar, atol=1e-7)
    assert np.array_equal(r['pred'], [0, 1, 1]) and r['accuracy'] == 1.0
    assert np.allclose(r['accuracy_curve'], [2 / 3, 1.0])         # draw 1 ties at point 2: the lowest label, 0
    assert abs(r['nll'] + (math.log(0.7) + math.log(0.575) + math.log(0.9)) / 3) < 1e-7
    assert abs(r['nll_curve'][0] + (math.log(0.8) + math.log(0.5) + math.log(0.9)) / 3) < 1e-7
    assert np.allclose(r['brier_i'], [0.18, 2 * 0.425 ** 2, 0.02], atol=1e-7)
    H = lambda p: -(p * np.log(p)).sum(-1)
    assert np.allclose(r['entropy'], H(pbar), atol=1e-7)
    assert np.allclose(r['expected_entropy'], (H(p1) + H(p2)) / 2, atol=1e-7)
    assert np.allclose(r['mutual_info'], H(pbar) - (H(p1) + H(p2)) / 2, atol=1e-7)
    # confidences 0.7, 0.575, 0.9 land in bins 10, 8 and 13 (upper edges inclusive), all correct
    assert abs(r['ece'] - (0.3 + 0.425 + 0.1) / 3) < 1e-7
    assert r['reliability_sums'][[10, 8, 13], 0].tolist() == [1, 1, 1]


def test_two_draws_three_points_binary():
    p1, p2 = np.array([0.8, 0.3, 0.6]), np.array([0.6, 0.5, 0.2])
    f = np.log(np.stack([p1, p2]) / (1 - np.stack([p1, p2])))[None, :, :, None]
    y = [1, 0, 1]
    r = O.evaluate(f, y, 'binary_class_linear_output')
    assert np.allclose(r['probs'][:, 0], [0.7, 0.4, 0.4], atol=1e-7)
    assert abs(r['accuracy'] - 2 / 3) < 1e-12
    assert np.allclose(r['accuracy_curve'], [1.0, 2 / 3])          # draw 1 alone predicts 1, 0, 1
    assert abs(r['nll'] + (math.log(0.7) + math.log(0.6) + math.log(0.4)) / 3) < 1e-7
    assert np.allclose(r['brier_i'], [0.09, 0.16, 0.36], atol=1e-7)
    hb = lambda p: -(p * np.log(p) + (1 - p) * np.log(1 - p))
    assert np.allclose(r['entropy'], hb(np.array([0.7, 0.4, 0.4])), atol=1e-7)
    assert np.allclose(r['expected_entropy'], (hb(p1) + hb(p2)) / 2, atol=1e-7)


def test_two_draws_three_points_regression():
    f = np.array([[0.0, 1.0, 2.0], [1.0, 1.0, 0.0]])[None, :, :, None]
    y = np.array([0.5, 1.0, 1.0])
    tau = np.array([[1.0, 4.0]])
    r = O.evaluate(f, y, 'regression', tau)
    assert np.allclose(r['mean'][:, 0], [0.5, 1.0, 1.0])
    assert np.allclose(r['epistemic'][:, 0], [0.25, 0.0, 1.0])
    assert np.allclose(r['var'][:, 0], np.array([0.25, 0.0, 1.0]) + (1 + 0.25) / 2)
    dens = 0.5 * (norm.pdf(y, f[0, 0, :, 0], 1.0) + norm.pdf(y, f[0, 1, :, 0], 0.5))
    assert np.allclose(r['lppd'], np.log(dens))
    assert np.allclose(r['pit'][:, 0], 0.5 * (norm.cdf((y - f[0, 0, :, 0]) * 1.0) + norm.cdf((y - f[0, 1, :, 0]) * 2.0)))
    assert np.allclose(r['rmse_curve'], [math.sqrt((0.25 + 0 + 1) / 3), math.sqrt((0 + 0 + 0) / 3)])
    assert np.allclose(r['nll_curve'][0], -np.log(norm.pdf(y, f[0, 0, :, 0], 1.0)).mean())


def test_curves_of_one_chain_are_the_notebook_loop_cleaned_up():
    """The notebook's loop over s, with the ensemble of the first s draws averaging probabilities for both quantities
    and dividing by the number of draws it holds."""
    g = torch.Generator().manual_seed(0)
    n, N, K = 30, 50, 5
    pred_list = torch.randn(n, N, K, generator=g, dtype=torch.float64) * 2
    y = torch.randint(0, K, (N,), generator=g)
    acc, nll = [], []
    for s in range(n):
        ens = torch.softmax(pred_list[:s + 1], -1).sum(0) / (s + 1)
        acc.append(float((ens.argmax(-1) == y).double().mean()))
        nll.append(float(-ens.gather(1, y[:, None]).log().mean()))
    r = O.evaluate(pred_list.float().numpy()[None], y.numpy(), 'multi_class_linear_output')
    assert np.allclose(r['accuracy_curve'], acc, atol=1e-12) and np.allclose(r['nll_curve'], nll, atol=1e-6)
    yr = torch.randn(N, 1, generator=g, dtype=torch.float64)
    fr = pred_list[..., :1].float().double()
    rmse = [float(((fr[:s + 1].mean(0) - yr) ** 2).mean().sqrt()) for s in range(n)]
    rr = O.evaluate(fr.float().numpy()[None], yr.numpy(), 'regression', 1.0)
    assert np.allclose(rr['rmse_curve'], rmse, atol=1e-12)


def test_identical_draws_carry_no_epistemic_uncertainty():
    f = np.repeat(np.random.default_rng(1).normal(size=(1, 1, 20, 3)), 8, axis=1).repeat(2, axis=0)
    r = O.evaluate(f, np.random.default_rng(2).integers(0, 3, 20), 'multi_class_linear_output')
    assert np.allclose(r['mutual_info'], 0.0, atol=1e-12)
    rr = O.evaluate(f, np.zeros((20, 3)), 'regression', 2.0)
    assert np.allclose(rr['epistemic'], 0.0, atol=1e-12) and np.allclose(rr['var'], 0.5)


def test_conjugate_regression_matches_the_exact_predictive():
    tgt, mu, L, _ = _conjugate()
    d, tau_out, M, S = 3, 4.0, 2000, 4000
    th = _posterior_draws(mu, L, S, seed=3)
    g = torch.Generator().manual_seed(7)
    xt = torch.randn(M, d, generator=g, dtype=torch.float64)
    X1 = torch.cat([xt, torch.ones(M, 1, dtype=torch.float64)], 1)
    y = xt @ torch.tensor([0.8, -0.5, 0.3], dtype=torch.float64) + 0.2 + \
        torch.randn(M, generator=g, dtype=torch.float64) / math.sqrt(tau_out)
    f = (th @ X1.t()).float().numpy()[None, :, :, None]              # (1, S, M, 1)
    r = O.evaluate(f, y.numpy(), 'regression', tau_out)
    Sig = L @ L.t()
    m_exact = (X1 @ mu).numpy()
    v_epi = ((X1 @ Sig) * X1).sum(1).numpy()
    assert np.all(np.abs(r['mean'][:, 0] - m_exact) <= 5 * np.sqrt(v_epi / S) + 1e-6)
    assert np.all(np.abs(r['var'][:, 0] - (1 / tau_out + v_epi)) <= 5 * v_epi * math.sqrt(2 / S) + 1e-6)
    for lv in O.LEVELS:
        assert abs(r['coverage'][lv] - lv) <= 4 * math.sqrt(lv * (1 - lv) / M) + 0.01, (lv, r['coverage'][lv])


# ------------------------------------------------------------------------------------------------------------------
# host-side refusals (before any CUDA work)
# ------------------------------------------------------------------------------------------------------------------
def test_evaluate_refuses_bad_inputs_on_the_host():
    tgt, th = _loss_target('multi_class_linear_output', 1.0)
    with pytest.raises(TypeError):
        P.evaluate(th[None].repeat(4, 1), object())
    nodata = T.MLPTarget(tgt.widths, tgt.acts, None, None, tgt.tau_list)
    with pytest.raises(RuntimeError, match='no data'):
        P.evaluate(th[None].repeat(4, 1), nodata)
    bad = T.MLPTarget(tgt.widths, tgt.acts, tgt.x, torch.full((37,), 4.0), tgt.tau_list,
                      model_loss='multi_class_linear_output')
    with pytest.raises(ValueError, match='integers'):
        P.evaluate(th[None].repeat(4, 1), bad)
    frac = T.MLPTarget(tgt.widths, tgt.acts, tgt.x, torch.full((37,), 0.5), tgt.tau_list,
                       model_loss='multi_class_linear_output')
    with pytest.raises(ValueError, match='integers'):
        P.evaluate(th[None].repeat(4, 1), frac)
    with pytest.raises(RuntimeError, match='outputs'):
        P.evaluate(torch.zeros(2, 4, 37, 5), tgt)                    # the target has O = 4
    with pytest.raises(RuntimeError, match='y and model_loss'):
        P.evaluate(torch.zeros(2, 4, 37, 4))
    with pytest.raises(ValueError, match='integers'):
        P.evaluate(torch.zeros(2, 4, 3, 4), y=[0, 1, 4], model_loss='multi_class_linear_output')
    blk = torch.zeros(2, 4, 3, 1)
    y = torch.zeros(3, 1)
    with pytest.raises(RuntimeError, match='needs tau_out'):
        P.evaluate(blk, y=y, model_loss='regression')
    with pytest.raises(RuntimeError, match='one value per draw'):
        P.evaluate(blk, y=y, model_loss='regression', tau_out=torch.ones(4, 2))
    for t in (0.0, -1.0, float('nan'), float('inf'), torch.tensor([[1.0, 1, 1, 1], [1, 1, -1, 1]])):
        with pytest.raises(ValueError, match='positive and finite'):
            P.evaluate(blk, y=y, model_loss='regression', tau_out=t)
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        P.evaluate(blk, y=y, model_loss='regression', tau_out=2.0)
    with pytest.raises(RuntimeError, match='CUDA'):                  # samples on the CPU, as diagnostics refuses them
        P.evaluate(th[None].repeat(4, 1), tgt)


# ------------------------------------------------------------------------------------------------------------------
# the C ABI
# ------------------------------------------------------------------------------------------------------------------
def test_predictive_entry_points_check_their_arguments(built_library):
    from hamiltorch_b200 import _native as N
    from hamiltorch_b200.engine import NativeTarget
    lib = N.load_library()
    assert lib.hmcx_abi_version() == 12
    tgt, _ = _loss_target('regression', 2.0)
    nt = NativeTarget(tgt, 'cpu')
    junk = C.c_void_p(16)
    args = lambda **kw: [kw.get(k, v) for k, v in (('t', nt.ref()), ('s', junk), ('cs', 8), ('ds', 64), ('C', 1),
                                                     ('n', 4), ('r0', 0), ('r1', 37), ('o', junk), ('ocs', 296),
                                                     ('ods', 74), ('st', None))]
    for bad in (dict(t=None), dict(s=None), dict(o=None), dict(C=0), dict(n=0), dict(cs=-1), dict(ds=-1),
                dict(ocs=-1), dict(ods=-1), dict(r0=-1), dict(r1=38), dict(r0=5, r1=5)):
        assert lib.hmcx_mlp_pointwise_out(*args(**bad)) == N.ERR_INVALID_ARG, bad
    gauss = N.TargetStruct()
    gauss.kind, gauss.dim = 0, 8
    assert lib.hmcx_mlp_pointwise_out(*args(t=C.byref(gauss))) == N.ERR_UNSUPPORTED
    nodata = NativeTarget(T.MLPTarget(tgt.widths, tgt.acts, None, None, tgt.tau_list), 'cpu')
    assert lib.hmcx_mlp_pointwise_out(*args(t=nodata.ref())) == N.ERR_INVALID_ARG

    for bad in ((0, 10, 1, 0, 1), (1, 0, 1, 0, 1), (2, 10, 1, 0, 0), (2, 10, 0, 0, 1), (2, 10, 1, 4, 1),
                (2, 10, 1, -1, 1)):
        assert lib.hmcx_pred_workspace_bytes(*bad) == 0, bad
    ws = lib.hmcx_pred_workspace_bytes(4, 100, 1, 0, 3)
    assert ws == 8 * (2 * 100 + 46 + 100 * (3 + 4)) * 3 and lib.hmcx_pred_workspace_bytes(4, 100, 1, 0, 6) == 2 * ws
    assert lib.hmcx_pred_workspace_bytes(4, 100, 10, 2, 1) == lib.hmcx_pred_workspace_bytes(4, 100, 10, 3, 1) == \
        8 * (246 + 100 * 14)
    pargs = lambda **kw: [kw.get(k, v) for k, v in (('f', junk), ('cs', 500), ('ds', 5), ('C', 4), ('n', 100),
                                                      ('O', 1), ('loss', 0), ('y', junk), ('tau', junk), ('tcs', 100),
                                                      ('tds', 1), ('N', 5), ('i0', 1), ('k', 3), ('pw', junk),
                                                      ('po', junk), ('nf', junk), ('part', junk), ('ws', junk),
                                                      ('wb', ws), ('st', None))]
    for bad in (dict(f=None), dict(y=None), dict(tau=None), dict(pw=None), dict(po=None), dict(nf=None),
                dict(part=None), dict(ws=None), dict(cs=-1), dict(ds=-1), dict(tcs=-1), dict(tds=-1), dict(C=0),
                dict(n=0), dict(O=0), dict(N=0), dict(i0=-1), dict(i0=3), dict(k=0), dict(loss=-1), dict(loss=4),
                dict(wb=ws - 1)):
        assert lib.hmcx_pred_pass(*pargs(**bad)) == N.ERR_INVALID_ARG, bad
    # running sums beyond one SM's shared memory: 128 threads x 4 sums x O doubles
    assert lib.hmcx_pred_pass(*pargs(O=100, wb=lib.hmcx_pred_workspace_bytes(4, 100, 100, 0, 3))) == N.ERR_UNSUPPORTED
    for bad in ((None, 10, 5, junk), (junk, 10, 5, None), (junk, 0, 5, junk), (junk, 10, 0, junk)):
        assert lib.hmcx_pred_totals(*bad, None) == N.ERR_INVALID_ARG, bad
