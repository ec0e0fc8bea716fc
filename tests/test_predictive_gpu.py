"""GPU: held-out evaluation (hamiltorch_b200.predictive) -- the outputs pass (hmcx_mlp_pointwise_out) against
predict_model's kernel bit for bit, the predictive pass (hmcx_pred_pass / hmcx_pred_totals) against the fp64 definition
of tests/predictive_oracle.py, byte-identical results across input routes, slab sizes and repeat calls, per-draw tau_out
of a hyperprior run, and agreement with loo.waic's lppd."""
import numpy as np
import pytest
import torch
import torch.nn as nn

from hamiltorch_b200 import engine, samplers
from hamiltorch_b200 import loo as LOO
from hamiltorch_b200 import predictive as P
from hamiltorch_b200 import targets as T
from tests import predictive_oracle as O
from tests.test_loo_gpu import _data, _draws, _net

pytestmark = pytest.mark.gpu

LOSSES = ['regression', 'binary_class_linear_output', 'multi_class_linear_output', 'multi_class_log_softmax_output']
TENSORS = ('nll_i', 'nll_curve', 'probs', 'pred', 'brier_i', 'entropy', 'expected_entropy', 'mutual_info',
           'accuracy_curve', 'reliability', 'mean', 'var', 'epistemic', 'pit', 'lppd', 'rmse_curve')
SCALARS = ('nll', 'nll_se', 'accuracy', 'accuracy_se', 'brier', 'brier_se', 'ece', 'rmse', 'coverage', 'num_nonfinite')


def _problem(loss, form, split):
    torch.manual_seed(1)
    if form == 'simt':
        model, O_ = _net(loss, 7, 24)
        N = 203
    else:
        model, O_ = _net(loss, 64, 128, nn.ReLU)
        N = 300
    x, y = _data(loss, N, model[0].in_features, O_, 2)
    tau = 2.5 if loss == 'regression' else 1.0
    if split:
        b = [0, 70, 190, N]
        tgt = [T.MLPTarget.from_model(model, x[i:j], y[i:j], None, tau, model_loss=loss) for i, j in zip(b, b[1:])]
    else:
        tgt = T.MLPTarget.from_model(model, x, y, None, tau, model_loss=loss)
    if form == 'tc':
        assert engine.native_target(tgt, 'cuda').mlp_struct.x_packed, 'the 64-128-O stack should take the tensor cores'
    return model, tgt, y, tau, _draws(model, 3, 6, 0.05, 3).cuda()


def _same(a, b):
    """Every result field the same bytes (NaN where NaN)."""
    for k in TENSORS:
        if hasattr(a, k):
            x, y = getattr(a, k), getattr(b, k)
            assert x.dtype == y.dtype and x.shape == y.shape, k
            assert torch.equal(x.view(torch.uint8) if x.dtype != torch.bool else x,
                               y.view(torch.uint8) if y.dtype != torch.bool else y), k
    for k in SCALARS:
        if hasattr(a, k):
            x, y = getattr(a, k), getattr(b, k)
            assert np.array_equal(np.asarray(list(x.values()) if isinstance(x, dict) else x),
                                  np.asarray(list(y.values()) if isinstance(y, dict) else y), equal_nan=True), k


def _close(got, want, name, skip=None):
    g = got.detach().cpu().double().numpy() if torch.is_tensor(got) else np.asarray(got, np.float64)
    w = np.asarray(want, np.float64)
    ok = (np.abs(g - w) <= 1e-10 * (1 + np.abs(w))) | (np.isnan(g) & np.isnan(w))
    if skip is not None:
        ok |= skip.reshape(skip.shape + (1,) * (ok.ndim - skip.ndim))
    assert ok.all(), (name, np.nanmax(np.abs(g - w)))


def _check_oracle(r, ref, loss):
    if loss == 'regression':
        for k in ('mean', 'var', 'epistemic', 'pit', 'lppd', 'nll_i', 'rmse_curve', 'nll_curve'):
            _close(getattr(r, k), ref[k], k)
        for k in ('rmse', 'nll', 'nll_se'):
            _close(getattr(r, k), ref[k], k)
        _close(list(r.coverage.values()), list(ref['coverage'].values()), 'coverage')
        return
    ok = ~np.isnan(ref['nll_i'])
    flip = None
    if 'top2_gap' in ref:
        flip = ref['top2_gap'] < 1e-12
        keep = ok & ~flip
        assert np.array_equal(r.pred.cpu().numpy()[keep], ref['pred'][keep])
    else:
        assert np.array_equal(r.pred.cpu().numpy()[ok], ref['pred'][ok])
    for k in ('probs', 'nll_i', 'brier_i', 'entropy', 'expected_entropy', 'mutual_info', 'nll_curve'):
        _close(getattr(r, k), ref[k], k)
    for k in ('nll', 'nll_se', 'brier', 'brier_se'):
        _close(getattr(r, k), ref[k], k)
    if flip is None or not flip.any():
        _close(r.accuracy_curve, ref['accuracy_curve'], 'accuracy_curve')
        _close(r.accuracy, ref['accuracy'], 'accuracy')
        _close(r.accuracy_se, ref['accuracy_se'], 'accuracy_se')
        _close(r.ece, ref['ece'], 'ece')
        sums = ref['reliability_sums']
        assert np.array_equal(r.reliability[:, 0].cpu().numpy(), sums[:, 0], equal_nan=True)


@pytest.mark.parametrize('split', [False, True])
@pytest.mark.parametrize('form', ['simt', 'tc'])
@pytest.mark.parametrize('loss', LOSSES)
def test_evaluate_matches_the_oracle_and_is_reproducible(loss, form, split):
    model, tgt, y, tau, draws = _problem(loss, form, split)
    out = P.pointwise_outputs(draws, tgt)
    pred, _ = engine.mlp_predict(tgt, draws.reshape(-1, draws.shape[-1]))
    torch.cuda.synchronize()
    assert torch.equal(out.reshape(pred.shape), pred), 'the outputs pass differs from predict_model'
    part = P.pointwise_outputs(draws, tgt, 61, 150)
    assert torch.equal(part, out[:, :, 61:150])

    r = P.evaluate(draws, tgt)
    ref = O.evaluate(out.cpu().numpy(), y.numpy(), loss, tau)
    assert r.num_nonfinite == 0 and ref['num_nonfinite'] == 0
    _check_oracle(r, ref, loss)

    blk = P.evaluate(out, y=y.cuda(), model_loss=loss, tau_out=tau if loss == 'regression' else None)
    _same(r, blk)
    _same(r, P.evaluate(out, tgt))
    _same(r, P.evaluate(draws, tgt))
    try:
        for k in (1, 7):
            P._slab_points_override = k
            _same(r, P.evaluate(draws, tgt))
    finally:
        P._slab_points_override = None


def test_per_draw_tau_out_of_a_hyperprior_run():
    torch.manual_seed(3)
    model, O_ = _net('regression', 6, 16)
    x, y = _data('regression', 150, 6, O_, 4)
    tgt = T.MLPTarget.from_model(model, x, y, None, 20.0)
    D = sum(p.numel() for p in model.parameters())
    q0 = torch.cat([p.detach().reshape(-1) for p in model.parameters()])[None] + \
        0.05 * torch.randn(2, D, generator=torch.Generator().manual_seed(2))
    res = samplers.sample_chains(tgt, q0, num_samples=30, num_steps_per_sample=3, step_size=0.004, burn=10,
                                 tau_prior=(2.0, 1.0), tau_out_prior=(2.0, 0.05), seed=4)
    torch.cuda.synchronize()
    assert not torch.equal(res.tau_out_trace[:, 1], res.tau_out_trace[:, 2])
    a = P.evaluate(res, tgt)
    b = P.evaluate(res.samples, tgt, tau_out=res.tau_out_trace)
    _same(a, b)
    c = P.evaluate(res.samples, tgt)                                 # the target's tau_out: a different predictive
    assert not torch.equal(a.var, c.var)
    out = P.pointwise_outputs(res.samples, tgt)
    ref = O.evaluate(out.cpu().numpy(), y.numpy(), 'regression', res.tau_out_trace.cpu().numpy())
    _check_oracle(a, ref, 'regression')
    w = LOO.waic(res, tgt)
    _close_ll(a.lppd, w.lppd)


def _close_ll(got, want):
    g, w = got.cpu().numpy(), want.cpu().numpy()
    assert np.all(np.abs(g - w) <= 1e-5 * (1 + np.abs(w))), np.abs(g - w).max()


@pytest.mark.parametrize('loss', LOSSES)
def test_lppd_agrees_with_waic(loss):
    _, tgt, _, _, draws = _problem(loss, 'simt', False)
    if loss == 'binary_class_linear_output':
        # each output is its own Bernoulli mixture, so only a one-output network has the joint lppd of loo.waic
        model = nn.Sequential(nn.Linear(7, 24), nn.Tanh(), nn.Linear(24, 1))
        x, y = _data(loss, 203, 7, 1, 2)
        tgt = T.MLPTarget.from_model(model, x, y, None, 1.0, model_loss=loss)
        draws = _draws(model, 3, 6, 0.05, 3).cuda()
    r = P.evaluate(draws, tgt)
    w = LOO.waic(draws, tgt)
    _close_ll(r.lppd if loss == 'regression' else -r.nll_i, w.lppd)


@pytest.mark.parametrize('loss', ['regression', 'multi_class_linear_output'])
def test_a_non_finite_draw_is_flagged(loss):
    _, tgt, y, tau, draws = _problem(loss, 'simt', False)
    out = P.pointwise_outputs(draws, tgt).clone()
    out[1, 2, 5, 0] = float('nan')
    out[0, 4, 9, 0] = float('inf')
    r = P.evaluate(out, tgt)
    ref = O.evaluate(out.cpu().numpy(), y.numpy(), loss, tau)
    assert r.num_nonfinite == 2 == ref['num_nonfinite']
    assert torch.isnan(r.nll_i[[5, 9]]).all() and not torch.isnan(r.nll_i[[0, 1, 6]]).any()
    curve = r.rmse_curve if loss == 'regression' else r.accuracy_curve
    assert not torch.isnan(curve[:2]).any() and torch.isnan(curve[2:]).all()     # draw 3 of chain 1 is the first bad
    assert not torch.isnan(r.nll_curve[:2]).any() and np.isnan(r.nll)
    _check_oracle(r, ref, loss)
