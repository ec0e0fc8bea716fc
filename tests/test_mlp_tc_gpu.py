"""GPU tests of the tensor-core (wgmma) first-layer path of the Bayesian-NN kernels: one-hidden-layer stacks
n0 -> 128 -> nL run H^T = W1 X^T and dW1 = dH^T X as 3xTF32 wgmmas (hmcx_mlp.cu, "First-layer GEMMs on the Hopper
tensor cores").  Checked against autograd through the reference's closure (targets.MLPTarget.__call__ restates
samplers.py:1141-1188 with the same torch ops), against the fp32 SIMT kernels of the same library
(hmcx_mlp_t.tensor_cores = HMCX_MLP_TC_OFF), and chain-by-chain against the oracle."""
import numpy as np
import pytest
import torch

import hamiltorch_b200 as hb
from hamiltorch_b200 import engine, targets as T, _native as N
from oracle import cases, hmc_oracle as O
from tests import parity

pytestmark = pytest.mark.gpu
TC_GRAD_RTOL = 2e-5            # of max |grad|; 3xTF32 keeps ~fp32 accuracy (dropped lo*lo terms are 2^-22 relative)
LOSS = {'regression': 'regression', 'binary': 'binary_class_linear_output',
        'multiclass': 'multi_class_linear_output', 'logsoftmax': 'multi_class_log_softmax_output'}


def _autograd(f, q):
    q = q.detach().requires_grad_()
    lp = f(q)
    lp = lp.sum()
    return torch.autograd.grad(lp, q)[0], lp.detach()


def _problem(seed, n, n_in, n_out, act, task, splits, tc=True):
    model, x, y = cases.mlp_problem(seed=seed, n=n, n_in=n_in, hidden=128, n_out=n_out, act=act, task=task)
    bounds = np.linspace(0, n, splits + 1).astype(int)
    descs = [T.MLPTarget.from_model(model, x[a:b], y[a:b], None, 7., prior_scale=splits, model_loss=LOSS[task])
             for a, b in zip(bounds[:-1], bounds[1:])]
    if not tc:
        descs[0].tensor_cores = 1
    return model, descs


@pytest.mark.parametrize('n_in,n_out,act,task,n,splits', [
    (64, 1, 'ReLU', 'regression', 1024, 4),        # BASELINE config 4
    (64, 1, 'Tanh', 'regression', 200, 1),         # ragged: tiles of 64, 64, 64, 8 rows
    (32, 1, 'Sigmoid', 'binary', 130, 2),          # 65-row splits: a 1-row tail tile
    (16, 3, 'ReLU', 'multiclass', 96, 1),
    (48, 4, 'Tanh', 'logsoftmax', 150, 2),
])
def test_tc_gradient_and_log_prob_match_autograd_and_simt(n_in, n_out, act, task, n, splits):
    model, descs = _problem(21, n, n_in, n_out, act, task, splits)
    _, descs_simt = _problem(21, n, n_in, n_out, act, task, splits, tc=False)
    D = descs[0].dim
    torch.manual_seed(1)
    q = hb.util.flatten(model).detach()[None] + 0.05 * torch.randn(4, D)
    for m in range(splits):
        g, lp = engine.grad_log_prob(descs, q, split=m)
        gs, lps = engine.grad_log_prob(descs_simt, q, split=m)
        for c in range(q.shape[0]):
            gr, lr = _autograd(descs[m], q[c])
            scale = gr.abs().max().item()
            assert (g[c].cpu() - gr).abs().max().item() <= TC_GRAD_RTOL * scale, (m, c)
            assert (g[c] - gs[c]).abs().max().item() <= TC_GRAD_RTOL * scale, (m, c)
            assert abs(float(lp[c]) - float(lr)) <= 2e-5 * (abs(float(lr)) + 1)
    g, lp = engine.grad_log_prob(descs, q, split=-1)                  # all rows as one potential
    gs, lps = engine.grad_log_prob(descs_simt, q, split=-1)
    assert (g - gs).abs().max().item() <= TC_GRAD_RTOL * gs.abs().max().item()
    assert torch.allclose(lp, lps, rtol=2e-5, atol=1e-4)


def test_tc_gradient_and_log_prob_are_deterministic():
    """Two identical calls on the config-4 shape (64-128-1, four 256-row splits, i.e. four 64-row tiles per split) return
    the same bits: the tensor-core gradient has a fixed summation order, so any difference is a race.  One CTA per chain,
    so the 264 chains are 264 independent repetitions within one call."""
    model, descs = _problem(21, 1024, 64, 1, 'ReLU', 'regression', 4)
    D = descs[0].dim
    torch.manual_seed(3)
    q = hb.util.flatten(model).detach()[None] + 0.05 * torch.randn(264, D)
    q[1:] = q[0]                                      # identical inputs across chains as well
    for split in (0, 3, -1):
        g1, lp1 = engine.grad_log_prob(descs, q, split=split)
        g2, lp2 = engine.grad_log_prob(descs, q, split=split)
        assert torch.equal(g1, g2) and torch.equal(lp1, lp2), split
        assert bool((g1 == g1[0]).all()) and bool((lp1 == lp1[0]).all()), split


@pytest.mark.parametrize('scheme,rows_per_split', [(N.SCHEME_SPLIT_SYM, 64), (N.SCHEME_SPLIT_SYM, 256),
                                                   (N.SCHEME_PLAIN, 100), (N.SCHEME_SPLIT_KMID, 130)])
def test_tc_chain_parity_vs_live_oracle(scheme, rows_per_split):
    """64-128-1 chains on the tensor-core path == the oracle's chains from the same random stream (rows_per_split 256
    with 3 chains also runs 4 CTAs per chain through distributed shared memory)."""
    M, S, L, burn = 2, 8, 3, 1
    model, x, y = cases.mlp_problem(seed=13, n=M * rows_per_split, n_in=64, hidden=128)
    if scheme == N.SCHEME_PLAIN:                      # sample_model: one closure over all rows
        descs = T.MLPTarget.from_model(model, x, y, None, 20.)
        D = descs.dim
    else:
        descs = [T.MLPTarget.from_model(model, x[m * rows_per_split:(m + 1) * rows_per_split],
                                        y[m * rows_per_split:(m + 1) * rows_per_split], None, 20., prior_scale=M)
                 for m in range(M)]
        D = descs[0].dim
    C = 3
    inits, zs, lus = [], [], []
    for seed in range(C):
        init, z, logu, _ = O.reference_stream(60 + seed, D, S,
                                              prior=lambda: hb.util.flatten(model).detach() + 0.02 * torch.randn(D))
        inits.append(init), zs.append(z), lus.append(logu)
    res = engine.hmc_run(descs, torch.stack(inits), S, L, 0.002, burn=burn, normals=torch.stack(zs, 1),
                         log_uniforms=torch.stack(lus, 1), record_ham=True, scheme=scheme)
    torch.cuda.synchronize()
    assert int(res.diverged.sum()) == 0
    split = {N.SCHEME_PLAIN: None, N.SCHEME_SPLIT_SYM: O.SPLIT_SYM, N.SCHEME_SPLIT_KMID: O.SPLIT_KMID}[scheme]
    for c in range(C):
        o = O.sample_hmc(descs, inits[c], num_samples=S, num_steps_per_sample=L, step_size=0.002, burn=burn,
                         split_scheme=split, normals=zs[c], log_uniforms=lus[c])
        parity.assert_chain_parity(res.samples[c].cpu().numpy(), res.accepted[c].cpu().numpy(),
                                   res.ham[c].cpu().numpy(), torch.stack(o['samples']).numpy(), o['accepted'],
                                   o['ham_old'], o['ham_new'], lus[c].numpy(), burn, exact=False, rtol=2e-4)


@pytest.mark.parametrize('n_in,n_out,act,task,n,splits', [(64, 1, 'ReLU', 'regression', 200, 1),
                                                          (48, 4, 'Tanh', 'logsoftmax', 150, 2)])
def test_tc_predict_matches_the_model_and_the_simt_kernel(n_in, n_out, act, task, n, splits):
    """predict_model's forward over posterior samples on the tensor-core path: network outputs == the torch model
    evaluated at each sample (log-probabilities for a LogSoftmax model) == the fp32 SIMT kernel."""
    model, descs = _problem(31, n, n_in, n_out, act, task, splits)
    _, descs_simt = _problem(31, n, n_in, n_out, act, task, splits, tc=False)
    D = descs[0].dim
    torch.manual_seed(2)
    samples = hb.util.flatten(model).detach()[None] + 0.05 * torch.randn(5, D)
    pred, lp = engine.mlp_predict(descs, samples)
    pred_s, lp_s = engine.mlp_predict(descs_simt, samples)
    x = torch.cat([d.x for d in descs])
    for s in range(samples.shape[0]):
        ref = descs[0].forward(samples[s], x)
        assert torch.allclose(pred[s].cpu(), ref, rtol=2e-5, atol=2e-5), s
    assert torch.allclose(pred, pred_s, rtol=2e-5, atol=2e-5)
    assert torch.allclose(lp, lp_s, rtol=2e-5, atol=1e-4)
