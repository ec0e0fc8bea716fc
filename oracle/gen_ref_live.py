"""Stores what the reference-comparison tests compare against, so that they run without the reference tree:

    python -m oracle.gen_ref_live          (needs the unmodified reference, see oracle/ref_import.py)

  tests/golden/ref_signatures.json   parameter names and defaults of the reference's sampler functions
  tests/golden/ref_live_hmc.npz      hamiltorch.sample (HMC and HMC_NUTS) on a 12-D diagonal Gaussian, seed 99
  tests/golden/ref_live_cfg4.npz     hamiltorch.sample_split_model on BASELINE config 4 (oracle/cfg4.py), seed 5
"""
import inspect
import json
import os
import sys

import numpy as np
import torch
import torch.utils.data as tud

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.ref_import import import_reference     # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden')
SIGNATURE_FUNCTIONS = ('sample', 'leapfrog', 'hamiltonian', 'gibbs', 'acceptance', 'adaptation')


def live_hmc_target():
    from hamiltorch_b200 import targets as T
    return T.GaussianDiag(torch.linspace(-1, 1, 12), 0.3 + torch.rand(12, generator=torch.Generator().manual_seed(0)))


LIVE_HMC_KW = dict(num_samples=25, num_steps_per_sample=4, step_size=0.4, burn=8)


def signatures(ref):
    out = {}
    for fn in SIGNATURE_FUNCTIONS:
        params = []
        for p in inspect.signature(getattr(ref.samplers, fn)).parameters.values():
            d = p.default
            if d is inspect.Parameter.empty:
                d = {'empty': True}
            elif hasattr(d, 'name') and not isinstance(d, (int, float, str)):
                d = {'enum': d.name}
            params.append([p.name, d])
        out[fn] = params
    return out


def main():
    torch.set_num_threads(1)
    ref = import_reference()
    with open(os.path.join(GOLD, 'ref_signatures.json'), 'w') as f:
        json.dump(signatures(ref), f, indent=1)

    tgt, init, arrays = live_hmc_target(), torch.zeros(12), {}
    for nuts in (False, True):
        torch.manual_seed(99)
        r = ref.sample(log_prob_func=tgt, params_init=init, verbose=False, debug=2,
                       sampler=ref.Sampler.HMC_NUTS if nuts else ref.Sampler.HMC, **LIVE_HMC_KW)
        arrays['samples_nuts' if nuts else 'samples_hmc'] = torch.stack(r[0]).numpy()
        if nuts:
            arrays['step_size_nuts'] = np.float64(r[1])
    np.savez(os.path.join(GOLD, 'ref_live_hmc.npz'), **arrays)

    from oracle import cfg4
    model, X, y = cfg4.problem()
    D = cfg4.descriptors(model, X, y)[0].dim
    init = ref.util.flatten(model).detach().clone()
    loader = tud.DataLoader(tud.TensorDataset(X, y), batch_size=cfg4.N_ROWS // cfg4.M, shuffle=False)
    torch.manual_seed(5)
    r = ref.sample_split_model(model, loader, params_init=init, num_splits=cfg4.M, model_loss='regression',
                               tau_out=cfg4.TAU_OUT, integrator=ref.Integrator.SPLITTING, verbose=False, num_samples=4,
                               num_steps_per_sample=cfg4.L, step_size=cfg4.EPS, inv_mass=torch.ones(D))
    np.savez_compressed(os.path.join(GOLD, 'ref_live_cfg4.npz'), samples=torch.stack(r).numpy())


if __name__ == '__main__':
    main()
