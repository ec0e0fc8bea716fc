import sys, os, json
sys.path.insert(0, '/root/repo')
import torch
from hamiltorch_b200 import targets as T, engine
def timed(fn, reps=3):
    fn(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps
for C, D in ((4096, 2048), (8192, 1024)):
    g = torch.Generator().manual_seed(3)
    A = torch.randn(D, D, generator=g, dtype=torch.float64) / D ** 0.5
    tgt = engine.NativeTarget(T.GaussianFull(torch.zeros(D), cov=A @ A.t() + 0.5 * torch.eye(D, dtype=torch.float64)), 'cuda')
    init = torch.randn(C, D, generator=g).cuda()
    S, L = 10, 10
    ms = timed(lambda: engine.hmc_run(tgt, init, S, L, 0.1, seed=5))
    print(json.dumps(dict(C=C, D=D, us_per_step_launch=1e3 * ms / (S * (L + 1)), tflops=2.0*C*D*D*(L+1)*S/(ms*1e-3)/1e12)))
