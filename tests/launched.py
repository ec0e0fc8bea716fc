"""Which element-wise HMC kernel a run launched: the instantiation names the CUDA profiler records.

The dispatch in elem_hmc_run (hmcx_hmc.cu) picks the register geometry, RNG mode, NUTS support and producer warps from
ld, the chain count, the RNG and the tuning argument.  A test that claims to exercise one instantiation asserts its name
here, so that a change of the dispatch fails the test instead of quietly testing another form."""
import time

import torch

FAMILIES = ('hmc_run_kernel<', 'hmc_run_big_kernel<')


def ran(kernel, fn, attempts=3):
    """fn() under the profiler; asserts that every element-wise run kernel it launched names ``kernel`` (a substring of
    the instantiation, e.g. ', 4, 2, 128, false, true, 1, false, 2>').  Late in a long GPU session the profiler has come
    back with no record at all for a run that did launch one (it keeps only the device records it can place inside its
    host-side window).  So the window is padded on both sides, and a trace holding no run-kernel record is taken again
    (fn is deterministic); a trace that records another form fails at once."""
    names = []
    for _ in range(attempts):
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA], acc_events=True) as prof:
            time.sleep(0.05)
            res = fn()
            torch.cuda.synchronize()
            time.sleep(0.05)
        names = sorted({e.name for e in prof.events() if any(f in e.name for f in FAMILIES)})
        if names:
            break
    assert names and all(kernel in n for n in names), ('expected %s' % kernel, names)
    return res
