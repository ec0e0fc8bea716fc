"""CPU: the launch rule of the small-D flow kernel (flow_geometry in hamiltorch_b200/csrc/hmcx_flow.cu), as restated by
tests/test_flow_small_gpu._flow_geometry, over its whole domain, and the restatement against the constants of the C++.

The GPU tests choose their chain counts and name the expected flow_small_kernel<NJ, R> from the restatement, so the two
must not drift apart: the C++ constants are read from the source here, and changing the rule on one side only fails."""
import os
import re

import numpy as np
import pytest

from tests.test_flow_small_gpu import SMEM_OPTIN_H100, _flow_geometry

SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'hamiltorch_b200', 'csrc', 'hmcx_flow.cu')
SMS = (114, 132)                        # H100 PCIe, H100 SXM
C_MAX = 40000


def _src():
    with open(SRC) as f:
        return ' '.join(f.read().split())                   # whitespace-normalised


def _one(pattern):
    m = re.findall(pattern, _src())
    assert len(m) == 1, (pattern, m)
    return m[0]


@pytest.mark.parametrize('sms', SMS)
@pytest.mark.parametrize('nmat', [1, 2, 3])
def test_geometry_fits_over_the_whole_domain(nmat, sms):
    """D = 17..128, C = 1..40,000: shared memory within the opt-in limit, at most 256 threads (__launch_bounds__), enough
    slots for every chain, and a last CTA that holds at least one live warp."""
    C = np.arange(1, C_MAX + 1, dtype=np.int64)
    for D in range(17, 129):
        R, w, grid, smem = _flow_geometry(C, D, nmat, sms)
        warps = -(-C // R)
        assert int(smem.max()) <= SMEM_OPTIN_H100, D
        assert int((32 * w).max()) <= 256 and int(w.min()) >= 1, D
        assert bool((grid * w * R >= C).all()), D
        assert bool(((grid - 1) * w < warps).all()), D                  # the last CTA's first warp has a chain
        assert bool(((warps - 1) * R < C).all()), D                     # only the last warp carries dead slots


def test_largest_request_is_d128_with_three_matrices():
    """The largest shared-memory request of the rule: D = 128, GaussianFull target + full mass (3 x 64 KiB), R = 4 and
    CTAs of 8 warps: 229,376 B of the 232,448 B an H100 CTA may opt in to."""
    for sms in SMS:
        C = 28 * sms + 5
        R, w, grid, smem = _flow_geometry(C, 128, 3, sms)
        assert (R, w, smem) == (4, 8, 229376)
        assert grid == -(-(-(-C // 4)) // 8)
        biggest = max(int(_flow_geometry(np.arange(1, C_MAX + 1), D, n, sms)[3].max())
                      for D in range(17, 129) for n in (1, 2, 3))
        assert biggest == smem <= SMEM_OPTIN_H100
    assert _flow_geometry(3701, 128, 3, 132)[:3] == (4, 8, 116)


def test_restatement_matches_the_cpp_constants():
    # chains per warp: C <= a SMs -> 1, <= b SMs -> 2, else 4
    a, b = (int(x) for x in _one(r'\(C <= (\d+) \* sms\) \? 1 : \(C <= (\d+) \* sms\) \? 2 : 4;'))
    assert (a, b) == (4, 12)
    for sms in SMS:
        for C, R in ((1, 1), (a * sms, 1), (a * sms + 1, 2), (b * sms, 2), (b * sms + 1, 4), (C_MAX, 4)):
            assert _flow_geometry(C, 64, 1, sms)[0] == R, (sms, C)
    # warps per CTA: ceil(warps / SMs), capped at 4 while the matrices take at most `cap` KiB, else at 8
    cap, lo, hi = (int(x) for x in _one(r'wmax = fw > 0 \? fw : \(matrix_bytes <= (\d+) \* 1024 \? (\d+) : (\d+)\);'))
    assert (cap, lo, hi) == (100, 4, 8)
    _one(r'const size_t matrix_bytes = \(size_t\)nmat \* K4 \* DP \* sizeof\(float\);')
    for D in range(17, 129):
        for nmat in (1, 2, 3):
            K4, DP = (D + 3) // 4 * 4, (D + 31) // 32 * 32
            want = lo if nmat * K4 * DP * 4 <= cap * 1024 else hi
            assert _flow_geometry(C_MAX, D, nmat, 132)[1] == want, (D, nmat)
    assert _flow_geometry(C_MAX, 97, 2, 132)[1] == 4 and _flow_geometry(C_MAX, 101, 2, 132)[1] == 8   # 100 KiB exactly
    # the geometry of the shared memory and of the kernel's per-warp staging rows
    _one(r'const int NJ = \(a\.D \+ 31\) / 32, DP = NJ \* 32, K4 = \(a\.D \+ 3\) & ~3;')
    _one(r'const int nmat = \(a\.tk == HMCX_TARGET_GAUSS_FULL \? 1 : 0\) \+ \(a\.mk == HMCX_MASS_FULL \? 2 : 0\);')
    _one(r'smem = \(\(size_t\)nmat \* K4 \* DP \+ \(size_t\)w \* 2 \* R \* DP\) \* sizeof\(float\);')
    _one(r'\+ warp \* \(2 \* R \* DP\);')
    _one(r'int w = \(warps \+ sms - 1\) / sms;')
    _one(r'grid = \(warps \+ w - 1\) / w;')
    # the forced values: R in {1, 2, 4}, W in 1..8 = the 256 threads of __launch_bounds__
    _one(r'flow_env\("HMCX_FLOW_R", 1, 4\)')
    _one(r'if \(fr == 0 \|\| fr == 3 \|\| fw == 0\) return HMCX_ERR_INVALID_ARG;')
    w_hi = int(_one(r'flow_env\("HMCX_FLOW_W", 1, (\d+)\)'))
    threads = int(_one(r'__launch_bounds__\((\d+), 1\) flow_small_kernel'))
    assert w_hi * 32 == threads == 256
