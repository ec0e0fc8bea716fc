"""numpy restatement of simulation-based calibration (hamiltorch_b200/sbc.py, csrc/hmcx_sbc.cu): the Philox streams 6
(prior) and 7 (data) on tests/philox_ref.py's Philox, the prior scaling, the three simulators, and the rank histogram /
chi^2 / p-value with scipy's regularised upper incomplete gamma function.

    stream         counter (x, y, z, w)                  use
    sbc prior (6)  (v, j_lo, j_hi | 6 << 24, m_lo)       row j of sim m (j = 0 theta~, 1 + r chain r's start):
                                                         Box-Muller(x, y) -> elements 4v, 4v+1; (z, w) -> 4v+2, 4v+3
    sbc data  (7)  (v, 0, 7 << 24, m_lo)                 regression: the same normals over the flattened (N O) outputs;
                                                         binary: u01(word e mod 4) of vector e / 4 for output e;
                                                         multi-class: u01(word x) of vector = row

Key (seed_lo, seed_hi ^ m_hi) for both.  The GPU's normals go through the .approx instructions of box_muller, so the fp64
values here are for tolerance checks; uniforms are exact."""
import numpy as np
from scipy import special

from tests import philox_ref as P

STREAM_SBC_PRIOR, STREAM_SBC_DATA = 6, 7


def _normals(words, n):
    """(..., nv, 4) Philox words -> (..., n) fp64 canonical Box-Muller normals of elements 0 .. n-1."""
    r2, th = P.box_muller_pairs(words[..., 0::2], words[..., 1::2])     # (..., nv, 2)
    r = np.sqrt(r2)
    z = np.stack([r * np.cos(th), r * np.sin(th)], -1)                   # (..., nv, 2, 2): element 4v + 2i + j
    return z.reshape(z.shape[:-3] + (-1,))[..., :n]


def prior_words(seed, sims, rows, D):
    """(len(sims), rows, ceil(D / 4), 4) uint64 words of stream 6."""
    nv = (D + 3) // 4
    m = np.asarray(sims, dtype=np.uint64)[:, None, None]
    j = np.arange(rows, dtype=np.uint64)[None, :, None]
    v = np.arange(nv, dtype=np.uint64)[None, None, :]
    return P.draw(seed, m, j, v, STREAM_SBC_PRIOR)


def element_sd(target):
    """(D,) fp64 prior standard deviation of every parameter: sqrt(prior_scale / tau_k) of the tensor holding it."""
    ps = float(target.prior_scale)
    return np.concatenate([np.full(n, np.sqrt(ps / float(t))) for n, t in zip(target.sizes, target.tau_list)])


def prior(seed, sims, R, target):
    """(len(sims), 1 + R, D) fp64: row 0 theta~, rows 1 .. R the chain starts."""
    D = target.dim
    return _normals(prior_words(seed, sims, 1 + R, D), D) * element_sd(target)


def data_words(seed, sims, nvec):
    m = np.asarray(sims, dtype=np.uint64)[:, None]
    return P.draw(seed, m, 0, np.arange(nvec, dtype=np.uint64)[None, :], STREAM_SBC_DATA)


def simulate_regression(seed, sims, f, tau_out):
    """f (M, N, O) -> y (M, N, O) fp64 = f + z / sqrt(tau_out)."""
    f = np.asarray(f, dtype=np.float64)
    M, n = f.shape[0], f.shape[1] * f.shape[2]
    z = _normals(data_words(seed, sims, (n + 3) // 4), n)
    return f + (z / np.sqrt(tau_out)).reshape(f.shape)


def simulate_binary(seed, sims, f):
    """f (M, N, O) -> (y (M, N, O) fp64 0 / 1, |u - sigmoid(f)| the distance of every draw to its class boundary)."""
    f = np.asarray(f, dtype=np.float64)
    M, n = f.shape[0], f.shape[1] * f.shape[2]
    w = data_words(seed, sims, (n + 3) // 4).reshape(M, -1)[:, :n]
    u = P.u01(w).astype(np.float64).reshape(f.shape)
    p = 1.0 / (1.0 + np.exp(-f))
    return (u < p).astype(np.float64), np.abs(u - p)


def simulate_multiclass(seed, sims, f):
    """f (M, N, O) -> (labels (M, N) fp64, the distance of u to the nearest cumulative-probability boundary)."""
    f = np.asarray(f, dtype=np.float64)
    M, N_, O = f.shape
    u = P.u01(data_words(seed, sims, N_)[..., 0]).astype(np.float64)     # (M, N)
    e = np.exp(f - f.max(-1, keepdims=True))
    cdf = np.cumsum(e, -1) / e.sum(-1, keepdims=True)                   # (M, N, O)
    label = np.minimum((u[..., None] > cdf[..., :O - 1]).sum(-1), O - 1)
    dist = np.abs(u[..., None] - cdf[..., :O - 1]).min(-1) if O > 1 else np.full(u.shape, np.inf)
    return label.astype(np.float64), dist


def ranks(draws, truth):
    """draws (K, L, P), truth (K, P) -> (K, P) int64 #{draws < truth}."""
    return (np.asarray(draws) < np.asarray(truth)[:, None, :]).sum(1)


def histogram(rk, L, B):
    """rk (M, P) ranks in 0 .. L -> (hist (P, B), expected (B,), chi2 (P,), p (P,)): bin floor(rho B / (L + 1)), exact
    expected counts M |bin| / (L + 1), p = Q((B - 1) / 2, chi2 / 2)."""
    rk = np.asarray(rk, dtype=np.int64)
    M, Pn = rk.shape
    b = rk * B // (L + 1)
    hist = np.stack([np.bincount(b[:, p], minlength=B) for p in range(Pn)])
    width = np.bincount(np.arange(L + 1) * B // (L + 1), minlength=B)
    expected = M * width / (L + 1)
    chi2 = ((hist - expected) ** 2 / expected).sum(1)
    return hist, expected, chi2, special.gammaincc((B - 1) / 2.0, chi2 / 2.0)
