"""The canonical random stream of the in-kernel Philox mode, restated on the CPU (numpy, vectorised).

Every kernel that runs with ``rng='philox'`` draws, for global chain id ``c = chain_offset + local c``, iteration ``n``
and ``seed``, from Philox4x32-10 (Salmon et al. 2011) with

    stream        counter (x, y, z, w)                      use
    momentum (0)  (v,            n_lo, n_hi,          c_lo)  Box-Muller(x, y) -> elements 4v, 4v+1; (z, w) -> 4v+2, 4v+3
    accept   (1)  (0xFFFFFFFF,   n_lo, n_hi | 1 << 24, c_lo)  log(u01(x))
    jitter   (2)  (16 k + v,     n_lo, n_hi | 2 << 24, c_lo)  fisher() call k, element 4v+j: (word_j >> 8) * 2^-24
    perm     (3)  (s,            n_lo, n_hi | 3 << 24, c_lo)  Fisher-Yates, s = M-1 .. 1, j = x mod (s+1)

and key ``(seed_lo, seed_hi ^ c_hi)`` for all four.  ``u01(x) = fma((float)x, 2^-32, 2^-33)`` lies in (0, 1].

This module is the specification the GPU tests hold the kernels to: uniforms, log-uniforms, jitter rows and
permutations are exact here.  The momentum normals go through the GPU's approximate lg2 / sqrt / sin / cos, so the fp64
Box-Muller below is for tolerance checks only.
"""
import numpy as np

MASK = np.uint64(0xFFFFFFFF)
M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)

STREAM_MOMENTUM, STREAM_ACCEPT, STREAM_JITTER, STREAM_PERM = 0, 1, 2, 3
JITTER_STRIDE = 16            # counter vectors per fisher() call: covers D <= 64 elements
ACCEPT_VEC = 0xFFFFFFFF


def _u64(a):
    return np.asarray(a, dtype=np.uint64)


def philox4x32_10(ctr, key):
    """ctr (..., 4), key (..., 2): integer arrays of 32-bit words (broadcast against each other) -> (..., 4) uint64."""
    ctr, key = _u64(ctr), _u64(key)
    shape = np.broadcast_shapes(ctr.shape[:-1], key.shape[:-1])
    x, y, z, w = (np.broadcast_to(ctr[..., i], shape).copy() for i in range(4))
    k0, k1 = (np.broadcast_to(key[..., i], shape).copy() for i in range(2))
    for _ in range(10):
        p0, p1 = M0 * x, M1 * z                    # exact: both factors < 2^32
        x, y, z, w = ((p1 >> np.uint64(32)) ^ y ^ k0, p1 & MASK, (p0 >> np.uint64(32)) ^ w ^ k1, p0 & MASK)
        k0, k1 = (k0 + W0) & MASK, (k1 + W1) & MASK
    return np.stack([x, y, z, w], -1)


def counter(stream, vec, n, chain):
    """The (x, y, z, w) counter of a draw, broadcast over vec / n / chain (global chain ids)."""
    vec, n, chain = _u64(vec), _u64(n), _u64(chain)
    vec, n, chain = np.broadcast_arrays(vec, n, chain)
    return np.stack([vec & MASK, n & MASK, (n >> np.uint64(32)) | np.uint64(stream << 24), chain & MASK], -1)


def key(seed, chain):
    seed, chain = _u64(seed), _u64(chain)
    seed, chain = np.broadcast_arrays(seed, chain)
    return np.stack([seed & MASK, (seed >> np.uint64(32)) ^ (chain >> np.uint64(32))], -1)


def draw(seed, chain, n, vec, stream):
    """Philox words (..., 4) of one stream at (chain, n, vec), broadcast."""
    return philox4x32_10(counter(stream, vec, n, chain), key(seed, chain))


def u01(x):
    """fma((float)x, 2^-32, 2^-33) in float32: the product is exact, so one rounding as on the GPU."""
    return np.asarray(x, dtype=np.uint64).astype(np.float32) * np.float32(2.0 ** -32) + np.float32(2.0 ** -33)


def log_uniforms(seed, chains, iterations):
    """(len(iterations), len(chains)) float32: the accept stream's log(u), correctly rounded (CUDA logf: <= 1 ulp)."""
    r = draw(seed, _u64(chains)[None, :], _u64(iterations)[:, None], ACCEPT_VEC, STREAM_ACCEPT)
    return np.log(u01(r[..., 0]).astype(np.float64)).astype(np.float32)


def jitter_rows(seed, chains, iterations, J, D):
    """(len(iterations), len(chains), J, D) float32: the torch.rand(D) of fisher() calls k = 0..J-1 of every iteration."""
    nv = (D + 3) // 4
    vec = JITTER_STRIDE * np.arange(J, dtype=np.uint64)[:, None] + np.arange(nv, dtype=np.uint64)[None, :]
    r = draw(seed, _u64(chains)[None, :, None, None], _u64(iterations)[:, None, None, None], vec[None, None],
             STREAM_JITTER)                                              # (S, C, J, nv, 4)
    u = (r >> np.uint64(8)).astype(np.float32) * np.float32(2.0 ** -24)
    return u.reshape(u.shape[:3] + (4 * nv,))[..., :D]


def perms(seed, chains, iterations, M):
    """(len(iterations), len(chains), M) int64: the randperm(M) of SPLITTING_RAND, Fisher-Yates on the perm stream."""
    chains, iterations = _u64(chains), _u64(iterations)
    out = np.broadcast_to(np.arange(M), (len(iterations), len(chains), M)).copy()
    rows = np.arange(len(iterations))[:, None], np.arange(len(chains))[None, :]
    for s in range(M - 1, 0, -1):
        x = draw(seed, chains[None, :], iterations[:, None], s, STREAM_PERM)[..., 0]
        j = (x % np.uint64(s + 1)).astype(np.int64)
        a, b = out[rows + (s,)].copy(), out[rows + (j,)].copy()
        out[rows + (s,)], out[rows + (j,)] = b, a
    return out


def momentum_words(seed, chains, n, D):
    """(len(chains), ceil(D/4), 4) uint64: the momentum stream's words of iteration n."""
    nv = (D + 3) // 4
    return draw(seed, _u64(chains)[:, None], n, np.arange(nv, dtype=np.uint64)[None, :], STREAM_MOMENTUM)


def box_muller_pairs(a, b):
    """fp64 Box-Muller of word pairs (a, b): (r^2, angle) with r^2 = -2 ln u01(a), angle = 2 pi (b + 1/2) 2^-32 - pi."""
    u = u01(a).astype(np.float64)
    return -2.0 * np.log(u), 2.0 * np.pi * (np.asarray(b, dtype=np.float64) + 0.5) * 2.0 ** -32 - np.pi


def normals(seed, chains, n, D):
    """(len(chains), D) fp64 momentum normals of iteration n (the GPU's are within the .approx error bounds)."""
    w = momentum_words(seed, chains, n, D)
    r2, th = box_muller_pairs(w[..., 0::2], w[..., 1::2])               # (C, nv, 2): pair 0 = (x, y), pair 1 = (z, w)
    r = np.sqrt(r2)
    z = np.stack([r * np.cos(th), r * np.sin(th)], -1)                  # (C, nv, 2, 2): elements 4v + 2i + j
    return z.reshape(z.shape[0], -1)[:, :D]
