"""CPU: the restated Philox4x32-10 stream (tests/philox_ref.py) -- known answers, the u01 edges and the layout of the
counters.  The GPU side (tests/test_philox_stream_gpu.py) holds every kernel's Philox mode to this restatement."""
import numpy as np

from tests import philox_ref as P


def _hex(words):
    return ' '.join('%08x' % int(w) for w in words)


def test_known_answer_vectors():
    """Random123's Philox4x32-10 known-answer vectors."""
    assert _hex(P.philox4x32_10([0, 0, 0, 0], [0, 0])) == '6627e8d5 e169c58d bc57ac4c 9b00dbd8'
    ones = 0xFFFFFFFF
    assert _hex(P.philox4x32_10([ones] * 4, [ones] * 2)) == '408f276d 41c83b0e a20bc7c6 6d5451fd'
    assert _hex(P.philox4x32_10([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], [0xa4093822, 0x299f31d0])) == \
        'd16cfe09 94fdcceb 5001e420 24126ea1'


def test_vectorised_form_equals_one_call_at_a_time():
    ctr = np.array([[1, 2, 3, 4], [0xFFFFFFFF, 7, 1 << 24, 9], [5, 0, 0, 0]], dtype=np.uint64)
    key = np.array([[11, 12], [0xDEADBEEF, 0xFEEDFACE], [0, 0]], dtype=np.uint64)
    batch = P.philox4x32_10(ctr, key)
    for i in range(3):
        assert np.array_equal(batch[i], P.philox4x32_10(ctr[i], key[i]))


def test_counter_and_key_layout():
    seed, chain, n = 0x123456789ABCDEF0, (5 << 32) + 17, (3 << 32) + 99
    assert P.counter(P.STREAM_JITTER, 33, n, chain).tolist() == [33, 99, 3 | (2 << 24), 17]
    assert P.key(seed, chain).tolist() == [0x9ABCDEF0, 0x12345678 ^ 5]
    assert P.counter(P.STREAM_ACCEPT, P.ACCEPT_VEC, 4, 1).tolist() == [0xFFFFFFFF, 4, 1 << 24, 1]


def test_u01_edges():
    """Word 0 gives 2^-33 (never 0: the log stays finite), word 0xFFFFFFFF gives exactly 1.0f (log-uniform 0)."""
    u = P.u01(np.array([0, 1, 0xFFFFFFFF], dtype=np.uint64))
    assert u.dtype == np.float32
    assert u[0] == np.float32(2.0 ** -33) and np.isfinite(np.log(u[0]))
    assert u[1] == np.float32(2.0 ** -32 + 2.0 ** -33)
    assert u[2] == np.float32(1.0)
    assert np.float32(np.log(np.float64(u[2]))) == 0.0


def test_stream_values_are_in_range():
    lu = P.log_uniforms(7, np.arange(3), np.arange(50))
    assert lu.shape == (50, 3) and lu.dtype == np.float32 and np.all(lu <= 0) and np.all(np.isfinite(lu))
    u = P.jitter_rows(7, np.arange(3), np.arange(4), 5, 47)
    assert u.shape == (4, 3, 5, 47) and np.all((u >= 0) & (u < 1))
    assert np.all(u * 2 ** 24 == np.floor(u * 2 ** 24))                  # 24-bit uniforms, exact in float32
    pm = P.perms(7, np.arange(3), np.arange(6), 8)
    assert pm.shape == (6, 3, 8) and np.all(np.sort(pm, -1) == np.arange(8))
    assert len({tuple(r) for r in pm.reshape(-1, 8)}) > 10               # not one fixed permutation
    z = P.normals(7, np.arange(2), 3, 37)
    assert z.shape == (2, 37) and np.all(np.isfinite(z))


def test_counters_of_one_iteration_are_distinct():
    """One chain, one iteration, D = 64: the momentum vectors, the accept draw, 400 fisher() calls' jitter rows and
    M = 8 perm draws never share a counter (the key is common to all of them)."""
    D, calls, M, n, chain = 64, 400, 8, 12345, (1 << 32) + 6
    nv = D // 4
    ctrs = [P.counter(P.STREAM_MOMENTUM, np.arange(nv), n, chain),
            P.counter(P.STREAM_ACCEPT, [P.ACCEPT_VEC], n, chain),
            P.counter(P.STREAM_JITTER, (P.JITTER_STRIDE * np.arange(calls)[:, None] + np.arange(nv)).ravel(), n, chain),
            P.counter(P.STREAM_PERM, np.arange(M - 1, 0, -1), n, chain)]
    allc = np.concatenate(ctrs)
    assert len({tuple(c) for c in allc.tolist()}) == len(allc)
    # and the jitter uniforms of consecutive calls are different numbers
    u = P.jitter_rows(3, [chain], [n], calls, D)[0, 0]
    assert not np.any(np.all(u[1:, :32] == u[:-1, 32:], axis=1))


def test_stride_eight_reused_counters_at_d48():
    """Regression note: the RMHMC kernels used to place call k's jitter row at vectors 8k + v.  At D = 48 (12 vectors),
    elements 32..47 of call k were then the uniforms of elements 0..15 of call k+1."""
    nv, calls = 12, 10
    old = (8 * np.arange(calls)[:, None] + np.arange(nv)).ravel()
    assert len(set(old.tolist())) < len(old)
    new = (P.JITTER_STRIDE * np.arange(calls)[:, None] + np.arange(nv)).ravel()
    assert len(set(new.tolist())) == len(new)
