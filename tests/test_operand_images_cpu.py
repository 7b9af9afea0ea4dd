"""Host-built operand images (no GPU): the NAR refiner's exact three-way bf16 split of the weights (W6) decodes back to
the matrix it was built from."""
import ctypes as C

import numpy as np

from sopro_b200 import _lib
from sopro_b200.weights import hash_uniform


def _bf16_to_f32(u16):
    return (u16.astype(np.uint32) << 16).view(np.float32)


def _bf16_rne(x):
    u = x.astype(np.float32).view(np.uint32).astype(np.uint64)
    u = u + 0x7FFF + ((u >> 16) & 1)
    return ((u >> 16) & 0xFFFF).astype(np.uint16)


def test_w6_is_an_exact_three_term_split_in_the_pair_order():
    lib = _lib.load()
    N, K = 12, 64
    W = (hash_uniform(N * K, 4242) * np.float32(3.0)).astype(np.float32).reshape(N, K)
    W[0, 0], W[0, 1], W[0, 2] = 0.0, 1.0, -2.5e-3  # exactly representable / small
    out = np.zeros((N, 6, K), dtype=np.uint16)
    _lib.check(lib.sopro_debug_pack_w6(W.ctypes.data, N, K, out.ctypes.data))
    t = _bf16_to_f32(out).astype(np.float64)
    # pair order mm, lh, hl, mh, hm, hh -> the w term of pair j is [m, h, l, h, m, h]
    m, h, l = t[:, 0], t[:, 1], t[:, 2]
    assert np.array_equal(t[:, 3], h) and np.array_equal(t[:, 4], m) and np.array_equal(t[:, 5], h)
    assert np.array_equal((h + m + l).astype(np.float32), W)           # exact: 3 x 8 mantissa bits cover fp32's 24
    assert np.array_equal(out[:, 1], _bf16_rne(W))                     # h = round-to-nearest-even bf16 of w
    assert np.all(np.abs(m) <= np.abs(h) * 2.0 ** -8 + 1e-45) and np.all(np.abs(l) <= np.abs(h) * 2.0 ** -16 + 1e-45)
