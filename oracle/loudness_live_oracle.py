"""Live loudness in float64: the causal leveller sopro_b200/csrc/level.cu implements (include/sopro_b200.h), built on
loudness_oracle's K-weighting and block energies.

Sub-block k is x[k s, (k + 1) s).  For k >= 3, M_k is the integrated loudness over blocks 0 .. k - 3 (the one-shot L of
the prefix x[0, (k + 1) s)); a_k = min(10^((T - M_k) / 20), 10^(B / 20)), 1 when M_k = -inf, B = 30 dB.  Sub-blocks
0 .. 3 go out at a_3, sub-block k > 3 under the ramp a_{k-1} + (a_k - a_{k-1}) (i + 1) / s; each released range under
its own ceiling c = 10^(-1/20) / max|x|, the gain rounded to fp32 toward zero and applied with one fp32 multiply.  A row
of fewer than 4 sub-blocks goes out at gain 1; the partial tail at the last a (1 when none)."""
from __future__ import annotations

import math
from typing import Tuple

import numpy as np

from .loudness_oracle import ABS_GATE_E, CEILING, REL_FACTOR, block_energies, sub_block

MAX_BOOST_DB = 30.0
MAX_BOOST = 10.0 ** (MAX_BOOST_DB / 20.0)


def meters(x: np.ndarray, sr: int) -> np.ndarray:
    """M_k for every complete sub-block k (NaN for k < 3), float64 [floor(n / s)]."""
    s = sub_block(sr)
    nsb = np.asarray(x).size // s
    M = np.full(nsb, np.nan)
    z = block_energies(x, sr)
    for k in range(3, nsb):
        zz = z[: k - 2]
        g1 = zz[zz > ABS_GATE_E]
        if g1.size == 0:
            M[k] = -math.inf
            continue
        g2 = g1[g1 > g1.mean() * REL_FACTOR]
        M[k] = -math.inf if g2.size == 0 else -0.691 + 10.0 * math.log10(float(g2.mean()))
    return M


def gains(M: np.ndarray, target: float) -> np.ndarray:
    """a_k from M_k (NaN stays NaN)."""
    a = np.where(np.isfinite(M), np.minimum(10.0 ** ((target - np.where(np.isfinite(M), M, 0.0)) / 20.0), MAX_BOOST), 1.0)
    return np.where(np.isnan(M), np.nan, a)


def _rz32(g: np.ndarray) -> np.ndarray:
    """float64 -> float32 rounded toward zero (g >= 0)."""
    g32 = g.astype(np.float32)
    up = g32.astype(np.float64) > g
    g32[up] = np.nextafter(g32[up], np.float32(0.0))
    return g32


def _release(x32: np.ndarray, a0: float, a1: float, s: int) -> Tuple[np.ndarray, np.ndarray]:
    """One released range: (y f32, the gain before rounding, float64)."""
    m = float(np.abs(x32).max()) if x32.size else 0.0
    c = CEILING / m if m > 0 else math.inf
    i = np.arange(x32.size, dtype=np.float64)
    r = a0 + (a1 - a0) * ((i + 1.0) / float(s))
    g = np.minimum(r, c)
    return (_rz32(g).astype(np.float64) * x32.astype(np.float64)).astype(np.float32), g


def level_live(x: np.ndarray, sr: int, target: float, a: np.ndarray = None):
    """-> (y f32 [n], a_k float64 [floor(n / s)], M_k float64).  `a`: use these gains instead of the oracle's own (to
    check the release rules on the kernel's a_k alone)."""
    x32 = np.asarray(x, dtype=np.float32).reshape(-1)
    s = sub_block(sr)
    n = x32.size
    m = n // s
    M = meters(x32, sr)
    A = gains(M, target) if a is None else np.asarray(a, dtype=np.float64)
    y = np.zeros(n, dtype=np.float32)
    for q in range(m + 1):
        t0, t1 = q * s, (q + 1) * s if q < m else n
        if t1 <= t0:
            continue
        if m < 4:
            a0 = a1 = 1.0
        elif q == m:
            a0 = a1 = A[m - 1]
        elif q <= 3:
            a0 = a1 = A[3]
        else:
            a0, a1 = A[q - 1], A[q]
        y[t0:t1] = _release(x32[t0:t1], a0, a1, s)[0]
    return y, A, M
