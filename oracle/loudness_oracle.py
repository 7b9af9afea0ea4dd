"""ITU-R BS.1770-4 integrated loudness in float64: the definition sopro_b200/csrc/loudness.cu implements
(include/sopro_b200.h).

K-weighting: libebur128's two biquads, derived from the analog prototype at the rate (the same double operations as the
library's host code, so the coefficients agree bit for bit), run with scipy.signal.lfilter from zero state.  Sub-block
s = floor((sr + 5) / 10); block j = sub-blocks j .. j + 3, J = max(0, floor(n / s) - 3); z_j = sum y^2 / (4 s).  Gates
compare energies: absolute z > 10^((-70 + 0.691) / 10), relative z > 0.1 * mean z over the absolutely gated blocks.
L = -0.691 + 10 log10(mean z over the blocks past both), -inf when none.  Gain: min(10^((T - L) / 20),
10^(-1/20) / max|x|), 1 when L = -inf."""
from __future__ import annotations

import math
from typing import Tuple

import numpy as np
from scipy.signal import lfilter

ABS_GATE_E = 10.0 ** ((-70.0 + 0.691) / 10.0)
REL_FACTOR = 10.0 ** (-10.0 / 10.0)
CEILING = 10.0 ** (-1.0 / 20.0)


def filter_coeffs(sr: int) -> Tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
    """(b1, a1, b2, a2): the shelf and the high-pass, float64, a[0] = 1."""
    f0, G, Q = 1681.974450955533, 3.999843853973347, 0.7071752369554196
    K = math.tan(math.pi * f0 / sr)
    Vh = math.pow(10.0, G / 20.0)
    Vb = math.pow(Vh, 0.4996667741545416)
    a0 = 1.0 + K / Q + K * K
    b1 = np.array([(Vh + Vb * K / Q + K * K) / a0, 2.0 * (K * K - Vh) / a0, (Vh - Vb * K / Q + K * K) / a0])
    a1 = np.array([1.0, 2.0 * (K * K - 1.0) / a0, (1.0 - K / Q + K * K) / a0])
    f0, Q = 38.13547087602444, 0.5003270373238773
    K = math.tan(math.pi * f0 / sr)
    a0 = 1.0 + K / Q + K * K
    b2 = np.array([1.0, -2.0, 1.0])
    a2 = np.array([1.0, 2.0 * (K * K - 1.0) / a0, (1.0 - K / Q + K * K) / a0])
    return b1, a1, b2, a2


def sub_block(sr: int) -> int:
    return (int(sr) + 5) // 10


def k_weight(x: np.ndarray, sr: int) -> np.ndarray:
    b1, a1, b2, a2 = filter_coeffs(sr)
    return lfilter(b2, a2, lfilter(b1, a1, np.asarray(x, dtype=np.float64).reshape(-1)))


def block_energies(x: np.ndarray, sr: int) -> np.ndarray:
    """z_j for j in [0, J)."""
    s = sub_block(sr)
    y = k_weight(x, sr)
    nsb = y.size // s
    if nsb < 4:
        return np.zeros(0)
    e = (y[: nsb * s] ** 2).reshape(nsb, s).sum(axis=1)
    return (e[:-3] + e[1:-2] + e[2:-1] + e[3:]) / (4.0 * s)


def integrated(x: np.ndarray, sr: int) -> float:
    z = block_energies(x, sr)
    g1 = z[z > ABS_GATE_E]
    if g1.size == 0:
        return -math.inf
    g2 = g1[g1 > g1.mean() * REL_FACTOR]
    if g2.size == 0:
        return -math.inf
    return -0.691 + 10.0 * math.log10(float(g2.mean()))


def gain(L: float, peak: float, target: float) -> float:
    """g64 before its rounding to fp32."""
    if not math.isfinite(L):
        return 1.0
    return min(10.0 ** ((target - L) / 20.0), CEILING / peak)
