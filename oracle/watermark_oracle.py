"""The watermark in float64: the definition sopro_b200/csrc/watermark.cu implements (include/sopro_b200.h).

Pattern: P = 8192 samples at 24 kHz; the real-DFT bins k = 342 .. 1194 (1000 Hz <= k 24000 / P <= 3500 Hz) get unit
magnitude and phase 2 pi u_k, u_k = (z >> 11) 2^-53 for the splitmix64 outputs z seeded with the key, one per bin in bin
order; p[n] = sum_k cos(2 pi k n / P + 2 pi u_k), scaled to unit RMS.
Embed: 240-sample blocks from the first sample, r_j their RMS (a trailing partial block over its own samples),
g_j = a min(r_{j-1}, r_j), r_{-1} = 0, a = 10^(-30/20); y[n] = x[n] + g_{j(n)} p[n mod P].
Detect: w_j = 1 / r_j where r_j > max(10^(-40/20) max r, 1e-6), else 0; F[k] = sum over n = k (mod P) of w x[n];
c[l] = sum_k F[k] p[(k + l) mod P]; score = max c / sqrt(mean c^2) (0 when c = 0), offset = the first argmax."""
from __future__ import annotations

from typing import Tuple

import numpy as np

P, BLOCK, RATE = 8192, 240, 24000
LO_HZ, HI_HZ = 1000, 3500
LEVEL = 10.0 ** (-30.0 / 20.0)
FLOOR = 10.0 ** (-40.0 / 20.0)
MIN_RMS = 1e-6
THRESHOLD = 7.0
_M64 = (1 << 64) - 1


def bins() -> np.ndarray:
    return np.arange(-(-LO_HZ * P // RATE), HI_HZ * P // RATE + 1)


def phases(key: int) -> np.ndarray:
    """u_k in [0, 1) for each in-band bin, in bin order."""
    state, out = int(key), []
    for _ in bins():
        state = (state + 0x9E3779B97F4A7C15) & _M64
        z = state
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
        z ^= z >> 31
        out.append((z >> 11) * 2.0 ** -53)
    return np.array(out)


def pattern(key: int) -> np.ndarray:
    """p [P] float64, unit RMS."""
    k, n = bins(), np.arange(P)
    phi = 2 * np.pi * phases(key)
    p = np.zeros(P)
    for kk, ph in zip(k, phi):
        p += np.cos(2 * np.pi * ((kk * n) % P) / P + ph)
    return p / np.sqrt(np.mean(p * p))


def block_rms(x: np.ndarray) -> np.ndarray:
    x = np.asarray(x, dtype=np.float64)
    J = -(-len(x) // BLOCK)
    r = np.zeros(J)
    for j in range(J):
        b = x[j * BLOCK: (j + 1) * BLOCK]
        r[j] = np.sqrt(np.mean(b * b))
    return r


def gains(x: np.ndarray) -> np.ndarray:
    """g_j per block."""
    r = block_rms(x)
    return LEVEL * np.minimum(np.concatenate([[0.0], r[:-1]]), r) if len(r) else r


def embed(x: np.ndarray, p: np.ndarray) -> np.ndarray:
    """y float64 for x (one row, 24 kHz) and the pattern p."""
    x = np.asarray(x, dtype=np.float64)
    n = np.arange(len(x))
    return x + np.repeat(gains(x), BLOCK)[: len(x)] * p[n % P]


def fold(x: np.ndarray) -> np.ndarray:
    x = np.asarray(x, dtype=np.float64)
    r = block_rms(x)
    F = np.zeros(P)
    if not len(r):
        return F
    thr = max(FLOOR * r.max(), MIN_RMS)
    w = np.where(r > thr, 1.0 / np.where(r > 0, r, 1.0), 0.0)
    wx = np.repeat(w, BLOCK)[: len(x)] * x
    pad = np.zeros(-(-len(x) // P) * P)
    pad[: len(x)] = wx
    return pad.reshape(-1, P).sum(axis=0)


def correlate(F: np.ndarray, p: np.ndarray) -> np.ndarray:
    """c[l] = sum_k F[k] p[(k + l) mod P] for every lag (by the DFT: the same sums, in float64)."""
    return np.real(np.fft.ifft(np.conj(np.fft.fft(F)) * np.fft.fft(p)))


def detect(x: np.ndarray, p: np.ndarray) -> Tuple[float, int]:
    """(score, offset) of one 24 kHz row against the pattern p."""
    c = correlate(fold(x), p)
    ms = float(np.mean(c * c))
    if ms <= 0.0:
        return 0.0, 0
    l = int(np.argmax(c))
    return float(c[l] / np.sqrt(ms)), l
