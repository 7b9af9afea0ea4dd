"""WSOLA time-stretch in float64 numpy: the definition sopro_b200/csrc/stretch.cu implements (include/sopro_b200.h).

Frame N = 480, synthesis hop Hs = 240, search tolerance D = 160, periodic Hann window sin^2(pi n / N) rounded to fp32
once.  S = round(speed * 65536); M = ceil(L * 65536 / S); K = ceil(M / Hs) + 1 frames; a_k = floor((k Hs S + 32768) / 65536).
d_0 = 0; frame k >= 1 scores c_k(d) = sum_n x[p_{k-1} + n] x[a_k + d - N/2 + n] for d in [-D, D] and keeps the argmax
(ties: smallest |d|, then the negative one); y[m] = sum_k w[m - k Hs + N/2] x[p_k + m - k Hs], cut to [0, M).

``stretch(x, S, offsets=...)`` replays a given d path instead of searching (frame k's template then follows the
replayed d_{k-1}), and always returns every frame's scores, so a device's path can be judged frame by frame."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import numpy as np

N, HS, D = 480, 240, 160
HALF = N // 2


def window() -> np.ndarray:
    """sin^2(pi n / N) in float64, rounded to fp32 once, returned as float64."""
    n = np.arange(N, dtype=np.float64)
    return (np.sin(np.pi * n / N) ** 2).astype(np.float32).astype(np.float64)


def quantise(speed: float) -> int:
    return int(round(float(speed) * 65536))


def out_len(S: int, L: int) -> int:
    return -(-int(L) * 65536 // int(S))


def n_frames(M: int) -> int:
    return 0 if M == 0 else -(-int(M) // HS) + 1


def pos_a(k: int, S: int) -> int:
    return (int(k) * HS * int(S) + 32768) // 65536


@dataclass
class Result:
    y: np.ndarray          # [M] float64
    deltas: np.ndarray     # [K] int64: d_k (searched, or the replayed path)
    scores: np.ndarray     # [K, 2 D + 1] float64: c_k(d) for d = -D .. D (row 0 is NaN: frame 0 does not search)
    score_mag: np.ndarray  # [K]: max over d of sum_n |t_k[n] x[a_k + d - N/2 + n]|
    y_mag: np.ndarray      # [M]: sum_k |w x| of each output


def best_delta(c: np.ndarray) -> int:
    """The argmax of c over d = -D .. D with the tie rule (smallest |d|, then the negative one)."""
    top = np.flatnonzero(c == c.max()) - D
    return int(sorted(top.tolist(), key=lambda d: (abs(d), d))[0])


def stretch(x: np.ndarray, S: int, offsets: Optional[np.ndarray] = None, w: Optional[np.ndarray] = None) -> Result:
    x = np.asarray(x, dtype=np.float64).reshape(-1)
    L = x.size
    w = window() if w is None else np.asarray(w, dtype=np.float64)
    M = out_len(S, L)
    K = n_frames(M)
    pad = HALF + 2 * D + N + 4 * HS + 8  # every read outside [0, L) lands in the zero padding
    xp = np.concatenate([np.zeros(pad), x, np.zeros(pad)])

    def seg(i0: int, n: int) -> np.ndarray:
        return xp[pad + i0: pad + i0 + n]

    y = np.zeros(max(K, 1) * HS + HS)
    ymag = np.zeros_like(y)
    deltas = np.zeros(K, dtype=np.int64)
    scores = np.full((K, 2 * D + 1), np.nan)
    smag = np.zeros(K)
    p = 0
    for k in range(K):
        a = pos_a(k, S)
        if k == 0:
            d = 0
        else:
            t = seg(p, N)
            cand = np.lib.stride_tricks.sliding_window_view(seg(a - D - HALF, 2 * D + N), N)  # [2D + 1, N]
            c = cand @ t
            scores[k] = c
            smag[k] = float((np.abs(cand) @ np.abs(t)).max())
            d = best_delta(c)
        if offsets is not None:
            d = int(offsets[k])
        deltas[k] = d
        p = a + d
        lo = (k - 1) * HS  # frame k covers outputs [(k - 1) Hs, (k + 1) Hs)
        contrib = w * seg(p - HALF, N)
        if lo < 0:
            y[: HS] += contrib[HALF:]
            ymag[: HS] += np.abs(contrib[HALF:])
        else:
            y[lo: lo + N] += contrib
            ymag[lo: lo + N] += np.abs(contrib)
    return Result(y[:M].copy(), deltas, scores, smag, ymag[:M].copy())
