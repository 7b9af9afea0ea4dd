"""Long-form synthesis's two GPU stages restated in numpy (sopro_b200/csrc/longform.cu, include/sopro_b200.h):
  - the speech extent of a 24 kHz row, the energy trim of sopro_b200.audio.trim_silence_energy, in float64;
  - the join of extents with raised-cosine edges and a fixed pause, replayed with the kernel's fp32 multiplies, so given
    the same extents it reproduces the kernel bit for bit."""
from __future__ import annotations

import math
from typing import List, Sequence, Tuple

import numpy as np

FRAME, HOP, PAD, MIN_ROW, MIN_KEEP, FLOOR_DB = 600, 240, 720, 2400, 12000, -40.0
FADE = 240


def frame_db(x: np.ndarray) -> np.ndarray:
    """dB_k = 10 log10(sum x^2 / 600 + 1e-10) of the K = (n - 600) // 240 + 1 frames, float64 [K]."""
    x = np.asarray(x, dtype=np.float64)
    K = (x.size - FRAME) // HOP + 1
    idx = np.arange(K)[:, None] * HOP + np.arange(FRAME)[None, :]
    return 10.0 * np.log10((x[idx] ** 2).sum(axis=1) / FRAME + 1e-10)


def extent_detail(x: np.ndarray) -> dict:
    """The extent of one row and how it was reached: start, end, and (for a row long enough to be framed) dB, thr,
    first and last voiced frame (-1 when none)."""
    n = int(np.asarray(x).size)
    out = {"start": 0, "end": n, "db": None, "thr": None, "first": -1, "last": -1}
    if n < MIN_ROW or n < FRAME:
        return out
    db = frame_db(x)
    thr = max(float(db.max()) + FLOOR_DB, FLOOR_DB)
    voiced = np.nonzero(db > thr)[0]
    out.update(db=db, thr=thr)
    if voiced.size == 0:
        return out
    first, last = int(voiced[0]), int(voiced[-1])
    start, end = max(0, first * HOP - PAD), min(n, last * HOP + FRAME + PAD)
    out.update(first=first, last=last)
    if end - start >= MIN_KEEP:
        out.update(start=start, end=end)
    return out


def extent(x: np.ndarray) -> Tuple[int, int]:
    d = extent_detail(x)
    return d["start"], d["end"]


def fade(F: int) -> np.ndarray:
    """f[i] = 0.5 - 0.5 cos(pi (i + 0.5) / F) in double, rounded to fp32 once."""
    return np.array([0.5 - 0.5 * math.cos(math.pi * (i + 0.5) / F) for i in range(F)], dtype=np.float64).astype(np.float32)


def pause_samples(pause_ms: float) -> int:
    return int(round(float(pause_ms) * 24))


def join(rows: Sequence[np.ndarray], extents: Sequence[Tuple[int, int]], pause: int) -> np.ndarray:
    """The joined fp32 waveform: each non-empty x[start, end) with its first and last F = min(240, span // 2) samples
    multiplied (fp32) by the fade, `pause` zeros between consecutive spans."""
    parts: List[np.ndarray] = []
    for x, (s, e) in zip(rows, extents):
        s, e = int(s), int(e)
        if e <= s:
            continue
        seg = np.asarray(x, dtype=np.float32)[s:e].copy()
        F = min(FADE, (e - s) // 2)
        if F:
            f = fade(F)
            seg[:F] = seg[:F] * f
            seg[e - s - F:] = seg[e - s - F:] * f[::-1]
        if parts:
            parts.append(np.zeros(int(pause), dtype=np.float32))
        parts.append(seg)
    return np.concatenate(parts) if parts else np.zeros(0, dtype=np.float32)
