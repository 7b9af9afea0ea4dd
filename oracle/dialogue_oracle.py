"""The dialogue join restated in numpy (sopro_b200/csrc/longform.cu, sopro_longform_join_gaps in include/sopro_b200.h):
oracle/longform_oracle.py's join with a pause per gap and a gain per span, replayed with the kernel's fp32 multiplies
in the kernel's order (the fade first, rounded, then the gain), so given the same extents it reproduces the kernel bit
for bit.  The gap rule is restated from its definition: the gap before a non-empty span is the turn pause when the
previous non-empty span belongs to another turn, the sentence pause otherwise."""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np

from .longform_oracle import FADE, fade


def gaps(extents: Sequence[Tuple[int, int]], turn_of: Sequence[int], pause: int, turn_pause: int) -> List[int]:
    """The zeros before each non-empty span after the first."""
    turns = [int(t) for (s, e), t in zip(extents, turn_of) if int(e) > int(s)]
    return [int(turn_pause) if b != a else int(pause) for a, b in zip(turns, turns[1:])]


def join(rows: Sequence[np.ndarray], extents: Sequence[Tuple[int, int]], pauses: Sequence[int],
         gains: Optional[Sequence[float]] = None) -> np.ndarray:
    """Each non-empty x[start, end) with its first and last F = min(240, span // 2) samples multiplied (fp32) by the
    fade, then, with `gains`, every sample of span i multiplied (fp32) by gains[i]; pauses[m] zeros before the
    (m + 1)-th non-empty span."""
    parts: List[np.ndarray] = []
    m = 0
    for i, (x, (s, e)) in enumerate(zip(rows, extents)):
        s, e = int(s), int(e)
        if e <= s:
            continue
        seg = np.asarray(x, dtype=np.float32)[s:e].copy()
        F = min(FADE, (e - s) // 2)
        if F:
            f = fade(F)
            seg[:F] = seg[:F] * f
            seg[e - s - F:] = seg[e - s - F:] * f[::-1]
        if gains is not None:
            seg = np.float32(gains[i]) * seg
        if parts:
            parts.append(np.zeros(int(pauses[m]), dtype=np.float32))
            m += 1
        parts.append(seg.astype(np.float32))
    assert m == len(pauses), (m, len(pauses))
    return np.concatenate(parts) if parts else np.zeros(0, dtype=np.float32)
