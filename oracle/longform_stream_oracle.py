"""The streaming trim of SoproTTS.stream_long (sopro_b200/csrc/longform.cu, include/sopro_b200.h) restated causally
in numpy, beside oracle/longform_oracle.py's one-shot extent and join: a row pushed in a chunk schedule -> the status
after every push (its certain prefix) and its final extent, under the causal rule; and the join of such extents."""
from __future__ import annotations

import math
from typing import List, Sequence, Tuple

import numpy as np

from .longform_oracle import FADE, FLOOR_DB, FRAME, HOP, MIN_KEEP, MIN_ROW, PAD, frame_db, join


def _pushes(n: int, schedule) -> List[int]:
    """A chunk schedule -> the push sizes over n samples: an int is a fixed size (the last push takes the rest), a
    sequence is taken as given (it must sum to n)."""
    if isinstance(schedule, (int, np.integer)):
        size = max(1, int(schedule))
        return [min(size, n - a) for a in range(0, n, size)] or [0]
    sizes = [int(c) for c in schedule]
    assert sum(sizes) == n and all(c >= 0 for c in sizes), (sizes, n)
    return sizes or [0]


def stream_extent(x: np.ndarray, schedule) -> dict:
    """The streaming trim of one row pushed in `schedule`'s pieces (the last one final) -> {"status": one
    (n, decided, start, available bound, final) per push, "start", "end": the final extent}.
    Causal rule: frame k is classified once, as it completes, against thr_k = max(M_k - 40, -40), M_k the largest dB of
    frames 0 .. k.  Certain prefix: with f, l the first and last voiced frames so far and n the samples so far, start =
    max(0, 240 f - 720), end_p = min(n, 240 l + 1320); once end_p - start >= 12000 the available bound is end_p - 240
    (nothing is available before).  At the final push the extent is the one-shot rule's over f and l, the whole row when
    n < 2400, nothing is voiced or the span is under 12000, and the bound is its end."""
    x = np.asarray(x, dtype=np.float32)
    N = int(x.size)
    db = frame_db(x) if N >= FRAME else np.zeros(0)
    M, first, last, K, n = -math.inf, -1, -1, 0, 0
    status = []
    sizes = _pushes(N, schedule)
    for i, c in enumerate(sizes):
        n += c
        final = i == len(sizes) - 1
        K_new = (n - FRAME) // HOP + 1 if n >= FRAME else 0
        for k in range(K, K_new):
            M = max(M, float(db[k]))
            if db[k] > max(M + FLOOR_DB, FLOOR_DB):
                first = k if first < 0 else first
                last = k
        K = K_new
        start = max(0, first * HOP - PAD)
        end = min(n, last * HOP + FRAME + PAD) if last >= 0 else 0
        if final:
            if n < MIN_ROW or last < 0 or end - start < MIN_KEEP:
                start, end = 0, n
            status.append((n, 1, start, end, 1))
        elif last >= 0 and end - start >= MIN_KEEP:
            status.append((n, 1, start, end - FADE, 0))
        else:
            status.append((n, 0, 0, 0, 0))
    _n, _d, start, end, _f = status[-1]
    return {"status": status, "start": start, "end": end}


def stream_join(rows: Sequence[np.ndarray], schedules, pause: int) -> Tuple[np.ndarray, List[dict]]:
    """The joined passage of rows trimmed by the streaming rule and each row's stream_extent; `schedules`: one schedule
    per row, or one int for every row.  When no frame of any row is above 0 dB this is join(rows, [extent(x)], pause)."""
    if isinstance(schedules, (int, np.integer)):
        schedules = [schedules] * len(rows)
    det = [stream_extent(x, s) for x, s in zip(rows, schedules)]
    return join(rows, [(d["start"], d["end"]) for d in det], pause), det
