"""Voice ingestion's preparation restated in numpy float64 (sopro_b200/csrc/ingest.cu, include/sopro_b200.h): the energy
trim extent of a clip at its own rate (the reference's trim_silence_energy, audio.py:30-87) and encode_file's centre-crop
plan (codec/mimi.py:52-57, audio.py center_crop_audio)."""
from __future__ import annotations

from typing import Tuple

import numpy as np

FLOOR_DB = -40.0


def geometry(sr: int) -> dict:
    """The reference's frame geometry at rate sr, in its own double arithmetic (int() truncates)."""
    return {"flen": max(1, int(sr * 25.0 / 1000.0)), "hop": max(1, int(sr * 10.0 / 1000.0)),
            "pad": int(sr * 30.0 / 1000.0), "min_row": int(sr * 0.1), "min_keep": int(0.5 * sr)}


def frame_db(x: np.ndarray, sr: int) -> np.ndarray:
    """dB_k = 10 log10(sum x^2 / flen + 1e-10) of the K = (n - flen) // hop + 1 frames, float64 [K]."""
    g = geometry(sr)
    x = np.asarray(x, dtype=np.float64).reshape(-1)
    K = (x.size - g["flen"]) // g["hop"] + 1
    idx = np.arange(K)[:, None] * g["hop"] + np.arange(g["flen"])[None, :]
    return 10.0 * np.log10((x[idx] ** 2).sum(axis=1) / g["flen"] + 1e-10)


def trim_detail(x: np.ndarray, sr: int) -> dict:
    """The extent of one clip and how it was reached: start, end, and (for a clip long enough to be framed) dB, thr,
    first and last voiced frame (-1 when none)."""
    g = geometry(sr)
    n = int(np.asarray(x).size)
    out = {"start": 0, "end": n, "db": None, "thr": None, "first": -1, "last": -1}
    if n < g["min_row"] or n < g["flen"]:
        return out
    db = frame_db(x, sr)
    thr = max(float(db.max()) + FLOOR_DB, FLOOR_DB)
    voiced = np.nonzero(db > thr)[0]
    out.update(db=db, thr=thr)
    if voiced.size == 0:
        return out
    first, last = int(voiced[0]), int(voiced[-1])
    start, end = max(0, first * g["hop"] - g["pad"]), min(n, last * g["hop"] + g["flen"] + g["pad"])
    out.update(first=first, last=last)
    if end - start >= g["min_keep"]:
        out.update(start=start, end=end)
    return out


def trim_extent(x: np.ndarray, sr: int) -> Tuple[int, int]:
    d = trim_detail(x, sr)
    return d["start"], d["end"]


def crop_window(crop_seconds) -> int:
    """encode_file's window in 24 kHz samples: max(1, round(s * 12.5)) * 1920, or 0 (no crop) for None / s <= 0."""
    if crop_seconds is None or not crop_seconds > 0:
        return 0
    return max(1, int(round(float(crop_seconds) * 12.5))) * 1920


def crop_plan(n: int, win: int) -> Tuple[int, int]:
    """(offset, length) of center_crop_audio over n samples."""
    if win <= 0 or n <= win:
        return 0, n
    return (n - win) // 2, win
