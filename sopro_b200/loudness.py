"""Loudness normalisation on the GPU (no reference counterpart: the reference's output level follows its reference
recording).

``measure_loudness(wav, sample_rate)`` is the ITU-R BS.1770-4 integrated loudness of each row in LUFS (float64, on the
device; -inf for a row with no gated block), ``normalize_loudness(wav, sample_rate, target)`` scales each row to the
target under a fixed -1 dBFS sample-peak ceiling.  Both take one row or a ragged batch in one call, and neither
synchronises with the host.  A target is a real number in [-60, 0] LUFS; ``check_loudness`` refuses anything else.  The
kernels are sopro_b200/csrc/loudness.cu, the contract is in include/sopro_b200.h."""
from __future__ import annotations

import numbers
from typing import Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import _lib
from .resample import _rate


def check_loudness(target) -> Optional[float]:
    """None for None (no normalisation), else the target as a float; ValueError for anything but a real number in
    [-60, 0].  Host only, nothing allocated."""
    if target is None:
        return None
    if isinstance(target, (bool, np.bool_)) or not isinstance(target, numbers.Real):
        raise ValueError(f"loudness must be a real number in [-60, 0] LUFS, got {target!r}")
    _lib.check_arg(_lib.load().sopro_loudness_target(float(target)))
    return float(target)


def loudness_filter(sample_rate: int) -> Tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
    """The K-weighting biquads the kernels use at this rate, in float64: (b1, a1, b2, a2), each [3] with a[0] = 1.
    Host only."""
    c = np.zeros(10, dtype=np.float64)
    _lib.check_arg(_lib.load().sopro_loudness_filter(_rate(sample_rate), c.ctypes.data))
    one = np.ones(1)
    return c[0:3].copy(), np.concatenate([one, c[3:5]]), c[5:8].copy(), np.concatenate([one, c[8:10]])


def workspace_bytes(rows: int, max_len: int, sample_rate: int) -> int:
    """Device workspace of one call over `rows` rows of at most max_len samples.  Host only."""
    n = int(_lib.load().sopro_loudness_workspace(int(rows), int(max_len), _rate(sample_rate)))
    if n < 0:
        loudness_filter(sample_rate)  # raises with the reason when the rate is refused
        raise ValueError(f"bad geometry: {rows} rows of {max_len} samples")
    return n


def _rows(wav: torch.Tensor, lens: Optional[Sequence[int]]):
    """-> the rows (see _lib.rows) and the longest row's valid samples, which sizes the workspace."""
    x, lead, lp = _lib.rows(wav, lens, "loudness metering")
    most = int(x.shape[1]) if lp is None else max(lp, default=0)
    return x, lead, lp, most


def measure_loudness(wav: torch.Tensor, sample_rate: int, lens: Optional[Sequence[int]] = None) -> torch.Tensor:
    """wav [..., L] on a CUDA device (rows = the leading dims flattened) -> float64 [...] LUFS on the device, -inf for a
    row with no gated block.  `lens`: valid samples per row (a ragged batch); samples past lens[b] are not read."""
    sr = _rate(sample_rate)
    x, lead, lp, most = _rows(wav, lens)
    B, L = x.shape
    lufs = torch.empty(B, dtype=torch.float64, device=x.device)
    if B:
        ws = torch.empty(workspace_bytes(B, most, sr), dtype=torch.uint8, device=x.device)
        with torch.cuda.device(x.device):
            _lib.check_arg(_lib.load().sopro_loudness_measure(x.data_ptr(), B, L, lp, sr, ws.data_ptr(), lufs.data_ptr(),
                                                              _lib.stream_ptr(x.device)))
    return lufs.reshape(lead)


def normalize_loudness(wav: torch.Tensor, sample_rate: int, target, lens: Optional[Sequence[int]] = None,
                       return_gain: bool = False) -> Union[torch.Tensor, Tuple[torch.Tensor, torch.Tensor]]:
    """wav [..., L] on a CUDA device -> [..., L] f32: each row times its gain g = fp32(min(10^((target - L) / 20),
    10^(-1/20) / max|x|)) rounded toward zero, 1 for a row with L = -inf (returned bit for bit).  `lens`: valid samples per row; samples past
    lens[b] are not read and row b's outputs past lens[b] are zero.  `return_gain` (a test hook) also returns every
    row's g, f32 [...] on the device."""
    T = check_loudness(target)
    if T is None:
        raise ValueError("loudness target is None: there is nothing to normalise to")
    sr = _rate(sample_rate)
    x, lead, lp, most = _rows(wav, lens)
    B, L = x.shape
    y = (torch.empty if lp is None else torch.zeros)((B, L), dtype=torch.float32, device=x.device)
    gain = torch.empty(B, dtype=torch.float32, device=x.device)
    if B:
        ws = torch.empty(workspace_bytes(B, most, sr), dtype=torch.uint8, device=x.device)
        with torch.cuda.device(x.device):
            _lib.check_arg(_lib.load().sopro_loudness_normalize(x.data_ptr(), B, L, lp, sr, T, y.data_ptr(), L,
                                                                ws.data_ptr(), None, gain.data_ptr(),
                                                                _lib.stream_ptr(x.device)))
    y = y.reshape(*lead, L)
    return (y, gain.reshape(lead)) if return_gain else y
