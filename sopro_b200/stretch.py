"""Speaking-rate control on the GPU (no reference counterpart: the reference has no rate control).

``stretch(wav, speed)`` time-stretches 24 kHz waveforms by WSOLA, pitch preserved, one row or a ragged batch in one
launch; ``StretchStream`` does the same chunk by chunk, and its chunks concatenate to the one-shot result bit for bit.
A speed is a real number in [0.25, 4.0], quantised to S = round(speed * 65536); ``check_speed`` returns None for a
bypass (None, or S = 65536).  The kernels are sopro_b200/csrc/stretch.cu, the contract is in include/sopro_b200.h."""
from __future__ import annotations

import ctypes as C
import numbers
from typing import Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import _lib

FRAME, HOP, TOLERANCE = 480, 240, 160  # N, Hs, D of the kernels


def quantise(speed) -> int:
    """S = round(speed * 65536) for an accepted speed (a real number in [0.25, 4.0]); ValueError otherwise.  Host only."""
    if isinstance(speed, (bool, np.bool_)) or not isinstance(speed, numbers.Real):
        raise ValueError(f"speed must be a real number in [0.25, 4.0], got {speed!r}")
    S = C.c_int32()
    _lib.check_arg(_lib.load().sopro_stretch_speed(float(speed), C.byref(S)))
    return int(S.value)


def check_speed(speed) -> Optional[int]:
    """None for a bypass (speed None, or one that quantises to S = 65536), else S; ValueError for a refused speed.
    Host only, nothing allocated."""
    if speed is None:
        return None
    S = quantise(speed)
    return None if S == 65536 else S


def _S(speed) -> int:
    if speed is None:
        raise ValueError("speed is None: there is nothing to stretch")
    return quantise(speed)


def stretched_length(speed, n: int) -> int:
    """M = ceil(n * 65536 / S), the outputs of n input samples.  Host only."""
    m = int(_lib.load().sopro_stretched_length(_S(speed), int(n)))
    if m < 0:
        raise ValueError(f"cannot stretch {n} samples")
    return m


def frame_positions(speed, n: int) -> np.ndarray:
    """The nominal analysis positions a_k of the K frames of n input samples (int64 [K]).  Host only."""
    lib, S = _lib.load(), _S(speed)
    K = int(lib.sopro_stretch_positions(S, int(n), None))
    if K < 0:
        raise ValueError(f"cannot stretch {n} samples")
    a = np.zeros(K, dtype=np.int64)
    if K:
        lib.sopro_stretch_positions(S, int(n), a.ctypes.data)
    return a


def n_frames(n_out: int) -> int:
    """K = ceil(M / Hs) + 1 frames for M outputs (0 when M = 0)."""
    return 0 if n_out == 0 else -(-int(n_out) // HOP) + 1


def stretch_window() -> np.ndarray:
    """The 480 fp32 window taps the kernels use: sin^2(pi n / 480) in double, rounded once.  Host only."""
    w = np.zeros(FRAME, dtype=np.float32)
    _lib.check_arg(_lib.load().sopro_stretch_window(w.ctypes.data))
    return w


def stretch(wav: torch.Tensor, speed, lens: Optional[Sequence[int]] = None,
            return_offsets: bool = False) -> Union[torch.Tensor, Tuple[torch.Tensor, torch.Tensor]]:
    """wav [..., L] on a CUDA device (rows = the leading dims flattened) -> [..., M] f32, M = stretched_length(speed, L).
    `lens`: valid samples per row (a ragged batch); samples past lens[b] are not read, and row b's outputs past
    stretched_length(lens[b]) are zero.  Every accepted speed runs the kernel, 1.0 included (the public API bypasses
    S = 65536 itself).  `return_offsets` (a test hook) also returns every frame's d_k, int32 [rows, K_max]."""
    S = _S(speed)
    x, lead, lp = _lib.rows(wav, lens, "the time-stretch")
    dev = x.device
    B, L = x.shape
    M = stretched_length(speed, L)
    y = (torch.empty if lp is None else torch.zeros)((B, M), dtype=torch.float32, device=dev)
    m_max = max((stretched_length(speed, int(v)) for v in lens), default=0) if lens is not None else M
    offs = torch.zeros((B, n_frames(m_max)), dtype=torch.int32, device=dev) if return_offsets else None
    if B and M:
        with torch.cuda.device(dev):
            _lib.check_arg(_lib.load().sopro_stretch(x.data_ptr(), B, L, lp, S, y.data_ptr(), M,
                                                     offs.data_ptr() if offs is not None and offs.numel() else None,
                                                     _lib.stream_ptr(dev)))
    y = y.reshape(*lead, M)
    return (y, offs) if return_offsets else y


def stretch_rows(wav: torch.Tensor, speeds: Sequence, lens: Optional[Sequence[int]] = None,
                 return_offsets: bool = False) -> Union[torch.Tensor, Tuple[torch.Tensor, torch.Tensor]]:
    """stretch with a speed per row, in one launch: wav [..., L] on a CUDA device (rows = the leading dims flattened),
    `speeds` one accepted speed per row -> [..., M] f32, M the longest row's stretched_length(speeds[b], lens[b]).  Row
    b has stretched_length(speeds[b], lens[b]) outputs, zeros after them; a row whose speed quantises to S = 65536 is
    its input copied through, any other row equals stretch of that row alone at its speed, bit for bit.  Every speed is
    checked before any work.  `return_offsets` (a test hook) also returns every frame's d_k, int32 [rows, K_max]; a
    copied row's stay 0."""
    x, lead, lp = _lib.rows(wav, lens, "the time-stretch")
    dev = x.device
    B, L = x.shape
    speeds = list(speeds)
    if len(speeds) != B:
        raise ValueError(f"{len(speeds)} speeds for {B} rows")
    S = [_S(v) for v in speeds]
    n = [L] * B if lens is None else [int(v) for v in lens]
    M = max((stretched_length(v, k) for v, k in zip(speeds, n)), default=0)
    y = torch.zeros((B, M), dtype=torch.float32, device=dev)
    offs = torch.zeros((B, n_frames(M)), dtype=torch.int32, device=dev) if return_offsets else None
    if B and M:
        with torch.cuda.device(dev):
            _lib.check_arg(_lib.load().sopro_stretch_rows(x.data_ptr(), B, L, lp, (C.c_int32 * B)(*S), y.data_ptr(), M,
                                                          offs.data_ptr() if offs is not None else None,
                                                          _lib.stream_ptr(dev)))
    y = y.reshape(*lead, M)
    return (y, offs) if return_offsets else y


class StretchStream(_lib.ChunkStream):
    """One utterance time-stretched chunk by chunk: ``push(x)`` returns every output the frames its input completes
    have finished, ``finish()`` the rest.  Their concatenation equals ``stretch`` of the concatenated input bit for bit.
    ``reset(speed)`` starts a new utterance at any accepted speed, so one state serves every speed."""

    _ready, _push, _finish = "sopro_stretch_stream_ready", "sopro_stretch_push", "sopro_stretch_finish"
    _destroy = "sopro_stretch_stream_destroy"
    _not_ready = "stretch stream is finished or has no speed (reset it), or n_more < 0"

    def __init__(self, max_chunk: int, device: Union[int, str, torch.device] = 0, speed=None):
        self.lib = _lib.load()
        dev = torch.device(device if not isinstance(device, int) else f"cuda:{device}")
        if dev.type != "cuda":
            raise _lib.SoproError("StretchStream needs a CUDA device; there is no CPU path")
        self.device = torch.device("cuda", dev.index if dev.index is not None else torch.cuda.current_device())
        self.max_chunk = int(max_chunk)
        h = C.c_void_p()
        _lib.check_arg(self.lib.sopro_stretch_stream_create(self.max_chunk, self.device.index, C.byref(h)))
        self._h = h
        self.S = 0
        if speed is not None:
            self.reset(speed)

    def reset(self, speed) -> None:
        S = _S(speed)
        _lib.check_arg(self.lib.sopro_stretch_stream_reset(self._h, S))
        self.S = S
