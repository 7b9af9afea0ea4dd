"""Speaking-rate control on the GPU (no reference counterpart: the reference has no rate control).

``stretch(wav, speed)`` time-stretches 24 kHz waveforms by WSOLA, pitch preserved, one row or a ragged batch in one
launch; ``StretchStream`` does the same chunk by chunk, and its chunks concatenate to the one-shot result bit for bit.
A speed is a real number in [0.25, 4.0], quantised to S = round(speed * 65536); ``check_speed`` returns None for a
bypass (None, or S = 65536).  The kernels are sopro_b200/csrc/stretch.cu, the contract is in include/sopro_b200.h."""
from __future__ import annotations

import ctypes as C
import math
import numbers
from typing import List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import _lib

FRAME, HOP, TOLERANCE = 480, 240, 160  # N, Hs, D of the kernels


def _check(rc: int) -> None:
    """SOPRO_ERR_INVALID (a refused speed, an oversized push) is a ValueError; anything else a SoproError."""
    if rc == -1:
        msg = _lib.load().sopro_last_error()
        raise ValueError(msg.decode() if msg else "invalid argument")
    _lib.check(rc)


def quantise(speed) -> int:
    """S = round(speed * 65536) for an accepted speed (a real number in [0.25, 4.0]); ValueError otherwise.  Host only."""
    if isinstance(speed, (bool, np.bool_)) or not isinstance(speed, numbers.Real):
        raise ValueError(f"speed must be a real number in [0.25, 4.0], got {speed!r}")
    S = C.c_int32()
    _check(_lib.load().sopro_stretch_speed(float(speed), C.byref(S)))
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
    _check(_lib.load().sopro_stretch_window(w.ctypes.data))
    return w


def _stream_ptr(device: torch.device) -> int:
    return int(torch.cuda.current_stream(device).cuda_stream)


def _cuda(wav: torch.Tensor) -> torch.device:
    if wav.device.type != "cuda":
        raise _lib.SoproError("the time-stretch needs CUDA tensors; there is no CPU path")
    return wav.device


def stretch(wav: torch.Tensor, speed, lens: Optional[Sequence[int]] = None,
            return_offsets: bool = False) -> Union[torch.Tensor, Tuple[torch.Tensor, torch.Tensor]]:
    """wav [..., L] on a CUDA device (rows = the leading dims flattened) -> [..., M] f32, M = stretched_length(speed, L).
    `lens`: valid samples per row (a ragged batch); samples past lens[b] are not read, and row b's outputs past
    stretched_length(lens[b]) are zero.  Every accepted speed runs the kernel, 1.0 included (the public API bypasses
    S = 65536 itself).  `return_offsets` (a test hook) also returns every frame's d_k, int32 [rows, K_max]."""
    S = _S(speed)
    dev = _cuda(wav)
    L = int(wav.shape[-1])
    lead = tuple(wav.shape[:-1])
    B = math.prod(lead)
    x = wav.detach().to(dtype=torch.float32).reshape(B, L).contiguous()
    M = stretched_length(speed, L)
    if lens is None:
        y = torch.empty((B, M), dtype=torch.float32, device=dev)
        lp = None
    else:
        if len(lens) != B:
            raise ValueError(f"lens has {len(lens)} entries for {B} rows")
        lp = (C.c_int64 * B)(*[int(v) for v in lens])
        y = torch.zeros((B, M), dtype=torch.float32, device=dev)
    m_max = max((stretched_length(speed, int(v)) for v in lens), default=0) if lens is not None else M
    offs = torch.zeros((B, n_frames(m_max)), dtype=torch.int32, device=dev) if return_offsets else None
    if B and M:
        with torch.cuda.device(dev):
            _check(_lib.load().sopro_stretch(x.data_ptr(), B, L, lp, S, y.data_ptr(), M,
                                             offs.data_ptr() if offs is not None and offs.numel() else None, _stream_ptr(dev)))
    y = y.reshape(*lead, M)
    return (y, offs) if return_offsets else y


class StretchStream:
    """One utterance time-stretched chunk by chunk: ``push(x)`` returns every output the frames its input completes
    have finished, ``finish()`` the rest.  Their concatenation equals ``stretch`` of the concatenated input bit for bit.
    ``reset(speed)`` starts a new utterance at any accepted speed, so one state serves every speed."""

    def __init__(self, max_chunk: int, device: Union[int, str, torch.device] = 0, speed=None):
        self.lib = _lib.load()
        dev = torch.device(device if not isinstance(device, int) else f"cuda:{device}")
        if dev.type != "cuda":
            raise _lib.SoproError("StretchStream needs a CUDA device; there is no CPU path")
        self.device = torch.device("cuda", dev.index if dev.index is not None else torch.cuda.current_device())
        self.max_chunk = int(max_chunk)
        h = C.c_void_p()
        _check(self.lib.sopro_stretch_stream_create(self.max_chunk, self.device.index, C.byref(h)))
        self._h = h
        self.S = 0
        if speed is not None:
            self.reset(speed)

    def reset(self, speed) -> None:
        S = _S(speed)
        _check(self.lib.sopro_stretch_stream_reset(self._h, S))
        self.S = S

    def ready(self, n_more: int, final: bool = False) -> int:
        """Outputs a push of n_more samples (followed by finish when `final`) would write."""
        n = int(self.lib.sopro_stretch_stream_ready(self._h, int(n_more), 1 if final else 0))
        if n < 0:
            raise _lib.SoproError("stretch stream is finished or has no speed (reset it), or n_more < 0")
        return n

    def push(self, x: torch.Tensor) -> torch.Tensor:
        """x: the next samples (any shape, flattened; at most max_chunk) -> [k] f32 on the device."""
        dev = self.device
        x = x.detach().to(device=dev, dtype=torch.float32).reshape(-1).contiguous()
        n = int(x.numel())
        k = int(self.lib.sopro_stretch_stream_ready(self._h, n, 0))
        y = torch.empty(max(k, 0), dtype=torch.float32, device=dev)
        _check(self.lib.sopro_stretch_push(self._h, x.data_ptr() if n else None, n, y.data_ptr() if k > 0 else None,
                                           _stream_ptr(dev)))
        return y

    def finish(self) -> torch.Tensor:
        """The remaining outputs (the input's end zero padded) -> [k]; the stream then takes no push until reset()."""
        dev = self.device
        k = int(self.lib.sopro_stretch_stream_ready(self._h, 0, 1))
        y = torch.empty(max(k, 0), dtype=torch.float32, device=dev)
        _check(self.lib.sopro_stretch_finish(self._h, y.data_ptr() if k > 0 else None, _stream_ptr(dev)))
        return y

    def close(self) -> None:
        if getattr(self, "_h", None):
            self.lib.sopro_stretch_stream_destroy(self._h)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class StretchPool:
    """Idle stream states of one device, reused by the next utterance at any speed (a new one allocates nothing)."""

    def __init__(self, device: torch.device):
        self.device = device
        self._idle: List[StretchStream] = []

    def checkout(self, max_chunk: int, speed) -> StretchStream:
        for i, s in enumerate(self._idle):
            if s.max_chunk >= max_chunk:
                del self._idle[i]
                s.reset(speed)
                return s
        return StretchStream(max_chunk, self.device, speed)

    def release(self, s: Optional[StretchStream]) -> None:
        if s is not None and len(self._idle) < 4:
            self._idle.append(s)
