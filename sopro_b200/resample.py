"""Output resampling on the GPU (no reference counterpart: the reference always returns 24 kHz).

``Resampler(sr_in, sr_out, device)`` resamples waveforms, one row or a ragged batch in one launch; ``.stream(max_chunk)``
gives a ``ResamplerStream`` whose pushed chunks concatenate to the one-shot result bit for bit.  The filter is
torchaudio.functional.resample's default (sinc_interp_hann, lowpass_filter_width 6, rolloff 0.99); the kernels are
sopro_b200/csrc/resample.cu, the contract is in include/sopro_b200.h."""
from __future__ import annotations

import ctypes as C
import numbers
from typing import List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import _lib


def _check(rc: int) -> None:
    """SOPRO_ERR_INVALID (a refused rate, an oversized push) is a ValueError; anything else a SoproError."""
    if rc == -1:
        msg = _lib.load().sopro_last_error()
        raise ValueError(msg.decode() if msg else "invalid argument")
    _lib.check(rc)


def _rate(sr) -> int:
    if isinstance(sr, bool) or not isinstance(sr, numbers.Integral):
        if not (isinstance(sr, numbers.Real) and float(sr).is_integer()):
            raise ValueError(f"sample rates are integers in Hz, got {sr!r}")
    return int(sr)


def filter_taps(sr_in: int, sr_out: int) -> Tuple[int, int, int, np.ndarray, np.ndarray, np.ndarray]:
    """-> (o, n, width, first [n], span [n], taps [n, S]): phase p's nonzero fp32 taps are taps[p, :span[p]], at
    positions first[p] .. first[p] + span[p] of torchaudio's kernel row of 2 * width + o taps.  Host only."""
    lib = _lib.load()
    sr_in, sr_out = _rate(sr_in), _rate(sr_out)
    geo = np.zeros(4, dtype=np.int32)
    _check(lib.sopro_resampler_filter(sr_in, sr_out, geo.ctypes.data_as(_lib._I32P), None, None, None))
    o, n, width, S = (int(v) for v in geo)
    first, span = np.zeros(n, dtype=np.int32), np.zeros(n, dtype=np.int32)
    taps = np.zeros((n, S), dtype=np.float32)
    _check(lib.sopro_resampler_filter(sr_in, sr_out, geo.ctypes.data_as(_lib._I32P), first.ctypes.data_as(_lib._I32P),
                                      span.ctypes.data_as(_lib._I32P), taps.ctypes.data))
    return o, n, width, first, span, taps


def resampled_length(sr_in: int, sr_out: int, n_in: int) -> int:
    """ceil(n * n_in / o): the outputs of n_in input samples (ValueError for a refused rate pair).  Host only."""
    sr_in, sr_out = _rate(sr_in), _rate(sr_out)
    n = int(_lib.load().sopro_resampled_length(sr_in, sr_out, int(n_in)))
    if n < 0:
        filter_taps(sr_in, sr_out)  # raises with the reason when the rates are refused
        raise ValueError(f"cannot resample {n_in} samples")
    return n


def check_rates(sr_in: int, sr_out: int) -> Tuple[int, int]:
    """(sr_in, sr_out) as ints, or ValueError when the pair is not supported.  Host only, nothing allocated."""
    sr_in, sr_out = _rate(sr_in), _rate(sr_out)
    _check(_lib.load().sopro_resampler_filter(sr_in, sr_out, (C.c_int32 * 4)(), None, None, None))
    return sr_in, sr_out


def _stream_ptr(device: torch.device) -> int:
    return int(torch.cuda.current_stream(device).cuda_stream)


class Resampler:
    """sr_in -> sr_out on one CUDA device; the tap table lives on the device."""

    def __init__(self, sr_in: int, sr_out: int, device: Union[int, str, torch.device] = 0):
        self.sr_in, self.sr_out = check_rates(sr_in, sr_out)
        self.lib = _lib.load()
        dev = torch.device(device if not isinstance(device, int) else f"cuda:{device}")
        if dev.type != "cuda":
            raise _lib.SoproError("Resampler needs a CUDA device; there is no CPU path")
        self.device = torch.device("cuda", dev.index if dev.index is not None else torch.cuda.current_device())
        h = C.c_void_p()
        _check(self.lib.sopro_resampler_create(self.sr_in, self.sr_out, self.device.index, C.byref(h)))
        self._h = h
        self._idle: List[ResamplerStream] = []

    def length(self, n: int) -> int:
        """Output samples for n input samples: ceil(n * sr_out / sr_in)."""
        return resampled_length(self.sr_in, self.sr_out, n)

    def __call__(self, wav: torch.Tensor, lens: Optional[Sequence[int]] = None) -> torch.Tensor:
        """wav [..., N] (rows = the leading dims flattened) -> [..., length(N)] f32 on the device.  `lens`: valid samples
        per row (a ragged batch); samples past lens[b] are not read, and row b's outputs past length(lens[b]) are zero."""
        N = int(wav.shape[-1])
        lead = tuple(wav.shape[:-1])
        x = wav.detach().to(device=self.device, dtype=torch.float32).reshape(-1, N).contiguous()
        B = int(x.shape[0])
        L = self.length(N)
        if lens is None:
            y = torch.empty((B, L), dtype=torch.float32, device=self.device)
            lp = None
        else:
            if len(lens) != B:
                raise ValueError(f"lens has {len(lens)} entries for {B} rows")
            lp = (C.c_int64 * B)(*[int(v) for v in lens])
            y = torch.zeros((B, L), dtype=torch.float32, device=self.device)
        if B and L:
            _check(self.lib.sopro_resample(self._h, x.data_ptr(), B, N, lp, y.data_ptr(), L, _stream_ptr(self.device)))
        return y.reshape(*lead, L)

    def stream(self, max_chunk: int) -> "ResamplerStream":
        return ResamplerStream(self, max_chunk)

    def checkout_stream(self, max_chunk: int) -> "ResamplerStream":
        """A reset stream state: a released one when one is idle, so a new utterance allocates nothing."""
        for i, s in enumerate(self._idle):
            if s.max_chunk >= max_chunk:
                del self._idle[i]
                s.reset()
                return s
        return self.stream(max_chunk)

    def release_stream(self, s: Optional["ResamplerStream"]) -> None:
        if s is not None and len(self._idle) < 4:
            self._idle.append(s)

    def close(self) -> None:
        for s in self._idle:
            s.close()
        self._idle = []
        if getattr(self, "_h", None):
            self.lib.sopro_resampler_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class ResamplerStream:
    """One utterance resampled chunk by chunk: ``push(x)`` returns every output whose filter window has arrived,
    ``finish()`` the rest.  Their concatenation equals ``Resampler`` on the concatenated input, bit for bit."""

    def __init__(self, resampler: Resampler, max_chunk: int):
        self.resampler, self.lib = resampler, resampler.lib
        self.max_chunk = int(max_chunk)
        h = C.c_void_p()
        _check(self.lib.sopro_resampler_stream_create(resampler._h, self.max_chunk, C.byref(h)))
        self._h = h

    def ready(self, n_more: int, final: bool = False) -> int:
        """Outputs a push of n_more samples (followed by finish when `final`) would write."""
        n = int(self.lib.sopro_resampler_stream_ready(self._h, int(n_more), 1 if final else 0))
        if n < 0:
            raise _lib.SoproError("resampler stream is finished (reset it) or n_more < 0")
        return n

    def push(self, x: torch.Tensor) -> torch.Tensor:
        """x: the next samples (any shape, flattened; at most max_chunk) -> [k] f32 on the device."""
        dev = self.resampler.device
        x = x.detach().to(device=dev, dtype=torch.float32).reshape(-1).contiguous()
        n = int(x.numel())
        k = int(self.lib.sopro_resampler_stream_ready(self._h, n, 0))
        y = torch.empty(max(k, 0), dtype=torch.float32, device=dev)
        _check(self.lib.sopro_resampler_push(self._h, x.data_ptr() if n else None, n, y.data_ptr() if k > 0 else None,
                                             _stream_ptr(dev)))
        return y

    def finish(self) -> torch.Tensor:
        """The remaining outputs (the input's end zero padded) -> [k]; the stream then takes no push until reset()."""
        dev = self.resampler.device
        k = int(self.lib.sopro_resampler_stream_ready(self._h, 0, 1))
        y = torch.empty(max(k, 0), dtype=torch.float32, device=dev)
        _check(self.lib.sopro_resampler_finish(self._h, y.data_ptr() if k > 0 else None, _stream_ptr(dev)))
        return y

    def reset(self) -> None:
        _check(self.lib.sopro_resampler_stream_reset(self._h))

    def close(self) -> None:
        if getattr(self, "_h", None) and getattr(self.resampler, "_h", None):
            self.lib.sopro_resampler_stream_destroy(self._h)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
