"""Output resampling on the GPU (no reference counterpart: the reference always returns 24 kHz).

``Resampler(sr_in, sr_out, device)`` resamples waveforms, one row or a ragged batch in one launch; ``.stream(max_chunk)``
gives a ``ResamplerStream`` whose pushed chunks concatenate to the one-shot result bit for bit.  The filter is
torchaudio.functional.resample's default (sinc_interp_hann, lowpass_filter_width 6, rolloff 0.99); the kernels are
sopro_b200/csrc/resample.cu, the contract is in include/sopro_b200.h."""
from __future__ import annotations

import ctypes as C
import numbers
from typing import Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import _lib


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
    _lib.check_arg(lib.sopro_resampler_filter(sr_in, sr_out, geo.ctypes.data_as(_lib._I32P), None, None, None))
    o, n, width, S = (int(v) for v in geo)
    first, span = np.zeros(n, dtype=np.int32), np.zeros(n, dtype=np.int32)
    taps = np.zeros((n, S), dtype=np.float32)
    _lib.check_arg(lib.sopro_resampler_filter(sr_in, sr_out, geo.ctypes.data_as(_lib._I32P),
                                              first.ctypes.data_as(_lib._I32P), span.ctypes.data_as(_lib._I32P),
                                              taps.ctypes.data))
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
    _lib.check_arg(_lib.load().sopro_resampler_filter(sr_in, sr_out, (C.c_int32 * 4)(), None, None, None))
    return sr_in, sr_out


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
        _lib.check_arg(self.lib.sopro_resampler_create(self.sr_in, self.sr_out, self.device.index, C.byref(h)))
        self._h = h
        self.pool = _lib.StatePool(self.stream)  # idle stream states: a new utterance allocates nothing

    def length(self, n: int) -> int:
        """Output samples for n input samples: ceil(n * sr_out / sr_in)."""
        return resampled_length(self.sr_in, self.sr_out, n)

    def __call__(self, wav: torch.Tensor, lens: Optional[Sequence[int]] = None) -> torch.Tensor:
        """wav [..., N] (rows = the leading dims flattened) -> [..., length(N)] f32 on the device.  `lens`: valid samples
        per row (a ragged batch); samples past lens[b] are not read, and row b's outputs past length(lens[b]) are zero."""
        x, lead, lp = _lib.rows(wav.to(device=self.device), lens, "Resampler")
        B, N = x.shape
        L = self.length(N)
        y = (torch.empty if lp is None else torch.zeros)((B, L), dtype=torch.float32, device=self.device)
        if B and L:
            _lib.check_arg(self.lib.sopro_resample(self._h, x.data_ptr(), B, N, lp, y.data_ptr(), L,
                                                   _lib.stream_ptr(self.device)))
        return y.reshape(*lead, L)

    def stream(self, max_chunk: int) -> "ResamplerStream":
        return ResamplerStream(self, max_chunk)

    def close(self) -> None:
        if getattr(self, "pool", None):
            self.pool.close()
        if getattr(self, "_h", None):
            self.lib.sopro_resampler_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class ResamplerStream(_lib.ChunkStream):
    """One utterance resampled chunk by chunk: ``push(x)`` returns every output whose filter window has arrived,
    ``finish()`` the rest.  Their concatenation equals ``Resampler`` on the concatenated input, bit for bit."""

    _ready, _push, _finish = "sopro_resampler_stream_ready", "sopro_resampler_push", "sopro_resampler_finish"
    _destroy = "sopro_resampler_stream_destroy"
    _not_ready = "resampler stream is finished (reset it) or n_more < 0"

    def __init__(self, resampler: Resampler, max_chunk: int):
        self.resampler, self.lib = resampler, resampler.lib
        self._owner, self.device = resampler, resampler.device
        self.max_chunk = int(max_chunk)
        h = C.c_void_p()
        _lib.check_arg(self.lib.sopro_resampler_stream_create(resampler._h, self.max_chunk, C.byref(h)))
        self._h = h

    def reset(self) -> None:
        _lib.check_arg(self.lib.sopro_resampler_stream_reset(self._h))
