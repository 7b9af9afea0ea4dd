"""Watermarking on the GPU (no reference counterpart: the reference's output carries no mark).

``embed_watermark(wav, key)`` adds a keyed spread-spectrum mark to 24 kHz rows, 30 dB below the local signal level, one
row or a ragged batch in two launches; ``WatermarkStream`` does the same chunk by chunk, and its chunks concatenate to
the one-shot result bit for bit.  ``detect_watermark(wav, sample_rate, key)`` scores rows at any rate the resampler
accepts against a key.  A key is an integer in [0, 2^32); ``check_watermark`` refuses anything else.  The kernels are
sopro_b200/csrc/watermark.cu, the definition is in include/sopro_b200.h and, in float64, oracle/watermark_oracle.py."""
from __future__ import annotations

import ctypes as C
import functools
import numbers
from typing import Dict, NamedTuple, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import _lib
from .config import TARGET_SR

PERIOD, BLOCK = 8192, 240  # SOPRO_WATERMARK_PERIOD, SOPRO_WATERMARK_BLOCK
THRESHOLD = 7.0  # SOPRO_WATERMARK_THRESHOLD: the score at and above which a row is detected
_resamplers: Dict[Tuple[int, int], object] = {}  # (input rate, device index) -> Resampler to 24 kHz


class Detection(NamedTuple):
    """Per row, on the device: ``score`` f32, ``offset`` i64 (the pattern's phase at the clip's first sample),
    ``detected`` bool (score >= THRESHOLD)."""
    score: torch.Tensor
    offset: torch.Tensor
    detected: torch.Tensor


def check_watermark(key) -> Optional[int]:
    """None for None (no mark), else the key as an int; ValueError for anything but an integer in [0, 2^32) (bools
    included).  Host only, nothing allocated."""
    if key is None:
        return None
    if isinstance(key, (bool, np.bool_)) or not isinstance(key, numbers.Integral) or not 0 <= int(key) < 1 << 32:
        raise ValueError(f"watermark must be an integer key in [0, 2^32), got {key!r}")
    return int(key)


def _key(key) -> int:
    k = check_watermark(key)
    if k is None:
        raise ValueError("watermark key is None: there is no pattern")
    return k


def watermark_pattern(key) -> np.ndarray:
    """The key's P fp32 pattern samples, computed on the host by the library.  Host only."""
    p = np.zeros(PERIOD, dtype=np.float32)
    _lib.check_arg(_lib.load().sopro_watermark_pattern(_key(key), p.ctypes.data))
    return p


@functools.lru_cache(maxsize=64)
def _pattern_on(key: int, device: torch.device) -> torch.Tensor:
    return torch.from_numpy(watermark_pattern(key)).to(device)


def pattern_tensor(key, device: torch.device) -> torch.Tensor:
    """The key's pattern on the device, cached per (key, device)."""
    dev = torch.device(device)
    if dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    return _pattern_on(_key(key), dev)


def _sizes(rows: int, most: int) -> Tuple[int, int]:
    e, d = C.c_int64(), C.c_int64()
    _lib.check_arg(_lib.load().sopro_watermark_sizes(int(rows), int(most), C.byref(e), C.byref(d)))
    return max(int(e.value), 1), max(int(d.value), 1)


def _rows(wav: torch.Tensor, lens: Optional[Sequence[int]], what: str):
    x, lead, lp = _lib.rows(wav, lens, what)
    most = int(x.shape[1]) if lp is None else max(lp, default=0)
    return x, lead, lp, most


def embed_watermark(wav: torch.Tensor, key, lens: Optional[Sequence[int]] = None) -> torch.Tensor:
    """wav [..., L] 24 kHz on a CUDA device (rows = the leading dims flattened) -> [..., L] f32, marked with the key.
    `lens`: valid samples per row (a ragged batch); samples past lens[b] are not read and row b's outputs past lens[b]
    are zero."""
    k = _key(key)
    x, lead, lp, most = _rows(wav, lens, "the watermark")
    B, L = x.shape
    y = (torch.empty if lp is None else torch.zeros)((B, L), dtype=torch.float32, device=x.device)
    if B and most:
        p = pattern_tensor(k, x.device)
        ws = torch.empty(_sizes(B, most)[0], dtype=torch.uint8, device=x.device)
        with torch.cuda.device(x.device):
            _lib.check_arg(_lib.load().sopro_watermark_embed(x.data_ptr(), B, L, lp, p.data_ptr(), y.data_ptr(), L,
                                                             ws.data_ptr(), _lib.stream_ptr(x.device)))
    return y.reshape(*lead, L)


def _to_24k(wav: torch.Tensor, sample_rate, lens: Optional[Sequence[int]]):
    from .resample import Resampler, _rate, check_rates

    if _rate(sample_rate) == TARGET_SR:
        return wav, lens
    sr = check_rates(sample_rate, TARGET_SR)[0]
    dev = wav.device
    idx = dev.index if dev.index is not None else torch.cuda.current_device()
    rs = _resamplers.get((sr, idx))
    if rs is None:
        rs = _resamplers[(sr, idx)] = Resampler(sr, TARGET_SR, idx)
    out = rs(wav, lens=lens)
    return out, None if lens is None else [rs.length(int(n)) for n in lens]


def detect_watermark(wav: torch.Tensor, sample_rate: int, key, lens: Optional[Sequence[int]] = None) -> Detection:
    """wav [..., L] at `sample_rate` on a CUDA device (rows = the leading dims flattened; `lens`: valid samples per row)
    -> Detection of tensors shaped [...], on the device.  Rows at another rate are resampled to 24 kHz first.  Detection
    is not promised below 8 kHz: the pattern's band reaches 3.5 kHz."""
    k = _key(key)
    if wav.device.type != "cuda":
        raise _lib.SoproError("watermark detection needs CUDA tensors; there is no CPU path")
    wav, lens = _to_24k(wav, sample_rate, lens)
    x, lead, lp, most = _rows(wav, lens, "watermark detection")
    B, L = x.shape
    dev = x.device
    score = torch.zeros(B, dtype=torch.float32, device=dev)
    offset = torch.zeros(B, dtype=torch.int64, device=dev)
    detected = torch.zeros(B, dtype=torch.bool, device=dev)
    if B:
        p = pattern_tensor(k, dev)
        ws = torch.empty(_sizes(B, most)[1], dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            _lib.check_arg(_lib.load().sopro_watermark_detect(x.data_ptr() if L else None, B, L, lp, p.data_ptr(),
                                                              ws.data_ptr(), score.data_ptr(), offset.data_ptr(),
                                                              detected.data_ptr(), _lib.stream_ptr(dev)))
    return Detection(score.reshape(lead), offset.reshape(lead), detected.reshape(lead))


class WatermarkStream(_lib.ChunkStream):
    """One utterance marked chunk by chunk: ``push(x)`` returns every complete 240-sample block of what it has been
    given, ``finish()`` the held partial block.  Their concatenation equals ``embed_watermark`` of the concatenated
    input bit for bit.  ``reset(key)`` starts a new utterance with any key, so one state serves every key."""

    _ready, _push, _finish = "sopro_watermark_stream_ready", "sopro_watermark_push", "sopro_watermark_finish"
    _destroy = "sopro_watermark_stream_destroy"
    _not_ready = "watermark stream is finished or has no key (reset it), or n_more < 0"

    def __init__(self, max_chunk: int, device: Union[int, str, torch.device] = 0, key=None):
        self.lib = _lib.load()
        dev = torch.device(device if not isinstance(device, int) else f"cuda:{device}")
        if dev.type != "cuda":
            raise _lib.SoproError("WatermarkStream needs a CUDA device; there is no CPU path")
        self.device = torch.device("cuda", dev.index if dev.index is not None else torch.cuda.current_device())
        self.max_chunk = int(max_chunk)
        h = C.c_void_p()
        _lib.check_arg(self.lib.sopro_watermark_stream_create(self.max_chunk, self.device.index, C.byref(h)))
        self._h = h
        self.pattern = None
        if key is not None:
            self.reset(key)

    def reset(self, key) -> None:
        p = pattern_tensor(key, self.device)
        _lib.check_arg(self.lib.sopro_watermark_stream_reset(self._h, p.data_ptr()))
        self.pattern = p  # the state reads it on the device until the next reset
