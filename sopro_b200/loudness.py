"""Loudness normalisation on the GPU (no reference counterpart: the reference's output level follows its reference
recording).

``measure_loudness(wav, sample_rate)`` is the ITU-R BS.1770-4 integrated loudness of each row in LUFS (float64, on the
device; -inf for a row with no gated block), ``normalize_loudness(wav, sample_rate, target)`` scales each row to the
target under a fixed -1 dBFS sample-peak ceiling.  Both take one row or a ragged batch in one call, and neither
synchronises with the host.  A target is a real number in [-60, 0] LUFS; ``check_loudness`` refuses anything else.  The
kernels are sopro_b200/csrc/loudness.cu, the contract is in include/sopro_b200.h.

Live loudness, for audio that is still arriving: ``LiveLeveller`` levels one stream chunk by chunk, ``level_live`` is its
one-shot form over a ragged batch, and ``level_stream`` / ``level_stream_batch`` wrap the items of ``SoproTTS.stream``,
``stream_long``, ``stream_dialogue`` and ``stream_batch``.  Its gain follows the integrated loudness of the audio so far
(a passage level, not an AGC: a quiet voice late in a long stream barely moves it), capped at +30 dB, under the same -1
dBFS ceiling; audio goes out in whole 100 ms sub-blocks once the first 400 ms have been metered.  The gain converges on
normalize_loudness's as the stream goes on, but it is a different, causal definition (include/sopro_b200.h): a stream's
levelled output equals ``level_live`` of its concatenation, not ``normalize_loudness``.  The kernels are
sopro_b200/csrc/level.cu, the oracle is oracle/loudness_live_oracle.py."""
from __future__ import annotations

import numbers
import ctypes as C
from typing import Iterable, Iterator, Optional, Sequence, Tuple, Union

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


def _level_target(target) -> float:
    T = check_loudness(target)
    if T is None:
        raise ValueError("loudness target is None: there is nothing to level to")
    return T


def level_live(wav: torch.Tensor, sample_rate: int, target, lens: Optional[Sequence[int]] = None,
               return_gains: bool = False) -> Union[torch.Tensor, Tuple[torch.Tensor, torch.Tensor, torch.Tensor]]:
    """wav [..., L] on a CUDA device -> [..., L] f32: each row levelled by the causal leveller (include/sopro_b200.h),
    exactly what ``LiveLeveller`` releases for that row, whatever its chunks.  `lens`: valid samples per row; samples
    past lens[b] are not read and row b's outputs past lens[b] are zero.  `return_gains` (a test hook) also returns
    every complete sub-block's a_k and M_k, float64 [..., floor(max lens / s)] on the device (NaN for k < 3 and past a
    row's sub-blocks)."""
    T = _level_target(target)
    sr = _rate(sample_rate)
    workspace_bytes(1, 0, sr)  # refuses the rate
    x, lead, lp, most = _rows(wav, lens)
    B, L = x.shape
    nsb = most // ((sr + 5) // 10)
    y = (torch.empty if lp is None else torch.zeros)((B, L), dtype=torch.float32, device=x.device)
    gains = meter = None
    if return_gains:
        gains = torch.full((B, nsb), float("nan"), dtype=torch.float64, device=x.device)
        meter = torch.full((B, nsb), float("nan"), dtype=torch.float64, device=x.device)
    if B:
        lib = _lib.load()
        n = int(lib.sopro_level_workspace(B, most, sr))
        if n < 0:
            raise ValueError(f"bad geometry: {B} rows of {most} samples")
        ws = torch.empty(max(n, 1), dtype=torch.uint8, device=x.device)
        with torch.cuda.device(x.device):
            _lib.check_arg(lib.sopro_level(x.data_ptr(), B, L, lp, sr, T, y.data_ptr(), L, ws.data_ptr(),
                                           None if meter is None else meter.data_ptr(),
                                           None if gains is None else gains.data_ptr(), _lib.stream_ptr(x.device)))
    y = y.reshape(*lead, L)
    if return_gains:
        return y, gains.reshape(*lead, nsb), meter.reshape(*lead, nsb)
    return y


class LiveLeveller(_lib.ChunkStream):
    """One stream levelled as it arrives: ``push(chunk) -> [1, k]`` returns the samples the chunk completes (none
    before the first 400 ms, then whole 100 ms sub-blocks), ``finish() -> [1, k]`` the rest.  Their concatenation
    equals ``level_live`` of the concatenated input bit for bit, whatever the chunk sizes.  ``reset(target)`` starts
    a new stream.  Each push that completes a sub-block is one launch; nothing synchronises with the host."""

    _ready, _push, _finish = "sopro_level_stream_ready", "sopro_level_push", "sopro_level_finish"
    _destroy = "sopro_level_stream_destroy"
    _not_ready = "live leveller is finished (reset it), or n_more < 0"
    max_chunk = 1 << 20  # samples per launch; a longer chunk is pushed in pieces (the output does not depend on them)

    def __init__(self, sample_rate: int, target, device: Optional[Union[int, str, torch.device]] = None):
        T = _level_target(target)
        self.sample_rate = _rate(sample_rate)
        workspace_bytes(1, 0, self.sample_rate)  # refuses the rate
        self.lib = _lib.load()
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(
            device if not isinstance(device, int) else f"cuda:{device}")
        if dev.type != "cuda":
            raise _lib.SoproError("LiveLeveller needs a CUDA device; there is no CPU path")
        self.device = torch.device("cuda", dev.index if dev.index is not None else torch.cuda.current_device())
        h = C.c_void_p()
        _lib.check_arg(self.lib.sopro_level_stream_create(self.max_chunk, self.sample_rate, self.device.index, C.byref(h)))
        self._h = h
        self.reset(T)

    def reset(self, target) -> None:
        self.target = _level_target(target)
        _lib.check_arg(self.lib.sopro_level_stream_reset(self._h, self.target))

    def push(self, chunk: torch.Tensor) -> torch.Tensor:
        if not isinstance(chunk, torch.Tensor) or chunk.device.type != "cuda":
            raise _lib.SoproError("live levelling needs CUDA tensors; there is no CPU path")
        if chunk.device != self.device:
            raise ValueError(f"chunk on {chunk.device}, the leveller on {self.device}")
        x = chunk.detach().to(dtype=torch.float32).reshape(-1)
        with torch.cuda.device(self.device):
            if x.numel() <= self.max_chunk:
                return super().push(x).reshape(1, -1)
            return torch.cat([super(LiveLeveller, self).push(x[i: i + self.max_chunk])
                              for i in range(0, int(x.numel()), self.max_chunk)]).reshape(1, -1)

    def finish(self) -> torch.Tensor:
        with torch.cuda.device(self.device):
            return super().finish().reshape(1, -1)


_POOLS: dict = {}


def _leveller(sr: int, T: float, device: torch.device) -> Tuple["LiveLeveller", "_lib.StatePool"]:
    """An idle leveller of this rate and device reset to T, or a new one (creating one allocates and synchronises)."""
    key = (torch.device(device), sr)
    pool = _POOLS.get(key)
    if pool is None:
        pool = _POOLS[key] = _lib.StatePool(lambda _max_chunk, T: LiveLeveller(sr, T, device=key[0]))
    return pool.checkout(LiveLeveller.max_chunk, T), pool


def level_stream(items: Iterable, sample_rate: int = 24000, *, target) -> Iterator:
    """The chunks of ``SoproTTS.stream``, ``stream_long`` or ``stream_dialogue`` ([1, n] on the device at
    `sample_rate`), levelled live to `target` LUFS: the same kind of items, each holding what its chunk completes, then
    the held tail.  ``stream(word_timestamps=True)``'s ``(wav, words)`` pairs keep their words unchanged (a gain moves
    no time).  Items with neither samples nor words are not yielded.  The yielded audio concatenates to
    ``level_live`` of the unwrapped stream's concatenation bit for bit.  A refused rate or target raises here, before
    the stream is read."""
    T = _level_target(target)
    sr = _rate(sample_rate)
    workspace_bytes(1, 0, sr)

    def gen():
        lev = pool = None
        pairs = False
        try:
            for item in items:
                pairs = isinstance(item, tuple)
                wav, words = item if pairs else (item, None)
                if lev is None:
                    lev, pool = _leveller(sr, T, wav.device)
                y = lev.push(wav)
                if y.shape[-1] or (pairs and words):
                    yield (y, words) if pairs else y
            if lev is not None:
                y = lev.finish()
                if y.shape[-1]:
                    yield (y, []) if pairs else y
        finally:
            if pool is not None:
                pool.release(lev)

    return gen()


def level_stream_batch(items: Iterable[tuple], sample_rate: int = 24000, *, target) -> Iterator[tuple]:
    """The items of ``SoproTTS.stream_batch`` -- ``(i, wav, last)`` or ``(i, wav, last, words)`` -- levelled live to
    `target` LUFS, one leveller per row: row i's items hold what its chunks complete, and its last item (always
    yielded) carries the row's held tail.  Other items with neither samples nor words are not yielded; words pass
    through unchanged.  Row i's audio concatenates to ``level_live`` of that row's unwrapped concatenation bit for
    bit.  A refused rate or target raises here, before the stream is read.  Idle levellers are kept for the next call
    (as the streams' own output stages are), so a stream allocates nothing once one has run."""
    T = _level_target(target)
    sr = _rate(sample_rate)
    workspace_bytes(1, 0, sr)

    def gen():
        levs = {}
        try:
            for item in items:
                i, wav, last = item[0], item[1], item[2]
                if i not in levs:
                    levs[i] = _leveller(sr, T, wav.device)
                lev, pool = levs[i]
                y = lev.push(wav)
                if last:
                    y = torch.cat([y, lev.finish()], dim=-1)
                    pool.release(levs.pop(i)[0])
                if last or y.shape[-1] or (len(item) > 3 and item[3]):
                    yield (i, y, last) + tuple(item[3:])
        finally:
            for lev, pool in levs.values():
                pool.release(lev)

    return gen()
