"""Voice ingestion on the GPU: many reference voices prepared in one batched pass, from in-memory audio or files.

``SoproTTS.prepare_references(clips, sample_rates=..., ref_seconds=...)`` follows ``MimiCodec.encode_file`` (reference
codec/mimi.py:41-63) step for step: energy trim at the clip's own rate, resample to 24 kHz, centre crop, Mimi encode,
reference preparation.  The first four steps run on the device for the whole batch (``MimiCodec.prepare_wavs``,
``MimiCodec.encode_wavs``); the one host read is the B trim extents, which size the rest.  This module checks and loads
the clips (every refusal happens here, before any device work) and binds the two ingestion launches of
sopro_b200/csrc/ingest.cu; the definitions are in include/sopro_b200.h."""
from __future__ import annotations

import ctypes as C
import numbers
import os
from typing import List, Optional, Sequence, Tuple, Union

import torch

from . import _lib
from .config import TARGET_SR
from .resample import _rate, check_rates, resampled_length

ENC_MAX_SAMPLES = 24000 * 600  # the Mimi encoder's bound per call (kEncMaxSamples, mimi_engine.cu): ten minutes at 24 kHz
FRAME_SAMPLES = 1920           # 24 kHz samples per 12.5 Hz codec frame
DEFAULT_REF_SECONDS = 12.0     # prepare_reference's default crop

Clip = Union[str, os.PathLike, torch.Tensor]


def crop_samples(crop_seconds: Optional[float]) -> int:
    """encode_file's centre-crop window in 24 kHz samples, max(1, round(s * 12.5)) * 1920; 0 (no crop) for None or s <= 0."""
    if crop_seconds is None:
        return 0
    if isinstance(crop_seconds, bool) or not isinstance(crop_seconds, numbers.Real):
        raise TypeError(f"crop seconds must be a number, got {crop_seconds!r}")
    if not crop_seconds > 0:
        return 0
    return max(1, int(round(float(crop_seconds) * 12.5))) * FRAME_SAMPLES


def crop_plan(n: int, win: int) -> Tuple[int, int]:
    """(offset, length) of the reference's center_crop_audio over n samples: the middle `win` when n > win > 0."""
    if win <= 0 or n <= win:
        return 0, n
    return (n - win) // 2, win


def _is_path(c) -> bool:
    return isinstance(c, (str, os.PathLike))


def _check_wav(wav: torch.Tensor, sr, i: int) -> int:
    """A clip [n] or [C, n] of floats at rate sr, which the resampler takes and the encoder can hold once at 24 kHz ->
    its rate.  Reads no sample."""
    if wav.dtype == torch.bool or not (wav.dtype.is_floating_point):
        raise TypeError(f"clip {i}: audio must be a float tensor, got {wav.dtype}")
    if wav.ndim not in (1, 2):
        raise ValueError(f"clip {i}: expected [n] or [channels, n], got shape {tuple(wav.shape)}")
    n = int(wav.shape[-1])
    if n == 0 or wav.numel() == 0:
        raise ValueError(f"clip {i} is empty")
    if sr is None:
        raise ValueError(f"clip {i} is a tensor without a sample rate (pass sample_rates=...)")
    sr = _rate(sr)
    if sr != TARGET_SR:
        check_rates(sr, TARGET_SR)
    n24 = n if sr == TARGET_SR else resampled_length(sr, TARGET_SR, n)
    if n24 > ENC_MAX_SAMPLES:
        raise ValueError(f"clip {i} is {n24} samples at 24 kHz; the encoder takes at most {ENC_MAX_SAMPLES}")
    return sr


def check_finite(wav: torch.Tensor, what: str) -> None:
    """ValueError unless every sample of wav is finite.  A NaN or infinite sample (a float file can hold one; peak
    normalising a silent clip makes every sample NaN) has no meaning as audio, and the encoder's codes of it would be
    the codebooks' first entries, not a voice."""
    if not bool(torch.isfinite(wav).all()):
        raise ValueError(f"{what} holds non-finite samples (NaN or infinity)")


def load_clips(clips: Sequence[Clip], sample_rates=None) -> Tuple[List[torch.Tensor], List[int]]:
    """The clips checked, then the paths read on the host (audio.load_audio_file) -> (tensors, rates).  `sample_rates`:
    one rate per clip (None for a path, which supplies its own), or one int for every tensor clip.  Every tensor clip's
    shape, type and rate are checked before any file is read; then every clip's samples must be finite.  Nothing here
    launches the library's kernels (a clip on the device is read by one torch reduction)."""
    if _is_path(clips) or isinstance(clips, torch.Tensor) or not isinstance(clips, Sequence):
        raise TypeError("clips must be a list of paths and / or tensors")
    clips = list(clips)
    if not clips:
        raise ValueError("clips is empty")
    if sample_rates is None or isinstance(sample_rates, numbers.Number):
        rates = [sample_rates] * len(clips)
    else:
        rates = list(sample_rates)
        if len(rates) != len(clips):
            raise ValueError(f"sample_rates has {len(rates)} entries for {len(clips)} clips")
    for i, c in enumerate(clips):
        if _is_path(c):
            continue
        if not isinstance(c, torch.Tensor):
            raise TypeError(f"clip {i}: expected a path or a tensor, got {type(c).__name__}")
        rates[i] = _check_wav(c, rates[i], i)
    from .audio import load_audio_file

    wavs = []
    for i, c in enumerate(clips):
        if _is_path(c):
            w, sr = load_audio_file(os.fspath(c))
            rates[i] = _check_wav(w, sr, i)
            c = w
        wavs.append(c)
    for i, w in enumerate(wavs):
        check_finite(w, f"clip {i}")
    return wavs, rates


def mono_rows(wavs: Sequence[torch.Tensor], device: torch.device) -> List[torch.Tensor]:
    """Each clip as one contiguous fp32 row on the device; channels averaged as audio.load_audio_file does."""
    rows = []
    for w in wavs:
        w = w.detach().to(device=device, dtype=torch.float32)
        if w.ndim == 2:
            w = w.mean(dim=0) if w.shape[0] > 1 else w[0]
        rows.append(w.contiguous())
    return rows


def _ptrs(ptrs: Sequence[int]):
    return (C.c_void_p * len(ptrs))(*ptrs)


def trim_extents(rows: Sequence[torch.Tensor], rates: Sequence[int]) -> torch.Tensor:
    """(start, end) of each row's energy trim at its own rate -> [B, 2] int64 on the rows' device.  One launch per 64
    rows, no synchronisation."""
    B = len(rows)
    dev = rows[0].device
    ext = torch.empty((B, 2), dtype=torch.int64, device=dev)
    lens = (C.c_int64 * B)(*[int(r.numel()) for r in rows])
    srs = (C.c_int32 * B)(*[int(s) for s in rates])
    _lib.check_arg(_lib.load().sopro_ingest_trim(_ptrs([r.data_ptr() for r in rows]), B, lens, srs, ext.data_ptr(),
                                                 _lib.stream_ptr(dev)))
    return ext


def pack(src_ptrs: Sequence[int], lens: Sequence[int], out: torch.Tensor) -> torch.Tensor:
    """Row b of out [B, L] (fp32, contiguous, on the device) = lens[b] samples read at device address src_ptrs[b], then
    zeros."""
    B, L = out.shape
    _lib.check_arg(_lib.load().sopro_ingest_pack(_ptrs(src_ptrs), int(B), (C.c_int64 * B)(*[int(n) for n in lens]),
                                                 out.data_ptr(), int(L), _lib.stream_ptr(out.device)))
    return out
