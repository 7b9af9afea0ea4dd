"""Reference-voice denoising on the GPU (no reference counterpart): a stationary-noise Wiener suppressor with the
decision-directed a priori SNR estimate (Ephraim-Malah), for recordings that carry fan, hum, room or street noise.

``denoise(wav, lens=None)`` cleans 24 kHz rows, one row or a ragged batch, in five launches; each row's result is the
same alone and in any batch, bit for bit.  ``SoproTTS.prepare_references(..., denoise=True)`` runs it on every trimmed,
resampled clip before the centre crop and the encode.  The noise estimate is the mean spectrum of the quietest tenth of
the clip's frames, so it assumes stationary noise and a clip with pauses: a clip that never pauses loses some of its
own stationary content.  The kernels are sopro_b200/csrc/denoise.cu, the definition is in include/sopro_b200.h and, in
float64, oracle/denoise_oracle.py."""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence, Tuple

import torch

from . import _lib

FRAME, HOP = 512, 256  # SOPRO_DENOISE_FRAME, SOPRO_DENOISE_HOP


def check_denoise(flag) -> bool:
    """The `denoise=` switch: a bool, else TypeError.  Host only."""
    if not isinstance(flag, bool):
        raise TypeError(f"denoise must be True or False, got {flag!r}")
    return flag


def workspace_bytes(rows: int, most: int) -> int:
    n = C.c_int64()
    _lib.check_arg(_lib.load().sopro_denoise_sizes(int(rows), int(most), C.byref(n)))
    return max(int(n.value), 1)


def _run(wav: torch.Tensor, lens: Optional[Sequence[int]]) -> Tuple[torch.Tensor, torch.Tensor]:
    """-> (y [..., L], the workspace as the call left it)"""
    x, lead, lp = _lib.rows(wav, lens, "denoising")
    B, L = x.shape
    y = torch.empty((B, L), dtype=torch.float32, device=x.device)
    most = L if lp is None else max(lp, default=0)
    ws = torch.empty(workspace_bytes(max(B, 1), most), dtype=torch.uint8, device=x.device)
    if B and L:
        with torch.cuda.device(x.device):
            _lib.check_arg(_lib.load().sopro_denoise(x.data_ptr(), B, L, lp, ws.data_ptr(), y.data_ptr(), L,
                                                     _lib.stream_ptr(x.device)))
    return y.reshape(*lead, L), ws


def denoise(wav: torch.Tensor, lens: Optional[Sequence[int]] = None) -> torch.Tensor:
    """wav [..., L] at 24 kHz on a CUDA device (rows = the leading dims flattened) -> [..., L] f32, each row denoised on
    its own.  `lens`: valid samples per row (a ragged batch); samples past lens[b] are not read and row b's outputs past
    lens[b] are zero.  A row shorter than 512 samples, or one whose frames hold a non-finite value, comes back unchanged.
    Stationary noise only; a clip without pauses loses some stationary content of its own (DESIGN.md §5n)."""
    return _run(wav, lens)[0]
