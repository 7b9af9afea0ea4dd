"""Lossless FLAC output on the GPU (no reference counterpart: the reference's demo sends PCM16 in WAV or its own frames).

``encode_flac(wav, sample_rate, lens=None)`` encodes one row, a ragged batch ``[B, L]`` with ``lens``, or the list of
``[1, 1, N_i]`` waveforms ``synthesize_batch`` returns, all rows in one launch per kernel, to complete FLAC streams.
``FlacStreamEncoder`` / ``encode_stream_flac`` turn the chunks of ``SoproTTS.stream`` into one FLAC stream with no
added latency (variable blocking).  Decoding gives back exactly the PCM16 samples ``wire.float_to_pcm16le`` sends.  The
kernels are sopro_b200/csrc/flac.cu, the contract is in include/sopro_b200.h, the oracle in oracle/flac_oracle.py."""
from __future__ import annotations

import ctypes as C
import struct
from typing import Iterable, Iterator, List, Optional, Sequence, Union

import torch

from . import _lib
from .resample import _rate

BLOCK = 4096
STREAM_MIN_BLOCK = 16


def sizes(rows: int, max_len: int, sample_rate: int):
    """-> (workspace bytes, output bound in bytes) of one encode of `rows` rows of at most max_len samples.  Host only;
    ValueError for a refused rate or geometry."""
    ws, out = C.c_int64(0), C.c_int64(0)
    _lib.check_arg(_lib.load().sopro_flac_sizes(int(rows), int(max_len), _rate(sample_rate), C.byref(ws), C.byref(out)))
    return int(ws.value), int(out.value)


def stream_header(sample_rate: int) -> bytes:
    """The streaming encoder's header: fLaC and a STREAMINFO with blocks of 16 .. 4096 samples, frame sizes and total
    unknown (0), MD5 not computed (0)."""
    sr = _rate(sample_rate)
    sizes(1, 0, sr)  # refuses the rate
    v = (sr << 44) | (15 << 36)
    return b"fLaC" + bytes([0x80, 0, 0, 34]) + struct.pack(">HH", STREAM_MIN_BLOCK, BLOCK) + bytes(6) + v.to_bytes(8, "big") + bytes(16)


def _cuda(t: torch.Tensor) -> torch.Tensor:
    if not isinstance(t, torch.Tensor) or t.device.type != "cuda":
        raise _lib.SoproError("FLAC encoding needs CUDA tensors; there is no CPU path")
    return t.detach().to(dtype=torch.float32)


def _to_host(dev: torch.Tensor, n: int):
    """The first n bytes of dev, through pinned host memory -> a numpy uint8 view."""
    host = torch.empty(max(n, 1), dtype=torch.uint8, pin_memory=True)
    if n:
        host[:n].copy_(dev[:n], non_blocking=True)
        torch.cuda.current_stream(dev.device).synchronize()
    return host.numpy()[:n]


def encode_flac(wav: Union[torch.Tensor, Sequence[torch.Tensor]], sample_rate: int,
                lens: Optional[Sequence[int]] = None) -> Union[bytes, List[bytes]]:
    """-> one FLAC stream (bytes) for a single row (any shape with one row of samples, e.g. [1, 1, N] or [N]), or a list
    of streams for a batch: a [B, L] tensor with `lens` (valid samples per row; samples past lens[b] are not read) or a
    list of CUDA tensors (each one row).  All rows go through one launch per kernel; the only host synchronisation is
    the read of the byte counts and the copy of the bytes."""
    sr = _rate(sample_rate)
    single = isinstance(wav, torch.Tensor) and lens is None and (wav.dim() <= 1 or wav.shape[:-1].numel() == 1)
    if isinstance(wav, torch.Tensor):
        x, _lead, lp = _lib.rows(wav.reshape(1) if wav.dim() == 0 else wav, lens, "FLAC encoding")
        B, L = x.shape
        lv = [L] * B if lp is None else list(lp)
    else:
        if lens is not None:
            raise ValueError("lens goes with a [B, L] tensor, not a list of rows")
        rows = [_cuda(w).reshape(-1) for w in wav]
        if not rows:
            return []
        lv = [int(r.numel()) for r in rows]
        L = max(lv)
        x = torch.zeros((len(rows), max(L, 1)), dtype=torch.float32, device=rows[0].device)
        for i, r in enumerate(rows):
            x[i, : lv[i]] = r
        B, L = len(rows), max(L, 1)
    ws_n, out_n = sizes(B, max(lv, default=0), sr)
    for v in lv:
        if v < 0 or v > L:
            raise ValueError(f"lens entry {v} not in [0, {L}]")
    dev = x.device
    ws = torch.empty(max(ws_n, 1), dtype=torch.uint8, device=dev)
    out = torch.empty(max(out_n, 1), dtype=torch.uint8, device=dev)
    meta = torch.empty(2 * B, dtype=torch.int64, device=dev)  # row offsets, then row sizes
    with torch.cuda.device(dev):
        _lib.check_arg(_lib.load().sopro_flac_encode(x.data_ptr(), B, L, (C.c_int64 * B)(*lv), sr, ws.data_ptr(), out.data_ptr(),
                                                     meta.data_ptr(), meta.data_ptr() + 8 * B, _lib.stream_ptr(dev)))
        m = meta.cpu().tolist()
        total = m[B - 1] + m[2 * B - 1]
        blob = _to_host(out, total)
    res = [blob[m[b]: m[b] + m[B + b]].tobytes() for b in range(B)]
    return res[0] if single else res


class FlacStreamEncoder:
    """Streaming FLAC: header(), then push(chunk) -> the bytes of the frames that chunk completes, then finish() -> the
    last frame.  Each push is cut into 4096-sample frames and one remainder frame; a remainder under 16 samples is
    carried (on the device) to the next push.  Frames are numbered by their first sample (variable blocking)."""

    def __init__(self, sample_rate: int, device: Optional[torch.device] = None):
        self.sample_rate = _rate(sample_rate)
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        h = _lib._VP()
        with torch.cuda.device(self.device):
            _lib.check_arg(_lib.load().sopro_flac_stream_create(self.sample_rate, C.byref(h)))
        self._h = h
        self._nbytes = torch.zeros(1, dtype=torch.int64, device=self.device)

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            _lib.load().sopro_flac_stream_destroy(h)
            self._h = None

    def header(self) -> bytes:
        return stream_header(self.sample_rate)

    @property
    def carried(self) -> int:
        """Samples held back for the next push (0 .. 15)."""
        return int(_lib.load().sopro_flac_stream_carried(self._h))

    def _run(self, x: Optional[torch.Tensor], n: int) -> bytes:
        ws_n, out_n = sizes(1, n + STREAM_MIN_BLOCK - 1, self.sample_rate)
        ws = torch.empty(max(ws_n, 1), dtype=torch.uint8, device=self.device)
        out = torch.empty(max(out_n, 1), dtype=torch.uint8, device=self.device)
        lib = _lib.load()
        with torch.cuda.device(self.device):
            sp = _lib.stream_ptr(self.device)
            if x is None:
                _lib.check_arg(lib.sopro_flac_stream_finish(self._h, ws.data_ptr(), out.data_ptr(), self._nbytes.data_ptr(), sp))
            else:
                _lib.check_arg(lib.sopro_flac_stream_push(self._h, x.data_ptr(), n, ws.data_ptr(), out.data_ptr(),
                                                          self._nbytes.data_ptr(), sp))
            return _to_host(out, int(self._nbytes.item())).tobytes()

    def push(self, chunk: torch.Tensor) -> bytes:
        x = _cuda(chunk).reshape(-1).contiguous()
        if x.device != self.device:
            raise ValueError(f"chunk on {x.device}, the encoder on {self.device}")
        return self._run(x, int(x.numel()))

    def finish(self) -> bytes:
        """The carried samples as the last frame (b"" when none); the encoder then starts a new stream at sample 0."""
        return self._run(None, 0)


def encode_stream_flac(chunks: Iterable[torch.Tensor], sample_rate: int = 24000) -> Iterator[bytes]:
    """The header, then each chunk's frames, then the last frame: one FLAC stream from the chunks of
    ``SoproTTS.stream`` (wire.encode_stream's counterpart).  Empty pieces are not yielded."""
    enc = None
    for c in chunks:
        if enc is None:
            enc = FlacStreamEncoder(sample_rate, device=c.device)
            yield enc.header()
        b = enc.push(c)
        if b:
            yield b
    if enc is None:
        yield stream_header(sample_rate)
        return
    b = enc.finish()
    if b:
        yield b
