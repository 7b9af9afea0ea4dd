"""Host-side sampling helpers of the product path.

The reference draws its randomness inside ``torch.multinomial`` from the global CPU
generator, one call per frame (reference sampling.py:83,93).  ATen implements a
single-sample multinomial as ``argmax(p / q)`` with ``q = empty_like(p).exponential_(1)``,
so the whole random stream of an utterance is a [steps, V] tensor of Exp(1) draws that can be
produced up front and handed to the device sampler: ``noise_tape``.  Because top-k zeroes all
but the ``top_k`` best-ranked probabilities and the draw is indexed by sorted rank
(sampling.py:83-84), only the first ``top_k`` columns are ever needed on the device.

The AR drivers draw the tape block by block, just before each launch: ``NoiseTape`` is one utterance's tape and
``TapeFeed`` the tapes of one AR session, drawn into a host buffer and uploaded to the device tape the session reads."""
from __future__ import annotations

import os
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch


def noise_tape(steps: int, vocab: int, *, seed: Optional[int] = None, generator: Optional[torch.Generator] = None,
               keep: Optional[int] = None, pin: bool = False) -> torch.Tensor:
    """[steps, keep or vocab] Exp(1) draws, consumed exactly as `steps` successive
    ``torch.multinomial(p[1, vocab], 1)`` calls would.

    seed=None and generator=None -> the global CPU generator is consumed, which is what the
    reference API does (it has no seed kwarg; the CLI seeds globally, cli.py:72-75)."""
    if seed is not None:
        generator = torch.Generator().manual_seed(int(seed))
    full = torch.empty(int(steps), int(vocab))
    full.exponential_(1.0, generator=generator)
    out = full if keep is None else full[:, : int(keep)].contiguous()
    return out.pin_memory() if pin else out


_TAPE_POOL = None


def _tape_pool():
    """Host threads that draw noise tapes (the Exp(1) draws release the GIL)."""
    global _TAPE_POOL
    if _TAPE_POOL is None:
        from concurrent.futures import ThreadPoolExecutor

        _TAPE_POOL = ThreadPoolExecutor(max_workers=max(1, len(os.sched_getaffinity(0))))
    return _TAPE_POOL


_NATIVE_NOISE = None


def _native_noise_ok() -> bool:
    """The host-side mt19937 tape generator of the library (csrc/noise_host.cu) is used for private generators when it
    reproduces THIS torch build's CPU exponential_ bit for bit (checked once per process; a torch built with another
    sampling kernel falls back to torch itself)."""
    global _NATIVE_NOISE
    if _NATIVE_NOISE is None:
        try:
            import ctypes as C

            from . import _lib

            lib = _lib.load()
            h = C.c_void_p()
            _lib.check(lib.sopro_noise_create(C.c_uint64(987654321), C.byref(h)))
            got = torch.empty(3, 7)
            _lib.check(lib.sopro_noise_rows(h, 3, 97, 7, got.data_ptr()))
            lib.sopro_noise_destroy(h)
            want = torch.empty(3, 97).exponential_(1.0, generator=torch.Generator().manual_seed(987654321))[:, :7]
            _NATIVE_NOISE = bool(torch.equal(got, want))
        except Exception:
            _NATIVE_NOISE = False
    return _NATIVE_NOISE


class NoiseTape:
    """One utterance's `steps` x `vocab` tape, drawn block by block (a [n, V] draw equals n successive [V] draws), of
    which the first `keep` columns are kept, with the bookkeeping needed to leave the generator exactly where the
    reference would leave it.  `seed` makes the generator private (the library's mt19937 when it passes its self-check
    and the seed is >= 0: bit-equal to torch, and it skips the unkept draws); otherwise `generator`, or the global one."""

    def __init__(self, steps: int, vocab: int, keep: int, seed: Optional[int] = None,
                 generator: Optional[torch.Generator] = None):
        self.steps, self.vocab, self.keep = int(steps), int(vocab), int(keep)
        self.private = seed is not None
        self.gen = torch.Generator().manual_seed(int(seed)) if seed is not None else (generator or torch.default_generator)
        self.marks: List[Tuple[int, torch.Tensor]] = []  # (first row of a block, generator state before it)
        self.drawn = 0
        self._native = None
        if seed is not None and int(seed) >= 0 and _native_noise_ok():  # (negative seeds: torch's own remapping, torch's path)
            import ctypes as C

            from . import _lib

            self._lib = _lib.load()
            h = C.c_void_p()
            _lib.check(self._lib.sopro_noise_create(C.c_uint64(int(seed) & 0xFFFFFFFFFFFFFFFF), C.byref(h)))
            self._native = h

    def draw(self, upto: int, out: np.ndarray) -> None:
        """Rows [drawn, upto) into out[drawn:upto], `out` being this tape's C-contiguous float32 [steps, keep] array."""
        a, b = self.drawn, min(int(upto), self.steps)
        if b <= a:
            return
        if self._native is not None:
            from . import _lib

            assert out.flags["C_CONTIGUOUS"] and out.shape == (self.steps, self.keep) and out.dtype == np.float32
            _lib.check(self._lib.sopro_noise_rows(self._native, b - a, self.vocab, self.keep, out[a:b].ctypes.data))
        else:
            if not self.private:
                self.marks.append((a, self.gen.get_state()))
            out[a:b] = torch.empty(b - a, self.vocab).exponential_(1.0, generator=self.gen)[:, : self.keep].numpy()
        self.drawn = b

    def settle(self, steps_used: int) -> None:
        """Rewind to the state after exactly `steps_used` draws (the reference stops drawing when it stops stepping)."""
        if self.private or steps_used >= self.drawn:
            return
        start, state = [m for m in self.marks if m[0] <= steps_used][-1]
        self.gen.set_state(state)
        if steps_used > start:
            torch.empty(int(steps_used - start), self.vocab).exponential_(1.0, generator=self.gen)
        self.drawn = int(steps_used)

    def close(self) -> None:
        if self._native is not None:
            self._lib.sopro_noise_destroy(self._native)
            self._native = None


class TapeFeed:
    """The noise of one AR session: B tapes drawn into a host buffer [B, steps, keep] (pinned when CUDA is available)
    and uploaded, block by block, into `dev`, the device tape handed to the session's `begin`.  `seeds` gives utterance
    i the private generator of seeds[i]; without it every utterance draws from `generator` (or the global one)."""

    def __init__(self, batch: int, steps: int, vocab: int, keep: int, device, seeds: Optional[Sequence[int]] = None,
                 generator: Optional[torch.Generator] = None):
        self.batch, self.steps, self.drawn = int(batch), int(steps), 0
        self.private = seeds is not None
        self.tapes = [NoiseTape(steps, vocab, keep, None if seeds is None else int(seeds[i]), generator)
                      for i in range(self.batch)]
        self.host = torch.empty((self.batch, self.steps, int(keep)), dtype=torch.float32, pin_memory=torch.cuda.is_available())
        self.view = self.host.numpy()  # pool threads are outside the caller's inference_mode: they write through numpy
        self.dev = torch.empty((self.batch, self.steps, int(keep)), dtype=torch.float32, device=device)

    def fill(self, upto: int) -> None:
        """Draws rows [drawn, upto) of every tape and enqueues their upload on the current stream.  One utterance draws
        on the calling thread; private generators draw side by side on the shared pool; a shared generator is consumed
        utterance after utterance, full length each, so its first fill draws every row."""
        a = self.drawn
        b = min(int(upto), self.steps) if self.batch == 1 or self.private else self.steps
        if b <= a:
            return
        if self.batch == 1:
            self.tapes[0].draw(b, self.view[0])
        elif self.private:
            list(_tape_pool().map(lambda i: self.tapes[i].draw(b, self.view[i]), range(self.batch)))
        else:
            for tape, out in zip(self.tapes, self.view):
                tape.draw(b, out)
        self.dev[:, a:b].copy_(self.host[:, a:b], non_blocking=True)
        self.drawn = b

    def settle(self, steps_used: int) -> None:
        for tape in self.tapes:
            tape.settle(steps_used)

    def __enter__(self) -> "TapeFeed":
        return self

    def __exit__(self, *exc) -> None:
        for tape in self.tapes:
            tape.close()
