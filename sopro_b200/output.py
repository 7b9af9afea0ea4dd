"""The output chain every synthesis entry point runs on the decoded 24 kHz audio: time-stretch (``speed``), then the
watermark (``watermark``), then resample (``sample_rate``), then loudness normalisation (``loudness``).  A stage whose
argument is a bypass runs nothing and allocates nothing.  ``synthesize``, ``synthesize_batch`` and ``synthesize_long`` call the chain on whole rows; ``stream``
feeds each chunk through a per-utterance state of stream states, which concatenates to the one-shot result bit for bit
(loudness has no streaming form: it needs the whole utterance)."""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import torch

from .config import TARGET_SR
from .loudness import check_loudness, normalize_loudness
from .stretch import check_speed, stretch, stretched_length
from .watermark import check_watermark, embed_watermark


class OutputChain:
    """Built per call from the caller's arguments.  Construction checks them in a fixed order, rate, then speed, then
    loudness, then the watermark key, and raises ValueError for a refused one before any other work (no random draw, nothing read from `tts`
    but its resampler cache).  ``sample_rate``: the rate of the returned audio; ``S``: the stretch's fixed-point speed,
    None on a bypass (word timestamps scale their samples by it)."""

    def __init__(self, tts, sample_rate: Optional[int] = None, speed: Optional[float] = None,
                 loudness: Optional[float] = None, watermark: Optional[int] = None):
        self.rs = tts._resampler(sample_rate)
        self.S = check_speed(speed)
        self.target = check_loudness(loudness)
        self.key = check_watermark(watermark)
        self.tts, self.speed = tts, speed
        self.sample_rate = TARGET_SR if self.rs is None else self.rs.sr_out

    def __call__(self, wav: torch.Tensor, lens: Optional[Sequence[int]] = None
                 ) -> Tuple[torch.Tensor, Optional[List[int]]]:
        """wav [..., L] 24 kHz on the device (rows = the leading dims flattened; `lens`: valid samples per row of a
        ragged batch) -> (wav [..., L'] at sample_rate, the rows' valid samples or None), each stage one launch."""
        if self.S is not None:
            wav = stretch(wav, self.speed, lens=lens)
            lens = None if lens is None else [stretched_length(self.speed, n) for n in lens]
        if self.key is not None:
            wav = embed_watermark(wav, self.key, lens=lens)
        if self.rs is not None:
            wav = self.rs(wav, lens=lens)
            lens = None if lens is None else [self.rs.length(n) for n in lens]
        if self.target is not None:
            wav = normalize_loudness(wav, self.sample_rate, self.target, lens=lens)
        return wav, lens

    def stream(self, max_push: int) -> "ChainStream":
        """The chain's streaming part for one utterance whose chunks hold at most max_push samples."""
        return ChainStream(self, max_push)


class ChainStream:
    """One utterance's stretch, watermark and resampler stream states, checked out of their pools (none on a bypass) and given
    back by ``release``.  Pushes go to a state in pieces of at most max_push samples: a stretch push can yield up to 4x
    its input."""

    def __init__(self, chain: OutputChain, max_push: int):
        self.max_push = int(max_push)
        self._stages = []  # (state, its pool), in chain order
        if chain.S is not None:
            pool = chain.tts._stretch_pool
            self._stages.append((pool.checkout(self.max_push, chain.speed), pool))
        if chain.key is not None:
            pool = chain.tts._watermark_pool
            self._stages.append((pool.checkout(self.max_push, chain.key), pool))
        if chain.rs is not None:
            pool = chain.rs.pool
            self._stages.append((pool.checkout(self.max_push), pool))

    def push(self, wav: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
        """The next chunk, [1, n] 24 kHz -> [1, k] at the output rate (None in, None out)."""
        return self._run(wav, False)

    def finish(self, wav: Optional[torch.Tensor] = None) -> Optional[torch.Tensor]:
        """The last chunk (or None), then every state's tail -> [1, k]; the chunk itself when nothing is stateful."""
        return self._run(wav, True)

    def _run(self, wav: Optional[torch.Tensor], last: bool) -> Optional[torch.Tensor]:
        if wav is None and not last:
            return None
        n = self.max_push
        for st, _pool in self._stages:
            parts = [st.push(wav[:, i: i + n]) for i in range(0, wav.shape[1], n)] if wav is not None else []
            if last:
                parts.append(st.finish())
            wav = torch.cat(parts).unsqueeze(0) if len(parts) > 1 else parts[0].unsqueeze(0)
        return wav

    def release(self) -> None:
        """The states back to their pools; an abandoned utterance's state is reset by its next checkout."""
        for st, pool in self._stages:
            pool.release(st)
        self._stages = []
