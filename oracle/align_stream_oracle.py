"""CPU oracle for word timestamps in streams (no reference counterpart).  TEST INFRASTRUCTURE ONLY.

`StreamAlign` restates the streaming alignment of include/sopro_b200.h (fixed-lag Viterbi with binding commits;
sopro_b200/csrc/align.cu, sopro_align_stream_*) in float64 numpy, in the same order of IEEE double additions and
comparisons as the device, so its committed paths equal the device's bit for bit.  `stream_path` and
`stream_first_frames` run it over whole rows; `word_end_tokens` restates when a stream's word becomes final.  A and the
word list are those of oracle/align_oracle.py, which restates the one-shot alignment."""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np

from oracle.align_oracle import _owner, _word_list, accumulate


class StreamAlign:
    """The streaming alignment of include/sopro_b200.h (fixed-lag Viterbi with binding commits; sopro_align_stream_*)
    in the same order of IEEE double operations: one row of L tokens with a lag of D >= 1 frames, fed frame by frame.
    `push` takes new rows of A, `end` closes the row.  `first` (int64 [L], -1 until committed), `F` (frames committed) and `K` (tokens
    whose first frame is final) are the committed state after every call."""

    def __init__(self, L: int, D: int):
        assert L >= 1 and D >= 1
        self.L, self.D = int(L), int(D)
        self.S: Optional[np.ndarray] = None
        self.moves: List[np.ndarray] = []
        self.first = np.full(self.L, -1, dtype=np.int64)
        self.F = self.K = self.t = 0
        self.ended = False

    def _token_at(self, l: int, t: int, c: int) -> int:
        """The backtrack from (t, l) to frame c."""
        for tau in range(t, c, -1):
            if l > 0 and self.moves[tau][l]:
                l -= 1
        return l

    def push(self, A: np.ndarray) -> None:
        assert not self.ended
        for a in np.asarray(A, dtype=np.float64).reshape(-1, self.L):
            t = self.t
            if t == 0:
                S = np.full(self.L, -np.inf)
                S[0] = a[0]
                mv = np.zeros(self.L, dtype=bool)
            else:
                stay = self.S
                move = np.concatenate([[-np.inf], self.S[:-1]])
                mv = move > stay  # ties: stay
                S = a + np.where(mv, move, stay)
            self.moves.append(mv)
            self.S = S
            if t >= self.D:
                self._commit(t)
            self.t += 1

    def _commit(self, t: int) -> None:
        c = t - self.D
        S = self.S
        fin = S > -np.inf
        if not fin.any():
            return
        best = S[fin].max()
        lstar = int(np.nonzero(fin & (S == best))[0][0])
        anc = np.array([self._token_at(l, t, c) if fin[l] else -1 for l in range(self.L)])
        kc = int(anc[lstar])
        S[fin & (anc != kc)] = -np.inf
        if c == 0:
            self.first[0] = 0
        elif kc != self.K - 1:
            self.first[kc] = c
        self.F, self.K = c + 1, kc + 1

    def end(self) -> Optional[np.ndarray]:
        """Close the row -> its path (first, int64 [L]), or None when there is none (T == 0)."""
        assert not self.ended
        self.ended = True
        T = self.t
        fin = self.S > -np.inf if T > 0 else np.zeros(self.L, dtype=bool)
        if not fin.any():
            self.first[:] = -1
            self.F = self.K = 0
            return None
        l = self.L - 1 if fin[self.L - 1] else int(np.nonzero(fin)[0][-1])
        le = l
        for tau in range(T - 1, max(self.F - 1, 0), -1):
            if l > 0 and self.moves[tau][l]:
                self.first[l] = tau
                l -= 1
        self.first[0] = 0
        self.first[le + 1:] = T
        self.F, self.K = T, self.L
        return self.first.copy()


def stream_path(A: np.ndarray, D: int) -> Optional[np.ndarray]:
    """The streaming alignment of A [T, L] with lag D -> first (int64 [L]), or None when there is no path."""
    T, L = A.shape
    s = StreamAlign(L, D)
    s.push(A)
    return s.end()


def stream_first_frames(probs: np.ndarray, text_len: Sequence[int], frames: Sequence[int], D: int) -> np.ndarray:
    """probs [steps, n_attn, B, H, ld] f32 -> first [B, ld] int32 of the streaming alignment at the rows' ends, as the
    out region of sopro_align_stream's state holds it."""
    _steps, _n, B, _H, ld = probs.shape
    out = np.full((B, ld), -1, dtype=np.int32)
    for b in range(B):
        L, T = int(text_len[b]), int(frames[b])
        f = stream_path(accumulate(probs, b, T, L), D)
        if f is not None:
            out[b, :L] = f
    return out


def word_end_tokens(text: str, spans) -> List[int]:
    """Per word of `text`, the token whose committed first frame makes it final in a stream: one past the last token
    owned by it or by an earlier word (L: only the row's end does)."""
    words = _word_list(text)
    owners = [_owner(text, sp, words) for sp in spans]
    out, last = [], -1
    for k in range(len(words)):
        for l, o in enumerate(owners):
            if o == k:
                last = max(last, l)
        out.append(last + 1)
    return out
