"""Word timestamps (no reference counterpart: the reference says nothing about when a word is spoken).

At every AR step each text cross-attention weighs the text tokens the frame is about to speak.  With
``word_timestamps=True`` the AR kernel exports those weights (``ArSession.set_attn_trace``), ``align`` turns them into
a monotonic token -> frame path on the GPU (sopro_b200/csrc/align.cu; the definition is in include/sopro_b200.h), and
the host maps tokens to words and frames to seconds of the returned audio:

- a word is a maximal ``\\S+`` run of the text; a token belongs to the word holding the first non-whitespace character of
  its character span; BOS, EOS and whitespace-only tokens belong to no word (BOS and EOS absorb the edge silences);
- a word runs from the first frame of its first token to the end frame of its last token; a word no token landed in
  gets a zero-length span at the end of the previous word;
- frame f starts at 24 kHz sample f * hop; with ``speed`` the sample is scaled by 65536 / S in double (S: the stretch's
  fixed-point speed); ``sample_rate`` and ``loudness`` leave the seconds unchanged;
- in ``synthesize_long`` segment i's sample x lands at O_i + clamp(x, e0_i, e1_i) - e0_i (the join's layout: O_i is the
  sum of the earlier non-empty extents plus one pause each), before the speed scaling.  The words of a skipped segment
  sit at O_i with zero length.

A stream (``stream`` / ``stream_batch`` with ``word_timestamps=True``) cannot wait for the whole utterance: the AR kernel
writes the weights into a ring of one chunk's steps, and ``StreamAligner`` aligns them as they come with the causal
rule of include/sopro_b200.h (fixed-lag Viterbi with binding commits, lag ``STREAM_ALIGN_LAG`` frames).  A word is
final, and handed out, once the committed path has passed its last token (or at the row's end); its timing is then the
mapping above applied to the committed path, and never changes.  Unlike the one-shot alignment, a stream with fewer
frames than tokens still gets its committed words, then zero-length ones at its end.

The timings are as good as the checkpoint's attention is monotone; the alignment's mechanics are exact."""
from __future__ import annotations

import bisect
import ctypes as C
import dataclasses
import numbers
import re
from typing import List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import _lib

SAMPLE_RATE = 24000
MAX_TOKENS = 2048  # the longest text either alignment takes
# frames between a frame's generation and the commit of its token in a stream: 4 default chunks, 1.92 s of audio.
# Whether this trades latency for agreement with the one-shot path well on the released checkpoint is not measured.
STREAM_ALIGN_LAG = 24
_WORD = re.compile(r"\S+")
_NONSPACE = re.compile(r"\S")
Span = Optional[Tuple[int, int]]


@dataclasses.dataclass(frozen=True)
class WordTiming:
    """One word of the text: its string, when it is spoken (seconds of the returned audio) and its characters
    text[char_start:char_end]."""
    word: str
    start: float
    end: float
    char_start: int
    char_end: int


def check_word_timestamps(word_timestamps) -> bool:
    """The `word_timestamps` argument of an entry point that checks it; TypeError for anything but a bool.  Host only."""
    if not isinstance(word_timestamps, bool):
        raise TypeError(f"word_timestamps must be a bool, got {type(word_timestamps).__name__}")
    return word_timestamps


# ---- the device part

def trace_buffer(cfg, steps: int, batch: int, ld: int, device) -> torch.Tensor:
    """A zeroed attention trace [steps, n_attn, batch, H, ld] f32 for ArSession.set_attn_trace."""
    return torch.zeros((int(steps), len(cfg.ar_attn_layers()), int(batch), int(cfg.AR_HEADS), int(ld)),
                       dtype=torch.float32, device=device)


def align(probs: torch.Tensor, text_len: Sequence[int], frames: Sequence[int]) -> torch.Tensor:
    """probs [steps, n_attn, B, H, ld] f32 on a CUDA device, text_len / frames: B ints -> first [B, ld] int32 on the
    device: the first frame of each token (-1 past text_len[b], and the whole row when there is no path)."""
    if probs.device.type != "cuda":
        raise _lib.SoproError("the alignment needs CUDA tensors; there is no CPU path")
    if probs.dim() != 5 or probs.dtype != torch.float32 or not probs.is_contiguous():
        raise ValueError("probs must be a contiguous f32 tensor [steps, n_attn, B, H, ld]")
    steps, n_attn, B, H, ld = (int(x) for x in probs.shape)
    if len(text_len) != B or len(frames) != B:
        raise ValueError(f"{len(text_len)} text lengths and {len(frames)} frame counts for {B} utterances")
    lib = _lib.load()
    ws_bytes = C.c_int64()
    _lib.check_arg(lib.sopro_align_sizes(B, steps, ld, C.byref(ws_bytes)))
    lens = (C.c_int32 * B)(*[int(v) for v in text_len])
    fr = (C.c_int32 * B)(*[int(v) for v in frames])
    ws = torch.empty(int(ws_bytes.value), dtype=torch.uint8, device=probs.device)
    first = torch.empty((B, ld), dtype=torch.int32, device=probs.device)
    with torch.cuda.device(probs.device):
        _lib.check_arg(lib.sopro_align(probs.data_ptr(), steps, n_attn, B, H, ld, lens, fr, ws.data_ptr(), first.data_ptr(),
                                       _lib.stream_ptr(probs.device)))
    return first


# ---- the host part

def words(text: str) -> List[Tuple[int, int]]:
    """The (start, end) character spans of the words (maximal \\S+ runs) of `text`."""
    return [(m.start(), m.end()) for m in _WORD.finditer(text)]


def token_words(text: str, spans: Sequence[Span], word_spans: Sequence[Tuple[int, int]]) -> List[Optional[int]]:
    """The word index of each token: the word holding the first non-whitespace character of its span, or None."""
    starts = [a for a, _b in word_spans]
    out: List[Optional[int]] = []
    for sp in spans:
        k = None
        if sp is not None:
            m = _NONSPACE.search(text, int(sp[0]), int(sp[1]))
            if m is not None:
                i = bisect.bisect_right(starts, m.start()) - 1
                if i >= 0 and m.start() < word_spans[i][1]:
                    k = i
        out.append(k)
    return out


def word_frames(first: Sequence[int], T: int, owner: Sequence[Optional[int]], n_words: int) -> List[Tuple[int, int]]:
    """(first frame, end frame) of each word from the tokens' first frames (token l owns [first[l], first[l+1]),
    first[L] := T) and their word indices; a word no token landed in sits at the end of the previous one."""
    L = len(owner)
    lo: List[Optional[int]] = [None] * n_words
    hi: List[int] = [0] * n_words
    for l, k in enumerate(owner):
        if k is None:
            continue
        if lo[k] is None:
            lo[k] = int(first[l])
        hi[k] = int(first[l + 1]) if l + 1 < L else int(T)
    out, prev = [], 0
    for k in range(n_words):
        if lo[k] is None:
            out.append((prev, prev))
        else:
            out.append((lo[k], hi[k]))
            prev = hi[k]
    return out


def sample_seconds(x: int, S: Optional[int]) -> float:
    """A 24 kHz sample index of the unstretched audio -> seconds of the returned audio (`S`: the stretch's fixed-point
    speed, None without one)."""
    y = float(x)
    if S is not None:
        y = y * 65536.0 / float(S)
    return y / SAMPLE_RATE


def utterance_timings(text: str, spans: Sequence[Span], first: Optional[np.ndarray], T: int, hop: int,
                      S: Optional[int]) -> List[WordTiming]:
    """The words of one utterance; [] when it has no alignment (`first` None or a row of -1)."""
    L = len(spans)
    if first is None or L == 0 or int(first[0]) < 0:
        return []
    ws = words(text)
    return _timings(text, ws, token_words(text, spans, ws), first, T, hop, S)


def _timings(text: str, ws: Sequence[Tuple[int, int]], owner: Sequence[Optional[int]], first, T: int, hop: int,
             S: Optional[int]) -> List[WordTiming]:
    fr = word_frames([int(v) for v in first[:len(owner)]], T, owner, len(ws))
    return [WordTiming(text[a:b], sample_seconds(f0 * hop, S), sample_seconds(f1 * hop, S), a, b)
            for (a, b), (f0, f1) in zip(ws, fr)]


class WordEmitter:
    """One stream row's words, handed out in text order as they become final: word k is final once the first frame
    of end_tok[k] is committed (one past the last token of words <= k; L: only at the row's end)."""

    def __init__(self, text: str, spans: Sequence[Span], hop: int, S: Optional[int]):
        self.text, self.hop, self.S = text, int(hop), S
        self.ws = words(text)
        self.owner = token_words(text, spans, self.ws)
        last = [-1] * len(self.ws)
        for l, k in enumerate(self.owner):
            if k is not None:
                last[k] = l
        run, self.end_tok = -1, []
        for x in last:
            run = max(run, x)
            self.end_tok.append(run + 1)
        self.taken = 0

    def take(self, first: np.ndarray, K: int, T: int, ended: bool) -> List[WordTiming]:
        """The words that became final since the last take, from the committed path: `first` (first frames, -1 where
        not committed), `K` tokens committed, `T` frames so far, `ended` (then `first` is the whole path)."""
        if ended:
            n = len(self.ws) if len(self.owner) and int(first[0]) >= 0 else 0
        else:
            n = bisect.bisect_left(self.end_tok, int(K))  # end_tok is non-decreasing: the words with end_tok < K
        if n <= self.taken:
            return []
        out = _timings(self.text, self.ws, self.owner, first, int(T), self.hop, self.S)
        a, self.taken = self.taken, n
        return out[a:n]


class StreamAligner:
    """Word timestamps of a stream of B rows: the ring trace the AR session writes (``ring``, for
    ArSession.set_attn_trace(ring, ring=rows)), the streaming alignment's device state, and per row the words handed
    out so far.  Per launch: ``push`` (on the stream the trace's readers run on, once the launch's steps are in the
    ring) enqueues the alignment of each row's new frames and the copy of the committed paths to pinned host memory;
    after the caller has synchronised that stream, ``take(b)`` returns row b's words that became final since the last
    take, in text order.  `S`: the stretch's fixed-point speed (None without one)."""

    def __init__(self, cfg, texts: Sequence[str], spans: Sequence[Sequence[Span]], *, ring: int, max_frames: int, hop: int,
                 S: Optional[int], device):
        if torch.device(device).type != "cuda":
            raise _lib.SoproError("the streaming alignment needs a CUDA device; there is no CPU path")
        lens = [len(sp) for sp in spans]
        B, ld = len(lens), max(lens)
        self.lib = _lib.load()
        self.ring = trace_buffer(cfg, ring, B, ld, device)
        nb = C.c_int64()
        lag, mf = int(STREAM_ALIGN_LAG), int(max_frames)
        _lib.check_arg(self.lib.sopro_align_stream_sizes(B, ld, lag, mf, C.byref(nb)))
        self.state = torch.empty(int(nb.value), dtype=torch.uint8, device=device)
        h = C.c_void_p()
        _lib.check_arg(self.lib.sopro_align_stream_create(B, ld, lag, mf, self.state.data_ptr(), C.byref(h)))
        self._h = h
        self._out = self.state[: B * (2 + ld) * 4].view(torch.int32).view(B, 2 + ld)  # {F, K, first[ld]} per row
        self.host = torch.empty((B, 2 + ld), dtype=torch.int32, pin_memory=True)
        self.device = torch.device(device)
        self.B, self.ld = B, ld
        self.rows = [WordEmitter(t, sp, hop, S) for t, sp in zip(texts, spans)]
        self.frames = [0] * B
        self.ended = [False] * B
        lens_c = (C.c_int32 * B)(*lens)
        _lib.check_arg(self.lib.sopro_align_stream_begin(self._h, lens_c, _lib.stream_ptr(self.device)))

    def push(self, frames: Sequence[int], ends: Sequence[bool]) -> None:
        """Row b's next frames[b] frames are in the ring; ends[b]: the row ends after them."""
        B = self.B
        n = (C.c_int32 * B)(*[int(x) for x in frames])
        e = (C.c_int32 * B)(*[1 if x else 0 for x in ends])
        _, n_attn, _, H, ld = (int(x) for x in self.ring.shape)
        _lib.check_arg(self.lib.sopro_align_stream_push(self._h, self.ring.data_ptr(), int(self.ring.shape[0]), n_attn, B,
                                                        H, ld, n, e, _lib.stream_ptr(self.device)))
        for b in range(B):
            self.frames[b] += int(frames[b])
            self.ended[b] = self.ended[b] or bool(ends[b])
        self.host.copy_(self._out, non_blocking=True)

    def take(self, b: int) -> List[WordTiming]:
        """Row b's words that became final since the last take (the host copy of the last push must have landed)."""
        row = self.host[b].numpy()
        return self.rows[b].take(row[2:], int(row[1]), self.frames[b], self.ended[b])

    def close(self) -> None:
        if getattr(self, "_h", None):
            self.lib.sopro_align_stream_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def long_timings(text: str, segments: Sequence[str], seg_spans: Sequence[Sequence[Span]],
                 firsts: Sequence[Optional[np.ndarray]], Ts: Sequence[int], hop: int, extents,
                 pause: Union[int, Sequence[int]], S: Optional[int], start: int = 0) -> List[WordTiming]:
    """The words of a synthesize_long passage, their char spans in the original `text`.  extents: int [segments, 2],
    the join's (e0, e1) per segment; pause: samples between spans, or one per non-empty span, the zeros that follow it
    (a dialogue's gaps differ: the one after a turn's last span is the turn pause); start: the passage sample at which
    the first span begins (a dialogue turn's start).  A segment with an empty extent has its words at the sample where
    the audio continues."""
    ext = np.asarray(extents, dtype=np.int64).reshape(-1, 2)
    n_spans = int((ext[:, 1] > ext[:, 0]).sum())
    after = [int(pause)] * n_spans if isinstance(pause, numbers.Integral) else [int(p) for p in pause]
    if len(after) != n_spans:
        raise ValueError(f"{len(after)} pauses for {n_spans} non-empty spans")
    text_words = words(text)
    out: List[WordTiming] = []
    k, O, m = 0, int(start), 0
    for i, seg in enumerate(segments):
        e0, e1 = int(ext[i, 0]), int(ext[i, 1])
        ws = words(seg)
        first = firsts[i]
        if e1 > e0 and first is not None and len(seg_spans[i]) and int(first[0]) >= 0:
            L = len(seg_spans[i])
            fr = word_frames([int(v) for v in first[:L]], int(Ts[i]), token_words(seg, seg_spans[i], ws), len(ws))
            ys = [(O + min(max(f0 * hop, e0), e1) - e0, O + min(max(f1 * hop, e0), e1) - e0) for f0, f1 in fr]
        else:
            ys = [(O, O)] * len(ws)
        for (a, b), (y0, y1) in zip(ws, ys):
            ta, tb = text_words[k]
            assert text[ta:tb] == seg[a:b], (text[ta:tb], seg[a:b])
            out.append(WordTiming(text[ta:tb], sample_seconds(y0, S), sample_seconds(y1, S), ta, tb))
            k += 1
        if e1 > e0:
            O += (e1 - e0) + after[m]
            m += 1
    assert k == len(text_words), (k, len(text_words))
    return out
