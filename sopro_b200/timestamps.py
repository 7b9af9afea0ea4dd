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

The timings are as good as the checkpoint's attention is monotone; the alignment's mechanics are exact."""
from __future__ import annotations

import bisect
import ctypes as C
import dataclasses
import re
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib

SAMPLE_RATE = 24000
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
    fr = word_frames([int(v) for v in first[:L]], T, token_words(text, spans, ws), len(ws))
    return [WordTiming(text[a:b], sample_seconds(f0 * hop, S), sample_seconds(f1 * hop, S), a, b)
            for (a, b), (f0, f1) in zip(ws, fr)]


def long_timings(text: str, segments: Sequence[str], seg_spans: Sequence[Sequence[Span]],
                 firsts: Sequence[Optional[np.ndarray]], Ts: Sequence[int], hop: int, extents, pause: int,
                 S: Optional[int]) -> List[WordTiming]:
    """The words of a synthesize_long passage, their char spans in the original `text`.  extents: int [segments, 2],
    the join's (e0, e1) per segment; pause: samples between spans."""
    ext = np.asarray(extents, dtype=np.int64).reshape(-1, 2)
    text_words = words(text)
    out: List[WordTiming] = []
    k, O = 0, 0
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
            O += (e1 - e0) + int(pause)
    assert k == len(text_words), (k, len(text_words))
    return out
