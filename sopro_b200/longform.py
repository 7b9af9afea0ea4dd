"""Long-form synthesis (no reference counterpart: the reference speaks one utterance of at most max_frames, about 32 s).

``split_text`` cuts a text into segments the model can speak; ``SoproTTS.synthesize_long`` generates them side by side
through the batch path and joins them on the GPU.  The two GPU stages are public too, so a caller with their own
``synthesize_batch`` outputs can join them the same way: ``speech_extents`` finds each decoded row's speech (the energy
trim of sopro_b200.audio.trim_silence_energy at 24 kHz, one launch for a ragged batch) and ``join_segments`` joins the
extents with a fixed pause and raised-cosine edges.  The kernels are sopro_b200/csrc/longform.cu, the contract is in
include/sopro_b200.h."""
from __future__ import annotations

import ctypes as C
import math
import numbers
import re
from typing import List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import _lib

SAMPLE_RATE = 24000       # the codec's rate: both stages work on the decoded rows
FADE = 240                # the longest fade, 10 ms
MAX_PAUSE_MS = 2000.0
MIN_TOKENS = 4
SEGMENT_GROUP = 64        # segments per synthesize_batch pass of synthesize_long

_PARAGRAPH = re.compile(r"\n\s*\n")
_TERMINATOR = re.compile("[.!?…]+[\"'”’)\\]]*")   # a maximal run of . ! ? ..., then closing quotes / brackets
_CLAUSE = re.compile("[,;:—–](?= )")                   # a clause mark followed by whitespace


# ---- text segmentation (host)

def _sentences(par: str) -> List[str]:
    """A normalised paragraph (single spaces, stripped) -> its sentences.  A boundary follows a terminator run and its
    closing quotes or brackets when a space or the paragraph's end follows, unless the next character is lowercase."""
    out, a = [], 0
    for m in _TERMINATOR.finditer(par):
        e = m.end()
        if e < len(par) and (par[e] != " " or par[e + 1].islower()):
            continue
        out.append(par[a:e])
        a = e + 1
    if a < len(par):
        out.append(par[a:])
    return out


def _cut(sentence: str, fits) -> List[str]:
    """An over-long sentence -> pieces: at the last clause mark whose left piece fits, else at the last space whose left
    piece fits, repeated on the rest; a space-free run that does not fit on its own is a piece of its own.  Candidates
    are tried left to right up to the first that does not fit (with token counts that grow with the text, as for a
    tokenizer that splits on whitespace first, that is the last one that fits)."""
    pieces, rest = [], sentence
    while not fits(rest):
        cut = None
        for marks, keep in ((_CLAUSE, 1), (re.compile(" "), 0)):
            for m in marks.finditer(rest):
                if not fits(rest[: m.start() + keep]):
                    break
                cut = m.start() + keep
            if cut is not None:
                break
        if cut is None:  # the first word alone is over the budget
            sp = rest.find(" ")
            if sp < 0:
                break
            cut = sp
        pieces.append(rest[:cut])
        rest = rest[cut + 1:]  # (every cut is at a space of the normalised text)
    pieces.append(rest)
    return pieces


def split_text(text: str, tokenizer, max_tokens: int = 64) -> List[str]:
    """A text -> the segments ``synthesize_long`` speaks, in order.  Pure and deterministic:

    1. Paragraphs: the text splits on blank lines (``\\n\\s*\\n``); inside a paragraph whitespace runs collapse to one
       space and the ends are stripped; empty paragraphs are dropped.  No segment spans two paragraphs.
    2. Sentences: a boundary follows a maximal run of ``.``, ``!``, ``?`` or ``…`` plus any closing quotes or brackets
       (``"'”’)]``) when whitespace or the paragraph's end follows, except when the next non-space character is a
       lowercase letter ("e.g. this", "approx. five").  There is no abbreviation list, so "Dr. Smith" splits.
    3. Packing: consecutive sentences of a paragraph merge greedily while the merged segment's token count,
       ``len(tokenizer.encode(segment))`` (BOS and EOS included), stays <= max_tokens.
    4. A sentence over the budget is cut at the last clause mark (``,`` ``;`` ``:`` ``—`` ``–`` followed by whitespace)
       whose left piece fits, failing that at the last whitespace whose left piece fits, and again on the rest; its
       pieces are segments of their own.  A whitespace-free run over the budget is a segment of its own (its audio is
       bounded by max_frames, as in ``synthesize``).

    For each paragraph, ``" ".join(its segments)`` is the normalised paragraph; every segment is non-empty and fits the
    budget, except a whitespace-free run that does not fit alone."""
    budget = int(max_tokens)

    def fits(s: str) -> bool:
        return len(tokenizer.encode(s)) <= budget

    out: List[str] = []
    for raw in _PARAGRAPH.split(text):
        par = " ".join(raw.split())
        if not par:
            continue
        cur: Optional[str] = None
        for s in _sentences(par):
            if not fits(s):
                if cur is not None:
                    out.append(cur)
                    cur = None
                out.extend(_cut(s, fits))
            elif cur is None:
                cur = s
            elif fits(cur + " " + s):
                cur = cur + " " + s
            else:
                out.append(cur)
                cur = s
        if cur is not None:
            out.append(cur)
    return out


def passage_segments(text: str, tokenizer, max_tokens: int) -> List[str]:
    """split_text for synthesize_long and stream_long; ValueError when the text has nothing to speak.  Host only."""
    segments = split_text(text, tokenizer, max_tokens)
    if not segments:
        raise ValueError("the text has nothing to speak (it is empty or whitespace only)")
    return segments


def check_pause(pause_ms) -> float:
    """The pause between segments in ms as a float; ValueError for anything but a real number in [0, 2000].  Host only."""
    if isinstance(pause_ms, (bool, np.bool_)) or not isinstance(pause_ms, numbers.Real) or \
            not (0.0 <= float(pause_ms) <= MAX_PAUSE_MS):
        raise ValueError(f"pause_ms must be a real number in [0, {MAX_PAUSE_MS:g}], got {pause_ms!r}")
    return float(pause_ms)


def check_max_tokens(max_tokens, limit: int) -> int:
    """The segment budget as an int; ValueError for anything but an integer in [4, limit] (limit: the prefill's
    max_text_len).  Host only."""
    if isinstance(max_tokens, (bool, np.bool_)) or not isinstance(max_tokens, numbers.Integral) or \
            not (MIN_TOKENS <= int(max_tokens) <= int(limit)):
        raise ValueError(f"max_tokens must be an integer in [{MIN_TOKENS}, {int(limit)}], got {max_tokens!r}")
    return int(max_tokens)


def pause_samples(pause_ms) -> int:
    """P = round(pause_ms * 24), the pause in samples at 24 kHz (half to even)."""
    return int(round(check_pause(pause_ms) * 24))


def fade_length(span: int) -> int:
    """F = min(240, floor(span / 2))."""
    return min(FADE, int(span) // 2)


def fade_window(F: int) -> np.ndarray:
    """The F fp32 fade taps the join uses: 0.5 - 0.5 cos(pi (i + 0.5) / F) in double, rounded once.  Host only."""
    f = np.zeros(int(F), dtype=np.float32)
    _lib.check_arg(_lib.load().sopro_longform_fade(int(F), f.ctypes.data if F else None))
    return f


def joined_length(extents, pause: int) -> int:
    """sum(spans) + (spans - 1) * P over the non-empty extents (host int64 [n, 2]); 0 when every extent is empty."""
    spans = [int(e) - int(s) for s, e in np.asarray(extents, dtype=np.int64).reshape(-1, 2) if int(e) > int(s)]
    return sum(spans) + max(0, len(spans) - 1) * int(pause)


def speech_extents(wav: torch.Tensor, lens: Optional[Sequence[int]] = None) -> torch.Tensor:
    """wav [..., L] 24 kHz on a CUDA device (rows = the leading dims flattened) -> int64 [rows, 2] (start, end) of each
    row's speech, on the device (nothing synchronises).  `lens`: valid samples per row (a ragged batch); samples past
    lens[b] are not read."""
    x, _lead, lp = _lib.rows(wav, lens, "speech extents")
    B, L = x.shape
    ext = torch.empty((B, 2), dtype=torch.int64, device=x.device)
    if B == 0:
        return ext
    with torch.cuda.device(x.device):
        _lib.check_arg(_lib.load().sopro_longform_extents(x.data_ptr(), B, L, lp, ext.data_ptr(), _lib.stream_ptr(x.device)))
    return ext


def _rows(rows_or_chunks) -> List[torch.Tensor]:
    """A tensor [..., L] (its rows) or a sequence of tensors (each one's rows, in order) -> 1-D fp32 CUDA rows."""
    parts = [rows_or_chunks] if isinstance(rows_or_chunks, torch.Tensor) else list(rows_or_chunks)
    out = []
    for t in parts:
        if t.device.type != "cuda":
            raise _lib.SoproError("the join needs CUDA tensors; there is no CPU path")
        t = t.detach().to(dtype=torch.float32)
        t = t.reshape(1, -1) if t.dim() <= 1 or math.prod(tuple(t.shape[:-1])) == 1 else t.reshape(-1, t.shape[-1])
        if t.numel() and t.stride(-1) != 1:
            t = t.contiguous()
        out.extend(t[i] for i in range(t.shape[0]))
    return out


def gap_pauses(extents, pause: int, turn_of: Optional[Sequence[int]] = None, turn_pause: int = 0) -> List[int]:
    """The zeros before each non-empty span after the first, over the non-empty extents (host int64 [n, 2]): `pause`,
    or `turn_pause` when the previous non-empty span belongs to another turn (`turn_of`: the turn of each segment;
    None = one turn).  Empty extents take no part: they have neither a span nor a gap."""
    ext = np.asarray(extents, dtype=np.int64).reshape(-1, 2)
    out: List[int] = []
    prev = None
    for i, (s, e) in enumerate(ext):
        if int(e) <= int(s):
            continue
        t = 0 if turn_of is None else int(turn_of[i])
        if prev is not None:
            out.append(int(turn_pause) if t != prev else int(pause))
        prev = t
    return out


def join_segments(rows_or_chunks: Union[torch.Tensor, Sequence[torch.Tensor]], extents, pause_ms) -> torch.Tensor:
    """Segment rows and their extents -> one waveform [1, 1, N] f32 on the rows' device: each non-empty extent in order,
    its first and last F = min(240, span // 2) samples faded by a raised cosine, round(pause_ms * 24) zeros between
    consecutive spans.  `rows_or_chunks`: a tensor whose rows are the segments (padded decode chunks [rows, 1, L]), or a
    sequence of them and of single rows; each row is read in place.  `extents`: int64 [segments, 2]; on the device, it
    is copied to the host here, the one synchronisation."""
    P = pause_samples(pause_ms)
    ext = (extents.detach().to("cpu") if isinstance(extents, torch.Tensor) else torch.as_tensor(extents)).to(torch.int64)
    ext = ext.numpy().reshape(-1, 2)
    return join_gaps(rows_or_chunks, ext, gap_pauses(ext, P))


def join_gaps(rows_or_chunks: Union[torch.Tensor, Sequence[torch.Tensor]], extents, pauses: Sequence[int],
              gain: Optional[torch.Tensor] = None) -> torch.Tensor:
    """join_segments with a pause per gap and a gain per span: `extents` on the host (int [segments, 2]), `pauses`
    the zeros before each non-empty span after the first (gap_pauses), each in [0, 48000]; `gain`: f32 [segments] on
    the rows' device or None.  Span i's samples are gain[i] times its faded samples, so spans that share a gain equal
    their own join scaled by it as normalize_loudness scales a row, bit for bit.  Nothing synchronises."""
    rows = _rows(rows_or_chunks)
    ext = np.ascontiguousarray(np.asarray(extents, dtype=np.int64).reshape(-1, 2))
    n = len(rows)
    if n == 0 or ext.shape[0] != n:
        raise ValueError(f"{ext.shape[0]} extents for {n} segment rows")
    spans = [int(e) - int(s) for s, e in ext if int(e) > int(s)]
    if len(pauses) != max(0, len(spans) - 1):
        raise ValueError(f"{len(pauses)} pauses for {len(spans)} non-empty spans")
    dev = rows[0].device
    if gain is not None:
        if gain.device != dev or gain.dtype != torch.float32 or gain.numel() != n:
            raise ValueError(f"gain must be f32 [{n}] on {dev}, got {gain.dtype} [{gain.numel()}] on {gain.device}")
        gain = gain.reshape(-1).contiguous()
    gaps = np.ascontiguousarray(np.asarray(list(pauses) or [0], dtype=np.int64))
    N = sum(spans) + int(gaps[: len(pauses)].sum())
    y = torch.empty((1, 1, N), dtype=torch.float32, device=dev)
    src = (C.c_void_p * n)(*[r.data_ptr() if r.numel() else None for r in rows])
    lens = (C.c_int64 * n)(*[int(r.numel()) for r in rows])
    with torch.cuda.device(dev):
        _lib.check_arg(_lib.load().sopro_longform_join_gaps(src, n, lens, ext.ctypes.data, gaps.ctypes.data,
                                                            None if gain is None else gain.data_ptr(),
                                                            y.data_ptr() if N else None, N, _lib.stream_ptr(dev)))
    return y


def join_padded(rows: Sequence[torch.Tensor], extents, pauses: Sequence[int], gain: Optional[torch.Tensor], lead: int,
                trail: int, device) -> torch.Tensor:
    """join_gaps with gaps of any length and `lead` / `trail` zeros around the passage -> [1, 1, N] f32 on `device`.
    The spans between two gaps longer than the kernel's 2 s are joined by join_gaps and the long gaps are zeros laid
    between those joins, so the samples equal one join with those gaps.  Nothing synchronises."""
    ext = np.asarray(extents, dtype=np.int64).reshape(-1, 2)
    spoken = [k for k in range(ext.shape[0]) if ext[k, 1] > ext[k, 0]]
    if len(pauses) != max(0, len(spoken) - 1):
        raise ValueError(f"{len(pauses)} pauses for {len(spoken)} non-empty spans")
    longest = pause_samples(MAX_PAUSE_MS)

    def zeros(n: int) -> torch.Tensor:
        return torch.zeros((1, 1, int(n)), dtype=torch.float32, device=device)

    parts = [zeros(lead)] if lead else []
    a = 0
    for m, p in enumerate(list(pauses) + [None] if spoken else []):
        if p is not None and p <= longest:
            continue
        idx = spoken[a: m + 1]
        parts.append(join_gaps([rows[k] for k in idx], ext[idx], pauses[a: m], None if gain is None else gain[idx]))
        if p is not None:
            parts.append(zeros(p))
        a = m + 1
    if trail:
        parts.append(zeros(trail))
    if not parts:
        return zeros(0)
    return parts[0] if len(parts) == 1 else torch.cat(parts, dim=-1)


def mix(rows: Sequence[torch.Tensor], offsets: Sequence[int], length: int, device=None) -> torch.Tensor:
    """Rows placed at absolute sample offsets on one timeline and summed where they overlap -> [1, 1, length] f32 on
    the rows' device (SoproTTS.synthesize_timed's placement).  Sample t is the first covering row's sample, then each
    later covering row's added in one fp32 add, in row order; 0 where no row covers t.  `rows`: 1-D tensors (others
    are flattened) on one CUDA device, read in place; an empty row covers nothing.  Every row must end by `length`
    (include/sopro_b200.h, sopro_timeline_mix); `device`: the output's device when there is no row (default: the
    current CUDA device).  Nothing synchronises."""
    flat = []
    for r in rows:
        if r.device.type != "cuda":
            raise _lib.SoproError("the mix needs CUDA tensors; there is no CPU path")
        flat.append(r.detach().to(dtype=torch.float32).reshape(-1).contiguous())
    n = len(flat)
    offs = [int(o) for o in offsets]
    if len(offs) != n:
        raise ValueError(f"{len(offs)} offsets for {n} rows")
    dev = flat[0].device if flat else torch.device(device if device is not None else "cuda")
    if dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    if any(r.device != dev for r in flat):
        raise ValueError("the rows are on different devices")
    L = int(length)
    y = torch.empty((1, 1, max(L, 0)), dtype=torch.float32, device=dev)
    src = (C.c_void_p * max(n, 1))(*[r.data_ptr() if r.numel() else None for r in flat])
    lens = (C.c_int64 * max(n, 1))(*[int(r.numel()) for r in flat])
    offp = (C.c_int64 * max(n, 1))(*offs)
    with torch.cuda.device(dev):
        _lib.check_arg(_lib.load().sopro_timeline_mix(src, n, lens, offp, y.data_ptr() if L > 0 else None, L,
                                                      _lib.stream_ptr(dev)))
    return y


# ---- the streaming trim and join (SoproTTS.stream_long)

class StreamJoin:
    """The streaming form of speech_extents + join_segments over one passage's segments, as their rows are decoded
    (the causal rule and the certain prefix: include/sopro_b200.h).  The device state holds the rows of at most two
    groups of `group` segments, segment i in slot (i // group) % 2, so one group can be emitted while the next one is
    generated; its buffers take rows x max_len x 4 bytes.

    ``begin`` starts a passage, ``start_group`` a group's rows (on the current stream), ``push`` appends one chunk-loop
    launch's decoded block and copies the status into pinned host memory (both on the current stream, with no host
    synchronisation: the reader synchronises that stream before ``take``), and ``take`` emits the next piece of the
    joined passage that is certain, at most `limit` samples, pause zeros included.  The pause before a span goes out
    only once that span has samples to follow it.  Allocation happens at construction only, so a pooled state serves the
    next passage without allocating on its first-item path."""

    def __init__(self, rows: int, max_len: int, device):
        self.device = torch.device(device)
        self.rows, self.max_len = int(rows), int(max_len)
        h = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check_arg(_lib.load().sopro_longform_stream_create(self.rows, self.max_len, self.device.index, C.byref(h)))
        self._h = h.value
        self._status = torch.zeros((self.rows, 5), dtype=torch.int64, pin_memory=True)
        self._st = self._status.numpy()
        self.begin(1, 0, 1)

    @staticmethod
    def rows_for(segments: int, group: int) -> int:
        """Device rows a passage of `segments` needs: one group's worth, or two slots of `group`."""
        return int(segments) if segments <= group else 2 * int(group)

    def begin(self, segments: int, pause: int, group: int, turn_of: Optional[Sequence[int]] = None,
              turn_pause: int = 0) -> None:
        """A passage of `segments` segments in groups of `group`; the gap before a span is `pause`, or `turn_pause`
        when the previous span belongs to another turn (gap_pauses; `turn_of`: the turn of each segment, None = one)."""
        if self.rows_for(segments, group) > self.rows:
            raise ValueError(f"{segments} segments in groups of {group} need {self.rows_for(segments, group)} rows, "
                             f"the state has {self.rows}")
        if turn_of is not None and len(turn_of) != int(segments):
            raise ValueError(f"{len(turn_of)} turns for {int(segments)} segments")
        self.B, self.P, self.G = int(segments), int(pause), int(group)
        self.TP, self.turn_of = int(turn_pause), None if turn_of is None else [int(t) for t in turn_of]
        self.prev_turn = None      # the turn of the last span begun
        self.cur, self.pos, self.pause_left, self.spans = 0, -1, 0, 0  # the segment being emitted, its next sample
        self.started = 0           # segments [0, started) have begun
        self.row0 = self.n_rows = 0  # the rows the pushes go to
        self.pushes = 0

    def _row(self, seg: int) -> int:
        return seg if self.B <= self.G else ((seg // self.G) % 2) * self.G + seg % self.G

    def can_start(self, g0: int) -> bool:
        """Whether the slot of the group starting at segment g0 is free: the group it held has been emitted."""
        return g0 < self.B and g0 == self.started and self.cur >= g0 - self.G

    def start_group(self, g0: int, n: int) -> None:
        """Segments [g0, g0 + n) take their slot's rows, reset on the current stream."""
        if not self.can_start(g0):
            raise _lib.SoproError(f"the group at segment {g0} cannot start yet")
        self.row0, self.n_rows = self._row(g0), int(n)
        self._st[self.row0: self.row0 + self.n_rows] = 0  # (no copy into them is in flight: their last one was read)
        _lib.check_arg(_lib.load().sopro_longform_stream_reset(self._h, self.row0, self.n_rows, _lib.stream_ptr(self.device)))
        self.started = g0 + int(n)

    def push(self, wav: Optional[torch.Tensor], counts: Sequence[int], final: Sequence[bool]) -> None:
        """One launch's block: wav [n_rows, L] f32 on the device (None when no row has samples), counts[i] new samples
        of the group's row i (0 = it did not run), final[i] when the row ends with this push."""
        n = self.n_rows
        if len(counts) != n or len(final) != n:
            raise ValueError(f"{len(counts)} counts and {len(final)} flags for {n} rows")
        if wav is not None:
            wav = wav.detach().reshape(n, -1)
            if wav.dtype != torch.float32 or (wav.numel() and wav.stride(-1) != 1):
                wav = wav.to(torch.float32).contiguous()
        cnt = (C.c_int64 * n)(*[int(c) for c in counts])
        fin = (C.c_int32 * n)(*[1 if f else 0 for f in final])
        lib, st = _lib.load(), _lib.stream_ptr(self.device)
        _lib.check_arg(lib.sopro_longform_stream_push(self._h, wav.data_ptr() if wav is not None and wav.numel() else None,
                                                      int(wav.stride(0)) if wav is not None else 0, self.row0, n, cnt, fin, st))
        _lib.check_arg(lib.sopro_longform_stream_status(self._h, self.row0, n, self._status[self.row0].data_ptr(), st))
        self.pushes += 1

    def status(self, seg: int) -> Tuple[int, int, int, int, int]:
        """(n, decided, start, available bound, final) of segment seg as of the last push read (zeros before its group
        starts)."""
        if seg >= self.started:
            return (0, 0, 0, 0, 0)
        n, d, s, a, f = (int(v) for v in self._st[self._row(seg)])
        return n, d, s, a, f

    def group_final(self) -> bool:
        """Every row of the group being pushed is final."""
        return all(self.status(self.started - self.n_rows + i)[4] for i in range(self.n_rows))

    def done(self) -> bool:
        return self.cur >= self.B

    def take(self, limit: int) -> Optional[torch.Tensor]:
        """The next certain piece of the passage, [1, m] f32 with 0 < m <= limit, written on the current stream; None
        when nothing is certain yet."""
        pieces, m = [], 0
        while m < limit and self.cur < self.B:
            n, decided, start, avail, final = self.status(self.cur)
            if not decided:
                break
            if final and avail == start:  # a segment with no samples: no span, no pause
                self.cur += 1
                continue
            if self.pos < 0:
                turn = 0 if self.turn_of is None else self.turn_of[self.cur]
                gap = self.P if turn == self.prev_turn else self.TP
                self.pos, self.pause_left = start, (gap if self.spans else 0)
                self.spans, self.prev_turn = self.spans + 1, turn
            if self.pause_left:
                z = min(self.pause_left, limit - m)
                pieces.append((-1, 0, z, 0, -1))
                m, self.pause_left = m + z, self.pause_left - z
                continue
            k = min(avail - self.pos, limit - m)
            if k > 0:
                pieces.append((self._row(self.cur), self.pos, self.pos + k, start, avail if final else -1))
                m, self.pos = m + k, self.pos + k
            if final and self.pos == avail:
                self.cur, self.pos = self.cur + 1, -1
                continue
            break
        if m == 0:
            return None
        q = np.ascontiguousarray(np.asarray(pieces, dtype=np.int64).reshape(-1, 5))
        y = torch.empty((1, m), dtype=torch.float32, device=self.device)
        _lib.check_arg(_lib.load().sopro_longform_stream_emit(self._h, q.ctypes.data, len(pieces), y.data_ptr(), m,
                                                              _lib.stream_ptr(self.device)))
        return y

    def close(self) -> None:
        if getattr(self, "_h", None):
            _lib.load().sopro_longform_stream_destroy(self._h)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class StreamJoinPool:
    """Idle StreamJoin states, reused by the next passage (like MimiStreamDecoder's stream states): ``checkout`` takes
    one with enough rows and capacity, ``release`` keeps at most MAX_IDLE, the oldest going first."""

    MAX_IDLE = 2

    def __init__(self, device):
        self.device = device
        self._idle: List[StreamJoin] = []

    def checkout(self, rows: int, max_len: int) -> StreamJoin:
        for i in range(len(self._idle) - 1, -1, -1):
            s = self._idle[i]
            if s.rows >= rows and s.max_len >= max_len:
                return self._idle.pop(i)
        return StreamJoin(rows, max_len, self.device)

    def release(self, s: Optional[StreamJoin]) -> None:
        if s is None:
            return
        self._idle.append(s)
        while len(self._idle) > self.MAX_IDLE:
            self._idle.pop(0).close()
