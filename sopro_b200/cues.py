"""Subtitle cues for timed synthesis (SoproTTS.synthesize_timed): a reader for SRT and WebVTT files, the records of a
track, and the rule that fits each cue into its slot.  Host only: nothing here draws a random number or touches a
device.

``parse(text)`` reads WebVTT when the text starts with ``WEBVTT`` (after an optional byte-order mark), SRT otherwise,
and returns the cues in input order.

- SRT: blocks separated by blank lines; a block is an optional numeric index line, a timing line
  ``hh:mm:ss,mmm --> hh:mm:ss,mmm`` (``.`` is accepted before the milliseconds, anything after the end time is
  ignored), then the text lines.  ``<i> <b> <u> <font ...>`` tags and ``{\\...}`` override blocks are removed.
- WebVTT: the header block is skipped, and so are ``NOTE``, ``STYLE`` and ``REGION`` blocks.  A cue is an optional
  identifier line, a timing line ``[hh:]mm:ss.ttt --> [hh:]mm:ss.ttt`` whose cue settings after the end time are
  ignored, then the text lines.  ``<v Name>`` (or ``<v.class Name>``) names the cue's voice; ``<rt>`` content is
  dropped; every other tag is removed (``<c>``, ``<i>``, ``<b>``, ``<u>``, ``<lang>``, ``<ruby>``, inline timestamps
  such as ``<00:00:01.000>``); ``&amp; &lt; &gt; &nbsp; &lrm; &rlm;`` are decoded (``&nbsp;`` to a space, the
  direction marks to nothing).

A cue's lines are joined with one space; CRLF and CR line ends are accepted.  A cue whose text is empty after the tags
are removed is kept: it speaks nothing.  Refused with ValueError, naming the line number: a malformed timing line,
an end not after its start, a time past MAX_SECONDS, a WebVTT cue with two different ``<v>`` names, and a file with no
cue.

Times map to 24 kHz samples as round(t * 24000) in double, half to even (``to_samples``); a time read from a file is
its milliseconds / 1000, so every millisecond time maps to exactly ms * 24 samples."""
from __future__ import annotations

import dataclasses
import math
import numbers
import re
from typing import Any, List, Mapping, Optional, Sequence, Tuple

MAX_SECONDS = 4 * 3600.0
SAMPLE_RATE = 24000


@dataclasses.dataclass(frozen=True)
class Cue:
    """One line of a track: `start` and `end` in seconds, 0 <= start < end <= MAX_SECONDS, the `text` to speak, and
    `voice`, a name of SoproTTS.synthesize_timed's `voices` (None: the call's `ref`).  ValueError / TypeError for
    anything else."""

    start: float
    end: float
    text: str
    voice: Optional[str] = None

    def __post_init__(self):
        for what in ("start", "end"):
            v = getattr(self, what)
            if isinstance(v, bool) or not isinstance(v, numbers.Real) or not math.isfinite(float(v)):
                raise ValueError(f"cue {what} must be a finite number of seconds, got {v!r}")
        if not 0.0 <= float(self.start) < float(self.end) <= MAX_SECONDS:
            raise ValueError(f"a cue needs 0 <= start < end <= {MAX_SECONDS:g} s, got [{self.start!r}, {self.end!r}]")
        if not isinstance(self.text, str):
            raise TypeError(f"cue text must be a str, got {type(self.text).__name__}")
        if self.voice is not None and not isinstance(self.voice, str):
            raise TypeError(f"cue voice must be a name (str) or None, got {type(self.voice).__name__}")


@dataclasses.dataclass(frozen=True)
class CueFit:
    """How cue `index` (input order) was fitted: `rate`, the speed-up S / 65536 it was spoken at (1: not stretched),
    `spoken`, its speech's length in seconds after the stretch, and `overrun`, the seconds its speech runs past the
    cue's end (0 unless the speed-up hit max_rate).  A cue that produced no speech has rate 1, spoken 0, overrun 0."""

    index: int
    rate: float
    spoken: float
    overrun: float


def to_samples(t: float) -> int:
    """round(t * 24000), half to even: a time in seconds as a 24 kHz sample index."""
    return int(round(float(t) * SAMPLE_RATE))


_SRT_TIME = r"(\d+):(\d{2}):(\d{2})[,.](\d{3})"
_SRT_TIMING = re.compile(rf"^\s*{_SRT_TIME}\s*-->\s*{_SRT_TIME}(?:\s.*)?$")
_VTT_TIME = r"(?:(\d+):)?(\d{2}):(\d{2})\.(\d{3})"
_VTT_TIMING = re.compile(rf"^\s*{_VTT_TIME}[ \t]+-->[ \t]+{_VTT_TIME}(?:[ \t].*)?$")
_SRT_TAG = re.compile(r"</?(?:i|b|u|font)(?:\s[^>]*)?>", re.IGNORECASE)
_SRT_OVERRIDE = re.compile(r"\{\\[^}]*\}")
_VTT_VOICE = re.compile(r"<v(?:\.[^\s>]*)?(?:[ \t]+([^>]*))?>")
_VTT_RT = re.compile(r"<rt(?:[.\s][^>]*)?>.*?</rt>", re.DOTALL)
_TAG = re.compile(r"<[^>]*>")
_ENTITY = re.compile(r"&(amp|lt|gt|nbsp|lrm|rlm);")
_ENTITIES = {"amp": "&", "lt": "<", "gt": ">", "nbsp": " ", "lrm": "", "rlm": ""}


def _ms(h: Optional[str], m: str, s: str, ms: str, line: int) -> int:
    if int(m) > 59 or int(s) > 59:
        raise ValueError(f"line {line}: minutes and seconds must be below 60")
    return ((int(h or 0) * 60 + int(m)) * 60 + int(s)) * 1000 + int(ms)


def _times(groups: Tuple[str, ...], line: int) -> Tuple[float, float]:
    a, b = _ms(*groups[:4], line), _ms(*groups[4:], line)
    if b <= a:
        raise ValueError(f"line {line}: the cue's end is not after its start")
    if b > MAX_SECONDS * 1000:
        raise ValueError(f"line {line}: a time past {MAX_SECONDS / 3600:g} h")
    return a / 1000, b / 1000


def _blocks(text: str) -> List[List[Tuple[int, str]]]:
    """The text's blocks of non-blank lines, each line with its 1-based number."""
    out: List[List[Tuple[int, str]]] = []
    cur: List[Tuple[int, str]] = []
    for n, raw in enumerate(text.replace("\r\n", "\n").replace("\r", "\n").split("\n"), 1):
        if raw.strip():
            cur.append((n, raw))
        elif cur:
            out.append(cur)
            cur = []
    if cur:
        out.append(cur)
    return out


def _join(lines: List[str]) -> str:
    return " ".join(s for s in (x.strip() for x in lines) if s)


def _srt(text: str) -> List[Cue]:
    cues = []
    for block in _blocks(text):
        k = 1 if block[0][1].strip().isdigit() and len(block) > 1 else 0
        line, timing = block[k]
        m = _SRT_TIMING.match(timing)
        if m is None:
            raise ValueError(f"line {line}: expected an SRT timing line 'hh:mm:ss,mmm --> hh:mm:ss,mmm', got {timing.strip()!r}")
        start, end = _times(m.groups(), line)
        body = [_SRT_OVERRIDE.sub("", _SRT_TAG.sub("", t)) for _n, t in block[k + 1:]]
        cues.append(Cue(start, end, _join(body)))
    return cues


def _vtt(text: str) -> List[Cue]:
    cues = []
    blocks = _blocks(text)
    for block in blocks[1:]:  # the first block is the header
        head = block[0][1].strip()
        if re.match(r"(NOTE|STYLE|REGION)(\s|$)", head):
            continue
        k = 0 if "-->" in block[0][1] else 1
        if k >= len(block):
            raise ValueError(f"line {block[0][0]}: expected a WebVTT timing line after the cue identifier {head!r}")
        line, timing = block[k]
        m = _VTT_TIMING.match(timing)
        if m is None:
            raise ValueError(f"line {line}: expected a WebVTT timing line '[hh:]mm:ss.ttt --> [hh:]mm:ss.ttt', "
                             f"got {timing.strip()!r}")
        start, end = _times(m.groups(), line)
        voice: Optional[str] = None
        for n, t in block[k + 1:]:
            for v in _VTT_VOICE.finditer(t):
                name = (v.group(1) or "").strip() or None
                if name is not None and voice is not None and name != voice:
                    raise ValueError(f"line {n}: a cue with two voices, {voice!r} and {name!r}")
                voice = voice or name
        body = "\n".join(t for _n, t in block[k + 1:])
        body = _TAG.sub("", _VTT_RT.sub("", body))
        body = _ENTITY.sub(lambda e: _ENTITIES[e.group(1)], body)
        cues.append(Cue(start, end, _join(body.split("\n")), voice))
    return cues


def parse(text: str) -> List[Cue]:
    """An SRT or WebVTT file's text -> its cues in input order (the module's docstring is the contract)."""
    if not isinstance(text, str):
        raise TypeError(f"the cues must be a str, got {type(text).__name__}")
    body = text[1:] if text.startswith("\ufeff") else text
    cues = _vtt(body) if body.startswith("WEBVTT") else _srt(body)
    if not cues:
        n = len(body.replace("\r\n", "\n").replace("\r", "\n").split("\n"))
        raise ValueError(f"line {n}: the file has no cue")
    return cues


# ---- the track as SoproTTS.synthesize_timed takes it, and the fit rule

ONE = 65536               # the stretch's fixed-point speed of rate 1
MIN_RATE, MAX_RATE = 1.0, 4.0


def track(cues) -> List[Cue]:
    """synthesize_timed's `cues`: a str goes through parse, a sequence must hold Cue records -> the cues, each cue's
    end on a later 24 kHz sample than its start.  TypeError / ValueError before any work."""
    if isinstance(cues, str):
        out = parse(cues)
    elif isinstance(cues, Sequence):
        out = list(cues)
        for i, c in enumerate(out):
            if not isinstance(c, Cue):
                raise TypeError(f"cue {i} is a {type(c).__name__}, not a Cue")
        if not out:
            raise ValueError("the track has no cue")
    else:
        raise TypeError(f"cues must be a str (SRT or WebVTT) or a sequence of Cue, got {type(cues).__name__}")
    for i, c in enumerate(out):
        if to_samples(c.end) <= to_samples(c.start):
            raise ValueError(f"cue {i}: its start and end map to the same 24 kHz sample")
    return out


def cue_voices(cues: Sequence[Cue], voices: Optional[Mapping[str, Any]], ref: Any) -> list:
    """Each cue's voice: `ref` for a cue without one, else voices[name].  ValueError for an unknown name, TypeError for a
    `voices` that is not a mapping."""
    if voices is None:
        voices = {}
    if not isinstance(voices, Mapping):
        raise TypeError(f"voices must be a mapping of names to voices, got {type(voices).__name__}")
    for i, c in enumerate(cues):
        if c.voice is not None and c.voice not in voices:
            raise ValueError(f"cue {i}: no voice named {c.voice!r} (the voices are {sorted(voices)})")
    return [ref if c.voice is None else voices[c.voice] for c in cues]


def check_max_rate(max_rate) -> int:
    """The largest speed-up as the stretch's fixed-point speed, round(max_rate * 65536); ValueError for anything but a
    real number in [1, 4] (speech is never slowed down)."""
    if isinstance(max_rate, bool) or not isinstance(max_rate, numbers.Real) or \
            not MIN_RATE <= float(max_rate) <= MAX_RATE:
        raise ValueError(f"max_rate must be a real number in [{MIN_RATE:g}, {MAX_RATE:g}], got {max_rate!r}")
    return int(round(float(max_rate) * ONE))


def fit_speed(n: int, slot: int, S_max: int) -> int:
    """The fit rule: S = 65536 when the n joined samples fit the slot's samples, else min(S_max, ceil(n * 65536 /
    slot)), the least speed-up that fits, capped."""
    n, slot = int(n), int(slot)
    if n <= slot:
        return ONE
    return min(int(S_max), -(-n * ONE // slot))


def groups(counts: Sequence[int], group: int) -> List[Tuple[int, int]]:
    """Consecutive cue ranges [a, b) whose segment counts sum to at most `group` (a cue with more segments than that is
    a range of its own; cues without segments join the range they fall in)."""
    out: List[Tuple[int, int]] = []
    a, filled = 0, 0
    for i, c in enumerate(counts):
        if filled and filled + int(c) > group:
            out.append((a, i))
            a, filled = i, 0
        filled += int(c)
    if a < len(counts):
        out.append((a, len(counts)))
    return out
