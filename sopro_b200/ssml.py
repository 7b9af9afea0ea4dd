"""Speech markup (no reference counterpart: the reference speaks plain text): an SSML subset read into a plan that
``SoproTTS.synthesize_ssml`` speaks through one batch and joins on the GPU.  Host only: parsing draws nothing and
touches no device, so a caller can inspect the plan before generating it.

The subset, parsed with the standard library's ``xml.etree.ElementTree`` (elements in the SSML namespace or in none):

- ``<speak>``: the root; text with no ``<speak>`` root is parsed as its content.  ``version`` and ``xml:lang`` are
  accepted on it and ignored.
- ``<p>``, ``<s>``: a segment boundary at their start and end.  The text between boundaries is cut as synthesize_long
  cuts a text (longform.split_text with `max_tokens`).
- ``<break time="350ms" | "1.5s">`` (each in [0, 10 s]) or ``<break strength="none | x-weak | weak | medium | strong |
  x-strong">`` (0, 50, 150, `pause_ms`, 500, 1000 ms; a bare ``<break/>`` is medium): the gap at this boundary.
- ``<prosody rate="x-slow | slow | medium | fast | x-fast" | "80%" | "1.2">``: multiplies the enclosing rate by 0.5,
  0.75, 1, 1.25, 1.5, the percentage or the factor.  ``<prosody volume="silent | x-soft | soft | medium | loud |
  x-loud" | "+3dB">``: adds -12, -6, 0, +6, +12 or the given dB to the enclosing level; ``silent`` (and everything
  inside it) has gain 0 and keeps its length.
- ``<voice name="...">``: a voice of the `voices` mapping; outside every ``<voice>``, `default_voice`.
- ``<sub alias="...">``: the alias is spoken instead of the element's text.

A change of voice, rate or volume starts a new segment where it happens.  The gap at a boundary, in samples at
24 kHz (round(ms * 24), half to even), is the sum of the breaks there (each rounded on its own) when there is one,
and otherwise its default: `paragraph_pause_ms` at a ``<p>`` edge, else `pause_ms` at an ``<s>`` edge, between two
segments split_text cut, or after text that ends a sentence (a run of ``.!?…`` and closing quotes or brackets), else
0 (a split inside a sentence; the join's raised-cosine edges still apply).  Breaks before the first segment or after
the last are the leading and trailing silence; the passage's edges have no default gap.

A segment that produces no speech (no frames, or an empty trim) takes no part in the join, and the gaps on either side
of it merge into the larger of the two (``Plan.pauses``); at the passage's edges the leading or trailing silence stays
as it is and the gap to the missing segment goes with it.  Segment k is generated with seed + k.

Refused with ValueError, naming the element or attribute: any other element or attribute (``<emphasis>``,
``<say-as>``, ``<phoneme>``, ``<audio>``, ``<mark>``, ``<prosody pitch>``, ...), malformed XML, an unknown voice name,
an effective rate (nested rates times the call's `speed`) outside [0.25, 4], an effective volume outside [-60, +12]
dB, and a script with nothing to speak.  A span's gain is fp32(10^(dB / 20)), evaluated in double and rounded once."""
from __future__ import annotations

import math
import numbers
import re
import xml.etree.ElementTree as ET
from dataclasses import dataclass
from typing import Any, Dict, List, Mapping, Optional, Sequence, Tuple

import numpy as np

from . import longform as LF

MIN_RATE, MAX_RATE = 0.25, 4.0
MIN_DB, MAX_DB = -60.0, 12.0
MAX_BREAK_MS = 10000.0
RATES = {"x-slow": 0.5, "slow": 0.75, "medium": 1.0, "fast": 1.25, "x-fast": 1.5}
VOLUMES = {"silent": -math.inf, "x-soft": -12.0, "soft": -6.0, "medium": 0.0, "loud": 6.0, "x-loud": 12.0}
STRENGTHS = {"none": 0.0, "x-weak": 50.0, "weak": 150.0, "medium": None, "strong": 500.0, "x-strong": 1000.0}  # None: pause_ms

_NS = "{http://www.w3.org/2001/10/synthesis}"
_XML_LANG = "{http://www.w3.org/XML/1998/namespace}lang"
_ATTRS = {"speak": {"version", _XML_LANG}, "p": set(), "s": set(), "break": {"time", "strength"},
          "prosody": {"rate", "volume"}, "voice": {"name"}, "sub": {"alias"}}
_SENTENCE_END = re.compile("[.!?…]+[\"'”’)\\]]*$")
_TIME = re.compile(r"^\s*(\d+(?:\.\d*)?|\.\d+)\s*(ms|s)\s*$")
_PERCENT = re.compile(r"^\s*(\d+(?:\.\d*)?|\.\d+)\s*%\s*$")
_FACTOR = re.compile(r"^\s*(\d+(?:\.\d*)?|\.\d+)\s*$")
_DB = re.compile(r"^\s*([+-]?(?:\d+(?:\.\d*)?|\.\d+))\s*dB\s*$")


@dataclass(frozen=True)
class Segment:
    text: str
    voice: Any       # a PreparedReference
    rate: float      # the speaking rate, the call's speed folded in, in [0.25, 4]
    db: float        # the level in dB relative to the model's own; -inf for silent

    @property
    def gain(self) -> float:
        """fp32(10^(db / 20)) evaluated in double and rounded once; 0 when silent."""
        return 0.0 if self.db == -math.inf else float(np.float32(10.0 ** (self.db / 20.0)))


@dataclass(frozen=True)
class Plan:
    segments: List[Segment]
    gaps: List[int]     # zeros between segment k and segment k + 1, at 24 kHz
    lead: int           # zeros before the first segment
    trail: int          # zeros after the last segment

    def pauses(self, spoken: Sequence[bool]) -> List[int]:
        """The zeros before each spoken segment after the first, given which segments produced speech: the gaps around
        a silent segment merge into the larger one, and a gap next to the passage's edge goes with the missing
        segment."""
        if len(spoken) != len(self.segments):
            raise ValueError(f"{len(spoken)} flags for {len(self.segments)} segments")
        out: List[int] = []
        seen, acc = False, 0
        for k, s in enumerate(spoken):
            if k:
                acc = max(acc, self.gaps[k - 1])
            if s:
                if seen:
                    out.append(acc)
                seen, acc = True, 0
        return out


def _ms_samples(ms: float) -> int:
    return int(round(float(ms) * 24))


def _real(v, what: str, lo: float, hi: float) -> float:
    if isinstance(v, (bool, np.bool_)) or not isinstance(v, numbers.Real) or not (lo <= float(v) <= hi):
        raise ValueError(f"{what} must be a real number in [{lo:g}, {hi:g}], got {v!r}")
    return float(v)


def _root(ssml: str) -> ET.Element:
    if not isinstance(ssml, str):
        raise TypeError(f"ssml must be a str, got {type(ssml).__name__}")
    try:
        root = ET.fromstring(ssml)
        if root.tag in ("speak", _NS + "speak"):
            return root
    except ET.ParseError:
        pass
    try:
        return ET.fromstring("<speak>" + ssml + "</speak>")
    except ET.ParseError as e:
        raise ValueError(f"the markup is not well-formed XML: {e}") from None


def _tag(el: ET.Element) -> str:
    t = el.tag if isinstance(el.tag, str) else ""
    if t.startswith(_NS):
        t = t[len(_NS):]
    if t not in _ATTRS:
        raise ValueError(f"<{t}> is not supported (the subset: {', '.join('<%s>' % k for k in _ATTRS)})")
    for a in el.attrib:
        if a not in _ATTRS[t]:
            name = "xml:lang" if a == _XML_LANG else a
            raise ValueError(f"<{t} {name}> is not supported")
    return t


def _break_ms(el: ET.Element, pause_ms: float) -> float:
    t = el.get("time")
    if t is not None:
        m = _TIME.match(t)
        if not m:
            raise ValueError(f"<break time={t!r}>: expected a time such as '350ms' or '1.5s'")
        ms = float(m.group(1)) * (1.0 if m.group(2) == "ms" else 1000.0)
        if not ms <= MAX_BREAK_MS:
            raise ValueError(f"<break time={t!r}> is over {MAX_BREAK_MS / 1000:g} s")
        return ms
    s = el.get("strength", "medium")
    if s not in STRENGTHS:
        raise ValueError(f"<break strength={s!r}>: expected one of {', '.join(STRENGTHS)}")
    return pause_ms if STRENGTHS[s] is None else STRENGTHS[s]


def _rate(v: str) -> float:
    if v in RATES:
        return RATES[v]
    m = _PERCENT.match(v)
    if m:
        return float(m.group(1)) / 100.0
    m = _FACTOR.match(v)
    if m:
        return float(m.group(1))
    raise ValueError(f"<prosody rate={v!r}>: expected {', '.join(RATES)}, a percentage or a factor")


def _volume(v: str) -> float:
    if v in VOLUMES:
        return VOLUMES[v]
    m = _DB.match(v)
    if m:
        return float(m.group(1))
    raise ValueError(f"<prosody volume={v!r}>: expected {', '.join(VOLUMES)} or a change in dB such as '+3dB'")


class _Builder:
    """Text runs of one style between boundaries -> segments, gaps and edge silences."""

    def __init__(self, tokenizer, max_tokens: int, P: int, PP: int):
        self.tok, self.max_tokens, self.P, self.PP = tokenizer, max_tokens, P, PP
        self.segments: List[Segment] = []
        self.gaps: List[int] = []
        self.lead = 0
        self.run: List[str] = []
        self.style: Optional[Tuple[Any, float, float]] = None
        self.kinds: set = set()            # the <p> / <s> edges at the pending boundary
        self.breaks: Optional[int] = None  # the pending boundary's breaks, None = no break
        self.ended = False                 # the last spoken run ended a sentence

    def text(self, s: Optional[str], style: Tuple[Any, float, float]) -> None:
        if not s:
            return
        if s.strip():
            if self.style is not None and "".join(self.run).strip() and not _same(style, self.style):
                self.close()
            if not "".join(self.run).strip():
                self.style = style
        self.run.append(s)

    def edge(self, kind: str) -> None:
        self.close()
        self.kinds.add(kind)

    def pause(self, samples: int) -> None:
        self.close()
        self.breaks = (self.breaks or 0) + samples

    def close(self) -> None:
        text, style = "".join(self.run), self.style
        self.run, self.style = [], None
        segs = LF.split_text(text, self.tok, self.max_tokens)
        if not segs:
            return
        if self.segments:
            if self.breaks is not None:
                gap = self.breaks
            elif "p" in self.kinds:
                gap = self.PP
            elif "s" in self.kinds or self.ended:
                gap = self.P
            else:
                gap = 0
            self.gaps.append(gap)
        else:
            self.lead = self.breaks or 0
        self.kinds, self.breaks = set(), None
        self.gaps += [self.P] * (len(segs) - 1)
        self.segments += [Segment(t, style[0], style[1], style[2]) for t in segs]
        self.ended = bool(_SENTENCE_END.search(text.rstrip()))


def _same(a, b) -> bool:
    return a[0] is b[0] and a[1] == b[1] and a[2] == b[2]


def parse(ssml: str, voices: Optional[Mapping[str, Any]], default_voice: Any, pause_ms=250, paragraph_pause_ms=500,
          speed=None, max_tokens: int = 64, tokenizer=None) -> Plan:
    """The markup -> its Plan (the module's docstring is the contract).  `voices`: {name: PreparedReference} for
    ``<voice name>`` (None = none); `default_voice`: the voice outside every ``<voice>``; `pause_ms` and
    `paragraph_pause_ms` in [0, 2000]; `speed` (None = 1) multiplies every segment's rate; `max_tokens` and
    `tokenizer`: split_text's budget and tokenizer.  ValueError (TypeError for a non-str `ssml` or a `voices` that is
    not a mapping) before anything else happens."""
    P, PP = LF.pause_samples(pause_ms), LF.pause_samples(paragraph_pause_ms)
    pause_ms = LF.check_pause(pause_ms)
    speed = 1.0 if speed is None else _real(speed, "speed", MIN_RATE, MAX_RATE)
    if voices is None:
        voices = {}
    if not isinstance(voices, Mapping):
        raise TypeError(f"voices must be a mapping of names to voices, got {type(voices).__name__}")
    b = _Builder(tokenizer, int(max_tokens), P, PP)

    def walk(el: ET.Element, style: Tuple[Any, float, float], top: bool) -> None:
        t = _tag(el)
        voice, rate, db = style
        if t == "speak" and not top:
            raise ValueError("<speak> inside <speak>")
        if t == "break":
            b.pause(_ms_samples(_break_ms(el, pause_ms)))
            return
        if t == "sub":
            alias = el.get("alias")
            if alias is None:
                raise ValueError("<sub> needs an alias")
            b.text(alias, style)
            return
        if t == "voice":
            name = el.get("name")
            if name not in voices:
                raise ValueError(f"<voice name={name!r}>: no such voice (the voices are {sorted(voices)})")
            voice = voices[name]
        if t == "prosody":
            if "rate" in el.attrib:
                rate = rate * _rate(el.get("rate"))
                if not MIN_RATE <= rate * speed <= MAX_RATE:
                    raise ValueError(f"<prosody rate={el.get('rate')!r}>: the effective rate {rate * speed:g} (nested "
                                     f"rates times speed) is outside [{MIN_RATE:g}, {MAX_RATE:g}]")
            if "volume" in el.attrib:
                db = db + _volume(el.get("volume"))
                if db != -math.inf and not MIN_DB <= db <= MAX_DB:
                    raise ValueError(f"<prosody volume={el.get('volume')!r}>: the effective volume {db:+g} dB is "
                                     f"outside [{MIN_DB:g}, {MAX_DB:+g}] dB")
        inner = (voice, rate, db)
        if t in ("p", "s"):
            b.edge(t)
        b.text(el.text, inner)
        for child in el:
            walk(child, inner, False)
            b.text(child.tail, inner)
        if t in ("p", "s"):
            b.edge(t)

    walk(_root(ssml), (default_voice, 1.0, 0.0), True)
    b.close()
    if not b.segments:
        raise ValueError("the markup has nothing to speak")
    segments = [Segment(s.text, s.voice, s.rate * speed, s.db) for s in b.segments]
    return Plan(segments, b.gaps, b.lead, b.breaks or 0)
