"""The speech-markup plan and assembly restated from their definitions (sopro_b200/ssml.py, SoproTTS.synthesize_ssml),
for markup the parser accepts; it checks nothing.

The markup flattens to a list of items in document order: text (with the voice, the rate and the dB in force),
``<p>`` / ``<s>`` edges (at an element's start and end), and breaks.  Text runs are maximal stretches of text of one
style with no edge or break inside (whitespace belongs to any run); each run is cut by the caller's split_text.

Gaps, at 24 kHz (round(ms * 24), half to even):
- between two segments of one run: the sentence pause P;
- between two runs: the sum of the breaks between them if there is any break (each break rounded on its own),
  else the paragraph pause at a ``<p>`` edge, else P at an ``<s>`` edge or after a run whose text ends a sentence
  (``[.!?…]+`` and closing quotes / brackets at its end), else 0;
- before the first segment and after the last: the breaks there, else nothing.
Rates multiply down the nesting and are multiplied by the call's speed; volumes add in dB (silent = -inf, gain 0);
a gain is fp32(10^(dB / 20)) from double.

Merging: a segment that produced no speech takes no part; between two consecutive spoken segments the gap is the
largest of the gaps between them, and the gaps between the passage's edge and the first (last) spoken segment are
dropped, the edge silences kept.

The assembly: lead zeros, then dialogue_oracle.join of the (already stretched) rows with the merged gaps and the
gains, then trail zeros."""
from __future__ import annotations

import math
import re
import xml.etree.ElementTree as ET
from typing import Callable, List, Sequence, Tuple

import numpy as np

from .dialogue_oracle import join

RATE = {"x-slow": 0.5, "slow": 0.75, "medium": 1.0, "fast": 1.25, "x-fast": 1.5}
VOLUME = {"silent": -math.inf, "x-soft": -12.0, "soft": -6.0, "medium": 0.0, "loud": 6.0, "x-loud": 12.0}
STRENGTH = {"none": 0.0, "x-weak": 50.0, "weak": 150.0, "strong": 500.0, "x-strong": 1000.0}
END = re.compile("[.!?…]+[\"'”’)\\]]*$")
NS = "{http://www.w3.org/2001/10/synthesis}"


def samples(ms: float) -> int:
    return int(round(float(ms) * 24))


def gain(db: float) -> np.float32:
    return np.float32(0.0) if db == -math.inf else np.float32(10.0 ** (db / 20.0))


def items(ssml: str, voices, default_voice, pause_ms: float) -> list:
    """("text", str, (voice, rate, db)) | ("edge", "p" | "s") | ("break", samples), in document order."""
    s = ssml.strip()
    try:
        root = ET.fromstring(s)
        if root.tag.replace(NS, "") != "speak":
            raise ET.ParseError
    except ET.ParseError:
        root = ET.fromstring("<speak>" + ssml + "</speak>")
    out: list = []

    def walk(el, voice, rate, db):
        tag = el.tag.replace(NS, "")
        if tag == "break":
            if el.get("time") is not None:
                t = el.get("time").strip()
                ms = float(t[:-2]) if t.endswith("ms") else float(t[:-1]) * 1000.0
            else:
                ms = STRENGTH.get(el.get("strength", "medium"), pause_ms)
            out.append(("break", samples(ms)))
            return
        if tag == "sub":
            out.append(("text", el.get("alias"), (voice, rate, db)))
            return
        if tag == "voice":
            voice = voices[el.get("name")]
        if tag == "prosody":
            r = el.get("rate")
            if r is not None:
                rate *= RATE[r] if r in RATE else (float(r.strip()[:-1]) / 100.0 if r.strip().endswith("%") else float(r))
            v = el.get("volume")
            if v is not None:
                db += VOLUME[v] if v in VOLUME else float(v.strip()[:-2])
        if tag in ("p", "s"):
            out.append(("edge", tag))
        out.append(("text", el.text or "", (voice, rate, db)))
        for c in el:
            walk(c, voice, rate, db)
            out.append(("text", c.tail or "", (voice, rate, db)))
        if tag in ("p", "s"):
            out.append(("edge", tag))

    walk(root, default_voice, 1.0, 0.0)
    return out


def plan(ssml: str, voices, default_voice, pause_ms: float, paragraph_pause_ms: float, speed,
         split: Callable[[str], List[str]]) -> Tuple[List[Tuple[str, object, float, float]], List[int], int, int]:
    """-> (segments as (text, voice, rate with speed, dB), gaps between consecutive segments, lead, trail)."""
    P, PP = samples(pause_ms), samples(paragraph_pause_ms)
    sp = 1.0 if speed is None else float(speed)
    # runs and the boundary items between them
    seq: list = []   # ("run", text, style) | item
    cur_text, cur_style = "", None
    for it in items(ssml, voices, default_voice, pause_ms):
        if it[0] == "text":
            t, st = it[1], it[2]
            if t.strip() and cur_text.strip() and not (st[0] is cur_style[0] and st[1:] == cur_style[1:]):
                seq.append(("run", cur_text, cur_style))
                cur_text, cur_style = "", None
            if t.strip() and not cur_text.strip():
                cur_style = st
            cur_text += t
        else:
            seq.append(("run", cur_text, cur_style))
            cur_text, cur_style = "", None
            seq.append(it)
    seq.append(("run", cur_text, cur_style))
    segs: list = []
    gaps: List[int] = []
    between: list = []     # the boundary items since the last spoken run
    last_text = None
    lead = 0
    for it in seq:
        if it[0] != "run":
            between.append(it)
            continue
        pieces = split(it[1])
        if not pieces:
            continue
        brk = [b[1] for b in between if b[0] == "break"]
        kinds = {b[1] for b in between if b[0] == "edge"}
        if last_text is None:
            lead = sum(brk)
        elif brk:
            gaps.append(sum(brk))
        elif "p" in kinds:
            gaps.append(PP)
        elif "s" in kinds or END.search(last_text.rstrip()):
            gaps.append(P)
        else:
            gaps.append(0)
        gaps += [P] * (len(pieces) - 1)
        voice, rate, db = it[2]
        segs += [(p, voice, rate * sp, db) for p in pieces]
        between, last_text = [], it[1]
    trail = sum(b[1] for b in between if b[0] == "break")
    return segs, gaps, lead, trail


def merged_pauses(gaps: Sequence[int], spoken: Sequence[bool]) -> List[int]:
    """The gap before each spoken segment after the first: the largest gap between it and the previous spoken one."""
    idx = [k for k, s in enumerate(spoken) if s]
    return [max(gaps[a:b]) for a, b in zip(idx, idx[1:])]


def assemble(rows: Sequence[np.ndarray], gaps: Sequence[int], dbs: Sequence[float], lead: int, trail: int) -> np.ndarray:
    """The stretched rows of the segments (each row all speech: its extent is the whole row) -> the passage."""
    spoken = [len(r) > 0 for r in rows]
    body = join(rows, [(0, len(r)) for r in rows], merged_pauses(gaps, spoken), [gain(d) for d in dbs])
    return np.concatenate([np.zeros(lead, np.float32), body, np.zeros(trail, np.float32)])
