"""Timed synthesis restated from its definition (sopro_b200/cues.py, SoproTTS.synthesize_timed, sopro_timeline_mix in
include/sopro_b200.h), independently of the package; it checks only what it needs to read.

- The cue reader: SRT, or WebVTT when the text starts with "WEBVTT" after an optional BOM.  Blocks are runs of
  non-blank lines.  SRT: [index], hh:mm:ss,mmm --> hh:mm:ss,mmm, text; <i> <b> <u> <font> tags and {\\...} blocks
  removed.  WebVTT: header, NOTE / STYLE / REGION blocks skipped; [id], [hh:]mm:ss.ttt --> [hh:]mm:ss.ttt [settings],
  text; <v Name> names the voice, <rt> content dropped, other tags removed, six entities decoded.  Lines join with one
  space.  Times are integer milliseconds; seconds = ms / 1000.
- The fit rule, per cue: off = round(start * 24000), slot = round(end * 24000) - off; S = 65536 when n <= slot, else
  min(round(max_rate * 65536), ceil(n * 65536 / slot)); M = ceil(n * 65536 / S); overrun = max(0, off + M - end
  sample); N = max over cues of max(end sample, off + M).
- The mix: items in (off, index) order, each sample the first covering item's value, then fp32 adds in item order."""
from __future__ import annotations

import re
from typing import List, Optional, Sequence, Tuple

import numpy as np

SR = 24000
ONE = 65536


def samples(t: float) -> int:
    return int(round(float(t) * SR))


def _lines(text: str) -> List[Tuple[int, str]]:
    return list(enumerate(text.replace("\r\n", "\n").replace("\r", "\n").split("\n"), 1))


def _blocks(text: str):
    out, cur = [], []
    for n, s in _lines(text):
        if s.strip():
            cur.append((n, s))
        elif cur:
            out.append(cur)
            cur = []
    if cur:
        out.append(cur)
    return out


def _ms(parts) -> int:
    h, m, s, ms = parts
    return ((int(h or 0) * 60 + int(m)) * 60 + int(s)) * 1000 + int(ms)


def parse(text: str) -> List[Tuple[float, float, str, Optional[str]]]:
    """-> [(start s, end s, text, voice name or None)] for text the reader accepts."""
    if text.startswith("\ufeff"):
        text = text[1:]
    cues = []
    if text.startswith("WEBVTT"):
        t = r"(?:(\d+):)?(\d\d):(\d\d)\.(\d\d\d)"
        timing = re.compile(rf"\s*{t}[ \t]+-->[ \t]+{t}")
        for block in _blocks(text)[1:]:
            first = block[0][1].strip()
            if first.split(" ")[0].split("\t")[0] in ("NOTE", "STYLE", "REGION"):
                continue
            k = 0 if "-->" in block[0][1] else 1
            g = timing.match(block[k][1]).groups()
            body = "\n".join(s for _n, s in block[k + 1:])
            names = [x.strip() for x in re.findall(r"<v(?:\.[^\s>]*)?[ \t]+([^>]*)>", body) if x.strip()]
            body = re.sub(r"<rt[^>]*>.*?</rt>", "", body, flags=re.S)
            body = re.sub(r"<[^>]*>", "", body)
            ent = {"&amp;": "&", "&lt;": "<", "&gt;": ">", "&nbsp;": " ", "&lrm;": "", "&rlm;": ""}
            body = re.sub("|".join(ent), lambda m: ent[m.group(0)], body)
            words = " ".join(x.strip() for x in body.split("\n") if x.strip())
            cues.append((_ms(g[:4]) / 1000, _ms(g[4:]) / 1000, words, names[0] if names else None))
        return cues
    t = r"(\d+):(\d\d):(\d\d)[,.](\d\d\d)"
    timing = re.compile(rf"\s*{t}\s*-->\s*{t}")
    for block in _blocks(text):
        k = 1 if block[0][1].strip().isdigit() and len(block) > 1 else 0
        g = timing.match(block[k][1]).groups()
        lines = []
        for _n, s in block[k + 1:]:
            s = re.sub(r"</?(i|b|u|font)(\s[^>]*)?>", "", s, flags=re.I)
            s = re.sub(r"\{\\[^}]*\}", "", s).strip()
            if s:
                lines.append(s)
        cues.append((_ms(g[:4]) / 1000, _ms(g[4:]) / 1000, " ".join(lines), None))
    return cues


def fit(n: Sequence[int], starts: Sequence[float], ends: Sequence[float], max_rate: float):
    """The joined lengths and times of a track's cues -> (S, M, overrun in samples, offsets, N)."""
    cap = int(round(max_rate * ONE))
    S, M, over, offs = [], [], [], []
    N = 0
    for nk, a, b in zip(n, starts, ends):
        off, end = samples(a), samples(b)
        slot = end - off
        s = ONE if nk <= slot else min(cap, -(-nk * ONE // slot))
        m = -(-nk * ONE // s)
        S.append(s)
        M.append(m)
        over.append(max(0, off + m - end))
        offs.append(off)
        N = max(N, end, off + m)
    return S, M, over, offs, N


def mix(rows: Sequence[np.ndarray], offsets: Sequence[int], length: int) -> np.ndarray:
    """A sequential fp32 accumulation in item order: y[t] starts as the first covering item's sample."""
    y = np.zeros(int(length), dtype=np.float32)
    have = np.zeros(int(length), dtype=bool)
    for r, o in zip(rows, offsets):
        r = np.asarray(r, dtype=np.float32)
        o = int(o)
        seg = slice(o, o + r.size)
        y[seg] = np.where(have[seg], y[seg] + r, r).astype(np.float32)
        have[seg] = True
    return y
