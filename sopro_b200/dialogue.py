"""Dialogue synthesis (no reference counterpart: the reference speaks one utterance in one voice): a script of
``(voice, text)`` turns spoken through one batch, each turn in its own voice, and joined on the GPU.

The script's segments are synthesize_long's: each turn's text is cut with ``split_text`` and the segments of every
turn are flattened in script order, segment k seeded ``seed + k`` and spoken in its turn's voice (turns that pass the
same PreparedReference object share one prefill slot, sopro_b200/voices.py).  The join places a sentence pause between
spans of one turn and a turn pause between spans of different turns (longform.gap_pauses), and can scale each turn to
a common loudness: turn j's gain is normalize_loudness's gain for that turn's own join at 24 kHz, applied inside the
join kernel (longform.join_gaps), so a levelled turn equals normalize_loudness of its solo join bit for bit.  The
entry points are SoproTTS.synthesize_dialogue and stream_dialogue.  Host planning lives here; the kernels are
sopro_b200/csrc/longform.cu."""
from __future__ import annotations

from typing import List, Sequence, Tuple

import numpy as np
import torch

from . import longform as LF
from . import voices
from .loudness import normalize_loudness
from .prefill import PreparedReference


def check_turns(turns) -> List[Tuple[PreparedReference, str]]:
    """The script as a list of (voice, text) pairs; TypeError for anything but a non-empty sequence of
    (PreparedReference, str) pairs (ValueError when it is empty).  Host only."""
    if isinstance(turns, (str, bytes)) or not isinstance(turns, Sequence):
        raise TypeError(f"turns must be a sequence of (PreparedReference, str) pairs, got {type(turns).__name__}")
    out = []
    for j, t in enumerate(turns):
        if isinstance(t, (str, bytes)) or not isinstance(t, Sequence) or len(t) != 2 or \
                not isinstance(t[0], PreparedReference) or not isinstance(t[1], str):
            raise TypeError(f"turn {j} is not a (PreparedReference, str) pair")
        out.append((t[0], t[1]))
    if not out:
        raise ValueError("turns is empty: a dialogue needs at least one turn")
    return out


def plan(turns: Sequence[Tuple[PreparedReference, str]], tokenizer, max_tokens: int
         ) -> Tuple[List[str], List[int], List[PreparedReference]]:
    """-> (the script's segments in order, the turn of each, the voice of each).  ValueError when no turn has anything
    to speak; a turn whose text is empty or whitespace only has no segments.  Host only."""
    segments: List[str] = []
    turn_of: List[int] = []
    voice_of: List[PreparedReference] = []
    for j, (voice, text) in enumerate(turns):
        segs = LF.split_text(text, tokenizer, max_tokens)
        segments += segs
        turn_of += [j] * len(segs)
        voice_of += [voice] * len(segs)
    if not segments:
        raise ValueError("the script has nothing to speak (every turn is empty or whitespace only)")
    return segments, turn_of, voice_of


def segment_voices(voice_of: Sequence[PreparedReference]):
    """One PreparedReference when every segment has the same voice object (the one-voice path of synthesize_long),
    else the per-segment list."""
    return voice_of[0] if all(v is voice_of[0] for v in voice_of) else list(voice_of)


def check_script(tts, turns, pause_ms, turn_pause_ms, max_tokens):
    """Every refusal that does not depend on the output chain, before any device work or random draw -> (turns,
    segments, turn of each, voice of each, P, turn P in samples)."""
    turns = check_turns(turns)
    geom = voices.geometry(tts.cfg)
    for r in voices.voice_slots([v for v, _ in turns], len(turns))[0]:
        voices.check_voice(r, **geom)
    P = LF.pause_samples(pause_ms)
    TP = LF.pause_samples(turn_pause_ms)
    budget = LF.check_max_tokens(max_tokens, tts.model.prefill.max_text_len)
    segments, turn_of, voice_of = plan(turns, tts.tokenizer, budget)
    return turns, segments, turn_of, voice_of, P, TP


def turn_segments(turn_of: Sequence[int], n_turns: int) -> List[List[int]]:
    """The segment indices of each turn, in order (empty for a turn with nothing to speak)."""
    out: List[List[int]] = [[] for _ in range(n_turns)]
    for k, j in enumerate(turn_of):
        out[int(j)].append(k)
    return out


def turn_gains(rows: Sequence[torch.Tensor], ext: np.ndarray, turn_of: Sequence[int], n_turns: int, P: int,
               target: float) -> torch.Tensor:
    """Each segment's loudness gain, f32 [segments] on the rows' device: turn j's spans joined alone with P (what
    synthesize_long joins for that turn), every such join metered in one ragged normalize_loudness launch at 24 kHz,
    and segment k takes its turn's gain (1 for a turn with no span).  Nothing synchronises."""
    dev = rows[0].device
    solo = []  # (turn, its own join)
    for j, idx in enumerate(turn_segments(turn_of, n_turns)):
        if idx and (ext[idx, 1] > ext[idx, 0]).any():
            solo.append((j, LF.join_gaps([rows[k] for k in idx], ext[idx], LF.gap_pauses(ext[idx], P)).reshape(-1)))
    g_turn = torch.ones(n_turns, dtype=torch.float32, device=dev)
    if solo:
        lens = [int(w.numel()) for _, w in solo]
        batch = torch.zeros((len(solo), max(lens)), dtype=torch.float32, device=dev)
        for b, (_j, w) in enumerate(solo):
            batch[b, : lens[b]] = w
        _y, g = normalize_loudness(batch, LF.SAMPLE_RATE, target, lens=lens, return_gain=True)
        g_turn[torch.tensor([j for j, _ in solo], device=dev)] = g
    return g_turn[torch.tensor(list(turn_of), device=dev)]


def turn_placement(ext: np.ndarray, turn_of: Sequence[int], n_turns: int, pauses: Sequence[int]
                   ) -> Tuple[List[int], List[List[int]]]:
    """Where each turn sits in the joined passage -> (the sample at which it begins, the zeros after each of its
    non-empty spans: the sentence pause, the gap to the next turn's first span after its last, 0 at the passage's
    end).  A turn with no span begins where the audio continues after the spans before it."""
    starts, after = [0] * n_turns, [[] for _ in range(n_turns)]
    O, m = 0, 0
    for j, idx in enumerate(turn_segments(turn_of, n_turns)):
        starts[j] = O  # empty segments do not move O: this is the turn's first span's start
        for k in idx:
            if int(ext[k, 1]) > int(ext[k, 0]):
                gap = int(pauses[m]) if m < len(pauses) else 0
                after[j].append(gap)
                O += int(ext[k, 1]) - int(ext[k, 0]) + gap
                m += 1
    return starts, after
