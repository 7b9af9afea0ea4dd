"""A voice per text: the host side of ``synthesize_batch(texts, ref=[...])`` and of the prefill's voice table.

``ref`` is either one ``PreparedReference`` for every text or a sequence with one per text.  The prefill reads a table
of distinct voices: texts that pass the same object share one slot (identity, not content: two equal references
prepared separately take two slots, which costs memory traffic, never correctness).  Every check here runs before any
device work or random draw, so a refused call leaves the device and the global generator untouched.  Host only.

Voice blends (``SoproTTS.blend_voices``).  A blend of voices v_1..v_n with weights w_i > 0 uses the normalised weights
ŵ_i = w_i / Σw, computed in float64 and each rounded once to float32; the prefill and the float64 oracle
(oracle/blend_oracle.py) both use those float32 values.  A voice enters generation only in the prefill, so the blend is
defined there:

- speaker vector: sv = normalize(Σ ŵ_i sv_i), in float64 on the host, rounded once to float32.  A blend of one
  component keeps that component's sv_ref unchanged (no renormalisation, so no last-bit change);
- each reference cross-attention layer: each component's read-out a_i is the row's query attending to that component's
  own K / V (its own softmax, non-finite entries zeroed), and a = Σ ŵ_i a_i in component order; only then come the RMS
  match clamp(rms(x) / rms(a), 0, 10), out_proj and the gate.  This is a mixture of per-voice read-outs, not one softmax
  over the union of the keys, in which whichever voice matches the query better would take over.  The next layer's
  queries come from this mixed output;
- everything else (text encoder, FiLM arithmetic, cond_norm) is unchanged.

A ``VoiceBlend`` is a ``PreparedReference`` whose reference fields are its components' concatenated along the frame
axis, so it goes wherever a voice goes; ``segments`` (frames per component) and ``weights`` (ŵ) tell the prefill where
each component's frames are (``segment_table``, ``sopro_prefill_run_blends``).  Whether a blend sounds between its
voices on the released checkpoint has not been measured."""
from __future__ import annotations

import math
import numbers
from dataclasses import dataclass
from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch

from .prefill import PreparedReference

MAX_REF_FRAMES = 4096  # the prefill's cross-attention limit (sopro_prefill_run_voices)
MAX_BLEND_SEGMENTS = 16  # segments of one blend (SOPRO_PREFILL_MAX_BLEND_SEGMENTS)


@dataclass
class VoiceBlend(PreparedReference):
    """A blended voice (see the module docstring).  ref_tokens_btq, ref_seq and each layer's K / V hold the components'
    frames one after another; segment s covers ``segments[s]`` frames and weighs ``weights[s]`` (float32 values that
    sum to 1 up to rounding).  ``segment_sv`` [n_segments, sv_dim] (float32, on the CPU) keeps each component's speaker
    vector, so that a blend of blends is the blend of their segments.  It holds no reference to its components."""
    segments: Tuple[int, ...]
    weights: Tuple[float, ...]
    segment_sv: torch.Tensor


def geometry(cfg) -> dict:
    """The voice geometry the prefill takes for this config (check_voice's keyword arguments)."""
    heads = int(cfg.ref_xattn_heads)
    return dict(layers=int(cfg.ref_xattn_layers), heads=heads, head_dim=int(cfg.d_model) // heads, sv_dim=int(cfg.sv_student_dim))


def voice_slots(ref, n_rows: int) -> Tuple[List[PreparedReference], List[int]]:
    """-> (the distinct voices in first-use order, the slot of each of the n_rows texts).  One PreparedReference is one
    slot for every text.  A sequence must hold n_rows PreparedReferences (ValueError on its length, TypeError on an
    element or on anything else)."""
    if isinstance(ref, PreparedReference):
        return [ref], [0] * int(n_rows)
    if isinstance(ref, (str, bytes)) or not isinstance(ref, Sequence):
        raise TypeError(f"ref must be a PreparedReference or a sequence of them, got {type(ref).__name__}")
    if len(ref) != int(n_rows):
        raise ValueError(f"ref holds {len(ref)} voices for {int(n_rows)} texts; pass one PreparedReference or one per text")
    slots: List[PreparedReference] = []
    index = {}
    of: List[int] = []
    for i, r in enumerate(ref):
        if not isinstance(r, PreparedReference):
            raise TypeError(f"ref[{i}] is a {type(r).__name__}, not a PreparedReference")
        k = id(r)
        if k not in index:
            index[k] = len(slots)
            slots.append(r)
        of.append(index[k])
    return slots, of


def check_voice(ref: PreparedReference, *, layers: int, heads: int, head_dim: int, sv_dim: int) -> int:
    """A voice's geometry against the engine's -> its reference frames Tr.  ValueError on a layer count, head count, head
    dim or sv_dim that differs, or Tr outside [1, 4096]; NotImplementedError on a key padding mask (prepare_reference
    never makes one)."""
    sv = ref.sv_ref
    if int(sv.numel()) != int(sv_dim):
        raise ValueError(f"a voice's sv_ref holds {int(sv.numel())} values; the engine takes {int(sv_dim)}")
    caches = ref.ref_kv_caches
    if len(caches) != int(layers):
        raise ValueError(f"a voice has {len(caches)} reference layers; the engine has {int(layers)}")
    Tr = None
    for i, c in enumerate(caches):
        if c.get("key_padding_mask") is not None:
            raise NotImplementedError("prepared references with a key padding mask are not produced by prepare_reference")
        k, v = c["k"], c["v"]
        shape = tuple(k.shape[1:]) if k.dim() == 4 and int(k.shape[0]) == 1 else tuple(k.shape)
        if len(shape) != 3 or tuple(v.shape) != tuple(k.shape) or shape[0] != int(heads) or shape[2] != int(head_dim):
            raise ValueError(f"reference layer {i}: K {tuple(k.shape)} / V {tuple(v.shape)}; the engine takes "
                             f"[1, {int(heads)}, Tr, {int(head_dim)}]")
        if Tr is None:
            Tr = shape[1]
        elif shape[1] != Tr:
            raise ValueError(f"reference layer {i} has {shape[1]} frames, layer 0 {Tr}")
    if Tr is not None and not 1 <= Tr <= MAX_REF_FRAMES:
        raise ValueError(f"a voice of {Tr} reference frames; the prefill takes [1, {MAX_REF_FRAMES}]")
    return 1 if Tr is None else int(Tr)


def check_voices(ref, n_rows: int, **geom) -> Tuple[List[PreparedReference], List[int]]:
    """voice_slots, and check_voice on every slot when `ref` is a sequence (one PreparedReference keeps the refusals it
    has always had, raised by the prefill itself)."""
    slots, of = voice_slots(ref, n_rows)
    if not isinstance(ref, PreparedReference):
        for r in slots:
            check_voice(r, **geom)
    return slots, of


def _frames_first(t: torch.Tensor) -> torch.Tensor:
    """A [T, C] or [1, T, C] reference tensor as [1, T, C]."""
    return t.unsqueeze(0) if t.dim() == 2 else t


def _kv4(t: torch.Tensor, heads: int, head_dim: int) -> torch.Tensor:
    """A cached K or V, [H, Tr, dh] or [1, H, Tr, dh], as [1, H, Tr, dh]."""
    return t.reshape(1, heads, -1, head_dim)


def _check_weights(weights, n: int) -> List[float]:
    if weights is None:
        return [1.0] * n
    if isinstance(weights, (str, bytes)) or not isinstance(weights, Sequence):
        raise TypeError(f"weights must be a sequence of numbers, got {type(weights).__name__}")
    ws = list(weights)
    if len(ws) != n:
        raise ValueError(f"{len(ws)} weights for {n} voices")
    out = []
    for i, w in enumerate(ws):
        if isinstance(w, (bool, np.bool_)) or not isinstance(w, numbers.Real):
            raise TypeError(f"weights[{i}] is a {type(w).__name__}, not a number")
        w = float(w)
        if not math.isfinite(w) or w <= 0.0:
            raise ValueError(f"weights[{i}] = {w}; a weight must be finite and > 0")
        out.append(w)
    return out


def blend(voices: Sequence[PreparedReference], weights=None, *, device, layers: int, heads: int, head_dim: int,
          sv_dim: int) -> VoiceBlend:
    """SoproTTS.blend_voices: the voices mixed with `weights` (None = equal) -> a VoiceBlend on `device`.
    The same object passed twice is one component whose weights add up; a VoiceBlend is flattened into its segments, its
    weights scaled by its own.  Every check runs before any device work; the only device access before the result is
    built is one read of the components' speaker vectors.  TypeError on `voices` that is not a sequence of
    PreparedReference or on a weight that is not a number (or a bool); ValueError on an empty sequence, weights of
    another length, a weight that is not finite and > 0, a voice of another geometry (check_voice) or with more than one
    speaker vector, more than MAX_BLEND_SEGMENTS segments or MAX_REF_FRAMES frames in all, or a weighted mean speaker
    vector of norm < 1e-6."""
    if isinstance(voices, (str, bytes, PreparedReference)) or not isinstance(voices, Sequence):
        raise TypeError(f"voices must be a sequence of PreparedReference, got {type(voices).__name__}")
    if len(voices) == 0:
        raise ValueError("voices is empty; a blend needs at least one voice")
    for i, r in enumerate(voices):
        if not isinstance(r, PreparedReference):
            raise TypeError(f"voices[{i}] is a {type(r).__name__}, not a PreparedReference")
    ws = _check_weights(weights, len(voices))
    geom = dict(layers=layers, heads=heads, head_dim=head_dim, sv_dim=sv_dim)
    # flatten and merge: a segment is (component, index of its segment or -1 for a plain voice, frames, first frame)
    merged: Dict[Tuple[int, int], list] = {}
    for i, (r, w) in enumerate(zip(voices, ws)):
        sv = r.sv_ref
        if sv.dim() >= 2 and int(sv.shape[0]) > 1:
            raise ValueError(f"voices[{i}] has {int(sv.shape[0])} speaker vectors; a blend takes voices with one")
        Tr = check_voice(r, **geom)
        if isinstance(r, VoiceBlend):
            if len(r.segments) != len(r.weights) or sum(r.segments) != Tr or int(r.segment_sv.shape[0]) != len(r.segments):
                raise ValueError(f"voices[{i}] is a VoiceBlend whose segments do not cover its {Tr} frames")
            parts, start = [], 0
            for k, (n, wk) in enumerate(zip(r.segments, r.weights)):
                parts.append(((id(r), k), w * float(wk), r, k, int(n), start))
                start += int(n)
        else:
            parts = [((id(r), -1), w, r, -1, Tr, 0)]
        for key, wk, comp, k, n, start in parts:
            if key in merged:
                merged[key][0] += wk
            else:
                merged[key] = [wk, comp, k, n, start]
    segs = list(merged.values())
    if len(segs) > MAX_BLEND_SEGMENTS:
        raise ValueError(f"a blend of {len(segs)} segments; the prefill takes at most {MAX_BLEND_SEGMENTS}")
    total = sum(s[3] for s in segs)
    if total > MAX_REF_FRAMES:
        raise ValueError(f"a blend of {total} reference frames; the prefill takes at most {MAX_REF_FRAMES}")
    wsum = math.fsum(s[0] for s in segs)
    what = [float(np.float32(s[0] / wsum)) for s in segs]
    # the speaker vectors: one read of every plain component's, the segment vectors a blend already keeps
    plain = {}
    for s in segs:
        if s[2] < 0 and id(s[1]) not in plain:
            plain[id(s[1])] = s[1].sv_ref.detach().to("cpu", torch.float32).reshape(-1)
    seg_sv = torch.stack([plain[id(s[1])] if s[2] < 0 else s[1].segment_sv[s[2]].to(torch.float32) for s in segs])
    if len(segs) == 1:
        comp = segs[0][1]
        sv_ref = (comp.sv_ref if segs[0][2] < 0 else seg_sv).detach().to(device, torch.float32).clone().reshape(1, -1)
    else:
        mix = (torch.tensor(what, dtype=torch.float64)[:, None] * seg_sv.double()).sum(dim=0)
        norm = float(mix.norm())
        if norm < 1e-6:
            raise ValueError(f"the weighted mean speaker vector has norm {norm:.3g}; those voices cancel out")
        sv_ref = (mix / norm).float().reshape(1, -1).to(device)

    def cat(pick) -> torch.Tensor:
        return torch.cat([pick(s).to(device) for s in segs], dim=-2).contiguous()

    def frames(t: torch.Tensor, s) -> torch.Tensor:
        return t if s[2] < 0 else t[..., s[4]: s[4] + s[3], :]

    caches = []
    for i in range(int(layers)):
        caches.append({"k": cat(lambda s: frames(_kv4(s[1].ref_kv_caches[i]["k"], heads, head_dim).float(), s)),
                       "v": cat(lambda s: frames(_kv4(s[1].ref_kv_caches[i]["v"], heads, head_dim).float(), s)),
                       "key_padding_mask": None})
    return VoiceBlend(ref_tokens_btq=cat(lambda s: frames(_frames_first(s[1].ref_tokens_btq), s)), sv_ref=sv_ref,
                      ref_seq=cat(lambda s: frames(_frames_first(s[1].ref_seq), s)), ref_kv_caches=caches,
                      segments=tuple(int(s[3]) for s in segs), weights=tuple(what), segment_sv=seg_sv.clone())


def segment_table(slots: Sequence[PreparedReference], trs: Sequence[int]) -> Tuple[List[int], List[int], List[float]]:
    """The prefill's voice slots (with their frames `trs`) -> sopro_prefill_run_blends's (n_seg, seg_frames, seg_w): a
    plain voice is one segment of weight 1, a VoiceBlend its own segments.  ValueError on a blend whose segments do not
    cover its frames."""
    n_seg: List[int] = []
    frames: List[int] = []
    ws: List[float] = []
    for r, tr in zip(slots, trs):
        if isinstance(r, VoiceBlend):
            if len(r.segments) != len(r.weights) or sum(r.segments) != int(tr):
                raise ValueError(f"a VoiceBlend of segments {r.segments} over {int(tr)} frames")
            n_seg.append(len(r.segments))
            frames += [int(n) for n in r.segments]
            ws += [float(w) for w in r.weights]
        else:
            n_seg.append(1)
            frames.append(int(tr))
            ws.append(1.0)
    return n_seg, frames, ws
