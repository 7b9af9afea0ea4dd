"""A voice per text: the host side of ``synthesize_batch(texts, ref=[...])`` and of the prefill's voice table.

``ref`` is either one ``PreparedReference`` for every text or a sequence with one per text.  The prefill reads a table
of distinct voices: texts that pass the same object share one slot (identity, not content: two equal references
prepared separately take two slots, which costs memory traffic, never correctness).  Every check here runs before any
device work or random draw, so a refused call leaves the device and the global generator untouched.  Host only."""
from __future__ import annotations

from typing import List, Sequence, Tuple

from .prefill import PreparedReference

MAX_REF_FRAMES = 4096  # the prefill's cross-attention limit (sopro_prefill_run_voices)


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
