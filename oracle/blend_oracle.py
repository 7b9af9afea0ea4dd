"""Float64 restatement of the prefill over a voice blend (sopro_b200/voices.py, DESIGN.md §5t), built from the
sopro_b200/prefill.py functions: ``prepare_conditioning`` with the reference cross-attention of every layer replaced by
the blend's mixture of per-segment read-outs.

Everything runs in float64 except where the shared prefill.py functions round through float32 themselves (their
rms_norm, inside the text encoder's blocks), as sopro_b200/prefill.py::prepare_conditioning does.  The segment weights
are used as given: VoiceBlend.weights already holds the float32 values the CUDA prefill uses."""
from __future__ import annotations

import math
from typing import List, Sequence, Tuple

import torch
import torch.nn.functional as F

from sopro_b200 import prefill as P

Tensor = torch.Tensor


def _rms_norm64(x: Tensor, w: Tensor, eps: float = 1e-6) -> Tensor:
    x = x.double()
    return x * torch.rsqrt(x.pow(2).mean(dim=-1, keepdim=True) + eps) * w.double()


def segments_of(ref: P.PreparedReference) -> Tuple[List[int], List[float]]:
    """(frames per segment, weight per segment): a VoiceBlend's own, a plain voice one segment of weight 1."""
    segs = getattr(ref, "segments", None)
    if segs is None:
        k = ref.ref_kv_caches[0]["k"]
        return [int(k.shape[-2])], [1.0]
    return [int(n) for n in segs], [float(w) for w in ref.weights]


def readout(q: Tensor, k: Tensor, v: Tensor) -> Tensor:
    """One segment's attention read-out: q [B, H, T, dh] against k / v [1 or B, H, Tr, dh] -> [B, H, T, dh], its own
    softmax over its Tr frames, non-finite entries zeroed (nn/ref.py:84-95)."""
    q, k, v = q.double(), k.double(), v.double()
    s = torch.matmul(q, k.transpose(-1, -2)) / math.sqrt(q.shape[-1])
    a = torch.matmul(torch.softmax(s, dim=-1), v)
    return torch.nan_to_num(a, nan=0.0, posinf=0.0, neginf=0.0)


def mixed_readout(q: Tensor, k: Tensor, v: Tensor, frames: Sequence[int], weights: Sequence[float]) -> Tensor:
    """a = sum_i w_i a_i in segment order, a_i the read-out of segment i (frames[i] frames of k / v, one after another)."""
    a, start = None, 0
    for n, w in zip(frames, weights):
        ai = float(w) * readout(q, k[..., start: start + n, :], v[..., start: start + n, :])
        a = ai if a is None else a + ai
        start += n
    return a


def blend_xattn(sd, cfg, x: Tensor, caches, frames: Sequence[int], weights: Sequence[float]) -> Tensor:
    """prefill.ref_xattn over a blend: per layer, the mixed read-out, then the RMS match, out_proj and the gate."""
    H = int(cfg.ref_xattn_heads)
    x = x.double()
    for i, c in enumerate(caches):
        p = f"ref_xattn.blocks.{i}."
        q = P._heads(F.linear(_rms_norm64(x, sd[p + "nq.weight"]), sd[p + "q_proj.weight"].double()), H)
        k, v = c["k"].double(), c["v"].double()
        if k.dim() == 3:
            k, v = k.unsqueeze(0), v.unsqueeze(0)
        a = mixed_readout(q, k, v, frames, weights)
        B, Hh, T, Dh = a.shape
        a = a.transpose(1, 2).reshape(B, T, Hh * Dh)
        rms = lambda t: torch.sqrt(t.pow(2).mean(dim=-1, keepdim=True) + 1e-6)  # noqa: E731
        a = a * (rms(x) / rms(a)).clamp(0.0, 10.0)
        a = F.linear(a, sd[p + "out_proj.weight"].double())
        x = x + float(cfg.ref_xattn_gmax) * math.tanh(float(sd[p + "gate"])) * a
    return x


def prepare_conditioning(sd, cfg, text_ids_1d: Tensor, ref: P.PreparedReference, *, max_frames: int, style_strength: float,
                         text_pos: Tensor, frame_pos: Tensor) -> dict:
    """prefill.prepare_conditioning of one text over `ref` (a VoiceBlend, or a plain voice as one segment of weight 1),
    on the CPU in float64 -> {"txt_seq", "txt_pool", "sv_ref", "cond_ar"}."""
    sd64 = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
    sv = ref.sv_ref.detach().to("cpu", torch.float64).reshape(1, -1)
    ids = text_ids_1d.to("cpu").reshape(1, -1)
    mask = torch.ones_like(ids, dtype=torch.bool)
    txt_seq, txt_pool = P.text_encoder(sd64, cfg, ids, mask, text_pos.double())
    T = int(max_frames) + 1
    cond = P.film(sd64, txt_pool[:, None, :] + frame_pos[:T].double().unsqueeze(0), sv, float(style_strength))
    caches = [{"k": c["k"].detach().cpu(), "v": c["v"].detach().cpu()} for c in ref.ref_kv_caches]
    frames, weights = segments_of(ref)
    cond = _rms_norm64(blend_xattn(sd64, cfg, cond, caches, frames, weights), sd64["cond_norm.weight"])
    return {"txt_seq": txt_seq, "txt_pool": txt_pool, "sv_ref": sv, "cond_ar": cond}
