"""Model configuration for the H100 Sopro engine.

Field names, defaults and meaning mirror the reference's ``SoproTTSConfig``
(reference: src/sopro/config.py:7-43) so that a ``cfg`` JSON blob read out of a
``model.safetensors`` header (reference: src/sopro/hub.py:38-48) populates this
dataclass unchanged.  Every kernel dimension is derived from an instance of
this class at engine-creation time; nothing is hard-coded in the CUDA code.
"""
from __future__ import annotations

import dataclasses
import json
from typing import Any, Dict, List, Tuple

TARGET_SR = 24000  # reference: src/sopro/constants.py:3


@dataclasses.dataclass
class SoproTTSConfig:
    # codec / framing
    num_codebooks: int = 32
    codebook_size: int = 2048
    mimi_fps: float = 12.5
    max_frames: int = 400
    audio_sr: int = TARGET_SR
    # trunk
    d_model: int = 384
    n_layers_text: int = 2
    dropout: float = 0.05
    pos_emb_max: int = 4096
    max_text_len: int = 2048
    # autoregressive RVQ-1 generator
    n_layers_ar: int = 6
    ar_kernel: int = 13
    ar_dilation_cycle: Tuple[int, ...] = (1, 2, 4, 1)
    ar_text_attn_freq: int = 2
    min_gen_frames: int = 12
    # non-autoregressive refiner
    n_layers_nar: int = 6
    nar_head_dim: int = 256
    nar_kernel_size: int = 11
    nar_dilation_cycle: Tuple[int, ...] = (1, 2, 4, 8)
    stage_B: Tuple[int, int] = (2, 4)
    stage_C: Tuple[int, int] = (5, 8)
    stage_D: Tuple[int, int] = (9, 16)
    stage_E: Tuple[int, int] = (17, 32)
    # speaker / reference conditioning
    sv_student_dim: int = 192
    style_strength: float = 1.0
    ref_enc_layers: int = 2
    ref_xattn_heads: int = 2
    ref_xattn_layers: int = 3
    ref_xattn_gmax: float = 0.35

    # ---- derived quantities used by the engine -------------------------
    AR_HEADS = 4  # reference: src/sopro/nn/generator.py:36 (heads=4 literal)

    def ar_dilations(self) -> Tuple[int, ...]:
        """Per-layer dilations (reference: src/sopro/nn/generator.py:16-20)."""
        cyc = [int(d) for d in self.ar_dilation_cycle]
        out: List[int] = []
        while len(out) < int(self.n_layers_ar):
            out.extend(cyc)
        return tuple(out[: int(self.n_layers_ar)])

    def nar_dilations(self) -> Tuple[int, ...]:
        cyc = [int(d) for d in self.nar_dilation_cycle] or [1]
        out: List[int] = []
        while len(out) < int(self.n_layers_nar):
            out.extend(cyc)
        return tuple(out[: int(self.n_layers_nar)])

    def ar_attn_layers(self) -> Tuple[int, ...]:
        """Block indices followed by a text cross-attention
        (reference: src/sopro/nn/generator.py:30-39)."""
        f = int(self.ar_text_attn_freq)
        return tuple(i for i in range(int(self.n_layers_ar)) if (i + 1) % f == 0)

    def ar_vocab(self) -> int:
        return int(self.codebook_size) + 1  # + EOS (reference: model.py:59,83)

    def stage_indices(self) -> Dict[str, List[int]]:
        """0-based codebook indices per NAR stage (reference: model.py:39-42,86-91)."""
        Q = int(self.num_codebooks)
        out = {}
        for name in ("B", "C", "D", "E"):
            lo, hi = getattr(self, f"stage_{name}")
            out[name] = [i for i in range(int(lo) - 1, int(hi)) if 1 <= i < Q]
        return out

    def rf_nar(self) -> int:
        """NAR receptive field (reference: model.py:125-131, sampling.py:100-101)."""
        return 1 + (int(self.nar_kernel_size) - 1) * int(sum(self.nar_dilations()))

    def rf_ar(self) -> int:
        return 1 + (int(self.ar_kernel) - 1) * int(sum(self.ar_dilations()))

    # ---- (de)serialisation ---------------------------------------------
    def to_json(self) -> str:
        return json.dumps(dataclasses.asdict(self))

    @classmethod
    def from_dict(cls, d: Dict[str, Any]) -> "SoproTTSConfig":
        """Unknown keys are dropped, as the reference does (hub.py:45-47)."""
        known = {f.name for f in dataclasses.fields(cls)}
        init = {}
        for k, v in d.items():
            if k in known:
                init[k] = tuple(v) if isinstance(v, list) else v
        return cls(**init)
