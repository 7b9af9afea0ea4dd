"""Host side of the CUDA NAR refiner (libsopro_b200.so: sopro_nar_*; reference model.py:307-347, nn/nar.py)."""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import torch

from . import _lib
from .config import SoproTTSConfig


def _f32(t: torch.Tensor) -> torch.Tensor:
    return t.detach().to(device="cpu", dtype=torch.float32).contiguous()


def fill_ssm_block(dst, sd: Dict[str, torch.Tensor], prefix: str, keep: list) -> None:
    """SSMLiteBlock tensors (nn/blocks.py:113-133) of `prefix` into a _lib.SsmBlockWeights."""
    names = (("norm_w", "norm.weight"), ("glu_w", "glu.pro.weight"), ("glu_b", "glu.pro.bias"), ("dw_w", "dw.dw.weight"),
             ("dw_b", "dw.dw.bias"), ("ffn_norm_w", "ff.0.weight"), ("ffn_w1", "ff.1.weight"), ("ffn_b1", "ff.1.bias"),
             ("ffn_w2", "ff.3.weight"), ("ffn_b2", "ff.3.bias"))
    for field, key in names:
        t = _f32(sd[prefix + key])
        keep.append(t)
        setattr(dst, field, C.cast(t.data_ptr(), C.POINTER(C.c_float)))


class NarEngine:
    """Device-resident NAR refiner.  ``refine(cond [B,T,D], rvq1 [B,T]) -> codes [B,T,Q]`` (int64, like the reference)."""

    def __init__(self, cfg: SoproTTSConfig, state_dict: Dict[str, torch.Tensor], device):
        self.lib = _lib.load()
        dev = torch.device(device if not isinstance(device, int) else f"cuda:{device}")
        if dev.type != "cuda":
            raise _lib.SoproError("NarEngine needs a CUDA device; there is no CPU path")
        self.device = torch.device("cuda", dev.index if dev.index is not None else 0)
        self.cfg = cfg
        sd = state_dict
        stages = [(n, idx) for n, idx in cfg.stage_indices().items() if len(idx) > 0]
        c = _lib.NarConfig()
        c.d_model, c.n_layers, c.kernel = int(cfg.d_model), int(cfg.n_layers_nar), int(cfg.nar_kernel_size)
        for i, d in enumerate(cfg.nar_dilations()):
            c.dilation[i] = int(d)
        c.n_codebooks, c.codebook_size, c.head_dim = int(cfg.num_codebooks), int(cfg.codebook_size), int(cfg.nar_head_dim)
        c.adapter_hidden = int(sd["nar.adapter.mlp.0.weight"].shape[0])
        c.n_stages = len(stages)
        keep: list = []

        def ptr(name: str):
            t = _f32(sd[name])
            keep.append(t)
            return C.cast(t.data_ptr(), C.POINTER(C.c_float))

        w = _lib.NarWeights()
        for i in range(c.n_layers):
            fill_ssm_block(w.block[i], sd, f"nar.blocks.{i}.", keep)
        w.norm_w, w.pre_w, w.pre_b = ptr("nar.norm.weight"), ptr("nar.pre.weight"), ptr("nar.pre.bias")
        w.stage_emb, w.adapter_norm_w = ptr("nar.stage_emb.weight"), ptr("nar.adapter.norm.weight")
        w.adapter_w0, w.adapter_b0 = ptr("nar.adapter.mlp.0.weight"), ptr("nar.adapter.mlp.0.bias")
        w.adapter_w2, w.adapter_b2 = ptr("nar.adapter.mlp.2.weight"), ptr("nar.adapter.mlp.2.bias")
        for s, (name, idx) in enumerate(stages):
            c.stage_first[s], c.stage_count[s] = int(idx[0]), len(idx)
            if list(idx) != list(range(idx[0], idx[0] + len(idx))):
                raise ValueError(f"NAR stage {name}: codebooks must be consecutive, got {idx}")
            for j, cb in enumerate(idx):
                w.head_w[cb], w.head_b[cb] = ptr(f"nar.heads.{name}.{j}.weight"), ptr(f"nar.heads.{name}.{j}.bias")
            w.head_id_emb[s], w.mix[s] = ptr(f"nar.head_id_emb.{name}.weight"), ptr(f"nar.mix.{name}")
        w.prev_cb_weights, w.cb_embed = ptr("nar_prev_cb_weights"), ptr("cb_embed.emb.weight")
        h = C.c_void_p()
        _lib.check(self.lib.sopro_nar_create(C.byref(c), C.byref(w), self.device.index, C.byref(h)))
        self._h = h
        self.Q = int(cfg.num_codebooks)
        del keep

    def refine(self, cond_btd: torch.Tensor, rvq1_bt: torch.Tensor, lens: Optional[torch.Tensor] = None) -> torch.Tensor:
        """cond [B, T, D] f32 (any strides along batch; rows contiguous), rvq1 [B, T] ints, lens [B] or None."""
        B, T, D = cond_btd.shape
        if lens is not None and lens.device.type == "cpu" and bool((lens == T).all()):
            # the kernels mask only the positions at or past a row's length, so lengths of T change nothing; without
            # them a one-row window replays its CUDA graph
            lens = None
        out = torch.empty((B, T, self.Q), dtype=torch.int32, device=self.device)
        if B == 0 or T == 0:
            return out.long()
        cond = cond_btd.to(device=self.device, dtype=torch.float32)
        if cond.stride(2) != 1 or cond.stride(1) != D:
            cond = cond.contiguous()
        bs = int(cond.stride(0)) if B > 1 else T * D
        if bs < T * D:
            cond = cond.contiguous()
            bs = T * D
        rvq1 = rvq1_bt.to(device=self.device, dtype=torch.int32).contiguous()
        ln = lens.to(device=self.device, dtype=torch.int32).contiguous() if lens is not None else None
        _lib.check(self.lib.sopro_nar_refine(self._h, cond.data_ptr(), bs, rvq1.data_ptr(), ln.data_ptr() if ln is not None else None,
                                             int(B), int(T), out.data_ptr(), int(torch.cuda.current_stream(self.device).cuda_stream)))
        return out.long()

    def set_contraction(self, mode: int) -> None:
        """-1 automatic (tensor cores with the exact six-product bf16 split above 16 rows), 0 fp32 FMA kernels only."""
        _lib.check(self.lib.sopro_nar_set_contraction(self._h, int(mode)))

    def set_graphs(self, enabled: bool) -> None:
        """CUDA-graph replay of single-utterance windows of <= 256 frames (default on; identical results)."""
        _lib.check(self.lib.sopro_nar_set_graphs(self._h, 1 if enabled else 0))

    def set_forced(self, forced_btq: Optional[torch.Tensor]) -> None:
        """Test hook: every stage conditions on these codes' previous codebooks (teacher forcing)."""
        self._forced = None if forced_btq is None else forced_btq.to(device=self.device, dtype=torch.int32).contiguous()
        _lib.check(self.lib.sopro_nar_set_forced(self._h, self._forced.data_ptr() if self._forced is not None else None))

    def set_trace(self, z: Optional[torch.Tensor]) -> None:
        """Test hook: every stage's pre-head activation z goes to z [n_stages, B, T, head_dim] f32 on the engine's device."""
        if z is not None and (z.device != self.device or z.dtype != torch.float32 or not z.is_contiguous()):
            raise ValueError("trace buffer must be a contiguous float32 tensor on the engine's device")
        self._trace = z
        _lib.check(self.lib.sopro_nar_set_trace(self._h, z.data_ptr() if z is not None else None))

    def close(self) -> None:
        if getattr(self, "_h", None):
            self.lib.sopro_nar_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
