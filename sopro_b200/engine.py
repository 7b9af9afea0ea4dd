"""Python host over the C-ABI AR engine.

``ArEngine`` owns the device copy of the AR step weights; ``ArSession`` is the
state of one batch of utterances (what ``ARRVQ1Generator.init_stream_state`` +
the locals of ``SoproTTSModel.ar_stream`` hold in the reference:
nn/generator.py:44-68, model.py:242-255).  torch is used for device memory and
streams only; all compute happens in libsopro_b200.so."""
from __future__ import annotations

import ctypes as C
import dataclasses
from typing import Dict, List, Optional, Sequence, Union

import numpy as np
import torch

from . import _lib
from .config import SoproTTSConfig


@dataclasses.dataclass
class Sampling:
    """kwargs of SoproTTSModel.ar_stream (reference model.py:218-231) + the literals
    it hands to sample_token (model.py:284-291)."""
    top_p: float = 0.9
    temperature: float = 1.05
    recovery_top_p: float = 0.85
    recovery_temp: float = 1.2
    repetition_penalty: float = 1.1
    top_k: int = 50
    anti_loop: bool = True
    loop_streak: int = 8
    min_gen_frames: int = 12
    stop_on_first_eos: bool = False

    def to_c(self) -> _lib.ArSampling:
        return _lib.ArSampling(
            float(self.top_p), float(self.temperature), float(self.recovery_top_p), float(self.recovery_temp),
            float(self.repetition_penalty), int(self.top_k), int(bool(self.anti_loop)), int(self.loop_streak),
            int(min(int(self.min_gen_frames), 2 ** 31 - 1)), int(bool(self.stop_on_first_eos)))

    def noise_cols(self, vocab: int) -> int:
        """Exp(1) draws per step the kernel reads: the top_k sorted ranks with top-p (sampling.py:83-84), every
        vocabulary id on the unsorted multinomial branch taken when top_p >= 1 (sampling.py:88-93)."""
        return int(self.top_k) if (self.top_p < 1.0 and self.recovery_top_p < 1.0) else int(vocab)


@dataclasses.dataclass(frozen=True)
class Generation:
    """The generation settings of one call, resolved once from the public keywords and carried to the AR launch:
    `max_frames` (the AR runs max_frames + 1 steps), the prefill's `style_strength` and the kernel's `sampling`."""
    max_frames: int
    style_strength: float
    sampling: Sampling

    @classmethod
    def resolve(cls, cfg: SoproTTSConfig, *, max_frames, top_p, temperature, anti_loop, style_strength,
                min_gen_frames) -> "Generation":
        """The public keywords -> the settings: style_strength=None and min_gen_frames=None take the config's,
        top_p=None is no top-p (legal in the reference, sampling.py:69: `top_p is not None and top_p < 1.0`)."""
        mg = int(cfg.min_gen_frames if min_gen_frames is None else min_gen_frames)
        samp = Sampling(top_p=1.0 if top_p is None else float(top_p), temperature=float(temperature),
                        anti_loop=bool(anti_loop), min_gen_frames=min(mg, 2 ** 31 - 1))
        return cls(int(max_frames), float(cfg.style_strength if style_strength is None else style_strength), samp)


def _f32(t: torch.Tensor) -> torch.Tensor:
    return t.detach().to(device="cpu", dtype=torch.float32).contiguous()


class ArEngine:
    def __init__(self, cfg: SoproTTSConfig, state_dict: Dict[str, torch.Tensor], device: Union[int, str, torch.device] = 0,
                 weight_dtype: str = "fp32"):
        self.lib = _lib.load()
        self.cfg = cfg
        dev = torch.device(device if not isinstance(device, int) else f"cuda:{device}")
        if dev.type != "cuda":
            raise _lib.SoproError("ArEngine needs a CUDA device; there is no CPU path")
        self.device = torch.device("cuda", dev.index if dev.index is not None else 0)
        if weight_dtype not in ("fp32", "bf16"):
            raise ValueError("weight_dtype must be 'fp32' or 'bf16'")
        self.weight_dtype = weight_dtype
        n = int(cfg.n_layers_ar)
        if n > _lib.MAX_AR_LAYERS:
            raise ValueError(f"n_layers_ar={n} > {_lib.MAX_AR_LAYERS}")
        c = _lib.ArConfig()
        c.d_model, c.n_layers, c.kernel, c.n_heads = int(cfg.d_model), n, int(cfg.ar_kernel), int(cfg.AR_HEADS)
        c.vocab, c.eos_id = cfg.ar_vocab(), int(cfg.codebook_size)
        attn = set(cfg.ar_attn_layers())
        for i, d in enumerate(cfg.ar_dilations()):
            c.dilation[i] = int(d)
            c.has_attn[i] = 1 if i in attn else 0
        c.weight_dtype = 0 if weight_dtype == "fp32" else 1
        keep: List[torch.Tensor] = []

        def ptr(name: str):
            t = _f32(state_dict[name])
            keep.append(t)
            return C.cast(t.data_ptr(), C.POINTER(C.c_float))

        w = _lib.ArWeights()
        for i in range(n):
            p, L = f"ar.blocks.{i}.", w.layer[i]
            L.norm_w, L.glu_w, L.glu_b = ptr(p + "norm.weight"), ptr(p + "glu.pro.weight"), ptr(p + "glu.pro.bias")
            L.dw_w, L.dw_b = ptr(p + "dw.dw.weight"), ptr(p + "dw.dw.bias")
            L.ffn_norm_w = ptr(p + "ff.0.weight")
            L.ffn_w1, L.ffn_b1 = ptr(p + "ff.1.weight"), ptr(p + "ff.1.bias")
            L.ffn_w2, L.ffn_b2 = ptr(p + "ff.3.weight"), ptr(p + "ff.3.bias")
            if i in attn:
                q = f"ar.x_attns.{i}."
                L.nq_w, L.nkv_w = ptr(q + "nq.weight"), ptr(q + "nkv.weight")
                L.q_w, L.k_w = ptr(q + "q_proj.weight"), ptr(q + "k_proj.weight")
                L.v_w, L.o_w = ptr(q + "v_proj.weight"), ptr(q + "out_proj.weight")
                # tanh in fp32 on the host, like torch.tanh(self.gate) (reference nn/text.py:131)
                L.gate_tanh = float(torch.tanh(_f32(state_dict[q + "gate"])))
        w.final_norm_w, w.head_w, w.head_b = ptr("ar.norm.weight"), ptr("ar.head.weight"), ptr("ar.head.bias")
        emb = _f32(state_dict["cb_embed.emb.weight"])
        keep.append(emb)
        w.cb_embed = C.cast(emb.data_ptr(), C.POINTER(C.c_float))
        w.cb_embed_rows = int(emb.shape[0])
        w.bos_row = int(cfg.num_codebooks) * int(cfg.codebook_size)
        h = C.c_void_p()
        _lib.check(self.lib.sopro_engine_create(C.byref(c), C.byref(w), self.device.index, C.byref(h)))
        self._h = h
        del keep

    @property
    def step_weight_bytes(self) -> int:
        return int(self.lib.sopro_engine_step_weight_bytes(self._h))

    @property
    def num_sms(self) -> int:
        return int(self.lib.sopro_engine_num_sms(self._h))

    def session(self, max_batch: int, max_steps: int, max_text_len: int) -> "ArSession":
        return ArSession(self, max_batch, max_steps, max_text_len)

    def close(self) -> None:
        if getattr(self, "_h", None):
            self.lib.sopro_engine_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class ArSession:
    def __init__(self, engine: ArEngine, max_batch: int, max_steps: int, max_text_len: int):
        self.engine, self.lib = engine, engine.lib
        self.max_batch, self.max_steps, self.max_text_len = int(max_batch), int(max_steps), int(max_text_len)
        h = C.c_void_p()
        _lib.check(self.lib.sopro_ar_session_create(engine._h, self.max_batch, self.max_steps, self.max_text_len, C.byref(h)))
        self._h = h
        self._keep: List[torch.Tensor] = []
        self.batch = 0
        self.steps = 0

    def set_team(self, utts_per_team: int) -> None:
        _lib.check(self.lib.sopro_ar_session_set_team(self._h, int(utts_per_team)))

    def _dev(self, t: torch.Tensor) -> torch.Tensor:
        t = t.to(device=self.engine.device, dtype=torch.float32).contiguous()
        self._keep.append(t)
        return t

    def begin(self, cond_ar: torch.Tensor, txt_seq: torch.Tensor, text_len: Sequence[int], noise: torch.Tensor,
              sampling: Union[Sampling, Sequence[Sampling]]) -> None:
        """cond_ar [B,steps,D], txt_seq [B,Ls,D], noise [B,steps,k] (device or host tensors)."""
        self._keep = []
        cond_ar, txt_seq, noise = self._dev(cond_ar), self._dev(txt_seq), self._dev(noise)
        B, steps, _D = cond_ar.shape
        samp = [sampling] * B if isinstance(sampling, Sampling) else list(sampling)
        arr = (_lib.ArSampling * B)(*[s.to_c() for s in samp])
        lens = (C.c_int32 * B)(*[int(x) for x in text_len])
        _lib.check(self.lib.sopro_ar_begin(
            self._h, B, steps, cond_ar.data_ptr(), txt_seq.data_ptr(), int(txt_seq.shape[1]), lens,
            noise.data_ptr(), int(noise.shape[2]), arr, _lib.stream_ptr(self.engine.device)))
        self.batch, self.steps = int(B), int(steps)

    def run(self, n_steps: Optional[int] = None) -> None:
        _lib.check(self.lib.sopro_ar_run(self._h, int(n_steps if n_steps is not None else self.steps),
                                         _lib.stream_ptr(self.engine.device)))

    def read(self):
        toks = np.zeros((self.batch, self.steps), dtype=np.int32)
        n = np.zeros((self.batch,), dtype=np.int32)
        done = np.zeros((self.batch,), dtype=np.int32)
        _lib.check(self.lib.sopro_ar_read(self._h, toks.ctypes.data, n.ctypes.data, done.ctypes.data,
                                          _lib.stream_ptr(self.engine.device)))
        return toks, n, done

    @property
    def position(self) -> int:
        return int(self.lib.sopro_ar_position(self._h))

    def generate_host(self, cond_ar: np.ndarray, txt_seq: np.ndarray, text_len: Sequence[int], noise: np.ndarray,
                      sampling: Union[Sampling, Sequence[Sampling]]):
        """Host-buffer path: numpy (or pinned torch CPU) in, numpy out; copies are inside the call."""
        def hp(a):
            if isinstance(a, torch.Tensor):
                assert a.device.type == "cpu" and a.dtype == torch.float32 and a.is_contiguous()
                return a.data_ptr(), tuple(a.shape)
            assert a.dtype == np.float32 and a.flags["C_CONTIGUOUS"]
            return a.ctypes.data, a.shape
        pc, sc = hp(cond_ar)
        pt, stx = hp(txt_seq)
        pn, sn = hp(noise)
        B, steps = int(sc[0]), int(sc[1])
        samp = [sampling] * B if isinstance(sampling, Sampling) else list(sampling)
        arr = (_lib.ArSampling * B)(*[s.to_c() for s in samp])
        lens = (C.c_int32 * B)(*[int(x) for x in text_len])
        toks = np.zeros((B, steps), dtype=np.int32)
        n = np.zeros((B,), dtype=np.int32)
        _lib.check(self.lib.sopro_ar_generate_host(
            self._h, B, steps, pc, pt, int(stx[1]), lens, pn, int(sn[2]), arr, toks.ctypes.data, n.ctypes.data,
            _lib.stream_ptr(self.engine.device)))
        self.batch, self.steps = B, steps
        return toks, n

    # ---- test hooks
    def set_forced(self, forced: Optional[torch.Tensor]) -> None:
        if forced is None:
            _lib.check(self.lib.sopro_ar_set_forced_tokens(self._h, None))
            return
        f = forced.to(device=self.engine.device, dtype=torch.int32).contiguous()
        self._forced = f
        _lib.check(self.lib.sopro_ar_set_forced_tokens(self._h, f.data_ptr()))

    def set_trace(self, blocks: Optional[torch.Tensor], logits: Optional[torch.Tensor]) -> None:
        self._trace = (blocks, logits)
        _lib.check(self.lib.sopro_ar_set_trace(self._h, blocks.data_ptr() if blocks is not None else None,
                                               logits.data_ptr() if logits is not None else None))

    def set_attn_trace(self, probs: Optional[torch.Tensor], ring: Optional[int] = None) -> None:
        """Word timestamps: later launches store their text cross-attention weights into `probs`, a device f32 tensor
        [steps, n_attn, batch, H, ld] (ld >= the batch's longest text); None turns the export off.  `ring` (streams):
        `probs` holds `ring` step rows [ring, n_attn, batch, H, ld], step t in row t % ring, and a launch of more than
        `ring` steps is refused."""
        if probs is None:
            self._attn_trace = None
            _lib.check(self.lib.sopro_ar_set_attn_trace(self._h, None, 0))
            return
        assert probs.dtype == torch.float32 and probs.is_contiguous() and probs.device == self.engine.device and probs.dim() == 5
        self._attn_trace = probs
        if ring is None:
            _lib.check(self.lib.sopro_ar_set_attn_trace(self._h, probs.data_ptr(), int(probs.shape[-1])))
        else:
            assert int(probs.shape[0]) >= int(ring)
            _lib.check(self.lib.sopro_ar_set_attn_trace_ring(self._h, probs.data_ptr(), int(probs.shape[-1]), int(ring)))

    def set_timing(self, buf: Optional[torch.Tensor], step: int = -1) -> None:
        self._timing = buf
        _lib.check(self.lib.sopro_ar_set_timing(self._h, buf.data_ptr() if buf is not None else None, int(step)))

    STAGE_KINDS = ("glu", "ffn1", "ffn2", "q", "o", "head", "att", "sample", "qatt")

    def set_task_shape(self, mode: int) -> None:
        """GEMV warp task shape of later launches: 0 = picked per stage (default), 1 = always wide, 2 = narrow wherever
        the kernel has it (every GEMV stage but GLU, teams of at least two utterances)."""
        _lib.check(self.lib.sopro_ar_session_set_task_shape(self._h, int(mode)))

    def stage_shapes(self):
        """[(kind, "wide" | "narrow")] of every stage of the last launch, in program order."""
        kinds, shapes, n = (C.c_int32 * 128)(), (C.c_int32 * 128)(), C.c_int32()
        _lib.check(self.lib.sopro_ar_session_stage_shapes(self._h, kinds, shapes, 128, C.byref(n)))
        return [(self.STAGE_KINDS[kinds[i]], ("wide", "narrow")[shapes[i]]) for i in range(n.value)]

    def sampled(self) -> torch.Tensor:
        out = torch.empty((self.batch, self.steps), dtype=torch.int32, device=self.engine.device)
        _lib.check(self.lib.sopro_ar_debug_sampled(self._h, out.data_ptr(), _lib.stream_ptr(self.engine.device)))
        return out

    def kv(self):
        cfg = self.engine.cfg
        n_attn = len(cfg.ar_attn_layers())
        Lp = (self.max_text_len + 3) // 4 * 4
        shape = (n_attn, self.batch, cfg.AR_HEADS, Lp, int(cfg.d_model) // cfg.AR_HEADS)
        ko = torch.empty(shape, dtype=torch.float32, device=self.engine.device)
        vo = torch.empty(shape, dtype=torch.float32, device=self.engine.device)
        _lib.check(self.lib.sopro_ar_debug_kv(self._h, ko.data_ptr(), vo.data_ptr(), _lib.stream_ptr(self.engine.device)))
        return ko, vo

    def close(self) -> None:
        if getattr(self, "_h", None):
            self.lib.sopro_ar_session_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
