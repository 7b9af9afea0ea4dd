"""Mimi codec boundary: the reference's ``MimiCodec`` / ``MimiStreamDecoder`` / ``MimiDecodeState``
(reference codec/mimi.py:18-181) over the CUDA decode engine in libsopro_b200.so.

DECODE (``decode_full`` / ``decode_step``) and ENCODE (``encode_file`` / ``encode_wav``: once per reference voice,
SURVEY.md §8f-4) both run entirely in our kernels; ``transformers`` is only the place the checkpoint's state_dict is
read from when none is passed in."""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from .config import TARGET_SR

UPSAMPLING_RATIOS = (8, 6, 5, 4)


def _f32(t: torch.Tensor) -> torch.Tensor:
    return t.detach().to(device="cpu", dtype=torch.float32).contiguous()


def _mimi_config(num_quantizers: int) -> "_lib.MimiConfigC":
    c = _lib.MimiConfigC()
    c.hidden, c.codebook_dim, c.n_q, c.n_sem, c.vocab = 512, 256, int(num_quantizers), 1, 2048
    c.n_layers, c.n_heads, c.ffn, c.window = 8, 8, 2048, 250
    c.num_filters, c.kernel, c.last_kernel, c.res_kernel, c.compress = 64, 7, 3, 3, 2
    c.n_ratios = len(UPSAMPLING_RATIOS)
    for i, r in enumerate(UPSAMPLING_RATIOS):
        c.ratios[i] = r
    c.norm_eps, c.rope_theta = 1e-5, 10000.0
    return c


def _codebooks(sd: Dict[str, torch.Tensor], num_quantizers: int) -> torch.Tensor:
    """embed = embed_sum / clamp(cluster_usage, eps)  (modeling_mimi.py:1192-1196); semantic first -> [Q, 2048, 256]"""
    embs = []
    for grp, n in (("semantic", 1), ("acoustic", int(num_quantizers) - 1)):
        for i in range(n):
            p = f"quantizer.{grp}_residual_vector_quantizer.layers.{i}.codebook."
            embs.append(_f32(sd[p + "embed_sum"]) / _f32(sd[p + "cluster_usage"]).clamp(min=1e-5)[:, None])
    return torch.stack(embs)


ENCODER_KEYS = ("encoder.layers.0.conv.weight", "encoder_transformer.layers.0.self_attn.q_proj.weight", "downsample.conv.weight",
                "quantizer.semantic_residual_vector_quantizer.input_proj.weight")


class MimiEncoderEngine:
    """Device-resident Mimi ENCODER (waveform -> codes), ``MimiModel.encode`` as ``MimiCodec.encode_file`` calls it
    (reference codec/mimi.py:41-63).  fp32, batch 1."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device, num_quantizers: int = 32):
        self.lib = _lib.load()
        dev = torch.device(device if not isinstance(device, int) else f"cuda:{device}")
        if dev.type != "cuda":
            raise _lib.SoproError("MimiEncoderEngine needs a CUDA device; there is no CPU path")
        self.device = torch.device("cuda", dev.index if dev.index is not None else 0)
        sd = state_dict
        missing = [k for k in ENCODER_KEYS if k not in sd]
        if missing:
            raise KeyError(f"state_dict has no Mimi encoder weights (e.g. {missing[0]})")
        self.num_quantizers = int(num_quantizers)
        c = _mimi_config(self.num_quantizers)
        keep = []

        def ptr(t: torch.Tensor):
            t = _f32(t)
            keep.append(t)
            return C.cast(t.data_ptr(), C.POINTER(C.c_float))

        w = _lib.MimiEncoderWeights()
        w.conv0_w, w.conv0_b = ptr(sd["encoder.layers.0.conv.weight"]), ptr(sd["encoder.layers.0.conv.bias"])
        li = 1
        for s in range(len(UPSAMPLING_RATIOS)):
            S, p = w.stage[s], f"encoder.layers.{li}.block."
            S.res1_w, S.res1_b = ptr(sd[p + "1.conv.weight"]), ptr(sd[p + "1.conv.bias"])
            S.res2_w, S.res2_b = ptr(sd[p + "3.conv.weight"]), ptr(sd[p + "3.conv.bias"])
            S.down_w, S.down_b = ptr(sd[f"encoder.layers.{li + 2}.conv.weight"]), ptr(sd[f"encoder.layers.{li + 2}.conv.bias"])
            li += 3
        w.last_w, w.last_b = ptr(sd[f"encoder.layers.{li + 1}.conv.weight"]), ptr(sd[f"encoder.layers.{li + 1}.conv.bias"])
        for l in range(8):
            p, L = f"encoder_transformer.layers.{l}.", w.layer[l]
            L.ln1_w, L.ln1_b = ptr(sd[p + "input_layernorm.weight"]), ptr(sd[p + "input_layernorm.bias"])
            L.q_w, L.k_w = ptr(sd[p + "self_attn.q_proj.weight"]), ptr(sd[p + "self_attn.k_proj.weight"])
            L.v_w, L.o_w = ptr(sd[p + "self_attn.v_proj.weight"]), ptr(sd[p + "self_attn.o_proj.weight"])
            L.ls1 = ptr(sd[p + "self_attn_layer_scale.scale"])
            L.ln2_w, L.ln2_b = ptr(sd[p + "post_attention_layernorm.weight"]), ptr(sd[p + "post_attention_layernorm.bias"])
            L.fc1_w, L.fc2_w = ptr(sd[p + "mlp.fc1.weight"]), ptr(sd[p + "mlp.fc2.weight"])
            L.ls2 = ptr(sd[p + "mlp_layer_scale.scale"])
        w.downsample_w = ptr(sd["downsample.conv.weight"])
        w.sem_in_proj = ptr(sd["quantizer.semantic_residual_vector_quantizer.input_proj.weight"].squeeze(-1))
        w.ac_in_proj = ptr(sd["quantizer.acoustic_residual_vector_quantizer.input_proj.weight"].squeeze(-1))
        w.embed = ptr(_codebooks(sd, self.num_quantizers))
        h = C.c_void_p()
        _lib.check(self.lib.sopro_mimi_encoder_create(C.byref(c), C.byref(w), self.device.index, C.byref(h)))
        self._h = h
        del keep

    def frames(self, n_samples: int) -> int:
        """MimiModel.get_encoded_length: every strided conv rounds up."""
        t = int(self.lib.sopro_mimi_encoded_frames(self._h, int(n_samples)))
        if t < 0:
            raise ValueError(f"cannot encode {n_samples} samples")
        return t

    def encode(self, wav: torch.Tensor, *, return_latent: bool = False):
        """wav [n] / [1, n] / [1, 1, n] f32 @24 kHz (any device) -> codes [Q, T] int64 on the engine's device
        (and, on request, the pre-quantizer embeddings [T, 512])."""
        wav = wav.reshape(-1).to(device=self.device, dtype=torch.float32).contiguous()
        n = int(wav.numel())
        T = self.frames(n)
        codes = torch.empty((self.num_quantizers, T), dtype=torch.int32, device=self.device)
        lat = torch.empty((T, 512), dtype=torch.float32, device=self.device) if return_latent else None
        _lib.check(self.lib.sopro_mimi_encode(self._h, wav.data_ptr(), n, codes.data_ptr(), lat.data_ptr() if lat is not None else None,
                                              int(torch.cuda.current_stream(self.device).cuda_stream)))
        codes = codes.to(torch.long)
        return (codes, lat) if return_latent else codes

    def encode_batch(self, wav_bl: torch.Tensor, lens: Sequence[int], *, return_latent: bool = False):
        """A ragged batch wav [B, L] f32 @24 kHz (row b's first lens[b] samples) -> codes: a list of [Q, T_b] int64 on
        the engine's device (and, on request, the latents [T_b, 512]).  Row b equals ``encode`` of its samples alone, bit
        for bit.  The rows run longest first in padded calls of at most ENC_MAX_SAMPLES samples each."""
        from .ingest import ENC_MAX_SAMPLES

        wav_bl = wav_bl.to(device=self.device, dtype=torch.float32)
        B, L = wav_bl.shape
        lens = [int(n) for n in lens]
        if len(lens) != B:
            raise ValueError(f"lens has {len(lens)} entries for {B} rows")
        if any(n < 1 or n > L for n in lens):
            raise ValueError(f"every length must be in [1, {L}]")
        Ts = [self.frames(n) for n in lens]
        unit = 2 * math.prod(UPSAMPLING_RATIOS)
        codes: List[Optional[torch.Tensor]] = [None] * B
        lats: List[Optional[torch.Tensor]] = [None] * B
        live = sorted(range(B), key=lambda i: -lens[i])
        st = int(torch.cuda.current_stream(self.device).cuda_stream)
        while live:
            pad = -(-lens[live[0]] // unit) * unit
            k = max(1, min(len(live), ENC_MAX_SAMPLES // pad))
            idx, live = live[:k], live[k:]
            if idx == list(range(idx[0], idx[0] + k)):
                x = wav_bl[idx[0]: idx[0] + k]
            else:
                x = wav_bl[torch.tensor(idx, device=self.device)]
            if x.stride(-1) != 1:
                x = x.contiguous()
            Tm = Ts[idx[0]]
            c = torch.empty((k, self.num_quantizers, Tm), dtype=torch.int32, device=self.device)
            lat = torch.empty((k, Tm, 512), dtype=torch.float32, device=self.device) if return_latent else None
            _lib.check_arg(self.lib.sopro_mimi_encode_batch(self._h, x.data_ptr(), k, int(x.stride(0)),
                                                            (C.c_int64 * k)(*[lens[i] for i in idx]), c.data_ptr(),
                                                            lat.data_ptr() if lat is not None else None, st))
            for j, i in enumerate(idx):
                codes[i] = c[j, :, : Ts[i]].to(torch.long)
                if lat is not None:
                    lats[i] = lat[j, : Ts[i]]
        return (codes, lats) if return_latent else codes

    def encode_host(self, wav: np.ndarray) -> np.ndarray:
        wav = np.ascontiguousarray(wav, dtype=np.float32).reshape(-1)
        T = self.frames(wav.size)
        codes = np.empty((self.num_quantizers, T), dtype=np.int32)
        _lib.check_arg(self.lib.sopro_mimi_encode_host(self._h, wav.ctypes.data, int(wav.size), codes.ctypes.data, None,
                                                       int(torch.cuda.current_stream(self.device).cuda_stream)))
        return codes

    def close(self):
        if getattr(self, "_h", None):
            self.lib.sopro_mimi_encoder_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class MimiEngine:
    """Device-resident Mimi decoder built from a ``MimiModel`` state_dict (decode-path tensors only)."""

    PRECISIONS = {"fp32": 0, "bf16_tc": 1}

    def __init__(self, state_dict: Dict[str, torch.Tensor], device, num_quantizers: int = 32, precision: str = "bf16_tc"):
        self.lib = _lib.load()
        dev = torch.device(device if not isinstance(device, int) else f"cuda:{device}")
        if dev.type != "cuda":
            raise _lib.SoproError("MimiEngine needs a CUDA device; there is no CPU path")
        self.device = torch.device("cuda", dev.index if dev.index is not None else 0)
        sd = state_dict
        c = _mimi_config(num_quantizers)
        self.num_quantizers = int(num_quantizers)
        keep = []

        def ptr(t: torch.Tensor):
            t = _f32(t)
            keep.append(t)
            return C.cast(t.data_ptr(), C.POINTER(C.c_float))

        w = _lib.MimiWeights()
        w.embed = ptr(_codebooks(sd, self.num_quantizers))
        w.sem_out_proj = ptr(sd["quantizer.semantic_residual_vector_quantizer.output_proj.weight"].squeeze(-1))
        w.ac_out_proj = ptr(sd["quantizer.acoustic_residual_vector_quantizer.output_proj.weight"].squeeze(-1))
        w.upsample_w = ptr(sd["upsample.conv.weight"])
        for l in range(8):
            p, L = f"decoder_transformer.layers.{l}.", w.layer[l]
            L.ln1_w, L.ln1_b = ptr(sd[p + "input_layernorm.weight"]), ptr(sd[p + "input_layernorm.bias"])
            L.q_w, L.k_w = ptr(sd[p + "self_attn.q_proj.weight"]), ptr(sd[p + "self_attn.k_proj.weight"])
            L.v_w, L.o_w = ptr(sd[p + "self_attn.v_proj.weight"]), ptr(sd[p + "self_attn.o_proj.weight"])
            L.ls1 = ptr(sd[p + "self_attn_layer_scale.scale"])
            L.ln2_w, L.ln2_b = ptr(sd[p + "post_attention_layernorm.weight"]), ptr(sd[p + "post_attention_layernorm.bias"])
            L.fc1_w, L.fc2_w = ptr(sd[p + "mlp.fc1.weight"]), ptr(sd[p + "mlp.fc2.weight"])
            L.ls2 = ptr(sd[p + "mlp_layer_scale.scale"])
        w.conv0_w, w.conv0_b = ptr(sd["decoder.layers.0.conv.weight"]), ptr(sd["decoder.layers.0.conv.bias"])
        li = 1
        for s in range(len(UPSAMPLING_RATIOS)):
            S = w.stage[s]
            S.convt_w, S.convt_b = ptr(sd[f"decoder.layers.{li + 1}.conv.weight"]), ptr(sd[f"decoder.layers.{li + 1}.conv.bias"])
            p = f"decoder.layers.{li + 2}.block."
            S.res1_w, S.res1_b = ptr(sd[p + "1.conv.weight"]), ptr(sd[p + "1.conv.bias"])
            S.res2_w, S.res2_b = ptr(sd[p + "3.conv.weight"]), ptr(sd[p + "3.conv.bias"])
            li += 3
        w.last_w, w.last_b = ptr(sd[f"decoder.layers.{li + 1}.conv.weight"]), ptr(sd[f"decoder.layers.{li + 1}.conv.bias"])
        h = C.c_void_p()
        _lib.check(self.lib.sopro_mimi_create(C.byref(c), C.byref(w), self.device.index, C.byref(h)))
        self._h = h
        self.hop = int(self.lib.sopro_mimi_samples_per_frame(h))
        del keep
        self.set_precision(precision)

    def set_precision(self, precision: str) -> None:
        """"bf16_tc": dense blocks on the tensor cores (wgmma) (bf16 operands, fp32 accumulate); "fp32": exact mode."""
        if precision not in self.PRECISIONS:
            raise ValueError(f"precision must be one of {sorted(self.PRECISIONS)}")
        _lib.check(self.lib.sopro_mimi_set_precision(self._h, self.PRECISIONS[precision]))
        self.precision = precision

    def set_graphs(self, enabled: bool) -> None:
        """CUDA-graph replay of small (<= 64 frame) decodes inside the library; on by default."""
        _lib.check(self.lib.sopro_mimi_set_graphs(self._h, 1 if enabled else 0))

    def _validated(self, codes: torch.Tensor, trusted: bool = False) -> torch.Tensor:
        """int32 codes on the device; like the reference's embedding lookup, a code outside [0, 2048) is an IndexError
        (an uncut EOS id would otherwise read past the codebook; the kernel itself clamps and flags).  `trusted`: codes
        this process produced itself (the NAR refiner's argmax over 2048 logits, clamped first codebook) skip the host
        check -- it is a device synchronisation in the middle of the streaming pipeline -- and rely on the device-side
        flag (``check()``)."""
        codes = codes.to(device=self.device, dtype=torch.int32).contiguous()
        if codes.numel() and not trusted:
            lo, hi = torch.aminmax(codes)
            lo, hi = int(lo), int(hi)
            if lo < 0 or hi >= 2048:
                raise IndexError(f"Mimi codes must be in [0, 2048), got values in [{lo}, {hi}]")
        return codes

    def decode(self, codes_bqt: torch.Tensor) -> torch.Tensor:
        """codes [B, Q, T] (any int dtype, any device) -> wav [B, 1, T*hop] f32 on the engine's device."""
        codes = self._validated(codes_bqt)
        B, Q, T = codes.shape
        if Q != self.num_quantizers:
            raise ValueError(f"expected {self.num_quantizers} codebooks, got {Q}")
        wav = torch.empty((B, 1, T * self.hop), dtype=torch.float32, device=self.device)
        if T == 0:
            return wav
        _lib.check(self.lib.sopro_mimi_decode(self._h, codes.data_ptr(), int(B), int(T), wav.data_ptr(),
                                              int(torch.cuda.current_stream(self.device).cuda_stream)))
        return wav

    def decode_host(self, codes_bqt: np.ndarray) -> np.ndarray:
        codes = np.ascontiguousarray(codes_bqt, dtype=np.int32)
        B, Q, T = codes.shape
        wav = np.empty((B, 1, T * self.hop), dtype=np.float32)
        _lib.check(self.lib.sopro_mimi_decode_host(self._h, codes.ctypes.data, int(B), int(T), wav.ctypes.data,
                                                   int(torch.cuda.current_stream(self.device).cuda_stream)))
        return wav

    def check(self) -> None:
        """Raises if any decode since the last check met an out-of-range code (device-side sticky flag)."""
        _lib.check(self.lib.sopro_mimi_check(self._h, int(torch.cuda.current_stream(self.device).cuda_stream)))

    def stream(self, max_chunk_frames: int = 16, rows: int = 1) -> "MimiStream":
        """A decode state of `rows` utterances stepped side by side (see MimiStream)."""
        return MimiStream(self, max_chunk_frames, rows)

    def close(self):
        if getattr(self, "_h", None):
            self.lib.sopro_mimi_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class MimiStream:
    """Persistent decode state of `rows` utterances on the device (per row: K/V rings, upsampler frame, conv context
    rows): ``step(codes [Q, n])`` (one row) or ``step(codes [rows, Q, n])`` returns the next n*hop samples of every row
    in O(rows * n) work.  Row b's samples equal a one-row stream fed row b's codes, bit for bit; a row whose utterance
    has ended can be fed code 0 and its samples dropped.  See include/sopro_b200.h."""

    def __init__(self, engine: MimiEngine, max_chunk_frames: int = 16, rows: int = 1):
        self.engine, self.lib = engine, engine.lib
        h = C.c_void_p()
        _lib.check(self.lib.sopro_mimi_stream_create_rows(engine._h, int(max_chunk_frames), int(rows), C.byref(h)))
        self._h = h
        self.rows = int(rows)

    @property
    def frames(self) -> int:
        return int(self.lib.sopro_mimi_stream_frames(self._h))

    @property
    def state_bytes(self) -> int:
        """Device bytes this state holds."""
        return int(self.lib.sopro_mimi_stream_bytes(self._h))

    def reset(self) -> None:
        _lib.check(self.lib.sopro_mimi_stream_reset(self._h, int(torch.cuda.current_stream(self.engine.device).cuda_stream)))

    def step(self, codes_qn: torch.Tensor, trusted: bool = False) -> torch.Tensor:
        """codes [Q, n] (a one-row state) or [rows, Q, n] -> wav [1, n*hop] or [rows, n*hop]."""
        codes = self.engine._validated(codes_qn, trusted)
        if codes.dim() == 2:
            codes = codes.unsqueeze(0)
        if codes.dim() != 3 or int(codes.shape[0]) != self.rows:
            raise ValueError(f"a stream of {self.rows} row(s) takes codes [{self.rows}, Q, n]"
                             + (" or [Q, n]" if self.rows == 1 else "") + f", got {tuple(codes_qn.shape)}")
        _rows, Q, n = codes.shape
        if Q != self.engine.num_quantizers:
            raise ValueError(f"expected {self.engine.num_quantizers} codebooks, got {Q}")
        wav = torch.empty((self.rows, n * self.engine.hop), dtype=torch.float32, device=self.engine.device)
        if n:
            _lib.check(self.lib.sopro_mimi_decode_step(self._h, codes.data_ptr(), int(n), wav.data_ptr(),
                                                       int(torch.cuda.current_stream(self.engine.device).cuda_stream)))
        return wav

    def step_host(self, codes_qn: np.ndarray) -> np.ndarray:
        """Host buffers: codes [Q, n] or [rows, Q, n] -> wav [rows, n*hop]."""
        codes = np.ascontiguousarray(codes_qn, dtype=np.int32).reshape(self.rows, self.engine.num_quantizers, -1)
        n = codes.shape[2]
        wav = np.empty((self.rows, n * self.engine.hop), dtype=np.float32)
        _lib.check(self.lib.sopro_mimi_decode_step_host(self._h, codes.ctypes.data, int(n), wav.ctypes.data,
                                                        int(torch.cuda.current_stream(self.engine.device).cuda_stream)))
        return wav

    def close(self):
        if getattr(self, "_h", None) and getattr(self.engine, "_h", None):
            self.lib.sopro_mimi_stream_destroy(self._h)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class MimiCodec:
    """reference codec/mimi.py:18-72.  ``hf_model`` (a transformers MimiModel) is only a source of the state_dict; both
    directions run on the CUDA engines.  The encoder engine is built on first use (a voice is encoded once)."""

    def __init__(self, num_quantizers: int, device: str = "cuda", model_id: str = "kyutai/mimi", *,
                 state_dict: Optional[Dict[str, torch.Tensor]] = None, hf_model=None, precision: str = "bf16_tc"):
        self.device = torch.device(device)
        self.model = hf_model
        if state_dict is None:
            if hf_model is None:
                from transformers import MimiConfig, MimiModel  # network / local HF cache, like the reference (:28-31)

                cfg = MimiConfig.from_pretrained(model_id, num_quantizers=int(num_quantizers))
                hf_model = MimiModel.from_pretrained(model_id, config=cfg).eval()
                self.model = hf_model
            state_dict = hf_model.state_dict()
        self._num_quantizers = int(num_quantizers)
        self.engine = MimiEngine(state_dict, self.device, num_quantizers=self._num_quantizers, precision=precision)
        self._encoder: Optional[MimiEncoderEngine] = None
        self._in_resamplers: Dict[int, "Resampler"] = {}  # clip rate -> 24 kHz (prepare_wavs)
        enc = ("encoder.", "encoder_transformer.", "downsample.", "quantizer.")
        self._encoder_sd = ({k: v for k, v in state_dict.items() if k.startswith(enc)}
                            if all(k in state_dict for k in ENCODER_KEYS) else None)

    @property
    def codebook_size(self) -> int:
        return 2048

    @property
    def num_quantizers(self) -> int:
        return self._num_quantizers

    @torch.no_grad()
    def encode_file(self, wav_path: str, *, crop_seconds: Optional[float] = None) -> torch.Tensor:
        """reference codec/mimi.py:41-63 (VAD trim -> resample -> centre crop -> MimiModel.encode)."""
        from .audio import center_crop_audio, load_audio_file, resample, trim_silence_energy

        from .ingest import check_finite

        wav, sr = load_audio_file(wav_path)
        check_finite(wav, wav_path)
        wav = trim_silence_energy(wav, sr)
        wav = resample(wav, sr, TARGET_SR)
        if crop_seconds is not None and crop_seconds > 0:
            hop = int(round(TARGET_SR / 12.5))
            wav = center_crop_audio(wav, max(1, int(round(crop_seconds * 12.5))) * hop)
        return self.encode_wav(wav)

    @property
    def encoder(self) -> MimiEncoderEngine:
        if self._encoder is None:
            if self._encoder_sd is None:
                raise RuntimeError("this MimiCodec was built from a decode-only state_dict: no Mimi encoder weights to encode with")
            self._encoder = MimiEncoderEngine(self._encoder_sd, self.device, num_quantizers=self._num_quantizers)
            self._encoder_sd = None
        return self._encoder

    @torch.no_grad()
    def encode_wav(self, wav: torch.Tensor) -> torch.Tensor:
        """mono waveform @24 kHz ([n], [1, n] or [1, 1, n]) -> codes [T, Q] int64 on the device: the model call of
        ``encode_file`` (reference codec/mimi.py:59-62), on the CUDA encoder.  A non-finite sample is a ValueError,
        raised before the encoder is built or launched."""
        from .ingest import check_finite

        check_finite(wav, "the waveform")
        return self.encoder.encode(wav).permute(1, 0).contiguous()

    @torch.no_grad()
    def prepare_wavs(self, wavs: Sequence[torch.Tensor], sample_rates: Sequence[int],
                     crop_seconds: Optional[float] = None, denoise: bool = False) -> Tuple[torch.Tensor, List[int]]:
        """``encode_file``'s preparation of a ragged batch on the device: clips [n] or [C, n] (any device, channels
        averaged), each at its own rate -> (wav [B, L] f32 @24 kHz on the device, valid samples per row; zeros past them).
        Per clip: energy trim at its rate (one launch for the batch), resample to 24 kHz (one launch per distinct rate;
        a 24 kHz clip is not resampled), centre crop to `crop_seconds` as encode_file does (None or <= 0: no crop).  The
        one host read is the B trim extents.  The trim sums in fp64 where the reference's torch ops sum in fp32, so only
        a frame within rounding of the threshold can be classified differently from ``encode_file``; the resampler is
        §5d's (DESIGN.md), not torchaudio's fp32 kernel.
        `denoise` (extension): after the resample, each trimmed clip goes through ``denoising.denoise`` (DESIGN.md §5n)
        before the crop, so that the noise estimate sees the whole clip; 24 kHz clips are then packed too, since the
        denoiser writes a new buffer.  The clips are denoised in groups of at most ENC_MAX_SAMPLES padded samples."""
        from . import ingest
        from .denoising import check_denoise
        from .resample import Resampler

        check_denoise(denoise)
        wavs, sample_rates = list(wavs), list(sample_rates)
        if not wavs or len(sample_rates) != len(wavs):
            raise ValueError(f"{len(wavs)} clips with {len(sample_rates)} sample rates")
        rates = [ingest._check_wav(w, sr, i) for i, (w, sr) in enumerate(zip(wavs, sample_rates))]
        win = ingest.crop_samples(crop_seconds)
        rows = ingest.mono_rows(wavs, self.device)
        ext = ingest.trim_extents(rows, rates).tolist()  # the one host read
        B = len(rows)
        src, n24 = [0] * B, [0] * B
        keep = []  # resampled rows, alive until the last pack has been enqueued
        by_rate: Dict[int, List[int]] = {}
        for b, (s, e) in enumerate(ext):
            if rates[b] == TARGET_SR and not denoise:
                src[b], n24[b] = rows[b].data_ptr() + 4 * s, e - s
            else:
                by_rate.setdefault(rates[b], []).append(b)
        for sr, idx in by_rate.items():
            lens = [ext[b][1] - ext[b][0] for b in idx]
            x = ingest.pack([rows[b].data_ptr() + 4 * ext[b][0] for b in idx], lens,
                            torch.empty((len(idx), max(lens)), dtype=torch.float32, device=self.device))
            if sr == TARGET_SR:
                y, n = x, lens
            else:
                rs = self._in_resamplers.get(sr)
                if rs is None:
                    rs = self._in_resamplers[sr] = Resampler(sr, TARGET_SR, self.device)
                y, n = rs(x, lens), [rs.length(v) for v in lens]
            if denoise:
                y = self._denoise_rows(y, n)
            keep.append(y)
            for j, b in enumerate(idx):
                src[b], n24[b] = y[j].data_ptr(), n[j]
        plan = [ingest.crop_plan(n, win) for n in n24]
        out = torch.empty((B, max(n for _, n in plan)), dtype=torch.float32, device=self.device)
        ingest.pack([src[b] + 4 * plan[b][0] for b in range(B)], [n for _, n in plan], out)
        return out, [n for _, n in plan]

    @staticmethod
    def _denoise_rows(y: torch.Tensor, lens: Sequence[int]) -> torch.Tensor:
        """denoising.denoise of the ragged batch y [k, L], in consecutive groups of at most ENC_MAX_SAMPLES padded
        samples (the rows' results do not depend on the grouping) -> a new [k, L]."""
        from .denoising import denoise
        from .ingest import ENC_MAX_SAMPLES

        out = torch.empty_like(y)
        per = max(1, ENC_MAX_SAMPLES // max(1, int(y.shape[1])))
        for i in range(0, int(y.shape[0]), per):
            out[i: i + per] = denoise(y[i: i + per], lens[i: i + per])
        return out

    @torch.no_grad()
    def encode_wavs(self, wav_bl: torch.Tensor, lens: Sequence[int]) -> List[torch.Tensor]:
        """A ragged batch @24 kHz (``prepare_wavs``' result) -> codes [T_b, Q] int64 per row on the device, each equal
        to ``encode_wav`` of the row's samples alone, bit for bit (batched Mimi encoder, sopro_mimi_encode_batch)."""
        return [c.permute(1, 0).contiguous() for c in self.encoder.encode_batch(wav_bl, lens)]

    @torch.no_grad()
    def decode_full(self, codes_tq: torch.Tensor) -> torch.Tensor:
        """[T, Q] -> [1, 1, T*1920] (reference codec/mimi.py:65-72)."""
        return self.engine.decode(codes_tq.permute(1, 0).unsqueeze(0))


@dataclass
class MimiDecodeState:
    """Fields of the reference's state (codec/mimi.py:75-80).  ``decoder_past_key_values`` holds the device-side
    stream (K/V rings of the transformer + the conv context rows) instead of a transformers cache object."""
    decoder_past_key_values: Optional[object] = None
    frames_seen: int = 0
    samples_emitted: int = 0
    tail_codes_tq: Optional[torch.Tensor] = None


class MimiStreamDecoder:
    """Chunked streaming decode (reference codec/mimi.py:83-181) over a persistent device state.

    The reference re-feeds the last ``overlap_frames`` frames on top of a transformers KV cache, with no conv
    context, and documents the result as "not bit-exact compared to the non-streaming version" (README.md:151); on
    transformers >= 5 its cache trimming silently does nothing (SURVEY.md §7.2) and later chunks drift by up to 0.7 of
    the waveform's peak from its own decode_full (measured: tests/golden/measure_stream_distance.py, DESIGN.md §5).
    Here the state carries everything a causal decoder needs (K/V rings, upsampler frame, the left context of every
    conv), so each chunk costs O(chunk) and the chunks concatenate to exactly the non-streaming waveform.
    ``overlap_frames`` is accepted for signature compatibility; nothing is re-decoded.

    A state can also hold several utterances stepped side by side (``new_state(rows)``, codes [rows, n, Q]; see
    MimiStream).  Released states are kept for reuse by their row count, at most MAX_IDLE_STATES of them holding at
    most MAX_IDLE_ROWS rows in all; the oldest go first."""

    MAX_IDLE_STATES = 4
    MAX_IDLE_ROWS = 256

    def __init__(self, codec: MimiCodec, max_chunk_frames: int = 16):
        self.codec = codec
        self.max_chunk_frames = int(max_chunk_frames)
        self._idle: list = []  # device streams of finished utterances, oldest first, reused after a reset

    def new_state(self, rows: int = 1) -> MimiDecodeState:
        """A fresh state of `rows` utterances; reuses the device buffers of a released one of that many rows when
        available (no allocation on the time-to-first-audio path)."""
        st = MimiDecodeState()
        for i in range(len(self._idle) - 1, -1, -1):
            if getattr(self._idle[i], "rows", 1) == int(rows):
                st.decoder_past_key_values = self._idle.pop(i)
                st.decoder_past_key_values.reset()
                break
        return st

    def release(self, state: Optional[MimiDecodeState]) -> None:
        """Hand a finished utterance's device buffers back for reuse."""
        if state is None or state.decoder_past_key_values is None:
            return
        dev, state.decoder_past_key_values = state.decoder_past_key_values, None
        self._idle.append(dev)
        while len(self._idle) > self.MAX_IDLE_STATES or sum(getattr(x, "rows", 1) for x in self._idle) > self.MAX_IDLE_ROWS:
            old = self._idle.pop(0)
            if hasattr(old, "close"):
                old.close()

    @torch.inference_mode()
    def decode_step(self, codes_chunk_tq: torch.Tensor, state: Optional[MimiDecodeState] = None, *,
                    overlap_frames: int = 2, _trusted: bool = False) -> Tuple[torch.Tensor, MimiDecodeState]:
        """codes [n, Q] of one utterance -> wav [1, n*hop]; or codes [rows, n, Q] of a state's rows -> wav [rows, n*hop]
        (the state takes its row count from the first chunk it decodes).  Codes [1, n, Q] are one utterance's: the state
        is a one-row stream, stepped with [Q, n] like any one-utterance chunk."""
        if state is None:
            state = MimiDecodeState()
        if codes_chunk_tq.dim() == 3 and codes_chunk_tq.size(0) == 1:
            codes_chunk_tq = codes_chunk_tq[0]
        rows = 1 if codes_chunk_tq.dim() == 2 else int(codes_chunk_tq.size(0))
        n_new = int(codes_chunk_tq.size(-2))
        if n_new == 0:
            return torch.zeros(rows, 0, device=self.codec.device), state
        if state.decoder_past_key_values is None:
            state.decoder_past_key_values = (self.codec.engine.stream(self.max_chunk_frames) if rows == 1 else
                                             self.codec.engine.stream(self.max_chunk_frames, rows))
        chunk = codes_chunk_tq.to(self.codec.device)
        wav_new = state.decoder_past_key_values.step(chunk.transpose(-1, -2), _trusted)
        state.frames_seen += n_new
        state.samples_emitted += int(wav_new.size(1))
        state.tail_codes_tq = chunk[..., -max(int(overlap_frames), 0):, :].detach() if overlap_frames > 0 else None
        return wav_new, state
