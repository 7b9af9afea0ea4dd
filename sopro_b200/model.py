"""Public API: ``SoproTTS`` with the reference's signatures (reference model.py:404-583) over the H100 engine.

``SoproTTS.model`` is a ``SoproModel``: it stands where the reference's ``SoproTTSModel`` stands
(model.py:53-401) and keeps its method names, but ``ar_stream`` drives the persistent CUDA kernel and the
codec decodes with the CUDA Mimi engine.  Prefill and the NAR refiner are torch ops on the same device
(sopro_b200/prefill.py).  There is no CPU path: constructing the model without a CUDA device raises.

Randomness: like the reference, sampling consumes the GLOBAL torch CPU generator (the reference has no seed
argument; its CLI calls torch.manual_seed, cli.py:72-75), one [V]-sized Exp(1) draw per generated frame, so
``torch.manual_seed(s); tts.synthesize(...)`` reproduces the reference's token ids.  Every generating method
additionally accepts ``seed=`` / ``generator=`` (an extension) to leave the global generator untouched.
"""
from __future__ import annotations

import contextlib
import dataclasses
import os
import threading
from typing import Dict, Iterator, List, Mapping, Optional, Sequence, Tuple, Union

import torch

from . import cues as CU
from . import dialogue as D
from . import ingest
from . import longform as LF
from . import prefill as P
from . import rerank
from . import ssml as SSML
from . import streaming as S
from . import timestamps as TS
from . import voices
from ._lib import StatePool
from .codec import MimiCodec, MimiStreamDecoder
from .config import TARGET_SR, SoproTTSConfig
from .denoising import check_denoise
from .engine import ArEngine, ArSession, Generation, Sampling
from .nar import NarEngine
from .prefill_cuda import PrefillEngine, RefPrepEngine
from .prefill import PreparedReference
from .output import OutputChain
from .resample import Resampler, check_rates
from .sampling import TapeFeed
from .stretch import StretchStream, stretch_rows, stretched_length
from .watermark import WatermarkStream
from .weights import load_safetensors, read_safetensors_cfg


def center_crop_tokens(ref_tq: torch.Tensor, win_frames: int) -> torch.Tensor:
    """reference sampling.py:8-13"""
    T = int(ref_tq.size(0))
    if T <= win_frames:
        return ref_tq
    s = (T - win_frames) // 2
    return ref_tq[s: s + win_frames]


def _complete_state_dict(cfg: SoproTTSConfig, sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """The reference loads with load_state_dict(strict=False) (model.py:443-446): tensors a checkpoint omits keep their
    module-init values.  The known omittable ones get those defaults here; anything else missing is ONE explicit error
    at construction instead of a KeyError deep inside the first synthesize call."""
    from .weights import param_specs

    Q = int(cfg.num_codebooks)
    tv = int(sd["text_enc.embed.emb.weight"].shape[0]) if "text_enc.embed.emb.weight" in sd else 0
    specs = param_specs(cfg, tv)
    out = dict(sd)
    missing = []
    for name, (shape, _kind, _fan) in specs.items():
        if name in out:
            continue
        if name in ("ref_cb_weights", "token2sv.cb_weights"):  # model.py:113-117, nn/speaker.py:22-23
            out[name] = torch.linspace(1.0, 0.1, Q)
        elif name == "nar_prev_cb_weights" or name.startswith("nar.head_id_emb."):  # model.py:70-72, nn/nar.py:79 (zeros)
            out[name] = torch.zeros(shape)
        else:
            missing.append(name)
    if missing:
        raise KeyError(f"checkpoint is missing {len(missing)} tensor(s) the engine needs: {missing[:12]}"
                       + (" ..." if len(missing) > 12 else ""))
    return out


def _growing_blocks(steps: int) -> List[Tuple[int, int]]:
    """Block edges of a seeded batch: the host draws block k+1 of the tapes while the device generates block k, so
    only the first, short block is exposed (and that one overlaps the prefill).  Block k+1 must be drawn faster than
    the device generates block k: the host draws ~10 steps per ms (64 utterances, 16 threads), the kernel runs ~6
    steps per ms -> blocks grow by 1.5x."""
    edges, a, step = [], 0, 24
    while a < steps:
        b = min(steps, a + step)
        if steps - b < 24:
            b = steps
        edges.append((a, b))
        a, step = b, (step * 3) // 2
    return edges


def _check_voices(cfg: SoproTTSConfig, voice_of: Sequence[PreparedReference]) -> None:
    """Every distinct voice of a segment list against the engine's geometry (TypeError for one that is not a
    PreparedReference)."""
    geom = voices.geometry(cfg)
    for r in voices.voice_slots(list(voice_of), len(voice_of))[0]:
        voices.check_voice(r, **geom)


def _check_texts(texts, seeds) -> Tuple[List[str], Optional[List[int]]]:
    """synthesize_batch's and stream_batch's `texts` and `seeds` -> (the texts, the seeds as ints or None), before any
    work: TypeError for a str or anything but a sequence, ValueError for no text or a seeds length that differs."""
    if isinstance(texts, str) or not isinstance(texts, Sequence):
        raise TypeError(f"texts must be a sequence of strings, got {type(texts).__name__}")
    texts = list(texts)
    if not texts:
        raise ValueError("texts is empty: give at least one text")
    if seeds is not None:
        seeds = [int(x) for x in seeds]
        if len(seeds) != len(texts):
            raise ValueError(f"{len(seeds)} seeds for {len(texts)} texts")
    return texts, seeds


class SoproModel:
    def __init__(self, cfg: SoproTTSConfig, state_dict: Dict[str, torch.Tensor], device, weight_dtype: str = "fp32"):
        dev = torch.device(device)
        if dev.type != "cuda":
            raise RuntimeError("sopro_b200 runs on CUDA devices only (sm_90a); there is no CPU fallback")
        self.cfg = cfg
        state_dict = _complete_state_dict(cfg, state_dict)
        self.device = torch.device("cuda", dev.index if dev.index is not None else torch.cuda.current_device())
        self.eos_id = int(cfg.codebook_size)
        self.weight_dtype = weight_dtype
        self.engine = ArEngine(cfg, state_dict, self.device, weight_dtype)
        # (every stage owns its device copy of the weights it needs inside its CUDA engine; no torch-side copy is kept)
        self.text_pos = P.sinusoid_table(int(cfg.max_text_len) + 8, int(cfg.d_model), self.device)
        self.frame_pos = P.sinusoid_table(int(cfg.pos_emb_max) + 8, int(cfg.d_model), self.device)
        # AR sessions are CHECKED OUT per generator / call and returned when it ends (ar_stream is a suspended
        # generator: two interleaved streams must never share a session's device state)
        self._sessions: Dict[Tuple[int, int, int], List[ArSession]] = {}
        self._sessions_busy: set = set()
        self._sessions_lock = threading.Lock()
        self.prefill = PrefillEngine(cfg, state_dict, self.device, self.text_pos, self.frame_pos)
        self.refprep = RefPrepEngine(cfg, state_dict, self.device)
        self.nar = NarEngine(cfg, state_dict, self.device)

    # ---- geometry helpers (reference model.py:119-131)
    def rf_ar(self) -> int:
        return self.cfg.rf_ar()

    def rf_nar(self) -> int:
        return self.cfg.rf_nar()

    def eval(self):
        return self

    @contextlib.contextmanager
    def _lease(self, batch: int, steps: int, text_len: int, attn_trace: Optional[torch.Tensor],
               attn_ring: Optional[int] = None) -> Iterator[ArSession]:
        """An idle session of this geometry (a fresh one when every cached one is in use), held for the `with` block,
        with `attn_trace` (word timestamps; a ring of `attn_ring` steps when given) set on it for that time: sessions
        are cached and shared."""
        key = (int(batch), int(steps), (int(text_len) + 63) // 64 * 64)
        with self._sessions_lock:
            ses = next((x for x in self._sessions.get(key, []) if id(x) not in self._sessions_busy), None)
            if ses is None:
                # evict idle sessions of other geometries beyond 8 cached (never one a live generator holds)
                idle = [(k, x) for k, v in self._sessions.items() for x in v if id(x) not in self._sessions_busy and k != key]
                total = sum(len(v) for v in self._sessions.values())
                while total >= 8 and idle:
                    k, x = idle.pop(0)
                    self._sessions[k].remove(x)
                    x.close()
                    total -= 1
                ses = self.engine.session(*key)
                self._sessions.setdefault(key, []).append(ses)
            self._sessions_busy.add(id(ses))
        try:
            if attn_trace is not None:
                ses.set_attn_trace(attn_trace, attn_ring)
            yield ses
        finally:
            if attn_trace is not None:
                ses.set_attn_trace(None)
            with self._sessions_lock:
                self._sessions_busy.discard(id(ses))

    @staticmethod
    def _launch_blocks(ses: ArSession, feed: TapeFeed, edges: Sequence[Tuple[int, int]], cond: torch.Tensor,
                       txt: torch.Tensor, lens: Sequence[int], samp: Sampling) -> Iterator[int]:
        """Runs the session block by block, (a, b) edges: each block's noise rows are drawn and queued for upload just
        before its launch.  The session is begun before the first block is drawn, so that the device work of `begin`
        (state resets, the text K/V) runs while the host draws.  Yields each block's end once it is enqueued."""
        for a, b in edges:
            if a == 0:
                ses.begin(cond, txt, lens, feed.dev, samp)
            feed.fill(b)
            ses.run(b - a)
            yield b

    # ---- prefill
    @torch.no_grad()
    def prepare_reference(self, ref_tokens_tq: torch.Tensor, *, device=None) -> PreparedReference:
        """reference model.py:152-170 on the CUDA reference-preparation engine (Token2SV, reference encoder, cached K/V)."""
        ref_btq = ref_tokens_tq.unsqueeze(0).to(device=self.device, dtype=torch.long)
        sv, seq, caches = self.refprep.run(ref_btq[0])
        return PreparedReference(ref_tokens_btq=ref_btq, sv_ref=sv, ref_seq=seq, ref_kv_caches=caches)

    @torch.no_grad()
    def speaker_vector(self, ref_tokens_tq: torch.Tensor) -> torch.Tensor:
        """Token2SV alone (SoproTTS.encode_speaker, reference model.py:458-475) -> [sv_dim]"""
        return self.refprep.run(ref_tokens_tq.to(self.device))[0].squeeze(0)

    @torch.no_grad()
    def prepare_conditioning(self, text_ids_1d: torch.Tensor, ref: PreparedReference, *, max_frames: int, device=None,
                             style_strength: float = 1.2) -> Dict[str, torch.Tensor]:
        """reference model.py:174-216 on the CUDA prefill engine (sopro_b200/csrc/nar_engine.cu: ~25 fused fp32 kernels)."""
        txt_seq, lens, txt_pool, cond = self.prefill.run([text_ids_1d], ref, n_frames=int(max_frames) + 1,
                                                         style_strength=float(style_strength))
        sv = ref.sv_ref.to(self.device)
        if sv.dim() == 1:
            sv = sv.unsqueeze(0)
        return {"txt_seq": txt_seq, "text_mask": torch.ones((1, lens[0]), dtype=torch.bool, device=self.device),
                "txt_pool": txt_pool, "sv_ref": sv, "cond_ar": cond}

    @torch.no_grad()
    def nar_refine(self, cond_seq: torch.Tensor, rvq1_1xT: torch.Tensor, lens: Optional[torch.Tensor] = None) -> torch.Tensor:
        """reference model.py:307-347 on the CUDA NAR engine (sopro_b200/csrc/nar_engine.cu): 4 stage passes of fused fp32
        kernels, ids equal to the reference's.  cond [B, T, D], rvq1 [B, T] -> [B, T, Q] int64.  `lens` (extension):
        valid frames per utterance of a ragged batch (the refiner is not causal)."""
        if int(cond_seq.size(1)) == 0:
            return torch.zeros((int(cond_seq.size(0)), 0, int(self.cfg.num_codebooks)), dtype=torch.long, device=self.device)
        return self.nar.refine(cond_seq, rvq1_1xT, lens)

    # ---- the hot path
    @torch.no_grad()
    def ar_chunk_rows(self, cond: torch.Tensor, txt: torch.Tensor, lens: Sequence[int], *, gen: Generation,
                      chunk_frames: int = 0, seeds: Optional[Sequence[int]] = None,
                      generator: Optional[torch.Generator] = None, progress: Optional[dict] = None,
                      attn_trace: Optional[torch.Tensor] = None, attn_ring: Optional[int] = None):
        """The persistent kernel over B utterances in one session (cond [B, >= steps, D], txt [B, Lmax, D], lens),
        driven `chunk_frames` frames per launch (0 = the whole utterance in one launch): every launch advances all of
        them by the same steps.  Yields ``(tokens, finished, prefetch)`` per launch: one list of new frames (ints) and
        one finished flag (EOS past the minimum frame count, or max_frames reached) per row, and a callable that
        enqueues the NEXT launch right away on the current CUDA stream -- a streaming consumer queues it behind its own
        NAR + Mimi work so it runs while the audio is handed out; without the call the next launch is enqueued when the
        generator is resumed.  `seeds` gives row i the private generator of seeds[i]; without them the rows draw from `generator`
        (None: the global one) as ar_generate_tensors does: one row's tape block by block, several rows' tapes in full,
        row after row, before the first launch.  One row's frames computed ahead of a consumer that stops early are
        abandoned: on exit its generator is settled to ``progress["consumed"]`` frames (default: every frame yielded),
        i.e. exactly the draws the reference would have made; several rows' are never settled.  `attn_trace` (word
        timestamps): a [max_frames + 1, n_attn, B, H, ld] buffer, ld >= max(lens), that receives the text
        cross-attention weights; with `attn_ring` (streams) a ring of that many step rows, at least `chunk_frames`."""
        B, steps = int(cond.size(0)), gen.max_frames + 1
        if cond.size(1) < steps:
            raise ValueError(f"cond_ar has {cond.size(1)} rows, need max_frames+1 = {steps}")
        samp = dataclasses.replace(gen.sampling, stop_on_first_eos=False)
        per = steps if chunk_frames <= 0 else int(chunk_frames)
        st = {"launched": 0, "read": 0, "yielded": 0}
        lens = [int(x) for x in lens]
        with TapeFeed(B, steps, self.cfg.ar_vocab(), samp.noise_cols(self.cfg.ar_vocab()), self.device,
                      None if seeds is None else [int(x) for x in seeds], generator) as feed, \
                self._lease(B, steps, max(lens), attn_trace, attn_ring) as ses:
            launches = self._launch_blocks(ses, feed, [(a, min(steps, a + per)) for a in range(0, steps, per)],
                                           cond[:, :steps], txt, lens, samp)

            def launch():
                """Enqueue the next launch (no-op while one is in flight)."""
                if st["launched"] < steps and st["launched"] <= st["read"]:
                    st["launched"] = next(launches)

            try:
                t = [0] * B
                over = [False] * B
                while not all(over):
                    launch()
                    toks, n, done = ses.read()  # synchronises the stream the launch ran on
                    st["read"] = st["launched"]
                    chunks, finished = [], []
                    for b in range(B):
                        upto = int(n[b])
                        chunks.append([] if over[b] else [int(x) for x in toks[b, t[b]:upto]])
                        over[b] = over[b] or bool(done[b]) or upto >= steps or upto < st["launched"]
                        finished.append(over[b])
                        t[b] = upto
                    st["yielded"] = max(t)
                    end = all(over)
                    yield chunks, finished, (launch if not end else (lambda: None))
            finally:
                if B == 1:
                    feed.settle(int(progress["consumed"]) if progress is not None and "consumed" in progress else st["yielded"])

    @torch.no_grad()
    def ar_stream(self, prep: Dict[str, torch.Tensor], *, max_frames: int, top_p: float = 0.9, temperature: float = 1.05,
                  anti_loop: bool = True, loop_streak: int = 8, recovery_top_p: float = 0.85, recovery_temp: float = 1.2,
                  min_gen_frames: Optional[int] = None, launch_frames: int = 0, seed: Optional[int] = None,
                  generator: Optional[torch.Generator] = None,
                  attn_trace: Optional[torch.Tensor] = None) -> Iterator[Tuple[int, int, bool]]:
        """Yields (t, token, is_eos) like the reference generator (model.py:218-305).  The persistent kernel runs
        `launch_frames` frames per launch (0 = the whole utterance in one launch); a consumer that stops iterating
        early simply abandons the frames computed ahead, and the RNG is settled to the frames actually consumed."""
        gen = Generation.resolve(self.cfg, max_frames=max_frames, top_p=top_p, temperature=temperature,
                                 anti_loop=anti_loop, style_strength=None, min_gen_frames=min_gen_frames)
        # top_p=None is no top-p (see Generation.resolve), and so is recovery_top_p=None
        samp = dataclasses.replace(gen.sampling, loop_streak=int(loop_streak), recovery_temp=float(recovery_temp),
                                   recovery_top_p=1.0 if recovery_top_p is None else float(recovery_top_p))
        progress = {"consumed": 0}
        chunks = self.ar_chunk_rows(prep["cond_ar"], prep["txt_seq"], [int(prep["txt_seq"].size(1))],
                                    gen=dataclasses.replace(gen, sampling=samp), chunk_frames=launch_frames,
                                    seeds=None if seed is None else [seed], generator=generator, progress=progress,
                                    attn_trace=attn_trace)
        t = 0
        try:
            for rows, _finished, _prefetch in chunks:
                for tok in rows[0]:
                    progress["consumed"] = t + 1
                    yield t, tok, tok == self.eos_id
                    t += 1
        finally:
            chunks.close()

    @torch.no_grad()
    def ar_generate_tensors(self, cond: torch.Tensor, txt: torch.Tensor, lens: Sequence[int], *, gen: Generation,
                            seeds: Optional[Sequence[int]] = None, attn_trace: Optional[torch.Tensor] = None,
                            generator: Optional[torch.Generator] = None, settle: bool = False):
        """B utterances in ONE persistent kernel run from batch tensors (cond [B, >=steps, D], txt [B, Lmax, D], lens).
        -> (tokens [B, steps] int32 numpy, n_tokens [B]); each row stops at its first EOS.  With `seeds` and at least 64
        steps the run is launched in growing blocks (the kernel resumes from its device state), each block's tapes drawn
        on host threads while the device generates the block before; otherwise in one launch.  `attn_trace` (word
        timestamps): a [steps, n_attn, B, H, ld] buffer, ld >= max(lens), that receives the text cross-attention
        weights.  Without `seeds` the tapes draw from `generator` (None: the global one), every tape in full, row after
        row; `settle` (one row) then leaves the generator after exactly the draws of the frames generated, up to and
        including the first EOS, as the reference's generate_tokens does."""
        B, steps = int(cond.shape[0]), gen.max_frames + 1
        samp = dataclasses.replace(gen.sampling, stop_on_first_eos=True)
        edges = _growing_blocks(steps) if seeds is not None and steps >= 64 else [(0, steps)]
        with TapeFeed(B, steps, self.cfg.ar_vocab(), samp.noise_cols(self.cfg.ar_vocab()), self.device, seeds, generator) as feed, \
                self._lease(B, steps, max(int(x) for x in lens), attn_trace) as ses:
            for _ in self._launch_blocks(ses, feed, edges, cond[:, :steps], txt, [int(x) for x in lens], samp):
                pass
            toks, n, _ = ses.read()
            if settle:
                feed.settle(int(n[0]))
        return toks, n

    @torch.no_grad()
    def generate_codes(self, text_ids: Sequence[torch.Tensor], ref, *, gen: Generation,
                       seeds: Optional[Sequence[int]] = None, generator: Optional[torch.Generator] = None,
                       settle: bool = False, attn_trace: Optional[torch.Tensor] = None,
                       info: Optional[dict] = None) -> Tuple[List[int], Optional[torch.Tensor]]:
        """NEW (the reference is batch-1): B texts with one prepared reference, or one each (`ref` as in
        SoproTTS.synthesize_batch): one batched prefill, one persistent AR run until each text's first EOS, one ragged
        NAR pass -> (frames before the first EOS per text, codes [B, Tmax, Q] on the device; None when every text has 0
        frames).  `seeds`, `generator`, `settle`, `attn_trace`: see ar_generate_tensors.  `info` (best-of-N): receives
        "stopped", whether each row sampled an EOS, and "text_lens"."""
        txt_seq, lens, _pool, cond = self.prefill.run(list(text_ids), ref, n_frames=gen.max_frames + 1,
                                                      style_strength=gen.style_strength)
        toks, n = self.ar_generate_tensors(cond, txt_seq, lens, gen=gen, seeds=seeds, attn_trace=attn_trace,
                                           generator=generator, settle=settle)
        eos = self.eos_id
        Ts, stopped = [], []
        for i in range(len(lens)):
            row = toks[i, : n[i]]
            hit = (row == eos).nonzero()[0]
            Ts.append(int(hit[0]) if hit.size else int(n[i]))
            stopped.append(bool(hit.size))
        if info is not None:
            info["stopped"], info["text_lens"] = stopped, [int(x) for x in lens]
        Tmax = max(Ts)
        if Tmax == 0:
            return Ts, None
        # NAR refiner over the ragged batch (not causal: `lens` makes the padding act as each utterance's zero padding)
        rvq1 = torch.from_numpy(toks[:, :Tmax].copy()).to(self.device)
        codes = self.nar_refine(cond[:, :Tmax], rvq1.clamp_(0, eos - 1), lens=torch.tensor(Ts, dtype=torch.int32))
        return Ts, codes

    @torch.no_grad()
    def generate_tokens(self, text_ids_1d: torch.Tensor, ref: PreparedReference, *, max_frames: int, device=None,
                        top_p: float = 0.9, temperature: float = 1.05, anti_loop: bool = True, style_strength: float = 1.2,
                        min_gen_frames: Optional[int] = None, seed: Optional[int] = None,
                        generator: Optional[torch.Generator] = None, attn_trace: Optional[torch.Tensor] = None) -> torch.Tensor:
        """reference model.py:349-401: prefill, AR until the first EOS, cut there, NAR refine -> [T, Q] int64; the
        one-text case of generate_codes, the generator settled as the reference leaves it.  `attn_trace`: see
        ar_generate_tensors."""
        gen = Generation.resolve(self.cfg, max_frames=max_frames, top_p=top_p, temperature=temperature,
                                 anti_loop=anti_loop, style_strength=style_strength, min_gen_frames=min_gen_frames)
        Ts, codes = self.generate_codes([text_ids_1d], ref, gen=gen, seeds=None if seed is None else [seed],
                                        generator=generator, settle=True, attn_trace=attn_trace)
        if codes is None:
            return torch.zeros((0, int(self.cfg.num_codebooks)), dtype=torch.long, device=self.device)
        return codes[0, : Ts[0]]


class SoproTTS:
    # idle Mimi stream states, made by the first stream (sopro_b200/streaming.py), replaced for larger chunks
    _stream_decoder: Optional[MimiStreamDecoder] = None

    def __init__(self, model: SoproModel, cfg: SoproTTSConfig, tokenizer, codec: MimiCodec, device: str):
        self.model = model
        self.cfg = cfg
        self.tokenizer = tokenizer
        self.codec = codec
        self.device = torch.device(device)
        self._resamplers: Dict[int, Resampler] = {}  # output rate -> its resampler (tap table on the device)
        dev = self.device
        self._stretch_pool = StatePool(lambda n, speed: StretchStream(n, dev, speed))  # idle time-stretch states, any speed
        self._watermark_pool = StatePool(lambda n, key: WatermarkStream(n, dev, key))  # idle watermark states, any key
        self._join_pool = LF.StreamJoinPool(dev)  # idle streaming-trim states of stream_long

    # ---- construction
    @classmethod
    def from_pretrained(cls, repo_id: str, *, revision: Optional[str] = None, cache_dir: Optional[str] = None,
                        token: Optional[str] = None, device: Optional[str] = None, weight_dtype: str = "fp32",
                        mimi_precision: str = "bf16_tc") -> "SoproTTS":
        """reference model.py:419-451: HF snapshot -> cfg from the safetensors header -> tokenizer -> weights -> Mimi."""
        from huggingface_hub import snapshot_download

        from .tokenizer import TextTokenizer

        device = device or "cuda"
        local_dir = repo_id if os.path.isdir(repo_id) else snapshot_download(repo_id=repo_id, revision=revision,
                                                                             cache_dir=cache_dir, token=token)
        model_path = os.path.join(local_dir, "model.safetensors")
        if not os.path.exists(model_path):
            raise FileNotFoundError(f"Expected {model_path} in repo snapshot.")
        cfg = read_safetensors_cfg(model_path)
        tokenizer = TextTokenizer(model_name=local_dir)
        model = SoproModel(cfg, load_safetensors(model_path), device, weight_dtype)
        codec = MimiCodec(num_quantizers=cfg.num_codebooks, device=device, precision=mimi_precision)
        return cls(model=model, cfg=cfg, tokenizer=tokenizer, codec=codec, device=device)

    @classmethod
    def from_state_dict(cls, cfg: SoproTTSConfig, state_dict: Dict[str, torch.Tensor], tokenizer,
                        mimi_state_dict: Dict[str, torch.Tensor], *, device: str = "cuda", weight_dtype: str = "fp32",
                        mimi_hf_model=None, mimi_precision: str = "bf16_tc") -> "SoproTTS":
        """Offline constructor (synthetic or locally stored checkpoints): no hub access."""
        model = SoproModel(cfg, state_dict, device, weight_dtype)
        codec = MimiCodec(int(cfg.num_codebooks), device=device, state_dict=mimi_state_dict, hf_model=mimi_hf_model,
                          precision=mimi_precision)
        return cls(model=model, cfg=cfg, tokenizer=tokenizer, codec=codec, device=device)

    # ---- reference plumbing (model.py:453-529)
    def encode_text(self, text: str) -> torch.Tensor:
        return torch.tensor(self.tokenizer.encode(text), dtype=torch.long, device=self.device)

    def encode_reference(self, *, ref_audio_path: Optional[str] = None, ref_tokens_tq: Optional[torch.Tensor] = None,
                         ref_seconds: Optional[float] = None) -> torch.Tensor:
        if ref_tokens_tq is None and ref_audio_path is None:
            raise RuntimeError("SoproTTS requires a reference. Provide ref_audio_path=... or ref_tokens_tq=...")
        if ref_tokens_tq is not None and ref_audio_path is not None:
            raise RuntimeError("Provide only one of ref_audio_path or ref_tokens_tq (not both).")
        if ref_seconds is None:
            ref_seconds = 12.0
        if ref_tokens_tq is not None:
            ref = ref_tokens_tq.to(self.device).long()
            if ref_seconds and ref_seconds > 0:
                ref = center_crop_tokens(ref, max(1, int(round(ref_seconds * float(self.cfg.mimi_fps)))))
            return ref
        crop = ref_seconds if ref_seconds is not None and ref_seconds > 0 else None
        return self.codec.encode_file(ref_audio_path, crop_seconds=crop).to(self.device).long()

    @torch.inference_mode()
    def encode_speaker(self, **kw) -> torch.Tensor:
        return self.model.speaker_vector(self.encode_reference(**kw)).detach()

    @torch.inference_mode()
    def prepare_reference(self, *, ref_audio_path: Optional[str] = None, ref_tokens_tq: Optional[torch.Tensor] = None,
                          ref_seconds: Optional[float] = None) -> PreparedReference:
        tokens_tq = self.encode_reference(ref_audio_path=ref_audio_path, ref_tokens_tq=ref_tokens_tq, ref_seconds=ref_seconds)
        return self.model.prepare_reference(tokens_tq, device=self.device)

    @torch.inference_mode()
    def prepare_references(self, clips: Sequence[ingest.Clip], *, sample_rates=None,
                           ref_seconds: Optional[float] = None, denoise: bool = False) -> List[PreparedReference]:
        """(extension) Many reference voices in one batched pass, from files or in-memory audio -> one PreparedReference
        per clip, in order.  `clips`: paths (read with audio.load_audio_file) and / or float tensors [n] or [C, n] on
        any device (channels averaged).  `sample_rates`: one rate per clip (None for a path, which has its own), or one
        int for every tensor clip.  `ref_seconds`: as in prepare_reference (None = 12 s, <= 0 = no crop).  One voice from
        memory: ``prepare_references([wav], sample_rates=[sr])[0]``.
        encode_file's steps run on the GPU for the whole batch (energy trim at each clip's rate, resample to 24 kHz,
        centre crop, a batched Mimi encode whose every row equals encode_wav of that row alone), then prepare_reference
        per voice.  Against prepare_reference(ref_audio_path=...) the trim decisions can differ only at a frame within
        rounding of the threshold, and the resampler is this library's (DESIGN.md §5d, §5l).  Every argument is checked,
        and the files read, before any device work.
        `denoise` (extension): remove stationary background noise (fans, hum, room tone) from each trimmed 24 kHz clip
        before the crop, with a CUDA Wiener suppressor whose noise estimate is the quietest tenth of the clip's frames
        (sopro_b200/denoising.py, DESIGN.md §5n).  It assumes the clip pauses: one that never does loses some of its own
        stationary content.  Whether it improves a clone has not been measured.  One denoised voice from a file:
        ``prepare_references([path], denoise=True)[0]`` (prepare_reference keeps the reference's signature)."""
        check_denoise(denoise)
        ingest.crop_samples(ref_seconds)
        wavs, rates = ingest.load_clips(clips, sample_rates)
        if ref_seconds is None:
            ref_seconds = ingest.DEFAULT_REF_SECONDS
        wav_bl, lens = self.codec.prepare_wavs(wavs, rates, ref_seconds, denoise=denoise)
        codes = self.codec.encode_wavs(wav_bl, lens)
        return [self.model.prepare_reference(c, device=self.device) for c in codes]

    @torch.inference_mode()
    def blend_voices(self, voices: Sequence[PreparedReference], weights: Optional[Sequence[float]] = None) -> PreparedReference:
        """(extension) A new voice mixed from prepared voices -> a voices.VoiceBlend (a PreparedReference) on the device,
        accepted wherever a voice is.  `weights`: one > 0 per voice, normalised to sum to 1 (None = equal).  The blend's
        speaker vector is the normalised weighted mean of the voices'; in each reference cross-attention layer every
        voice is read out on its own and the read-outs are mixed with the weights (DESIGN.md §5t).  The same object
        passed twice counts once with its weights added, so ``blend_voices([a])`` and ``blend_voices([a, a])`` speak as
        ``a``; a blend passed in is flattened into its voices.  Refusals (sopro_b200/voices.py::blend) raise before any
        device work.  Whether a blend sounds between its voices on the released checkpoint has not been measured."""
        from . import voices as V  # the `voices` argument shadows the module

        return V.blend(voices, weights, device=self.device, **V.geometry(self.cfg))

    # ---- synthesis (model.py:531-580)
    @torch.inference_mode()
    def synthesize(self, text: str, *, ref: Optional[PreparedReference] = None, ref_audio_path: Optional[str] = None,
                   ref_tokens_tq: Optional[torch.Tensor] = None, max_frames: int = 400, top_p: float = 0.9,
                   temperature: float = 1.05, anti_loop: bool = True, style_strength: Optional[float] = None,
                   ref_seconds: Optional[float] = None, min_gen_frames: Optional[int] = None, seed: Optional[int] = None,
                   generator: Optional[torch.Generator] = None, sample_rate: Optional[int] = None,
                   speed: Optional[float] = None, loudness: Optional[float] = None, word_timestamps: bool = False,
                   best_of: int = 1, watermark: Optional[int] = None):
        """-> [1, 1, N] f32 on the device.  `sample_rate` (extension): the output rate in Hz (None = 24 kHz, the codec's
        own); another rate resamples the decoded waveform on the GPU (sopro_b200/resample.py).  `speed` (extension): the
        speaking rate in [0.25, 4.0] (None = the model's own); the 24 kHz waveform is time-stretched on the GPU with its
        pitch kept (sopro_b200/stretch.py), then resampled when `sample_rate` is set.  `loudness` (extension): a target
        integrated loudness in LUFS, [-60, 0] (None = the level the model produced); the final waveform is measured per
        ITU-R BS.1770-4 and scaled on the GPU under a -1 dBFS sample-peak ceiling (sopro_b200/loudness.py).
        `word_timestamps` (extension): also return when each word is spoken, ``(wav, List[WordTiming])``, from the AR
        step's text cross-attention (sopro_b200/timestamps.py); the audio is the same as without it.
        `best_of` (extension): generate that many takes side by side in one batch (take k with seed + k) and keep the
        one rerank.choose picks: takes that ended with an EOS and have at least one frame per text token first, then
        the highest cosine between the take's speaker vector and the reference voice's; only that take is decoded.
        The result equals synthesize(seed=seed + k) for the picked k.  Without a seed the takes draw from the generator
        as synthesize_batch of the takes would.  That the cosine picks better-sounding takes is not measured.
        `watermark` (extension): a key, an integer in [0, 2^32) (None = no mark); the 24 kHz waveform, after the
        time-stretch, carries a keyed spread-spectrum mark 30 dB below the local signal level, which
        sopro_b200.detect_watermark finds with the same key (sopro_b200/watermark.py)."""
        post = OutputChain(self, sample_rate, speed, loudness, watermark)  # a refused argument raises before any work
        n_best = self._check_best_of(best_of, 1)
        gen = Generation.resolve(self.cfg, max_frames=max_frames, top_p=top_p, temperature=temperature,
                                 anti_loop=anti_loop, style_strength=style_strength, min_gen_frames=min_gen_frames)
        if ref is None:
            ref = self.prepare_reference(ref_audio_path=ref_audio_path, ref_tokens_tq=ref_tokens_tq, ref_seconds=ref_seconds)
        tr: Optional[dict] = {} if word_timestamps else None
        # one take settles the generator as the reference's generate_tokens does; best_of takes draw as synthesize_batch
        Ts, codes = self._best_codes([text], ref, n_best, seeds=None if seed is None else [int(seed)], trace_out=tr,
                                     gen=gen, generator=generator, settle=n_best == 1)
        words = None
        if word_timestamps:
            spans = self.tokenizer.encode_with_offsets(text)[1]
            words = self._timings([text], [spans], tr["probs"], tr["lens"], Ts, post.S)[0]
        wav = torch.zeros(1, 1, 0, device=self.device)
        for _chunk, w, lens in self._decode_chunks(codes, Ts):
            w, lens = post(w, lens)
            wav = w[:, :, : lens[0]]
        return (wav, words) if word_timestamps else wav

    @torch.inference_mode()
    def synthesize_batch(self, texts: Sequence[str], *, ref: Union[PreparedReference, Sequence[PreparedReference]],
                         max_frames: int = 400, top_p: float = 0.9,
                         temperature: float = 1.05, anti_loop: bool = True, style_strength: Optional[float] = None,
                         min_gen_frames: Optional[int] = None, seeds: Optional[Sequence[int]] = None,
                         sample_rate: Optional[int] = None, speed: Optional[float] = None,
                         loudness: Optional[float] = None, word_timestamps: bool = False, best_of: int = 1,
                         watermark: Optional[int] = None):
        """NEW: B texts -> B waveforms [1, 1, N_i].  `ref`: one prepared reference for every text, or a sequence of B, a
        voice per text (texts that pass the same object share its K / V; sopro_b200/voices.py).  One batched prefill,
        one persistent AR launch, one ragged NAR pass, padded Mimi decodes (each time-stretched, then resampled, then
        loudness-normalised, in one ragged launch when `speed` / `sample_rate` / `loudness` is given); utterance i equals
        synthesize(texts[i], ref=ref[i] (or ref), seed=seeds[i], sample_rate=sample_rate, speed=speed, loudness=loudness).
        `word_timestamps`: also return each utterance's word timings (see synthesize), ``(List[wav], List[List[WordTiming]])``.
        `best_of`: each text's takes are generated in the same pass (B x best_of rows, take k of text i with seed
        seeds[i] + k, in text i's voice) and only the picked take of each text is decoded (see synthesize; text i's takes
        are scored against its own voice's sv_ref).  `watermark`: every utterance carries the key's mark (see
        synthesize).  Refused before any device work or random draw: `texts` that is a str or not a sequence
        (TypeError), no text or `seeds` of another length (ValueError), a `ref` sequence of the wrong length
        (ValueError), an element that is not a PreparedReference (TypeError), a voice of another geometry or outside
        [1, 4096] reference frames (ValueError) or with a key padding mask (NotImplementedError)."""
        post = OutputChain(self, sample_rate, speed, loudness, watermark)
        texts, seeds = _check_texts(texts, seeds)
        n_best = self._check_best_of(best_of, len(texts))
        voices.check_voices(ref, len(texts), **voices.geometry(self.cfg))
        gen = Generation.resolve(self.cfg, max_frames=max_frames, top_p=top_p, temperature=temperature,
                                 anti_loop=anti_loop, style_strength=style_strength, min_gen_frames=min_gen_frames)
        tr: Optional[dict] = {} if word_timestamps else None
        Ts, codes = self._best_codes(texts, ref, n_best, seeds=seeds, trace_out=tr, gen=gen)
        words = None
        if word_timestamps:
            spans = [self.tokenizer.encode_with_offsets(t)[1] for t in texts]
            words = self._timings(texts, spans, tr["probs"], tr["lens"], Ts, post.S)
        out: List[torch.Tensor] = [torch.zeros(1, 1, 0, device=self.device) for _ in texts]
        for chunk, wav, lens in self._decode_chunks(codes, Ts):
            wav, lens = post(wav, lens)  # [rows, 1, L]: one ragged launch per stage
            for j, i in enumerate(chunk):
                out[i] = wav[j: j + 1, :, : lens[j]].clone()
        return (out, words) if word_timestamps else out

    @torch.inference_mode()
    def synthesize_long(self, text: str, *, ref: PreparedReference, max_frames: int = 400, max_tokens: int = 64,
                        pause_ms: float = 250, top_p: float = 0.9, temperature: float = 1.05, anti_loop: bool = True,
                        style_strength: Optional[float] = None, min_gen_frames: Optional[int] = None,
                        seed: Optional[int] = None, sample_rate: Optional[int] = None, speed: Optional[float] = None,
                        loudness: Optional[float] = None, word_timestamps: bool = False, best_of: int = 1,
                        watermark: Optional[int] = None):
        """NEW: a text of any length -> one waveform [1, 1, N] f32 on the device.  The text is cut into segments of at
        most `max_tokens` tokens (sopro_b200/longform.py::split_text: paragraphs, sentences, greedy packing); the
        segments are generated side by side through the batch path, SEGMENT_GROUP at a time (segment i equals
        synthesize(segment, seed=seed + i); without a seed the global generator is consumed segment after segment, as by
        synthesize_batch), each decoded row is trimmed to its speech on the GPU, and the rows are joined with
        `pause_ms` (in [0, 2000]) of silence between them and 10 ms raised-cosine edges.  The joined 24 kHz row then goes
        through the chain of synthesize: stretch (`speed`, pauses included), resample (`sample_rate`), loudness (one
        level for the whole passage).  Segments that produced no frames are skipped; if none did, the result is
        [1, 1, 0].  Every argument is checked before any work.  `word_timestamps`: also return the passage's word timings
        (see synthesize), ``(wav, List[WordTiming])``, their char spans in `text`.  `best_of`: each segment picks its own
        take (see synthesize; take k of segment i with seed seed + i + k) and the join sees only the picked ones; a
        group then holds fewer segments when group x best_of rows would exceed the batch limit.  `watermark`: the joined
        passage carries the key's mark (see synthesize)."""
        post = OutputChain(self, sample_rate, speed, loudness, watermark)
        n_best = self._check_best_of(best_of, 1)
        LF.check_pause(pause_ms)
        budget = LF.check_max_tokens(max_tokens, self.model.prefill.max_text_len)
        segments = LF.passage_segments(text, self.tokenizer, budget)
        gen = Generation.resolve(self.cfg, max_frames=max_frames, top_p=top_p, temperature=temperature,
                                 anti_loop=anti_loop, style_strength=style_strength, min_gen_frames=min_gen_frames)
        rows, ext, firsts, all_Ts = self._speak_segments(segments, ref, n_best, seed=seed, word_timestamps=word_timestamps,
                                                          gen=gen)
        wav = LF.join_segments(rows, ext, pause_ms)  # the one host read: the B extents
        words = None
        if word_timestamps:
            spans = [self.tokenizer.encode_with_offsets(t)[1] for t in segments]
            words = TS.long_timings(text, segments, spans, firsts, all_Ts, self.codec.engine.hop, ext.cpu().numpy(),
                                    LF.pause_samples(pause_ms), post.S)
        if wav.shape[-1] == 0:
            return (wav, words) if word_timestamps else wav
        wav, _ = post(wav)
        return (wav, words) if word_timestamps else wav

    @torch.inference_mode()
    def synthesize_dialogue(self, turns: Sequence[Tuple[PreparedReference, str]], *, seed: Optional[int] = None,
                            pause_ms: float = 250, turn_pause_ms: float = 500, max_frames: int = 400,
                            max_tokens: int = 64, top_p: float = 0.9, temperature: float = 1.05, anti_loop: bool = True,
                            style_strength: Optional[float] = None, min_gen_frames: Optional[int] = None,
                            sample_rate: Optional[int] = None, speed: Optional[float] = None,
                            loudness: Optional[float] = None, word_timestamps: bool = False, best_of: int = 1,
                            watermark: Optional[int] = None):
        """NEW: a script of ``(voice, text)`` turns, in speaking order -> one waveform [1, 1, N] f32 on the device, each
        turn in its own voice (sopro_b200/dialogue.py).  Each turn's text is cut as synthesize_long cuts a text and the
        segments of all turns go through the batch path together, SEGMENT_GROUP at a time: segment k of the script
        equals synthesize(segment, ref=its turn's voice, seed=seed + k) (without a seed the global generator is consumed
        segment after segment); turns that pass the same PreparedReference object share its prefill slot.  The trimmed
        segments are joined on the GPU with `pause_ms` between spans of one turn and `turn_pause_ms` between spans of
        different turns (both in [0, 2000]; consecutive turns by the same voice still get `turn_pause_ms`), then go
        through the chain of synthesize_long: stretch (`speed`), watermark, resample (`sample_rate`).  `loudness`
        levels each turn, not the passage: turn j is scaled by normalize_loudness's gain for its own 24 kHz join (what
        synthesize_long would join for that turn alone), inside the join, before the chain, and there is no
        passage-level loudness stage.  A turn whose text is empty or whitespace only speaks nothing; segments that
        produced no frames are skipped; if nothing was produced the result is [1, 1, 0].  `word_timestamps`: also
        return each turn's words, ``(wav, List[List[WordTiming]])``, their char spans in that turn's text and their
        times in seconds of the returned audio.  `best_of`: as in synthesize_long, each segment scored against its own
        voice.  Refused before any device work or random draw: `turns` that is not a non-empty sequence of
        (PreparedReference, str) pairs (TypeError; ValueError when empty), a script with nothing to speak, a voice of
        the wrong geometry, `pause_ms` / `turn_pause_ms` / `max_tokens` out of range, a refused sample_rate / speed /
        loudness / watermark / best_of, a non-bool `word_timestamps`."""
        turns, segments, turn_of, voice_of, pause, turn_pause = D.check_script(self, turns, pause_ms, turn_pause_ms,
                                                                               max_tokens)
        post = OutputChain(self, sample_rate, speed, loudness, watermark)
        target, post.target = post.target, None  # levelled per turn at 24 kHz, before the chain
        n_best = self._check_best_of(best_of, 1)
        TS.check_word_timestamps(word_timestamps)
        gen = Generation.resolve(self.cfg, max_frames=max_frames, top_p=top_p, temperature=temperature,
                                 anti_loop=anti_loop, style_strength=style_strength, min_gen_frames=min_gen_frames)
        rows, ext_dev, firsts, Ts = self._speak_segments(segments, D.segment_voices(voice_of), n_best, seed=seed,
                                                         word_timestamps=word_timestamps, gen=gen)
        ext = ext_dev.cpu().numpy()  # the one host read: the extents
        pauses = LF.gap_pauses(ext, pause, turn_of, turn_pause)
        gain = None if target is None else D.turn_gains(rows, ext, turn_of, len(turns), pause, target)
        wav = LF.join_gaps(rows, ext, pauses, gain)
        words = None
        if word_timestamps:
            starts, after = D.turn_placement(ext, turn_of, len(turns), pauses)
            hop = self.codec.engine.hop
            words = []
            for j, ((_voice, text), idx) in enumerate(zip(turns, D.turn_segments(turn_of, len(turns)))):
                segs = [segments[k] for k in idx]
                spans = [self.tokenizer.encode_with_offsets(t)[1] for t in segs]
                words.append(TS.long_timings(text, segs, spans, [firsts[k] for k in idx], [Ts[k] for k in idx], hop,
                                             ext[idx].reshape(-1, 2), after[j], post.S, start=starts[j]))
        if wav.shape[-1]:
            wav, _ = post(wav)
        return (wav, words) if word_timestamps else wav

    @torch.inference_mode()
    def synthesize_ssml(self, ssml: str, *, ref: PreparedReference, voices: Optional[Mapping[str, PreparedReference]] = None,
                        seed: Optional[int] = None, pause_ms: float = 250, paragraph_pause_ms: float = 500,
                        max_frames: int = 400, max_tokens: int = 64, top_p: float = 0.9, temperature: float = 1.05,
                        anti_loop: bool = True, style_strength: Optional[float] = None,
                        min_gen_frames: Optional[int] = None, sample_rate: Optional[int] = None,
                        speed: Optional[float] = None, loudness: Optional[float] = None,
                        watermark: Optional[int] = None, best_of: int = 1):
        """NEW: speech markup -> one waveform [1, 1, N] f32 on the device.  The markup is an SSML subset
        (sopro_b200/ssml.py: ``<speak>``, ``<p>``, ``<s>``, ``<break>``, ``<prosody rate / volume>``, ``<voice>``,
        ``<sub>``); ssml.parse turns it into segments, each with its text, voice, rate and volume, and the gaps between
        them.  The segments go through the batch path together, SEGMENT_GROUP at a time: segment k equals
        synthesize(segment, ref=its voice, seed=seed + k) (without a seed the global generator is consumed segment
        after segment).  `ref` speaks outside every ``<voice>``, `voices` maps ``<voice name>`` to prepared voices.
        Each decoded row is trimmed to its speech, the trimmed spans are time-stretched in one launch at each span's
        rate times `speed` (a span at rate 1 is copied), and the spans are joined on the GPU with the plan's gaps, each
        span scaled by its volume's gain, between the leading and trailing silence.  The join then goes through the
        chain of synthesize: watermark, resample (`sample_rate`), loudness (one level for the whole passage, so the
        spans' relative volumes survive).  Unlike synthesize_long, `speed` does not stretch the pauses: it is folded
        into the spans' rates, so a ``<break time="1s"/>`` lasts one second at any speed.  Markup that is plain text
        in a ``<speak>`` equals synthesize_long of that text.  Segments that produce no speech are skipped and the
        gaps around them merge into the larger one (ssml.Plan.pauses).  `best_of`: as in synthesize_long.  Refused
        before any device work or random draw: every refusal of ssml.parse, a voice of the wrong geometry,
        `pause_ms` / `paragraph_pause_ms` / `max_tokens` out of range, a refused sample_rate / speed / loudness /
        watermark / best_of."""
        post = OutputChain(self, sample_rate, None, loudness, watermark)
        n_best = self._check_best_of(best_of, 1)
        budget = LF.check_max_tokens(max_tokens, self.model.prefill.max_text_len)
        plan = SSML.parse(ssml, voices, ref, pause_ms, paragraph_pause_ms, speed, budget, self.tokenizer)
        voice_of = [s.voice for s in plan.segments]
        _check_voices(self.cfg, voice_of)
        gen = Generation.resolve(self.cfg, max_frames=max_frames, top_p=top_p, temperature=temperature,
                                 anti_loop=anti_loop, style_strength=style_strength, min_gen_frames=min_gen_frames)
        rows, ext_dev, _f, _T = self._speak_segments([s.text for s in plan.segments], D.segment_voices(voice_of),
                                                     n_best, seed=seed, word_timestamps=False, gen=gen)
        ext = ext_dev.cpu().numpy()  # the one host read: the extents
        spans = [max(0, int(e) - int(s)) for s, e in ext]
        rates = [s.rate for s in plan.segments]
        n_out = [stretched_length(r, n) for r, n in zip(rates, spans)]
        stretched: List[torch.Tensor] = [torch.zeros(0, device=self.device)] * len(spans)
        if max(spans):
            batch = torch.zeros((len(spans), max(spans)), dtype=torch.float32, device=self.device)
            for k, (s, n) in enumerate(zip(ext[:, 0], spans)):
                if n:
                    batch[k, :n] = rows[k][int(s): int(s) + n]
            y = stretch_rows(batch, rates, lens=spans)
            stretched = [y[k] for k in range(len(spans))]
        gains = [s.gain for s in plan.segments]
        gain = None if all(g == 1.0 for g in gains) else torch.tensor(gains, dtype=torch.float32, device=self.device)
        out_ext = [(0, n) for n in n_out]
        wav = LF.join_padded(stretched, out_ext, plan.pauses([n > 0 for n in n_out]), gain, plan.lead, plan.trail,
                             self.device)
        if wav.shape[-1]:
            wav, _ = post(wav)
        return wav

    @torch.inference_mode()
    def synthesize_timed(self, cues: Union[str, Sequence[CU.Cue]], *, ref: PreparedReference,
                         voices: Optional[Mapping[str, PreparedReference]] = None, seed: Optional[int] = None,
                         max_rate: float = 1.5, pause_ms: float = 250, max_frames: int = 400, max_tokens: int = 64,
                         top_p: float = 0.9, temperature: float = 1.05, anti_loop: bool = True,
                         style_strength: Optional[float] = None, min_gen_frames: Optional[int] = None,
                         sample_rate: Optional[int] = None, loudness: Optional[float] = None,
                         watermark: Optional[int] = None, best_of: int = 1) -> Tuple[torch.Tensor, List[CU.CueFit]]:
        """NEW: subtitle cues spoken at their times -> (one waveform [1, 1, N] f32 on the device, one CueFit per cue in
        input order).  `cues`: an SRT or WebVTT file's text (sopro_b200/cues.py::parse) or a sequence of Cue; a cue
        without a voice speaks in `ref`, a named one in voices[name].  Each cue's text is cut as synthesize_long cuts a
        text, and segment k of the track (cue order, then segment order) equals synthesize(segment, ref=its cue's
        voice, seed=seed + k) (without a seed the global generator is consumed segment after segment).  The cues are
        processed in groups whose segments fill at most one SEGMENT_GROUP pass (a cue with more segments is a group of
        its own): the group is generated and decoded, each cue's segments are trimmed and joined with `pause_ms` as by
        synthesize_long, and the cue rows are time-stretched in one launch; only the stretched rows outlive the group.
        Fit rule, with n the cue's joined 24 kHz length and slot = round(end * 24000) - round(start * 24000): a cue that
        fits is not stretched; a longer one is sped up by the least fixed-point speed S = ceil(n * 65536 / slot) that
        fits, at most round(max_rate * 65536) (`max_rate` in [1, 4]); speech is never slowed down, so a capped cue runs
        past its end.  Each stretched cue is placed at round(start * 24000) and the cues are summed, in ascending
        (start sample, input index) order, by one CUDA mix (longform.mix: overlaps add, unclipped; silence elsewhere).
        The timeline lasts to the later of the last cue's end and the end of its speech, then goes through the chain
        of synthesize_ssml: watermark, resample (`sample_rate`), loudness (whose -1 dBFS ceiling applies as everywhere).
        So a cue equals stretch_rows of synthesize_long(its text, ref=its voice, seed=seed + its first segment) at its
        S.  `best_of`: as in synthesize_long.  Refused before any device work or random draw: every refusal of
        cues.parse, a sequence element that is not a Cue (TypeError), a cue whose start and end round to one sample,
        an unknown voice name, a voice of the wrong geometry, `max_rate` / `pause_ms` / `max_tokens` out of range, a
        refused sample_rate / loudness / watermark / best_of, and a track with nothing to speak."""
        post = OutputChain(self, sample_rate, None, loudness, watermark)
        n_best = self._check_best_of(best_of, 1)
        P = LF.pause_samples(pause_ms)
        budget = LF.check_max_tokens(max_tokens, self.model.prefill.max_text_len)
        S_max = CU.check_max_rate(max_rate)
        track = CU.track(cues)
        voice_of = CU.cue_voices(track, voices, ref)
        _check_voices(self.cfg, voice_of)
        segs = [LF.split_text(c.text, self.tokenizer, budget) for c in track]
        if not any(segs):
            raise ValueError("the track has nothing to speak (every cue is empty)")
        gen = Generation.resolve(self.cfg, max_frames=max_frames, top_p=top_p, temperature=temperature,
                                 anti_loop=anti_loop, style_strength=style_strength, min_gen_frames=min_gen_frames)
        K = len(track)
        offs = [CU.to_samples(c.start) for c in track]
        ends = [CU.to_samples(c.end) for c in track]
        S, M = [CU.ONE] * K, [0] * K
        spoken: List[Optional[torch.Tensor]] = [None] * K
        k0 = 0  # the track's index of the group's first segment
        for a, b in CU.groups([len(s) for s in segs], self._segment_group(n_best)):
            part = [s for c in range(a, b) for s in segs[c]]
            if not part:
                continue
            rows, ext_dev, _f, _T = self._speak_segments(
                part, D.segment_voices([voice_of[c] for c in range(a, b) for _ in segs[c]]), n_best,
                seed=None if seed is None else int(seed) + k0, word_timestamps=False, gen=gen)
            ext = ext_dev.cpu().numpy()  # the group's one host read: the extents
            joined: List[Optional[torch.Tensor]] = []
            j = 0
            for c in range(a, b):
                e = ext[j: j + len(segs[c])]
                live = bool(len(e)) and bool((e[:, 1] > e[:, 0]).any())
                joined.append(LF.join_gaps(rows[j: j + len(segs[c])], e, LF.gap_pauses(e, P)).reshape(-1)
                              if live else None)
                j += len(segs[c])
            n = [0 if w is None else int(w.numel()) for w in joined]
            for i, c in enumerate(range(a, b)):
                S[c] = CU.fit_speed(n[i], ends[c] - offs[c], S_max)
                M[c] = stretched_length(S[c] / CU.ONE, n[i])
            if max(n):
                batch = torch.zeros((b - a, max(n)), dtype=torch.float32, device=self.device)
                for i, w in enumerate(joined):
                    if w is not None:
                        batch[i, : n[i]] = w
                y = stretch_rows(batch, [S[c] / CU.ONE for c in range(a, b)], lens=n)
                for i, c in enumerate(range(a, b)):
                    if M[c]:
                        spoken[c] = y[i, : M[c]].clone()
                del batch, y
            del rows, ext_dev, joined  # the group's decodes go before the next group's
            k0 += len(part)
        order = [c for c in sorted(range(K), key=lambda c: (offs[c], c)) if M[c]]
        N = max(max(e, o + m) for e, o, m in zip(ends, offs, M))
        wav = LF.mix([spoken[c] for c in order], [offs[c] for c in order], N, self.device)
        wav, _ = post(wav)
        fits = [CU.CueFit(index=c, rate=S[c] / CU.ONE, spoken=M[c] / CU.SAMPLE_RATE,
                          overrun=max(0, offs[c] + M[c] - ends[c]) / CU.SAMPLE_RATE) for c in range(K)]
        return wav, fits

    def _speak_segments(self, segments: Sequence[str], ref, n_best: int, *, seed: Optional[int], word_timestamps: bool,
                        **kw) -> Tuple[List[torch.Tensor], torch.Tensor, list, List[int]]:
        """The segments of a long-form passage or a dialogue, generated through the batch path SEGMENT_GROUP at a time
        (segment k with seed seed + k and its own voice when `ref` is a sequence of one voice per segment) and
        decoded -> (each segment's 24 kHz row, read in place by the join; their extents, int64 [K, 2] on the device;
        with word_timestamps each segment's first frames and frame count, else empty lists).  Nothing synchronises.
        `kw`: _best_codes's `gen`."""
        B, group = len(segments), self._segment_group(n_best)
        one = isinstance(ref, PreparedReference)
        ext = torch.zeros((B, 2), dtype=torch.int64, device=self.device)
        rows: List[torch.Tensor] = [torch.zeros(0, device=self.device)] * B
        firsts: List = []
        all_Ts: List[int] = []
        for g0 in range(0, B, group):
            part = segments[g0: g0 + group]
            seeds = None if seed is None else [int(seed) + g0 + i for i in range(len(part))]
            tr: Optional[dict] = {} if word_timestamps else None
            Ts, codes = self._best_codes(part, ref if one else list(ref[g0: g0 + group]), n_best, seeds=seeds,
                                         trace_out=tr, **kw)
            if word_timestamps:
                first = TS.align(tr["probs"], tr["lens"], Ts).cpu().numpy()
                firsts.extend(first[i] for i in range(len(part)))
                all_Ts.extend(Ts)
            for chunk, wav, lens in self._decode_chunks(codes, Ts):
                flat = wav.view(len(chunk), -1)
                ext[torch.tensor([g0 + i for i in chunk], device=self.device)] = LF.speech_extents(flat, lens=lens)
                for j, i in enumerate(chunk):
                    rows[g0 + i] = flat[j, : lens[j]]  # read in place by the join
        return rows, ext, firsts, all_Ts

    def _segment_group(self, n_best: int) -> int:
        """Segments per batch pass of the passage paths: SEGMENT_GROUP, fewer when their best_of takes would exceed
        the batch limit."""
        group = int(LF.SEGMENT_GROUP)
        if n_best > 1:
            limit = self._batch_limit()
            if limit is not None:
                group = max(1, min(group, limit // n_best))
        return group

    def _timings(self, texts: Sequence[str], spans, probs: torch.Tensor, lens: Sequence[int], Ts: Sequence[int],
                 S: Optional[int]) -> List[List[TS.WordTiming]]:
        """The word timings of each utterance from its exported attention weights (one alignment launch)."""
        first = TS.align(probs, lens, Ts).cpu().numpy()
        hop = self.codec.engine.hop
        return [TS.utterance_timings(t, sp, first[i], int(Ts[i]), hop, S) for i, (t, sp) in enumerate(zip(texts, spans))]

    def _best_codes(self, texts: Sequence[str], ref, best_of: int, *, seeds: Optional[Sequence[int]], gen: Generation,
                    trace_out: Optional[dict] = None, generator: Optional[torch.Generator] = None,
                    settle: bool = False) -> Tuple[List[int], Optional[torch.Tensor]]:
        """_batch_codes with `best_of` candidates per text (sopro_b200/rerank.py): text i's candidate k is row i*N + k
        of ONE _batch_codes pass, with seed seeds[i] + k and text i's voice; every take is scored with one Token2SV
        launch against its text's voice's sv_ref, rerank.choose picks one per text, and only the picked rows are returned
        (the trace too), so the caller decodes those alone.  best_of = 1 is _batch_codes itself (`settle` only then)."""
        N = int(best_of)
        if N == 1:
            return self._batch_codes(texts, ref, seeds=seeds, trace_out=trace_out, gen=gen, generator=generator,
                                     settle=settle)
        slots, of = voices.voice_slots(ref, len(texts))
        rows = [t for t in texts for _ in range(N)]
        row_ref = slots[0] if len(slots) == 1 else [slots[of[r // N]] for r in range(len(rows))]
        tr: Optional[dict] = {} if trace_out is not None else None
        info: dict = {}
        Ts, codes = self._batch_codes(rows, row_ref, seeds=rerank.candidate_seeds(seeds, N), trace_out=tr, gen=gen,
                                      generator=generator, info=info)
        cos = [0.0] * len(rows)
        live = [r for r in range(len(rows)) if Ts[r] > 0]
        if live:  # the takes with frames, in one launch
            sv_ref = slots[0].sv_ref if len(slots) == 1 else torch.cat(
                [slots[of[r // N]].sv_ref.to(codes.device, torch.float32).reshape(1, -1) for r in live])
            _sv, c = self.model.refprep.speaker_vectors(codes[torch.tensor(live, device=codes.device)], [Ts[r] for r in live],
                                                        sv_ref)
            for r, v in zip(live, c.tolist()):
                cos[r] = v
        picks = []
        for i in range(len(texts)):
            a = i * N
            picks.append(a + rerank.choose(Ts[a: a + N], info["stopped"][a: a + N], info["text_lens"][a], cos[a: a + N]))
        Ts = [Ts[p] for p in picks]
        if tr is not None:
            trace_out["probs"] = tr["probs"][:, :, picks].contiguous()
            trace_out["lens"] = [tr["lens"][p] for p in picks]
        if max(Ts) == 0:
            return Ts, None
        return Ts, codes[torch.tensor(picks, device=codes.device)]

    def _batch_limit(self) -> Optional[int]:
        """The AR session's batch limit (SMs x 16 utterances per team)."""
        dev = self.model.device
        return torch.cuda.get_device_properties(dev).multi_processor_count * 16 if dev.type == "cuda" else None

    def _check_best_of(self, best_of, rows: int) -> int:
        """best_of checked, and the rows it makes checked against the batch limit, before any work."""
        n = rerank.check_best_of(best_of)
        if n > 1:
            rerank.check_rows(rows * n, self._batch_limit())
        return n

    def _batch_codes(self, texts: Sequence[str], ref, *, seeds: Optional[Sequence[int]], gen: Generation,
                     trace_out: Optional[dict] = None, **kw) -> Tuple[List[int], Optional[torch.Tensor]]:
        """SoproModel.generate_codes of the texts (`ref` as in synthesize_batch) -> (frames before the first EOS per
        text, codes [B, Tmax, Q]; None when every text has 0 frames).  `trace_out` (word timestamps): receives "probs",
        the AR launch's attention weights, and "lens", the text lengths.  `kw`: generate_codes's `generator`, `settle`
        and `info`."""
        ids = [self.encode_text(t) for t in texts]
        trace = None
        if trace_out is not None:
            lens = [int(x.numel()) for x in ids]
            trace = TS.trace_buffer(self.cfg, gen.max_frames + 1, len(ids), max(lens), self.device)
            trace_out["probs"], trace_out["lens"] = trace, lens
        return self.model.generate_codes(ids, ref, gen=gen, seeds=seeds, attn_trace=trace, **kw)

    def _decode_chunks(self, codes: Optional[torch.Tensor], Ts: Sequence[int]) -> Iterator[Tuple[List[int], torch.Tensor, List[int]]]:
        """Padded Mimi decodes of the utterances with frames -> yields (indices, wav [rows, 1, L], valid samples per
        row), longest utterances first.  The padding past Ts[i] * hop holds decoded filler: every stage after the decode
        takes the lens so it never reads it."""
        if codes is None:
            return
        # Mimi decode is causal and per-utterance: right-pad to the longest of a chunk, decode together, cut
        live = sorted((i for i in range(len(Ts)) if Ts[i] > 0), key=lambda i: -Ts[i])
        hop = self.codec.engine.hop
        cap = 12800  # frames per decode call (workspace bound)
        while live:
            chunk, frames = [], 0
            while live and (not chunk or (len(chunk) + 1) * max(frames, Ts[live[0]]) <= cap):
                frames = max(frames, Ts[live[0]])
                chunk.append(live.pop(0))
            idx = torch.tensor(chunk, device=self.device)
            batch = codes[idx, :frames].permute(0, 2, 1).to(torch.int32)
            keep = torch.arange(frames, device=self.device)[None, :] < torch.tensor([Ts[i] for i in chunk], device=self.device)[:, None]
            batch = (batch * keep[:, None, :]).contiguous()  # padding frames decode code 0; their samples are cut by lens
            yield chunk, self.codec.engine.decode(batch), [Ts[i] * hop for i in chunk]

    # the reference's module-level streaming.stream (reference streaming.py:134-143), a method here
    stream = S.stream

    def stream_batch(self, texts: Sequence[str], *, ref: Union[PreparedReference, Sequence[PreparedReference]],
                     seeds: Optional[Sequence[int]] = None, max_frames: int = 400, top_p: float = 0.9,
                     temperature: float = 1.05, anti_loop: bool = True, style_strength: Optional[float] = None,
                     min_gen_frames: Optional[int] = None, chunk_frames: int = 6, nar_context_frames: Optional[int] = None,
                     sample_rate: Optional[int] = None, speed: Optional[float] = None,
                     watermark: Optional[int] = None, word_timestamps: bool = False) -> Iterator[tuple]:
        """NEW: many texts streamed side by side through one chunk loop (sopro_b200/streaming.py): one AR launch of
        `chunk_frames` frames for every row, one ragged NAR pass and one batched Mimi stream step per chunk.  Yields
        ``(i, wav [1, n] on the device at the output rate, last)``; within a chunk the rows come in index order.  Row i
        yields its non-empty chunks in order, then exactly one item with last=True, which carries the tails of its
        output chain and may be [1, 0].  `ref`: one prepared voice for every text, or one per text (as in
        synthesize_batch); the sampling settings are shared.  With `seeds`, row i's chunks equal
        ``list(stream(texts[i], ref=ref[i] (or ref), seed=seeds[i], ...))`` bit for bit, the last item being the stream's
        final chunk (or empty when the stream yielded nothing more).  Without seeds the rows draw their noise as
        synthesize_batch(texts) does, every tape in full, row after row, from the global generator; that draw happens
        before the first AR launch, so time to first audio wants seeds (one text behaves exactly as stream(), generator
        included).  There is no loudness (it needs the whole utterance) or best_of (see stream).  `word_timestamps=True`
        yields ``(i, wav, last, words)``: row i's words that became final since its previous item (see stream).
        Refused before any device work or random draw: empty `texts`, `seeds` of another length, a wrong `ref`
        sequence, `chunk_frames` outside [1, 256], a refused sample_rate / speed / watermark, more texts than
        min(the AR batch limit, 256), a non-bool `word_timestamps`, and with it a text over 2048 tokens.  Closing the generator early releases its AR session, noise tapes, Mimi state and
        output-chain states."""
        texts, seeds = _check_texts(texts, seeds)
        limit = self._batch_limit()
        limit = S.MAX_STREAM_ROWS if limit is None else min(int(limit), S.MAX_STREAM_ROWS)
        if len(texts) > limit:
            raise ValueError(f"{len(texts)} texts; stream_batch streams at most {limit} side by side on this device")
        voices.check_voices(ref, len(texts), **voices.geometry(self.cfg))
        S._check_chunk_frames(chunk_frames)
        spans = S._word_spans(self, texts, word_timestamps)
        post = OutputChain(self, sample_rate, speed, watermark=watermark)
        gen = Generation.resolve(self.cfg, max_frames=max_frames, top_p=top_p, temperature=temperature,
                                 anti_loop=anti_loop, style_strength=style_strength, min_gen_frames=min_gen_frames)
        dec = S._decoder(self, chunk_frames)

        def rows_of():
            ids = [self.encode_text(t) for t in texts]
            rows = S._chunk_loop(self, dec, ids, ref, post, gen=gen, chunk_frames=chunk_frames,
                                 nar_context_frames=nar_context_frames, seeds=seeds,
                                 word_texts=None if spans is None else texts, word_spans=spans)
            try:
                for i, wav, last, words in rows:
                    wav = wav if wav is not None else torch.zeros(1, 0, device=self.device)
                    yield (i, wav, last) if spans is None else (i, wav, last, words)
            finally:
                rows.close()

        return rows_of()

    def stream_long(self, text: str, *, ref: PreparedReference, seed: Optional[int] = None, max_frames: int = 400,
                    max_tokens: int = 64, pause_ms: float = 250, top_p: float = 0.9, temperature: float = 1.05,
                    anti_loop: bool = True, style_strength: Optional[float] = None, min_gen_frames: Optional[int] = None,
                    chunk_frames: int = 6, nar_context_frames: Optional[int] = None, sample_rate: Optional[int] = None,
                    speed: Optional[float] = None, watermark: Optional[int] = None) -> Iterator[torch.Tensor]:
        """NEW: a text of any length, streamed -> chunks [1, n] f32 on the device at the output rate.  The segments are
        synthesize_long's (split_text, `max_tokens`), streamed side by side SEGMENT_GROUP at a time through
        stream_batch's chunk loop (segment i with seed seed + i; without a seed each group draws from the global
        generator as stream_batch of the group does).  Each segment's decoded audio is trimmed as it arrives and the
        spans are joined with `pause_ms` of silence and 10 ms raised-cosine edges, on the GPU
        (sopro_b200/longform.py::StreamJoin); the joined 24 kHz passage goes through one stretch -> watermark ->
        resample stream (`speed`, `watermark`, `sample_rate`).  The chunks concatenate to synthesize_long's join of the
        segments' streamed audio bit for bit whenever no 25 ms frame of a segment is above full scale; a louder segment
        is trimmed by the causal rule of include/sopro_b200.h.  A segment's audio comes out once its trim is certain:
        about 0.5 s past its first voiced frame.  Each resumption runs at most one AR chunk; an item holds at most
        chunk_frames x 1920 samples of the 24 kHz passage.  There is no loudness (it needs the whole passage), best_of
        or word_timestamps.  Refused before any device work or random draw: a text with nothing to speak, `pause_ms`
        or `max_tokens` out of range, `chunk_frames` outside [1, 256], a refused sample_rate / speed / watermark.
        Closing the generator early releases its AR session, noise tapes, Mimi state, trim state and chain states."""
        post = OutputChain(self, sample_rate, speed, watermark=watermark)
        pause = LF.pause_samples(pause_ms)
        budget = LF.check_max_tokens(max_tokens, self.model.prefill.max_text_len)
        S._check_chunk_frames(chunk_frames)
        segments = LF.passage_segments(text, self.tokenizer, budget)
        gen = Generation.resolve(self.cfg, max_frames=max_frames, top_p=top_p, temperature=temperature,
                                 anti_loop=anti_loop, style_strength=style_strength, min_gen_frames=min_gen_frames)
        return S._stream_passage(self, segments, ref, post, pause, seed=seed, gen=gen, chunk_frames=chunk_frames,
                                 nar_context_frames=nar_context_frames)

    def stream_dialogue(self, turns: Sequence[Tuple[PreparedReference, str]], *, seed: Optional[int] = None,
                        pause_ms: float = 250, turn_pause_ms: float = 500, max_frames: int = 400, max_tokens: int = 64,
                        top_p: float = 0.9, temperature: float = 1.05, anti_loop: bool = True,
                        style_strength: Optional[float] = None, min_gen_frames: Optional[int] = None,
                        chunk_frames: int = 6, nar_context_frames: Optional[int] = None,
                        sample_rate: Optional[int] = None, speed: Optional[float] = None,
                        watermark: Optional[int] = None) -> Iterator[torch.Tensor]:
        """NEW: a script of ``(voice, text)`` turns, streamed -> chunks [1, n] f32 on the device at the output rate.
        stream_long's passage loop over synthesize_dialogue's segments, each streamed in its turn's voice (segment k
        with seed seed + k), joined as they arrive with synthesize_dialogue's gaps.  The chunks concatenate to the
        dialogue join of the segments' streamed audio bit for bit under stream_long's condition (no 25 ms frame of a
        segment above full scale).  There is no loudness (levelling needs a whole turn), best_of or word_timestamps.
        Refused before any device work or random draw: what synthesize_dialogue refuses, and `chunk_frames` outside
        [1, 256].  Closing the generator early releases its AR session, noise tapes, Mimi state, trim state and chain
        states."""
        _turns, segments, turn_of, voice_of, pause, turn_pause = D.check_script(self, turns, pause_ms, turn_pause_ms,
                                                                                max_tokens)
        S._check_chunk_frames(chunk_frames)
        post = OutputChain(self, sample_rate, speed, watermark=watermark)
        gen = Generation.resolve(self.cfg, max_frames=max_frames, top_p=top_p, temperature=temperature,
                                 anti_loop=anti_loop, style_strength=style_strength, min_gen_frames=min_gen_frames)
        return S._stream_passage(self, segments, D.segment_voices(voice_of), post, pause, turn_of=turn_of,
                                 turn_pause=turn_pause, seed=seed, gen=gen, chunk_frames=chunk_frames, nar_context_frames=nar_context_frames)

    def save_wav(self, path: str, wav_1xT: torch.Tensor, sample_rate: int = TARGET_SR) -> None:
        """`sample_rate`: the rate the waveform is at (the one passed to synthesize / stream)."""
        from .audio import save_audio

        save_audio(path, wav_1xT, sr=int(sample_rate))

    def save_flac(self, path: str, wav_1xT: torch.Tensor, sample_rate: int = TARGET_SR) -> None:
        """Writes the waveform (one row on the device) as a lossless 16-bit FLAC file, encoded on the GPU
        (sopro_b200/flac.py); `sample_rate`: the rate the waveform is at."""
        from .flac import encode_flac

        data = encode_flac(wav_1xT, sample_rate)
        with open(path, "wb") as f:
            f.write(data)

    def _resampler(self, sample_rate: Optional[int]) -> Optional[Resampler]:
        """None for the codec's own 24 kHz (no launch); otherwise this rate's cached resampler.  A refused rate raises
        ValueError here, before a caller has consumed any random draws."""
        if sample_rate is None or (not isinstance(sample_rate, bool) and sample_rate == TARGET_SR):
            return None
        sr = check_rates(TARGET_SR, sample_rate)[1]
        rs = self._resamplers.get(sr)
        if rs is None:
            rs = self._resamplers[sr] = Resampler(TARGET_SR, sr, self.device)
        return rs
