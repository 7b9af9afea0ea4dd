"""Chunked streaming synthesis (reference streaming.py:12-152): every ``chunk_frames`` AR tokens the NAR refiner
runs over the new frames plus ``rf_nar`` frames of left context and the Mimi stream decoder emits their audio.
The AR kernel is launched ``chunk_frames`` frames at a time, so time-to-first-audio is prefill + one short
persistent launch + one NAR window + one Mimi decode."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Iterator, List, Optional

import torch

from .codec import MimiDecodeState, MimiStreamDecoder
from .output import OutputChain
from .prefill import PreparedReference


@dataclass
class StreamConfig:
    chunk_frames: int = 16
    nar_context_frames: Optional[int] = None


class SoproTTSStreamer:
    """Pipelined chunk loop.  Per chunk k, in device order:  AR(k) -> [NAR window + Mimi step](k) -> AR(k+1) -> ...
    The host enqueues NAR + Mimi of chunk k on a side stream, then immediately enqueues AR(k+1) behind them (an event
    keeps the persistent kernel, which takes every SM, from cutting in front of chunk k's audio), and only then waits
    for chunk k's samples and yields them: the next AR launch runs while the consumer handles the audio, and the device
    never waits for the host between launches.  The reference runs the three stages strictly in turn on one thread
    (streaming.py:81-130)."""

    def __init__(self, tts, cfg: Optional[StreamConfig] = None):
        self.tts = tts
        self.cfg = cfg or StreamConfig()
        # one decoder (= one pool of device stream states) per SoproTTS: a finished utterance's state is reset and reused by
        # the next stream() instead of a 0.8 ms allocation + memset on the time-to-first-audio path
        need = max(16, int(self.cfg.chunk_frames))
        dec = getattr(tts, "_stream_decoder", None)
        if dec is None or dec.max_chunk_frames < need or dec.codec is not tts.codec:
            dec = MimiStreamDecoder(tts.codec, max_chunk_frames=need)
            try:
                tts._stream_decoder = dec
            except Exception:
                pass
        self.mimi_stream = dec

    @torch.inference_mode()
    def stream(self, text: str, *, ref_audio_path: Optional[str] = None, ref_tokens_tq: Optional[torch.Tensor] = None,
               ref: Optional[PreparedReference] = None, max_frames: int = 400, top_p: float = 0.9, temperature: float = 1.05,
               anti_loop: bool = True, style_strength: Optional[float] = None, ref_seconds: Optional[float] = None,
               chunk_frames: Optional[int] = None, nar_context_frames: Optional[int] = None,
               min_gen_frames: Optional[int] = None, seed: Optional[int] = None,
               generator: Optional[torch.Generator] = None, sample_rate: Optional[int] = None,
               speed: Optional[float] = None, watermark: Optional[int] = None) -> Iterator[torch.Tensor]:
        """`sample_rate` (extension): chunks at this rate (None = 24 kHz).  `speed` (extension): the speaking rate in
        [0.25, 4.0] (None = the model's own).  `watermark` (extension): a key in [0, 2^32) to mark the audio with (None =
        no mark).  Each chunk's audio goes through a time-stretch stream, a watermark stream, then a resampler stream,
        right after its Mimi step, so the chunks concatenate to the one-shot stretch, mark and resample of the 24 kHz
        stream bit for bit; the last chunk also carries their tails."""
        tts, model = self.tts, self.tts.model
        post = OutputChain(tts, sample_rate, speed, watermark=watermark)  # a refused argument raises before the prefill
        text_ids = tts.encode_text(text)
        if ref is None:
            ref = tts.prepare_reference(ref_audio_path=ref_audio_path, ref_tokens_tq=ref_tokens_tq, ref_seconds=ref_seconds)
        prep = model.prepare_conditioning(
            text_ids, ref, max_frames=max_frames,
            style_strength=float(style_strength if style_strength is not None else tts.cfg.style_strength))
        cf = int(chunk_frames if chunk_frames is not None else self.cfg.chunk_frames)
        ctx = nar_context_frames if nar_context_frames is not None else self.cfg.nar_context_frames
        ctx = int(model.rf_nar() if ctx is None else ctx)
        hist: List[int] = []
        emitted = 0
        state = self.mimi_stream.new_state()
        # the stretch / resampler states' pushes are bounded by one chunk's samples
        post_state = post.stream(self.mimi_stream.max_chunk_frames * tts.codec.engine.hop)
        on_gpu = tts.device.type == "cuda"
        main = torch.cuda.current_stream(tts.device) if on_gpu else None
        side = torch.cuda.Stream(tts.device) if on_gpu else None

        def refine_and_emit(end: int, last: bool) -> Optional[torch.Tensor]:
            """NAR over the new frames + `ctx` frames of left context, Mimi stream step on the new frames' codes
            (reference streaming.py:81-104), then the stretch and resampler pushes (and, on the last chunk, their
            finishes); enqueued on the side stream."""
            nonlocal emitted, state
            wav = None
            if end > emitted:
                lo = max(0, emitted - ctx)
                toks = torch.as_tensor(hist[lo:end], device=tts.device, dtype=torch.long).unsqueeze(0)
                win = model.nar_refine(prep["cond_ar"][:, lo:end, :], toks).squeeze(0)
                wav, state = self.mimi_stream.decode_step(win[emitted - lo:, :], state, _trusted=True)  # our own NAR's codes
                emitted = end
            wav = post_state.finish(wav) if last else post_state.push(wav)
            return wav if wav is not None and wav.numel() > 0 else None

        progress = {"consumed": 0}
        chunks = model.ar_chunks(prep, max_frames=max_frames, chunk_frames=cf, top_p=top_p, temperature=temperature,
                                 anti_loop=anti_loop, min_gen_frames=min_gen_frames, seed=seed, generator=generator,
                                 progress=progress)
        try:
            for toks, finished, prefetch in chunks:
                # the stream ends at the first EOS regardless of min_gen_frames (reference streaming.py:114-115)
                stop = model.eos_id in toks
                if stop:
                    toks = toks[: toks.index(model.eos_id)]
                progress["consumed"] += len(toks) + (1 if stop else 0)  # the reference also draws for the EOS step
                hist.extend(toks)
                last = stop or finished
                end = len(hist) if last else (len(hist) // cf) * cf
                wav = None
                if on_gpu:
                    side.wait_stream(main)
                    with torch.cuda.stream(side):
                        wav = refine_and_emit(end, last)
                    if not last:
                        main.wait_stream(side)  # AR(k+1) behind chunk k's NAR + Mimi, never in front of them
                        prefetch()
                    side.synchronize()
                    if wav is not None:
                        wav.record_stream(main)
                else:
                    wav = refine_and_emit(end, last)
                if wav is not None:
                    yield wav
                if last:
                    break
        finally:
            chunks.close()
            self.mimi_stream.release(state)
            post_state.release()


@torch.inference_mode()
def stream(tts, text: str, *, ref_audio_path: Optional[str] = None, ref_tokens_tq: Optional[torch.Tensor] = None,
           ref: Optional[PreparedReference] = None, chunk_frames: int = 6, sample_rate: Optional[int] = None,
           speed: Optional[float] = None, watermark: Optional[int] = None, **kwargs) -> Iterator[torch.Tensor]:
    OutputChain(tts, sample_rate, speed, watermark=watermark)  # a refused argument raises at the call, not at the first chunk
    streamer = SoproTTSStreamer(tts, StreamConfig(chunk_frames=chunk_frames))
    return streamer.stream(text, ref_audio_path=ref_audio_path, ref_tokens_tq=ref_tokens_tq, ref=ref,
                           chunk_frames=chunk_frames, sample_rate=sample_rate, speed=speed, watermark=watermark, **kwargs)
