"""Chunked streaming synthesis (reference streaming.py:12-152): every ``chunk_frames`` AR tokens the NAR refiner
runs over the new frames plus ``rf_nar`` frames of left context and the Mimi stream decoder emits their audio.
The AR kernel is launched ``chunk_frames`` frames at a time, so time-to-first-audio is prefill + one short
persistent launch + one NAR window + one Mimi decode.

``stream`` (SoproTTS.stream) and SoproTTS's other streaming entry points (sopro_b200/model.py) check and resolve their
arguments, then run the loops here.  ``stream`` and ``stream_batch`` run one chunk loop (``_chunk_loop``), pipelined.
Per chunk k, in device order: AR(k) -> [NAR window + Mimi step](k) -> AR(k+1) -> ...  The host enqueues NAR + Mimi of
chunk k on a side stream, then immediately enqueues AR(k+1) behind them (an event keeps the persistent kernel, which
takes every SM, from cutting in front of chunk k's audio), and only then waits for chunk k's samples and yields them:
the next AR launch runs while the consumer handles the audio, and the device never waits for the host between
launches.  The reference runs the three stages strictly in turn on one thread (streaming.py:81-130)."""
from __future__ import annotations

from typing import Callable, Iterator, List, Optional, Sequence, Tuple

import torch

from .codec import MimiStreamDecoder
from .engine import Generation
from .output import OutputChain
from .prefill import PreparedReference


def stream(tts, text: str, *, ref_audio_path: Optional[str] = None, ref_tokens_tq: Optional[torch.Tensor] = None,
           ref: Optional[PreparedReference] = None, max_frames: int = 400, top_p: float = 0.9,
           temperature: float = 1.05, anti_loop: bool = True, style_strength: Optional[float] = None,
           ref_seconds: Optional[float] = None, chunk_frames: int = 6, nar_context_frames: Optional[int] = None,
           min_gen_frames: Optional[int] = None, seed: Optional[int] = None,
           generator: Optional[torch.Generator] = None, sample_rate: Optional[int] = None,
           speed: Optional[float] = None, watermark: Optional[int] = None,
           word_timestamps: bool = False) -> Iterator[torch.Tensor]:
    """SoproTTS.stream: chunks [1, n] of one utterance as they are generated, through the chunk loop below.
    `sample_rate` (extension): chunks at this rate (None = 24 kHz).  `speed` (extension): the speaking rate in
    [0.25, 4.0] (None = the model's own).  `watermark` (extension): a key in [0, 2^32) to mark the audio with (None =
    no mark).  Each chunk's audio goes through a time-stretch stream, a watermark stream, then a resampler stream,
    right after its Mimi step, so the chunks concatenate to the one-shot stretch, mark and resample of the 24 kHz
    stream bit for bit; the last chunk also carries their tails.  A refused sample_rate / speed / watermark raises
    here, at the call, not at the first chunk.  There is no `best_of` here: a stream plays its take while it is
    generated, so it cannot choose among takes before playing one.  `word_timestamps=True` (extension) yields
    ``(wav, words)``: the words that became final since the previous item, aligned causally on the GPU
    (sopro_b200/timestamps.py, lag STREAM_ALIGN_LAG frames); times are seconds of this stream's audio, scaled by
    `speed` as in synthesize.  If words are still pending when the stream ends without more audio, the last item is
    ``([1, 0] wav, words)``.  The chunks are the same as without it."""
    spans = _word_spans(tts, [text], word_timestamps)
    post = OutputChain(tts, sample_rate, speed, watermark=watermark)
    gen = Generation.resolve(tts.cfg, max_frames=max_frames, top_p=top_p, temperature=temperature,
                             anti_loop=anti_loop, style_strength=style_strength, min_gen_frames=min_gen_frames)
    dec = _decoder(tts, chunk_frames)

    @torch.inference_mode()
    def chunks():
        voice = ref
        if voice is None:
            voice = tts.prepare_reference(ref_audio_path=ref_audio_path, ref_tokens_tq=ref_tokens_tq,
                                          ref_seconds=ref_seconds)
        rows = _chunk_loop(tts, dec, [tts.encode_text(text)], voice, post, gen=gen, chunk_frames=chunk_frames,
                           nar_context_frames=nar_context_frames, seeds=None if seed is None else [seed],
                           generator=generator, word_texts=None if spans is None else [text], word_spans=spans)
        try:
            for _i, wav, last, words in rows:
                if spans is None:
                    if wav is not None:
                        yield wav
                elif wav is not None:
                    yield wav, words
                elif last and words:
                    yield torch.zeros(1, 0, device=tts.device), words
        finally:
            rows.close()

    return chunks()


MAX_STREAM_ROWS = 256  # a Mimi stream state holds tens of MB per row (DESIGN.md §5o)


def _stream_passage(tts, segments: Sequence[str], ref, post: OutputChain, P: int, *,
                    turn_of: Optional[Sequence[int]] = None, turn_pause: int = 0, seed: Optional[int], gen: Generation,
                    chunk_frames: int, nar_context_frames: Optional[int]):
    """The passage loop of stream_long and stream_dialogue over checked arguments -> the generator of the passage's
    chunks.  `ref`: one voice, or one per segment; `turn_of` / `turn_pause`: the dialogue's gaps
    (longform.gap_pauses), None for one turn.

    The segments run SEGMENT_GROUP at a time, each group through one chunk loop whose decoded blocks go to the
    streaming trim (longform.StreamJoin) instead of an output chain; the joined 24 kHz passage goes through one
    output-chain stream.  Each resumption runs at most one AR chunk, then yields the next piece of the passage (at most
    chunk_frames x 1920 samples of it before the chain); it runs more chunks only while nothing is certain yet.  A
    group starts at the first resumption after the group before it has ended and the group before that has been
    emitted (the trim state holds two groups)."""
    from . import longform as LF

    B, G = len(segments), int(LF.SEGMENT_GROUP)
    one = isinstance(ref, PreparedReference)
    hop = tts.codec.engine.hop
    limit = int(chunk_frames) * hop
    dec = _decoder(tts, chunk_frames)
    bypass = OutputChain(tts)

    @torch.inference_mode()
    def passage():
        join = tts._join_pool.checkout(LF.StreamJoin.rows_for(B, G), (gen.max_frames + 1) * hop)
        join.begin(B, P, G, turn_of, turn_pause)
        out = post.stream(limit)
        main = torch.cuda.current_stream(tts.device)
        emit = torch.cuda.Stream(tts.device)  # the pieces and the chain: never queued behind the next AR launch
        loop = None

        def start(g0):
            part = segments[g0: g0 + G]
            join.start_group(g0, len(part))
            voice = ref if one else list(ref[g0: g0 + G])
            return _chunk_loop(tts, dec, [tts.encode_text(t) for t in part], voice, bypass, gen=gen,
                               chunk_frames=chunk_frames, nar_context_frames=nar_context_frames,
                               seeds=None if seed is None else [int(seed) + g0 + i for i in range(len(part))],
                               on_block=join.push)

        def chunk() -> bool:
            """One AR chunk of the group being generated (starting the next group when it may); False when there is
            nothing to run."""
            nonlocal loop
            if loop is None:
                if not join.can_start(join.started):
                    return False
                loop = start(join.started)
            k = join.pushes
            for _ in loop:  # the launch's items: the trim stage has its block (and the status is on the host)
                if join.pushes > k:
                    break
            if join.group_final():
                for _ in loop:  # the rest of the last launch's items; the loop then releases its session and state
                    pass
                loop.close()
                loop = None
            return join.pushes > k

        def piece() -> Optional[torch.Tensor]:
            """The next non-empty item through the chain, from what is certain now (None: nothing is)."""
            with torch.cuda.stream(emit):  # (what it reads was pushed on a stream the loop has synchronised)
                while True:
                    y = join.take(limit)
                    if y is None:
                        return None
                    y = out.push(y)
                    if y.numel():
                        break
            y.record_stream(main)
            main.wait_stream(emit)
            return y

        try:
            while True:
                chunk()
                y = piece()
                while y is None and not join.done():
                    if not chunk():
                        raise RuntimeError("the passage has nothing to run and nothing certain to emit")
                    y = piece()
                if y is None:
                    break
                yield y
            with torch.cuda.stream(emit):
                tail = out.finish()
            if tail is not None and tail.numel():
                tail.record_stream(main)
                main.wait_stream(emit)
                yield tail
        finally:
            if loop is not None:
                loop.close()
            out.release()
            tts._join_pool.release(join)

    return passage()


def _word_spans(tts, texts: Sequence[str], word_timestamps) -> Optional[list]:
    """`word_timestamps` checked -> the texts' token character spans (None without it).  Host work only."""
    from .timestamps import MAX_TOKENS, check_word_timestamps

    if not check_word_timestamps(word_timestamps):
        return None
    spans = [tts.tokenizer.encode_with_offsets(t)[1] for t in texts]
    for i, sp in enumerate(spans):
        if len(sp) > MAX_TOKENS:
            raise ValueError(f"text {i} has {len(sp)} tokens; word timestamps align at most {MAX_TOKENS}")
    return spans


def _check_chunk_frames(chunk_frames) -> None:
    if isinstance(chunk_frames, bool) or not isinstance(chunk_frames, int):
        raise TypeError(f"chunk_frames must be an int, got {type(chunk_frames).__name__}")
    if not 1 <= chunk_frames <= 256:
        raise ValueError(f"chunk_frames must be in [1, 256], got {chunk_frames}")


def _decoder(tts, chunk_frames) -> MimiStreamDecoder:
    """The SoproTTS's one stream decoder (one pool of device stream states: a finished utterance's state is reset and
    reused by the next stream instead of a 0.8 ms allocation + memset on the time-to-first-audio path), made on first
    use and replaced by a larger one when `chunk_frames` exceeds its chunk size."""
    need = max(16, int(chunk_frames))
    if tts._stream_decoder is None or tts._stream_decoder.max_chunk_frames < need:
        tts._stream_decoder = MimiStreamDecoder(tts.codec, max_chunk_frames=need)
    return tts._stream_decoder


@torch.inference_mode()
def _chunk_loop(tts, dec: MimiStreamDecoder, text_ids: Sequence[torch.Tensor], ref, post: OutputChain, *,
                gen: Generation, chunk_frames: int, nar_context_frames: Optional[int],
                seeds: Optional[Sequence[int]], generator: Optional[torch.Generator] = None,
                on_block: Optional[Callable[[Optional[torch.Tensor], List[int], List[bool]], None]] = None,
                word_texts: Optional[Sequence[str]] = None, word_spans: Optional[Sequence[Sequence]] = None
                ) -> Iterator[Tuple[int, Optional[torch.Tensor], bool, Optional[list]]]:
    """The chunk loop of B utterances (`ref`: one prepared voice, or one per text) -> ``(i, wav or None, last, words)``:
    per launch, in row order, each live row's chunk (None when it has no samples), the row's last item once with
    last=True.  All rows advance in lockstep, `chunk_frames` AR frames per launch, so the NAR window [lo, end) is
    shared by the live rows (only a row that ends in this launch has a shorter one) and runs as one ragged NAR pass;
    one Mimi step decodes every row (a row that has ended is fed code 0 and its samples are dropped), then each row's
    samples go through its own output-chain stream.  Row i's chunks are those of this loop over text i alone.
    `on_block` (stream_long's trim stage): called once per launch, on the stream the launch's Mimi step ran on, with
    the step's decoded block [B, L] (None when nothing was decoded), each row's new samples in it (0 for a row that
    did not run) and whether each row ends with this launch; the loop synchronises that stream before it yields the
    launch's items.  `word_texts` / `word_spans` (word timestamps): the texts and their tokens' character spans; the
    AR launches then write their attention weights into a ring of `chunk_frames` steps, each launch's new frames are
    aligned by one push of a timestamps.StreamAligner on the side stream ahead of that launch's NAR and Mimi step (the
    main stream's wait for the side stream orders it before the next launch overwrites the ring), and each item's
    fourth element is the list of the row's words that became final since its previous item (None without them)."""
    model = tts.model
    B = len(text_ids)
    txt, lens, _pool, cond = model.prefill.run(list(text_ids), ref, n_frames=gen.max_frames + 1,
                                               style_strength=gen.style_strength)
    cf = int(chunk_frames)
    ctx = int(model.rf_nar() if nar_context_frames is None else nar_context_frames)
    hop = tts.codec.engine.hop
    hist: List[List[int]] = [[] for _ in range(B)]
    ended = [False] * B
    emitted = 0
    state = dec.new_state(B)
    # the stretch / resampler states' pushes are bounded by one chunk's samples
    posts = []
    on_gpu = tts.device.type == "cuda"
    main = torch.cuda.current_stream(tts.device) if on_gpu else None
    side = torch.cuda.Stream(tts.device) if on_gpu else None

    def refine_and_emit(ends: List[int], last: List[bool], live: List[int]) -> List[Optional[torch.Tensor]]:
        """NAR over the new frames + `ctx` frames of left context, Mimi stream step on the new frames' codes
        (reference streaming.py:81-104), then each live row's stretch and resampler pushes (and, on its last chunk,
        their finishes); enqueued on the side stream."""
        nonlocal emitted, state
        out: List[Optional[torch.Tensor]] = [None] * B
        end = max(ends[b] for b in live)
        rows_wav = None
        if end > emitted:
            lo = max(0, emitted - ctx)
            run = [b for b in live if ends[b] > emitted]
            sel = slice(None) if len(run) == B else torch.tensor(run, device=tts.device)
            toks = torch.tensor([hist[b][lo:ends[b]] + [0] * (end - ends[b]) for b in run], dtype=torch.long,
                                device=tts.device)
            win = model.nar_refine(cond[sel, lo:end, :], toks,
                                   lens=torch.tensor([ends[b] - lo for b in run], dtype=torch.int32))
            codes = win[:, emitted - lo:, :]
            n = end - emitted
            if any(e < end for e in ends):  # a row ended before this window's end: its frames decode code 0
                keep = (torch.arange(n)[None, :] < torch.tensor([ends[b] - emitted for b in run])[:, None]).to(tts.device)
                codes, part = torch.zeros((B, n, win.shape[2]), dtype=torch.long, device=tts.device), codes
                codes[sel] = part * keep[:, :, None]
            rows_wav, state = dec.decode_step(codes, state, _trusted=True)  # our own NAR's codes
        if on_block is not None:
            on_block(rows_wav, [(ends[b] - emitted) * hop if rows_wav is not None and ends[b] > emitted else 0
                                for b in range(B)], last)
        for b in live:
            wav = rows_wav[b: b + 1, : (ends[b] - emitted) * hop] if rows_wav is not None and ends[b] > emitted else None
            wav = posts[b].finish(wav) if last[b] else posts[b].push(wav)
            out[b] = wav if wav is not None and wav.numel() > 0 else None
        emitted = end
        return out

    aligner = None
    if word_spans is not None:
        from .timestamps import StreamAligner

        aligner = StreamAligner(tts.cfg, word_texts, word_spans, ring=cf, max_frames=gen.max_frames + 1, hop=hop,
                                S=post.S, device=tts.device)
    pending: List[list] = [[] for _ in range(B)]
    progress = {"consumed": 0}
    chunks = model.ar_chunk_rows(cond, txt, lens, gen=gen, chunk_frames=cf, seeds=seeds, generator=generator,
                                 progress=progress,
                                 attn_trace=None if aligner is None else aligner.ring,
                                 attn_ring=None if aligner is None else cf)
    try:
        for _ in range(B):
            posts.append(post.stream(dec.max_chunk_frames * hop))
        for toks_rows, finished, prefetch in chunks:
            live = [b for b in range(B) if not ended[b]]
            ends, last, new = [0] * B, [False] * B, [0] * B
            for b in live:
                toks = toks_rows[b]
                # the stream ends at the first EOS, even before the minimum frame count (reference streaming.py:114-115)
                stop = model.eos_id in toks
                if stop:
                    toks = toks[: toks.index(model.eos_id)]
                progress["consumed"] += len(toks) + (1 if stop else 0)  # the reference also draws for the EOS step
                hist[b].extend(toks)
                new[b] = len(toks)
                last[b] = stop or finished[b]
                ends[b] = len(hist[b]) if last[b] else (len(hist[b]) // cf) * cf
            done = all(last[b] for b in live)
            if on_gpu:
                side.wait_stream(main)
                with torch.cuda.stream(side):
                    if aligner is not None:
                        aligner.push(new, last)
                    wavs = refine_and_emit(ends, last, live)
                if not done:
                    main.wait_stream(side)  # AR(k+1) behind chunk k's NAR + Mimi, never in front of them
                    prefetch()
                side.synchronize()
                for w in wavs:
                    if w is not None:
                        w.record_stream(main)
            else:
                wavs = refine_and_emit(ends, last, live)
            for b in live:
                if aligner is not None:
                    pending[b] += aligner.take(b)
                if wavs[b] is not None or last[b]:
                    words, pending[b] = (pending[b], []) if aligner is not None else (None, pending[b])
                    yield b, wavs[b], last[b], words
                ended[b] = last[b]
            if done:
                break
    finally:
        chunks.close()
        if aligner is not None:
            aligner.close()
        dec.release(state)
        for p in posts:
            p.release()
