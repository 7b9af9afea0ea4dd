"""Batched streaming on the GPU (bench.py's workload: synthetic seeded checkpoint, bf16 AR weights, EOS logit pushed
down so every utterance runs the full 401 AR steps, 52-id texts, one prepared voice; nothing is written):
  - stream_batch of B in {1, 8, 64} texts (400 frames, min_gen_frames=10**9, chunk_frames=6, seeded), and of 64 texts
    in 64 voices: time from the call to each row's first chunk (p50 / p90 over rows and runs), time to finish all
    rows, audio seconds produced per wall second;
  - the same B texts as B stream() generators served round-robin (how a server serves B clients with stream()), and as
    B stream() calls one after another;
  - one chunk split into AR launch, NAR window, Mimi step and output chain with CUDA events recorded around each call
    on the stream it is enqueued on (a separate, traced run; with and without a 16 kHz output rate);
  - the Mimi stream state's device bytes per row.
Host clock around calls that end in a device synchronise.  Prints one JSON object with the card's name, power limit
and SM clocks read in the same run.

  python tools/prof_stream_batch.py [--runs N] [--batches 1,8,64]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
FRAMES, CF = 400, 6


def card():
    import torch

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def build_tts():
    import torch

    import bench
    from sopro_b200 import SoproTTS
    from sopro_b200.config import SoproTTSConfig
    from sopro_b200.tokenizer import IdsTokenizer
    from sopro_b200.weights import synth_mimi_state_dict

    torch.set_grad_enabled(False)
    cfg = SoproTTSConfig()
    tts = SoproTTS.from_state_dict(cfg, bench.bench_state_dict(cfg), IdsTokenizer(bench.TEXT_VOCAB), synth_mimi_state_dict(),
                                   device="cuda:0", weight_dtype="bf16")
    return tts, bench


def run_batch(tts, texts, ref, seeds, **kw):
    """-> (first-chunk seconds per row, seconds to the end, audio seconds) of one stream_batch"""
    import torch

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    first, samples = [None] * len(texts), 0
    for i, w, _last in tts.stream_batch(texts, ref=ref, seeds=seeds, max_frames=FRAMES, min_gen_frames=10 ** 9,
                                        chunk_frames=CF, **kw):
        if first[i] is None and w.shape[1] > 0:
            first[i] = time.perf_counter() - t0
        samples += int(w.shape[1])
    torch.cuda.synchronize()
    return first, time.perf_counter() - t0, samples / 24000.0


def run_streams(tts, texts, ref, seeds, interleaved):
    """B stream() generators, round-robin or one after another -> same triple as run_batch"""
    import torch

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    first, samples = [None] * len(texts), 0
    gens = [tts.stream(t, ref=ref, seed=s, max_frames=FRAMES, min_gen_frames=10 ** 9, chunk_frames=CF) for t, s in zip(texts, seeds)]
    if interleaved:
        live = list(range(len(gens)))
        while live:
            for i in list(live):
                try:
                    w = next(gens[i])
                except StopIteration:
                    live.remove(i)
                    continue
                if first[i] is None:
                    first[i] = time.perf_counter() - t0
                samples += int(w.shape[1])
    else:
        for i, g in enumerate(gens):
            for w in g:
                if first[i] is None:
                    first[i] = time.perf_counter() - t0
                samples += int(w.shape[1])
    torch.cuda.synchronize()
    return first, time.perf_counter() - t0, samples / 24000.0


def summary(results):
    firsts = [f for r in results for f in r[0] if f is not None]
    ends = [r[1] for r in results]
    audio = results[0][2]
    return {"first_chunk_ms_p50": float(np.median(firsts)) * 1e3, "first_chunk_ms_p90": float(np.percentile(firsts, 90)) * 1e3,
            "all_rows_done_ms_p50": float(np.median(ends)) * 1e3, "audio_s": audio,
            "audio_s_per_wall_s": audio / float(np.median(ends)), "runs": len(results)}


def split(tts, texts, ref, seeds, **kw):
    """Device time per chunk of each stage, from CUDA events around every call on the stream it is enqueued on."""
    import torch

    from sopro_b200 import engine, output
    from sopro_b200.codec import MimiStreamDecoder

    marks = []

    def wrap(obj, name, cat):
        real = getattr(obj, name)

        def f(*a, **k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = real(*a, **k)
            e1.record()
            marks.append((cat, e0, e1))
            return r

        setattr(obj, name, f)
        return real

    saved = [(engine.ArSession, "run", wrap(engine.ArSession, "run", "ar_launch")),
             (MimiStreamDecoder, "decode_step", wrap(MimiStreamDecoder, "decode_step", "mimi_step")),
             (output.ChainStream, "push", wrap(output.ChainStream, "push", "output_chain")),
             (output.ChainStream, "finish", wrap(output.ChainStream, "finish", "output_chain"))]
    wrap(tts.model, "nar_refine", "nar_window")  # an instance attribute over the method, deleted afterwards
    try:
        run_batch(tts, texts, ref, seeds, **kw)
        torch.cuda.synchronize()
    finally:
        for obj, name, real in saved:
            setattr(obj, name, real)
        del tts.model.nar_refine
    chunks = -(-(FRAMES + 1) // CF)
    out = {}
    for cat, e0, e1 in marks:
        out[cat] = out.get(cat, 0.0) + e0.elapsed_time(e1)
    return {k: v / chunks for k, v in out.items()} | {"chunks": chunks}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--batches", default="1,8,64")
    args = ap.parse_args()
    import torch

    tts, bench = build_tts()
    out = {"card": card(), "workload": f"bench.py texts, {FRAMES} frames, chunk_frames={CF}, seeded, min_gen_frames=1e9"}
    one, two = tts.codec.engine.stream(16, rows=1), tts.codec.engine.stream(16, rows=2)
    out["mimi_state_bytes_per_row"] = {"rows1": one.state_bytes, "rows2_minus_rows1": two.state_bytes - one.state_bytes,
                                       "precision": tts.codec.engine.precision, "max_chunk_frames": 16}
    one.close()
    two.close()
    ref = tts.prepare_reference(ref_tokens_tq=bench.bench_ref_tokens())
    for B in [int(x) for x in args.batches.split(",")]:
        texts = bench.bench_texts(0, B)
        seeds = list(range(1234, 1234 + B))
        run_batch(tts, texts, ref, seeds)  # warm-up: sessions, pooled states
        row = {"stream_batch": summary([run_batch(tts, texts, ref, seeds) for _ in range(args.runs)])}
        n = 1 if B > 8 else args.runs
        run_streams(tts, texts[:1], ref, seeds[:1], True)
        row["stream_round_robin"] = summary([run_streams(tts, texts, ref, seeds, True) for _ in range(n)])
        row["stream_sequential"] = summary([run_streams(tts, texts, ref, seeds, False) for _ in range(n)])
        out[f"B{B}"] = row
        print(json.dumps({f"B{B}": row}), file=sys.stderr, flush=True)
    # 64 texts in 64 voices
    voices = [tts.prepare_reference(ref_tokens_tq=torch.randint(0, 2048, (bench.REF_FRAMES, 32), generator=torch.Generator().manual_seed(100 + i)))
              for i in range(64)]
    texts, seeds = bench.bench_texts(0, 64), list(range(1234, 1298))
    run_batch(tts, texts, voices, seeds)
    out["B64_64_voices"] = {"stream_batch": summary([run_batch(tts, texts, voices, seeds) for _ in range(args.runs)])}
    # per-chunk device split (traced runs, after the timed ones)
    for B in (1, 64):
        texts, seeds = bench.bench_texts(0, B), list(range(1234, 1234 + B))
        out[f"split_ms_per_chunk_B{B}"] = split(tts, texts, ref, seeds)
        out[f"split_ms_per_chunk_B{B}_16kHz"] = split(tts, texts, ref, seeds, sample_rate=16000)
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
