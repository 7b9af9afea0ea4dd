"""Long-form streaming on the GPU (bench.py's synthetic seeded checkpoint, bf16 AR weights, EOS logit pushed down so
every segment runs the full 401 AR steps, one prepared voice, chunk_frames=6; nothing is written):
  - stream_long of a passage of N in {1, 16, 64} segments (bench.py's 52-id texts as sentences): time from the call to
    the first item (p50 / p90 over runs), and to the end of the passage for a consumer that never waits;
  - synthesize_long of the same passage, and stream() of segment 0 alone (first chunk, end);
  - device time per chunk of the trim stage's push and emit at 64 rows, from CUDA events recorded around each call on
    the stream it is enqueued on (a separate, traced run).
Host clock around calls that end in a device synchronise.  Prints one JSON object with the card's name, power limit
and SM clocks read in the same run.

  python tools/prof_stream_long.py [--runs N] [--segments 1,16,64]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.prof_stream_batch import build_tts, card  # noqa: E402

FRAMES, CF = 400, 6
KW = dict(max_frames=FRAMES, min_gen_frames=10 ** 9)


def passage(bench, n):
    """n sentences of 52 ids: each one segment under the default 64-token budget"""
    return " ".join(t + "." for t in bench.bench_texts(0, n))


def timed(make):
    """-> (seconds to the first item, seconds to the end, items) of an iterator, consumed as fast as it comes"""
    import torch

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    first, n = None, 0
    for _ in make():
        if first is None:
            first = time.perf_counter() - t0
        n += 1
    torch.cuda.synchronize()
    return first, time.perf_counter() - t0, n


def stage_split(tts, text, ref):
    """Device ms per chunk of StreamJoin.push and of StreamJoin.take (the emit), at every push / take of one run."""
    import torch

    from sopro_b200.longform import StreamJoin

    marks = {"push": [], "emit": []}
    saved = {}

    def wrap(name, cat):
        real = getattr(StreamJoin, name)
        saved[name] = real

        def f(self, *a, **k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = real(self, *a, **k)
            e1.record()
            if cat == "push" or r is not None:
                marks[cat].append((e0, e1))
            return r

        setattr(StreamJoin, name, f)

    wrap("push", "push")
    wrap("take", "emit")
    try:
        for _ in tts.stream_long(text, ref=ref, seed=1234, chunk_frames=CF, **KW):
            pass
        torch.cuda.synchronize()
    finally:
        for k, v in saved.items():
            setattr(StreamJoin, k, v)
    out = {}
    for cat, ms in marks.items():
        t = [a.elapsed_time(b) for a, b in ms]
        out[cat] = {"calls": len(t), "ms_mean": float(np.mean(t)), "ms_p50": float(np.median(t)), "ms_p90": float(np.percentile(t, 90))}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--segments", default="1,16,64")
    args = ap.parse_args()

    tts, bench = build_tts()
    out = {"card": card(), "workload": f"bench.py texts as sentences, {FRAMES} frames per segment, chunk_frames={CF}, "
                                       "seeded, min_gen_frames=1e9, one voice"}
    ref = tts.prepare_reference(ref_tokens_tq=bench.bench_ref_tokens())
    for n in [int(x) for x in args.segments.split(",")]:
        text = passage(bench, n)
        seg0 = bench.bench_texts(0, 1)[0] + "."

        def long():
            return tts.stream_long(text, ref=ref, seed=1234, chunk_frames=CF, **KW)

        timed(long)  # warm-up: sessions, pooled states
        runs = [timed(long) for _ in range(args.runs)]
        firsts = [r[0] for r in runs]
        row = {"stream_long": {"first_item_ms_p50": float(np.median(firsts)) * 1e3,
                               "first_item_ms_p90": float(np.percentile(firsts, 90)) * 1e3,
                               "passage_done_ms_p50": float(np.median([r[1] for r in runs])) * 1e3,
                               "items": runs[0][2], "runs": len(runs)}}
        tts.synthesize_long(text, ref=ref, seed=1234, **KW)
        syn = []
        for _ in range(args.runs):
            t = timed(lambda: iter([tts.synthesize_long(text, ref=ref, seed=1234, **KW)]))
            syn.append(t[1])
        row["synthesize_long_ms_p50"] = float(np.median(syn)) * 1e3

        def solo():
            return tts.stream(seg0, ref=ref, seed=1234, chunk_frames=CF, **KW)

        timed(solo)
        s = [timed(solo) for _ in range(args.runs)]
        row["stream_segment0"] = {"first_chunk_ms_p50": float(np.median([r[0] for r in s])) * 1e3,
                                  "done_ms_p50": float(np.median([r[1] for r in s])) * 1e3}
        out[f"N{n}"] = row
        print(json.dumps({f"N{n}": row}), file=sys.stderr, flush=True)
    out["stage_ms_N64"] = stage_split(tts, passage(bench, 64), ref)
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
