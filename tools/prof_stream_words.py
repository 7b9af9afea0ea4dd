"""Word timestamps on streams, on the GPU (bench.py's workload: synthetic seeded checkpoint, bf16 AR weights, EOS logit
pushed down so every utterance runs the full 401 AR steps, 52-id texts, one prepared voice; nothing is written):
  - stream() of one text: time to first audio (p50 / p90) and the time of the whole 400-frame stream, with and without
    word_timestamps=True, the two alternating run by run;
  - stream_batch of 64 texts likewise (first chunk of each row, and the whole batch);
  - the streaming alignment's push kernel: CUDA events around each push on the stream it is enqueued on, B = 1 and 64.
Host clock around calls that end in a device synchronise.  Prints one JSON object with the card's name, power limit
and SM clocks read in the same run.

  python tools/prof_stream_words.py [--runs N]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from prof_stream_batch import CF, FRAMES, build_tts, card  # noqa: E402

KW = dict(max_frames=FRAMES, min_gen_frames=10 ** 9, chunk_frames=CF)


def one_stream(tts, text, ref, seed, words):
    import torch

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    first, n_words = None, 0
    for item in tts.stream(text, ref=ref, seed=seed, word_timestamps=words, **KW):
        if first is None:
            first = time.perf_counter() - t0
        if words:
            n_words += len(item[1])
    torch.cuda.synchronize()
    return first, time.perf_counter() - t0, n_words


def batch(tts, texts, ref, seeds, words):
    import torch

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    first, n_words = [None] * len(texts), 0
    for item in tts.stream_batch(texts, ref=ref, seeds=seeds, word_timestamps=words, **KW):
        i, w = item[0], item[1]
        if first[i] is None and w.shape[1] > 0:
            first[i] = time.perf_counter() - t0
        if words:
            n_words += len(item[3])
    torch.cuda.synchronize()
    return first, time.perf_counter() - t0, n_words


def stats(firsts, ends, n_words):
    return {"ttfa_ms_p50": float(np.median(firsts)) * 1e3, "ttfa_ms_p90": float(np.percentile(firsts, 90)) * 1e3,
            "total_ms_p50": float(np.median(ends)) * 1e3, "total_ms_min": float(np.min(ends)) * 1e3,
            "words_per_run": n_words, "runs": len(ends)}


def push_times(tts, texts, ref, seeds):
    """ms per push from CUDA events recorded around each StreamAligner.push on its stream."""
    import torch

    from sopro_b200 import timestamps as TS

    ev = []
    real = TS.StreamAligner.push

    def push(self, frames, ends):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        real(self, frames, ends)
        b.record()
        ev.append((a, b))

    TS.StreamAligner.push = push
    try:
        for _ in tts.stream_batch(texts, ref=ref, seeds=seeds, word_timestamps=True, **KW):
            pass
    finally:
        TS.StreamAligner.push = real
    torch.cuda.synchronize()
    ms = [a.elapsed_time(b) for a, b in ev]  # includes the pinned copy of the committed paths
    return {"pushes": len(ms), "push_ms_p50": float(np.median(ms)), "push_ms_max": float(np.max(ms)),
            "push_ms_total": float(np.sum(ms))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=10)
    args = ap.parse_args()
    tts, bench = build_tts()
    out = {"card": card(), "workload": f"bench.py texts, {FRAMES} frames, chunk_frames={CF}, seeded, min_gen_frames=1e9"}
    ref = tts.prepare_reference(ref_tokens_tq=bench.bench_ref_tokens())
    text = bench.bench_texts(0, 1)[0]
    for w in (False, True):  # warm-up
        one_stream(tts, text, ref, 1234, w)
    res = {False: [], True: []}
    for r in range(args.runs):
        for w in ((False, True) if r % 2 == 0 else (True, False)):
            res[w].append(one_stream(tts, text, ref, 1234, w))
    out["stream_B1"] = {("words" if w else "plain"): stats([x[0] for x in v], [x[1] for x in v], v[0][2])
                        for w, v in res.items()}
    texts, seeds = bench.bench_texts(0, 64), list(range(1234, 1298))
    for w in (False, True):
        batch(tts, texts, ref, seeds, w)
    res = {False: [], True: []}
    for r in range(max(2, args.runs // 2)):
        for w in ((False, True) if r % 2 == 0 else (True, False)):
            res[w].append(batch(tts, texts, ref, seeds, w))
    out["stream_batch_B64"] = {("words" if w else "plain"): stats([f for x in v for f in x[0]], [x[1] for x in v], v[0][2])
                               for w, v in res.items()}
    out["push_B1"] = push_times(tts, texts[:1], ref, seeds[:1])
    out["push_B64"] = push_times(tts, texts, ref, seeds)
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
