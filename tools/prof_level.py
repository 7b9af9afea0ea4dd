"""Cost of live loudness on the GPU, in one process:
  - device time per push of one LiveLeveller (11,520-sample chunks, stream()'s default chunk at 24 kHz), CUDA events
    over a 60 s row, early in the row and after 10 minutes have been metered (the meter's sum grows with the row);
  - device time per chunk across 64 levellers, one per stream_batch row, each pushed one 11,520-sample chunk;
  - level_live over 19.2 M samples (one row of 800 s at 24 kHz, and 64 rows of 300,000), CUDA events;
  - stream() time to first audio and whole-stream time on the synthetic checkpoint, with and without level_stream
    around it, alternated.
Prints one JSON object with the card's name and power limit, read in the same call (nothing is written)."""
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def event_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def pct(v, q):
    v = sorted(v)
    return v[min(len(v) - 1, int(round(q * (len(v) - 1))))]


def main():
    from sopro_b200 import SoproTTS
    from sopro_b200.config import SoproTTSConfig
    from sopro_b200.loudness import LiveLeveller, level_live, level_stream
    from sopro_b200.tokenizer import IdsTokenizer
    from sopro_b200.weights import synth_mimi_state_dict, synth_state_dict

    torch.set_grad_enabled(False)
    dev = torch.device("cuda:0")
    out = {"card": card()}
    g = torch.Generator(device=dev).manual_seed(3)
    C = 11520

    # one leveller: device time of each push, from CUDA events around the push alone
    x = 0.05 * torch.randn(24000 * 660, device=dev, generator=g)
    lev = LiveLeveller(24000, -16.0, device=dev)
    times, a = [], 0
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(x.numel() // C)]
    for e0, e1 in ev:
        e0.record()
        lev.push(x[a: a + C])
        e1.record()
        a += C
    torch.cuda.synchronize()
    times = [e0.elapsed_time(e1) for e0, e1 in ev]
    early, late = times[5:60], times[-55:]
    out["push_11520_24k_device_ms"] = {"first_minute_median": statistics.median(early), "after_10_min_median": statistics.median(late),
                                       "after_10_min_max": max(late)}
    lev.finish()

    # 64 levellers, one chunk each (what one stream_batch chunk asks for), after 2 s of each row
    levs = [LiveLeveller(24000, -16.0, device=dev) for _ in range(64)]
    rows = 0.05 * torch.randn(64, 4 * C, device=dev, generator=g)
    for i, l in enumerate(levs):
        l.push(rows[i, : 3 * C])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    e0.record()
    for i, l in enumerate(levs):
        l.push(rows[i, 3 * C:])
    e1.record()
    e1.synchronize()
    out["push_64_rows_one_chunk"] = {"device_ms": e0.elapsed_time(e1), "host_ms": (time.perf_counter() - t0) * 1e3}

    # the one-shot over 19.2 M samples
    one = 0.05 * torch.randn(19_200_000, device=dev, generator=g)
    out["level_live_19M2_one_row_ms"] = event_ms(lambda: level_live(one, 24000, -16.0), 3)
    many = one.reshape(64, 300_000)
    out["level_live_19M2_64_rows_ms"] = event_ms(lambda: level_live(many, 24000, -16.0), 5)

    # stream() with and without level_stream, alternated
    cfg = SoproTTSConfig()
    tts = SoproTTS.from_state_dict(cfg, synth_state_dict(cfg, 1000, 0), IdsTokenizer(1000), synth_mimi_state_dict(),
                                   device="cuda:0", weight_dtype="bf16")
    ref = tts.prepare_reference(ref_tokens_tq=torch.randint(0, 2048, (38, 32), generator=torch.Generator().manual_seed(7)))
    text = " ".join(str(17 * i + 5) for i in range(50))
    kw = dict(ref=ref, max_frames=200, seed=1, min_gen_frames=10 ** 9)

    def run(levelled):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        it = tts.stream(text, **kw)
        if levelled:
            it = level_stream(it, 24000, target=-16.0)
        first = None
        for c in it:
            if first is None:
                torch.cuda.current_stream().synchronize()
                first = time.perf_counter() - t0
        torch.cuda.synchronize()
        return first * 1e3, (time.perf_counter() - t0) * 1e3

    for v in (False, True):
        run(v)
    res = {"plain": [], "levelled": []}
    for _round in range(10):
        for v in (False, True):
            res["levelled" if v else "plain"].append(run(v))
    out["stream_200_frames_ms"] = {k: {"ttfa_p50": pct([t for t, _ in v], 0.5), "ttfa_p90": pct([t for t, _ in v], 0.9),
                                       "total_p50": pct([w for _, w in v], 0.5)} for k, v in res.items()}
    out["card_after"] = card()
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
