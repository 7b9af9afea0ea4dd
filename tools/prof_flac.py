"""Cost of FLAC encoding on the GPU, next to the work it serves, in one process:
  - `encode_flac` of 400-frame rows (a real Mimi decode of the synthetic checkpoint, 768,000 samples at 24 kHz,
    resampled to 48 kHz for the 48 kHz case) at B = 1 and B = 64, host wall time of the whole call (it ends with the
    copy of the bytes to the host), median of the repetitions;
  - the Mimi decode of those 400 frames, for scale (CUDA events);
  - `stream()` time to first audio, and to the first FLAC frame through `encode_stream_flac`, alternating;
  - the compression ratio against PCM16 of the synthetic checkpoint's output (random weights: not speech) and of the
    speech-like test signal of tests/test_flac_gpu.py.
Prints one JSON object with the card's name and power limit (nothing is written)."""
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


def wall_ms(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return {"median": statistics.median(ts), "min": min(ts), "max": max(ts)}


def main():
    import numpy as np

    from sopro_b200 import SoproTTS
    from sopro_b200.config import SoproTTSConfig
    from sopro_b200.flac import encode_flac, encode_stream_flac
    from sopro_b200.resample import Resampler
    from sopro_b200.tokenizer import IdsTokenizer
    from sopro_b200.weights import synth_mimi_state_dict, synth_state_dict
    from tests.test_flac_gpu import signal

    torch.set_grad_enabled(False)
    dev = torch.device("cuda:0")
    out = {"card": card()}
    cfg = SoproTTSConfig()
    tts = SoproTTS.from_state_dict(cfg, synth_state_dict(cfg, 1000, 0), IdsTokenizer(1000), synth_mimi_state_dict(),
                                   device="cuda:0", weight_dtype="bf16")
    codes = torch.randint(0, 2048, (1, 32, 400), generator=torch.Generator().manual_seed(5)).to(dev)
    wav = tts.codec.engine.decode(codes)
    out["mimi_decode_400_frames_ms"] = event_ms(lambda: tts.codec.engine.decode(codes), 10)
    enc = {}
    for sr in (24000, 48000):
        x = wav.reshape(-1).contiguous() if sr == 24000 else Resampler(24000, sr, dev)(wav.reshape(-1)).contiguous()
        rows = x.repeat(64, 1).contiguous()
        b = encode_flac(x, sr)
        enc[str(sr)] = {"samples": int(x.numel()), "ratio_vs_pcm16": len(b) / (2 * x.numel()),
                        "b1_ms": wall_ms(lambda: encode_flac(x, sr), 20),
                        "b64_ms": wall_ms(lambda: encode_flac(rows, sr, lens=[x.numel()] * 64), 5)}
    out["encode_400_frames"] = enc
    # device time per kernel of one B = 64 encode at 24 kHz (torch.profiler's CUDA activity)
    rows = wav.reshape(-1).repeat(64, 1).contiguous()
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        encode_flac(rows, 24000)
    per = {}
    for e in prof.events():
        if "flac" in e.name or "Memcpy" in e.name:
            per[e.name] = per.get(e.name, 0.0) + e.device_time_total / 1e3
    out["b64_24k_device_ms_per_kernel"] = per
    sp = signal("speech", 10 * 24000)
    out["speech_like_ratio_vs_pcm16"] = len(encode_flac(torch.from_numpy(sp).to(dev), 24000)) / (2 * sp.size)

    ref = tts.prepare_reference(ref_tokens_tq=torch.randint(0, 2048, (38, 32), generator=torch.Generator().manual_seed(7)))
    text = " ".join(str(17 * i + 5) for i in range(50))
    kw = dict(ref=ref, max_frames=64, seed=1, min_gen_frames=10 ** 9)

    def ttfa(flac):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        it = tts.stream(text, **kw)
        if flac:
            g = encode_stream_flac(it, 24000)
            next(g)  # the header
            next(g)  # the first chunk's frames
            t = time.perf_counter() - t0
            for _ in g:
                pass
        else:
            next(it)
            t = time.perf_counter() - t0
            for _ in it:
                pass
        return t * 1e3

    for flac in (False, True):
        ttfa(flac)
    res = {"pcm": [], "flac": []}
    for _round in range(5):
        for flac in (False, True):
            res["flac" if flac else "pcm"].append(ttfa(flac))
    out["stream_ttfa_ms"] = {k: {"median": statistics.median(v), "all": v} for k, v in res.items()}
    w = tts.synthesize(text, ref=ref, max_frames=400, seed=1, min_gen_frames=10 ** 9)
    out["synthetic_checkpoint_ratio_vs_pcm16"] = len(encode_flac(w, 24000)) / (2 * w.numel())
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
