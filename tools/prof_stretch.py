"""Cost of the time-stretch on the GPU, next to the work it serves, in one process:
  - CUDA-event time of the one-shot stretch of a 400-frame waveform (768,000 samples at 24 kHz, a real Mimi decode) at
    speeds 0.5, 1.25 and 2.0, at B = 1 and B = 64 rows, with the frame count of one row;
  - the Mimi decode of those 400 frames and `synthesize` of a 400-frame utterance, for scale;
  - stream() time-to-first-audio p50 and the 400-frame stream time, without and with speed=1.25, alternating.
Prints one JSON object with the card's name and power limit (synthetic seeded weights; nothing is written)."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
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


def main():
    from sopro_b200 import SoproTTS
    from sopro_b200.config import SoproTTSConfig
    from sopro_b200.stretch import n_frames, stretch, stretched_length
    from sopro_b200.tokenizer import IdsTokenizer
    from sopro_b200.weights import synth_mimi_state_dict, synth_state_dict

    torch.set_grad_enabled(False)
    dev = torch.device("cuda:0")
    out = {"card": card()}
    cfg = SoproTTSConfig()
    tts = SoproTTS.from_state_dict(cfg, synth_state_dict(cfg, 1000, 0), IdsTokenizer(1000), synth_mimi_state_dict(),
                                   device="cuda:0", weight_dtype="bf16")
    codes = torch.randint(0, 2048, (1, 32, 400), generator=torch.Generator().manual_seed(5)).to(dev)
    wav = tts.codec.engine.decode(codes)
    out["mimi_decode_400_frames_ms"] = event_ms(lambda: tts.codec.engine.decode(codes), 10)
    x = wav.reshape(-1).contiguous()  # 768,000 samples
    rows = x.repeat(64, 1).contiguous()
    one = {}
    for speed in (0.5, 1.25, 2.0):
        m = stretched_length(speed, x.numel())
        one[str(speed)] = {"frames": n_frames(m), "samples_out": m,
                           "b1_ms": event_ms(lambda: stretch(x, speed), 10),
                           "b64_ms": event_ms(lambda: stretch(rows, speed), 3)}
        one[str(speed)]["us_per_frame_b1"] = 1e3 * one[str(speed)]["b1_ms"] / one[str(speed)]["frames"]
    out["one_shot"] = one

    ref = tts.prepare_reference(ref_tokens_tq=torch.randint(0, 2048, (38, 32), generator=torch.Generator().manual_seed(7)))
    text = " ".join(str(17 * i + 5) for i in range(50))
    kw = dict(ref=ref, max_frames=400, seed=1, min_gen_frames=10 ** 9)

    def synth_ms(speed):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        w = tts.synthesize(text, speed=speed, **kw)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, int(w.numel())

    for speed in (None, 1.25):
        synth_ms(speed)
    syn = {"none": [], "1.25": []}
    for _round in range(3):
        for speed in (None, 1.25):
            t, n = synth_ms(speed)
            syn["none" if speed is None else "1.25"].append(t)
            syn[f"samples_{speed}"] = n
    out["synthesize_400_ms"] = syn

    def whole(speed):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        n = sum(c.numel() for c in tts.stream(text, speed=speed, **kw))
        torch.cuda.synchronize()
        return time.perf_counter() - t0, n

    def ttfa(speed):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        it = tts.stream(text, speed=speed, **kw)
        next(it).cpu()
        t1 = time.perf_counter()
        it.close()
        torch.cuda.synchronize()
        return t1 - t0

    for speed in (None, 1.25):  # warm-up: graphs, module loads, pools
        whole(speed)
        for _ in range(3):
            ttfa(speed)
    res = {"none": {"ttfa_p50_ms": [], "stream_400_ms": []}, "1.25": {"ttfa_p50_ms": [], "stream_400_ms": []}}
    for _round in range(3):
        for speed in (None, 1.25):
            key = "none" if speed is None else "1.25"
            t, n = whole(speed)
            res[key]["stream_400_ms"].append(t * 1e3)
            res[key]["samples"] = n
            res[key]["ttfa_p50_ms"].append(float(np.median([ttfa(speed) for _ in range(15)])) * 1e3)
    out["stream"] = res
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
