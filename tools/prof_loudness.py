"""Cost of the loudness meter and gain on the GPU, next to the work it serves, in one process:
  - CUDA-event time of one-shot `normalize_loudness` of a 400-frame utterance (a real Mimi decode, 768,000 samples at
    24 kHz, resampled to 48 kHz for the 48 kHz case) at B = 1 and B = 64 rows;
  - the same for the 19.2 M-sample (10k-frame) waveform at 24 kHz, as input bytes over time;
  - the Mimi decode of those 400 frames, for scale;
  - `synthesize` of a 400-frame utterance without and with loudness=-16, alternating.
Prints one JSON object with the card's name and power limit (synthetic seeded weights; nothing is written)."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
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
    from sopro_b200.loudness import normalize_loudness
    from sopro_b200.resample import Resampler
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
    one = {}
    for sr in (24000, 48000):
        x = wav.reshape(-1).contiguous() if sr == 24000 else Resampler(24000, sr, dev)(wav.reshape(-1)).contiguous()
        rows = x.repeat(64, 1).contiguous()
        one[str(sr)] = {"samples": int(x.numel()),
                        "b1_ms": event_ms(lambda: normalize_loudness(x, sr, -16.0), 20),
                        "b64_ms": event_ms(lambda: normalize_loudness(rows, sr, -16.0), 5)}
    out["one_shot_400_frames"] = one
    big = torch.randn(10000 * 1920, generator=torch.Generator().manual_seed(1)).mul_(0.1).to(dev)
    t = event_ms(lambda: normalize_loudness(big, 24000, -16.0), 5)
    out["one_shot_19.2M"] = {"ms": t, "input_GB_per_s": big.numel() * 4 / (t * 1e-3) / 1e9}

    ref = tts.prepare_reference(ref_tokens_tq=torch.randint(0, 2048, (38, 32), generator=torch.Generator().manual_seed(7)))
    text = " ".join(str(17 * i + 5) for i in range(50))
    kw = dict(ref=ref, max_frames=400, seed=1, min_gen_frames=10 ** 9)

    def synth_ms(loudness):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        w = tts.synthesize(text, loudness=loudness, **kw)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, int(w.numel())

    for loudness in (None, -16.0):
        synth_ms(loudness)
    syn = {"none": [], "-16": []}
    for _round in range(3):
        for loudness in (None, -16.0):
            t, n = synth_ms(loudness)
            syn["none" if loudness is None else "-16"].append(t)
            syn["samples"] = n
    out["synthesize_400_ms"] = syn
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
