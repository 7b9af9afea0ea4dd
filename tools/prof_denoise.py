"""Cost of reference-voice denoising on the GPU, in one process (synthetic seeded weights, clips already on the device):
  (a) `denoise` alone over 1, 8 and 64 clips of 10 s at 24 kHz (CUDA events around the call; the workspace
      allocation is inside the window, as a caller pays it);
  (b) `prepare_references` of 64 clips of 10 s at 44.1 kHz, alternating denoise=True and denoise=False (host clock
      around a call that ends in a device synchronise).
Five rounds after one warm-up; medians.  Prints one JSON object with the card's name, power limit, maximum SM clock and
SM clock, read in the same run."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

ROUNDS = 5


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def voice(sr, seed, secs=10.0):
    """speech-like bursts with pauses over white noise at about 10 dB SNR"""
    g = np.random.default_rng(seed)
    t = np.arange(int(sr * secs)) / sr
    f0 = 120 + 60 * np.sin(2 * np.pi * 0.3 * t + seed)
    env = np.clip(np.sin(2 * np.pi * 0.7 * t + seed), 0, None) * (0.5 + 0.5 * np.sin(2 * np.pi * 4.0 * t))
    x = 0.4 * env * np.sin(2 * np.pi * np.cumsum(f0) / sr) + 0.03 * g.standard_normal(t.size)
    return torch.from_numpy(x.astype(np.float32))


def med(v):
    return round(float(np.median(v)), 3)


def main():
    from sopro_b200 import SoproTTS
    from sopro_b200.config import SoproTTSConfig
    from sopro_b200.denoising import denoise
    from sopro_b200.tokenizer import IdsTokenizer
    from sopro_b200.weights import synth_mimi_encoder_state_dict, synth_mimi_state_dict, synth_state_dict

    torch.set_grad_enabled(False)
    out = {"card (name, power limit, max SM clock, SM clock)": card()}
    dev = torch.device("cuda", 0)

    x64 = torch.stack([voice(24000, 10 + i) for i in range(64)]).to(dev)

    def alone(B):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        denoise(x64[:B])
        b.record()
        b.synchronize()
        return a.elapsed_time(b)

    for B in (1, 8, 64):
        alone(B)
    res = {f"denoise {B} x 10 s (ms)": [] for B in (1, 8, 64)}
    for _ in range(ROUNDS):
        for B in (1, 8, 64):
            res[f"denoise {B} x 10 s (ms)"].append(alone(B))

    cfg = SoproTTSConfig()
    msd = dict(synth_mimi_state_dict())
    msd.update(synth_mimi_encoder_state_dict())
    tts = SoproTTS.from_state_dict(cfg, synth_state_dict(cfg, 1000, 0), IdsTokenizer(1000), msd, device="cuda:0")
    clips = [voice(44100, 200 + i).to(dev) for i in range(64)]

    def prep(flag):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        refs = tts.prepare_references(clips, sample_rates=44100, denoise=flag)
        torch.cuda.synchronize()
        assert len(refs) == 64
        return (time.perf_counter() - t0) * 1e3

    prep(True)
    prep(False)
    on, off = [], []
    for _ in range(ROUNDS):
        on.append(prep(True))
        off.append(prep(False))
    res["prepare_references 64 x 10 s @ 44.1 kHz, denoise=True (ms)"] = on
    res["prepare_references 64 x 10 s @ 44.1 kHz, denoise=False (ms)"] = off
    out[f"median of {ROUNDS} rounds"] = {k: med(v) for k, v in res.items()}
    out["all rounds"] = {k: [round(x, 3) for x in v] for k, v in res.items()}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
