"""Cost of the output resampler on the GPU, next to the work it serves, in one process:
  - CUDA-event time of the one-shot kernel on the 10k-frame waveform (19.2 M samples at 24 kHz, a real Mimi decode) to
    8, 16, 22.05, 44.1 and 48 kHz, with effective GB/s (4 bytes per input and per output sample);
  - the Mimi decode of those 10k frames (25 x 400, the bench's shape) for scale;
  - stream() time-to-first-audio p50 and the 400-frame stream time, without and with sample_rate=48000, alternating.
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
    from sopro_b200.resample import Resampler
    from sopro_b200.tokenizer import IdsTokenizer
    from sopro_b200.weights import synth_mimi_state_dict, synth_state_dict

    torch.set_grad_enabled(False)
    dev = torch.device("cuda:0")
    out = {"card": card()}
    cfg = SoproTTSConfig()
    tts = SoproTTS.from_state_dict(cfg, synth_state_dict(cfg, 1000, 0), IdsTokenizer(1000), synth_mimi_state_dict(),
                                   device="cuda:0", weight_dtype="bf16")
    codes = torch.randint(0, 2048, (25, 32, 400), generator=torch.Generator().manual_seed(5)).to(dev)
    wav = tts.codec.engine.decode(codes)
    out["mimi_decode_10k_frames_ms"] = event_ms(lambda: tts.codec.engine.decode(codes), 5)
    x = wav.reshape(-1).contiguous()  # 19.2 M samples
    one = {}
    for sr in (8000, 16000, 22050, 44100, 48000):
        rs = Resampler(24000, sr, dev)
        ms = event_ms(lambda: rs(x), 20)
        n_out = rs.length(x.numel())
        one[str(sr)] = {"ms": ms, "gb_per_s": 4 * (x.numel() + n_out) / (ms * 1e-3) / 1e9, "samples_out": n_out}
    rs48 = Resampler(24000, 48000, dev)
    rows = wav.reshape(25, -1)
    ms = event_ms(lambda: rs48(rows, lens=[rows.shape[1]] * 25), 20)
    one["48000_as_25_rows"] = {"ms": ms, "gb_per_s": 4 * 3 * x.numel() / (ms * 1e-3) / 1e9}
    out["one_shot"] = one
    out["hbm_datasheet_tb_per_s"] = 3.35

    ref = tts.prepare_reference(ref_tokens_tq=torch.randint(0, 2048, (38, 32), generator=torch.Generator().manual_seed(7)))
    text = " ".join(str(17 * i + 5) for i in range(50))

    def whole(sr):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        n = sum(c.numel() for c in tts.stream(text, ref=ref, max_frames=400, seed=1, min_gen_frames=10 ** 9, sample_rate=sr))
        torch.cuda.synchronize()
        return time.perf_counter() - t0, n

    def ttfa(sr):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        it = tts.stream(text, ref=ref, max_frames=400, seed=1, min_gen_frames=10 ** 9, sample_rate=sr)
        next(it).cpu()
        t1 = time.perf_counter()
        it.close()
        torch.cuda.synchronize()
        return t1 - t0

    for sr in (None, 48000):  # warm-up: graphs, module loads, pools
        whole(sr)
        for _ in range(3):
            ttfa(sr)
    res = {"24000": {"ttfa_p50_ms": [], "stream_400_ms": []}, "48000": {"ttfa_p50_ms": [], "stream_400_ms": []}}
    for _round in range(3):
        for sr in (None, 48000):
            key = "24000" if sr is None else "48000"
            t, n = whole(sr)
            res[key]["stream_400_ms"].append(t * 1e3)
            res[key]["samples"] = n
            res[key]["ttfa_p50_ms"].append(float(np.median([ttfa(sr) for _ in range(15)])) * 1e3)
    out["stream"] = res
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
