"""Cost of the watermark on the GPU, in one process:
  - CUDA-event time of one-shot `embed_watermark` of a 400-frame utterance (a real Mimi decode, 768,000 samples at
    24 kHz) at B = 1 and B = 64 rows;
  - `detect_watermark` of 64 clips of 10 s at 24 kHz;
  - `synthesize` of a 400-frame utterance without and with `watermark`, alternating;
  - `stream()` time to first audio, p50 of alternating runs without and with `watermark`.
Prints one JSON object with the card's name and power limit (synthetic seeded weights; nothing is written)."""
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
    from sopro_b200.tokenizer import IdsTokenizer
    from sopro_b200.watermark import detect_watermark, embed_watermark
    from sopro_b200.weights import synth_mimi_state_dict, synth_state_dict
    from tests.cases import e2e_inputs

    torch.set_grad_enabled(False)
    dev = torch.device("cuda:0")
    out = {"card": card()}
    key = 0xC0FFEE
    cfg = SoproTTSConfig()
    tts = SoproTTS.from_state_dict(cfg, synth_state_dict(cfg, 1000, 0), IdsTokenizer(1000), synth_mimi_state_dict(),
                                   device="cuda:0", weight_dtype="bf16")
    codes = torch.randint(0, 2048, (1, 32, 400), generator=torch.Generator().manual_seed(5)).to(dev)
    wav = tts.codec.engine.decode(codes).reshape(-1).contiguous()
    rows = wav.repeat(64, 1).contiguous()
    out["mimi_decode_400_frames_ms"] = event_ms(lambda: tts.codec.engine.decode(codes), 10)
    out["embed_400_frames_b1_ms"] = event_ms(lambda: embed_watermark(wav, key), 50)
    out["embed_400_frames_b64_ms"] = event_ms(lambda: embed_watermark(rows, key), 10)
    clips = embed_watermark(wav[:240000].repeat(64, 1).contiguous(), key)
    out["detect_64_clips_10s_ms"] = event_ms(lambda: detect_watermark(clips, 24000, key), 10)

    _c, _s, inp = e2e_inputs()
    ref = tts.prepare_reference(ref_tokens_tq=inp["ref_tokens_tq"])
    text = " ".join(str(7 * i + 3) for i in range(20))
    kw = dict(ref=ref, max_frames=400, min_gen_frames=10 ** 9, seed=1)
    for k in (None, key):
        tts.synthesize(text, watermark=k, **kw)
    times = {None: [], key: []}
    for _ in range(7):
        for k in (None, key):
            torch.cuda.synchronize()
            t = time.perf_counter()
            tts.synthesize(text, watermark=k, **kw)
            torch.cuda.synchronize()
            times[k].append(1e3 * (time.perf_counter() - t))
    out["synthesize_400_frames_ms"] = {"plain": statistics.median(times[None]), "watermark": statistics.median(times[key])}

    ttfa = {None: [], key: []}
    skw = dict(ref=ref, max_frames=64, min_gen_frames=10 ** 9, seed=2)
    for i in range(41):
        for k in (None, key):
            torch.cuda.synchronize()
            t = time.perf_counter()
            it = tts.stream(text, watermark=k, **skw)
            next(it)
            dt = 1e3 * (time.perf_counter() - t)
            for _ in it:
                pass
            if i:  # the first round warms up
                ttfa[k].append(dt)
    out["stream_ttfa_p50_ms"] = {"plain": statistics.median(ttfa[None]), "watermark": statistics.median(ttfa[key]),
                                 "runs": len(ttfa[key])}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
