"""Cost of long-form synthesis on the GPU, in one process (synthetic seeded weights; segment lengths forced with
min_gen_frames=10**9, so every round does the same work; nothing is written):
  - `synthesize_long` of a 16- and a 64-segment text against a host loop of `synthesize` over the same segments
    (seed + i each), alternating, three rounds each; the two outputs are checked equal;
  - CUDA-event time of the extents and join stages on 64 x 400-frame segments (a real Mimi decode), with the Mimi decode
    of those 64 x 400 frames beside it.
Prints one JSON object with the card's name and power limit."""
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
    from sopro_b200.longform import join_segments, speech_extents, split_text
    from sopro_b200.tokenizer import IdsTokenizer
    from sopro_b200.weights import synth_mimi_state_dict, synth_state_dict

    torch.set_grad_enabled(False)
    dev = torch.device("cuda:0")
    out = {"card": card()}
    cfg = SoproTTSConfig()
    tts = SoproTTS.from_state_dict(cfg, synth_state_dict(cfg, 1000, 0), IdsTokenizer(1000), synth_mimi_state_dict(),
                                   device="cuda:0", weight_dtype="bf16")
    ref = tts.prepare_reference(ref_tokens_tq=torch.randint(0, 2048, (38, 32), generator=torch.Generator().manual_seed(7)))
    F = 400
    kw = dict(ref=ref, max_frames=F, min_gen_frames=10 ** 9)

    # ---- the two stages at 64 x 400 frames, decoded as synthesize_long decodes them: two padded chunks of 32
    codes = [torch.randint(0, 2048, (32, 32, F), generator=torch.Generator().manual_seed(5 + c)).to(dev).to(torch.int32)
             for c in range(2)]
    chunks = [tts.codec.engine.decode(c).view(32, -1) for c in codes]  # 2 x [32, 400 * 1920]

    def extents():
        return torch.cat([speech_extents(c) for c in chunks])

    stages = {"segments": 64, "samples_per_segment": int(chunks[0].shape[1]),
              "mimi_decode_ms": event_ms(lambda: [tts.codec.engine.decode(c) for c in codes], 3),
              "extents_ms": event_ms(extents, 20)}
    ext_host = extents().cpu()
    views = [c[i] for c in chunks for i in range(32)]
    stages["join_ms"] = event_ms(lambda: join_segments(views, ext_host, 250), 20)
    stages["joined_samples"] = int(join_segments(views, ext_host, 250).shape[-1])
    out["stages_64x400_frames"] = stages

    # ---- synthesize_long against a serial loop of synthesize, alternating
    def text_of(n):
        return " ".join(" ".join(str((17 * i + 5 * j) % 997) for j in range(40)) + "." for i in range(n))

    res = {}
    for n_seg in (16, 64):
        text = text_of(n_seg)
        segs = split_text(text, tts.tokenizer, 64)
        assert len(segs) == n_seg, len(segs)

        def long_ms():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            w = tts.synthesize_long(text, seed=1, **kw)
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) * 1e3, w

        def serial_ms():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ws = [tts.synthesize(s, seed=1 + i, **kw) for i, s in enumerate(segs)]
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) * 1e3, ws

        _t, w = long_ms()
        _t, ws = serial_ms()
        e = torch.cat([speech_extents(x) for x in ws])
        assert torch.equal(w, join_segments(ws, e, 250)), "synthesize_long differs from its parts"
        r = {"long_ms": [], "serial_synthesize_ms": [], "audio_s": w.shape[-1] / 24000}
        for _round in range(3):
            r["long_ms"].append(long_ms()[0])
            r["serial_synthesize_ms"].append(serial_ms()[0])
        res[str(n_seg)] = r
    out["synthesize_long"] = res
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
