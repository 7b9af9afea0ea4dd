"""Cost of dialogue synthesis on the GPU, in one process (synthetic seeded weights; segment lengths forced with
min_gen_frames=10**9, so every round does the same work; nothing is written):
  - `synthesize_dialogue` of a 4-voice script of 16 turns, 64 segments, against a host loop of `synthesize_long` per
    turn (the turn's voice, seed + its first segment), alternating, three rounds each;
  - CUDA-event time of the dialogue join without and with per-turn levelling (the turns' own joins, one ragged
    loudness launch and the gained join) on 64 x 400-frame segments (a real Mimi decode), with the Mimi decode of
    those 64 x 400 frames beside it.
Prints one JSON object with the card's name and power limit."""
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
    from sopro_b200 import dialogue as D
    from sopro_b200.config import SoproTTSConfig
    from sopro_b200.longform import gap_pauses, join_gaps, speech_extents
    from sopro_b200.tokenizer import IdsTokenizer
    from sopro_b200.weights import synth_mimi_state_dict, synth_state_dict

    torch.set_grad_enabled(False)
    dev = torch.device("cuda:0")
    out = {"card": card()}
    cfg = SoproTTSConfig()
    tts = SoproTTS.from_state_dict(cfg, synth_state_dict(cfg, 1000, 0), IdsTokenizer(1000), synth_mimi_state_dict(),
                                   device="cuda:0", weight_dtype="bf16")
    voices = [tts.prepare_reference(ref_tokens_tq=torch.randint(0, 2048, (n, 32), generator=torch.Generator().manual_seed(s)))
              for n, s in ((38, 7), (25, 8), (50, 9), (44, 10))]
    F = 400
    kw = dict(max_frames=F, min_gen_frames=10 ** 9)
    P, TP = 6000, 12000

    # ---- the join stages at 64 x 400 frames, 16 turns of 4 segments
    codes = [torch.randint(0, 2048, (32, 32, F), generator=torch.Generator().manual_seed(5 + c)).to(dev).to(torch.int32)
             for c in range(2)]
    chunks = [tts.codec.engine.decode(c).view(32, -1) for c in codes]
    views = [c[i] for c in chunks for i in range(32)]
    ext = torch.cat([speech_extents(c) for c in chunks]).cpu().numpy()
    turn_of = [k // 4 for k in range(64)]
    pauses = gap_pauses(ext, P, turn_of, TP)
    stages = {"segments": 64, "turns": 16, "samples_per_segment": int(chunks[0].shape[1]),
              "mimi_decode_ms": event_ms(lambda: [tts.codec.engine.decode(c) for c in codes], 3),
              "join_ms": event_ms(lambda: join_gaps(views, ext, pauses), 20),
              "levelled_join_ms": event_ms(lambda: join_gaps(views, ext, pauses,
                                                             D.turn_gains(views, ext, turn_of, 16, P, -16.0)), 20)}
    out["stages_64x400_frames"] = stages

    # ---- synthesize_dialogue against a loop of synthesize_long per turn, alternating
    def turn_text(j):
        return " ".join(" ".join(str((17 * (4 * j + i) + 5 * w) % 997) for w in range(40)) + "." for i in range(4))

    script = [(voices[j % 4], turn_text(j)) for j in range(16)]
    segs, t_of, _v = D.plan(script, tts.tokenizer, 64)
    assert len(segs) == 64, len(segs)

    def dialogue_ms():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        w = tts.synthesize_dialogue(script, seed=1, **kw)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, w

    def per_turn_ms():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ws = [tts.synthesize_long(text, ref=v, seed=1 + 4 * j, **kw) for j, (v, text) in enumerate(script)]
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, ws

    _t, w = dialogue_ms()
    _t, ws = per_turn_ms()
    assert w.shape[-1] == sum(x.shape[-1] for x in ws) + 15 * TP, "the dialogue differs from its turns in length"
    r = {"dialogue_ms": [], "per_turn_synthesize_long_ms": [], "audio_s": w.shape[-1] / 24000}
    for _round in range(3):
        r["dialogue_ms"].append(dialogue_ms()[0])
        r["per_turn_synthesize_long_ms"].append(per_turn_ms()[0])
    r["median_ratio"] = float(np.median(r["per_turn_synthesize_long_ms"]) / np.median(r["dialogue_ms"]))
    out["synthesize_dialogue_4_voices_64_segments"] = r
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
