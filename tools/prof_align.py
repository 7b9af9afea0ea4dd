"""Cost of word timestamps: the alignment kernel alone (B = 64 at L = 66 over 401 steps; B = 8 at L = 2048, since a
64 x 2048 trace would be 2.5 GB, over 2400 steps, since 2048 tokens have no path through 401 frames), and
synthesize_batch of 64 texts with and without word_timestamps (synthetic checkpoint).  Prints the card and its power
limit from the same run.

    python tools/prof_align.py
"""
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def time_align(B, L, steps=401, reps=20):
    from sopro_b200.timestamps import align

    g = torch.Generator(device="cuda").manual_seed(0)
    p = torch.rand((steps, 3, B, 4, L), device="cuda", generator=g)
    lens, frames = [L] * B, [steps] * B
    for _ in range(3):
        align(p, lens, frames)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        align(p, lens, frames)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def time_batch(reps=5):
    from sopro_b200 import SoproTTS
    from sopro_b200.tokenizer import IdsTokenizer
    from oracle import mimi_oracle as M
    from tests.cases import e2e_inputs

    cfg, sd, inp = e2e_inputs()
    tts = SoproTTS.from_state_dict(cfg, sd, IdsTokenizer(1000), M.synth_mimi_state_dict(), device="cuda:0")
    ref = tts.prepare_reference(ref_tokens_tq=inp["ref_tokens_tq"])
    texts = [" ".join(str((7 * i + 3 * j) % 997) for j in range(64)) for i in range(64)]
    kw = dict(ref=ref, seeds=list(range(64)), max_frames=400, min_gen_frames=10 ** 9)
    out = {}
    for flag in (False, True, False, True):
        tts.synthesize_batch(texts, word_timestamps=flag, **kw)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(reps):
            tts.synthesize_batch(texts, word_timestamps=flag, **kw)
        torch.cuda.synchronize()
        out.setdefault(flag, []).append((time.perf_counter() - t0) / reps * 1e3)
    return out


if __name__ == "__main__":
    torch.set_grad_enabled(False)
    print(f"card: {card()}")
    print(f"align, 401 steps, B=64, L=66:   {time_align(64, 66):.3f} ms")
    print(f"align, 2400 steps, B=8, L=2048: {time_align(8, 2048, steps=2400, reps=5):.3f} ms")
    r = time_batch()
    print(f"synthesize_batch of 64 texts (L=66, 401 frames): without {r[False]} ms, with word_timestamps {r[True]} ms")
