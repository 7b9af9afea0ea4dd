"""Cost of voice blends on the GPU (bench.py's workload: synthetic seeded checkpoint, bf16 AR weights, EOS logit pushed
down so every utterance runs the full 401 AR steps, 52-id texts; nothing is written):
  - the prefill alone (PrefillEngine.run, 64 texts, 401 frames) in one plain voice of 150 reference frames, against one
    blend of 2, 4 and 16 such voices and against 64 distinct 2-voice blends, and against plain voices of the blends'
    total frames (300, 600, 2400), which separates the cost of more frames from the cost of mixing; CUDA events around
    20 calls, the cases alternated round by round;
  - synthesize_batch of the 64 texts in one 2-voice blend against the same texts in one plain voice, host clock around
    calls that end in a device synchronise, alternated after one warm-up of each.
Prints one JSON object with the card's name, power limit and SM clocks read in the same run.

  python tools/prof_blend.py [--rounds N]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
N_TEXTS, TR = 64, 150


def card():
    import torch

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def build_tts():
    import torch

    import bench
    from sopro_b200 import SoproTTS
    from sopro_b200.config import SoproTTSConfig
    from sopro_b200.tokenizer import IdsTokenizer
    from sopro_b200.weights import synth_mimi_state_dict

    torch.set_grad_enabled(False)
    cfg = SoproTTSConfig()
    tts = SoproTTS.from_state_dict(cfg, bench.bench_state_dict(cfg), IdsTokenizer(bench.TEXT_VOCAB), synth_mimi_state_dict(),
                                   device="cuda:0", weight_dtype="bf16")
    return tts, bench


def timed(fn):
    import torch

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def med(v):
    return sorted(v)[len(v) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("prof_blend.py measures on a CUDA device; there is none")
    out = {"card (name, power limit, max SM clock, SM clock)": card()}
    tts, bench = build_tts()
    g = torch.Generator().manual_seed(5)
    voices = [tts.prepare_reference(ref_tokens_tq=torch.randint(0, 2048, (TR, 32), generator=g)) for _ in range(16)]
    texts = bench.bench_texts(0, N_TEXTS)
    seeds = list(range(1234, 1234 + N_TEXTS))
    cases = {"1_plain_voice": voices[0],
             "1_blend_of_2": tts.blend_voices(voices[:2]),
             "1_blend_of_4": tts.blend_voices(voices[:4]),
             "1_blend_of_16": tts.blend_voices(voices),
             "64_distinct_blends_of_2": [tts.blend_voices([voices[i % 16], voices[(i // 16 + i + 1) % 16]], [1.0, 1.0 + i])
                                         for i in range(N_TEXTS)]}
    for n in (2, 4, 16):
        cases[f"1_plain_voice_of_{n * TR}_frames"] = tts.prepare_reference(
            ref_tokens_tq=torch.randint(0, 2048, (n * TR, 32), generator=g), ref_seconds=0)  # 0: no 12 s crop

    # ---- the prefill alone
    pe = tts.model.prefill
    ids = [tts.encode_text(t) for t in texts]

    def event_ms(ref, reps=20):
        pe.run(ids, ref, n_frames=401, style_strength=1.2)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            pe.run(ids, ref, n_frames=401, style_strength=1.2)
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) / reps

    pre = {k: [] for k in cases}
    for _ in range(args.rounds):
        for k, ref in cases.items():
            pre[k].append(event_ms(ref))
    out[f"prefill_64_texts_401_frames_voices_of_{TR}_frames_ms (CUDA events, incl. host copies of the voice table)"] = {
        k: {"median": med(v), "all": v} for k, v in pre.items()}

    # ---- synthesize_batch: one 2-voice blend against one plain voice
    kw = dict(max_frames=400, min_gen_frames=10 ** 9)
    refs = {"1_plain_voice": voices[0], "1_blend_of_2": cases["1_blend_of_2"]}
    for r in refs.values():
        timed(lambda: tts.synthesize_batch(texts, ref=r, seeds=seeds, **kw))  # warm-up: sessions, workspaces
    res = {k: [] for k in refs}
    for _ in range(args.rounds):
        for k, r in refs.items():
            res[k].append(timed(lambda: tts.synthesize_batch(texts, ref=r, seeds=seeds, **kw))[0])
    m = {k: med(v) for k, v in res.items()}
    out["synthesize_batch_64_texts_401_frames_ms (host clock)"] = {
        "median": m, "all": res, "blend_over_plain": m["1_blend_of_2"] / m["1_plain_voice"]}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
