"""Cost of timed synthesis on the GPU, in one process (synthetic seeded weights; every segment is forced to max_frames
frames with min_gen_frames=10**9, so every run does the same work; nothing is written):
  - `synthesize_timed` of a one-hour two-voice WebVTT track of 1,000 cues (one segment each, a quarter of them in slots
    that need a speed-up), against a host loop of `synthesize_long` per cue, `stretch_rows` at the cue's speed and
    torch placement into one buffer; and the peak device memory of the `synthesize_timed` call;
  - CUDA-event time of the mix kernel alone (longform.mix) at one hour / 1,000 cues and at four hours / 4,000 cues,
    with the bytes it must move (the rows read once, the timeline written once) over that time, against the H100 SXM
    data sheet's 3.35 TB/s.
Prints one JSON object with the card's name, power limit and maximum SM clock."""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from prof_dialogue import card, event_ms  # noqa: E402

HBM = 3.35e12


def _stamp(t):
    ms = int(round(t * 1000))
    return f"{ms // 3_600_000:02d}:{ms // 60_000 % 60:02d}:{ms // 1000 % 60:02d}.{ms % 1000:03d}"


def mix_case(hours, cues, dev):
    """Rows of 2 .. 5 s at random places in `hours` of timeline (overlaps included) -> the mix's timing."""
    from sopro_b200.longform import mix

    g = np.random.default_rng(int(hours * 10))
    N = int(hours * 3600 * 24000)
    lens = [int(v) for v in g.integers(48_000, 120_000, cues)]
    offs = sorted(int(g.integers(0, N - k)) for k in lens)
    base = torch.randn(130_000, generator=torch.Generator().manual_seed(3)).to(dev)
    rows = [base[: k] for k in lens]
    ms = event_ms(lambda: mix(rows, offs, N), 20)
    moved = 4 * (sum(lens) + N)
    return {"hours": hours, "cues": cues, "samples": N, "mix_ms": ms, "bytes": moved,
            "achieved_TB_per_s": moved / (ms * 1e-3) / 1e12, "share_of_3_35_TB_per_s": moved / (ms * 1e-3) / HBM}


def main():
    from sopro_b200 import SoproTTS
    from sopro_b200.config import SoproTTSConfig
    from sopro_b200.cues import parse
    from sopro_b200.stretch import stretch_rows
    from sopro_b200.tokenizer import IdsTokenizer
    from sopro_b200.weights import synth_mimi_state_dict, synth_state_dict

    torch.set_grad_enabled(False)
    dev = torch.device("cuda:0")
    out = {"card": card()}

    # ---- the mix kernel alone
    out["mix"] = [mix_case(1, 1000, dev), mix_case(4, 4000, dev)]

    # ---- a one-hour track
    cfg = SoproTTSConfig()
    tts = SoproTTS.from_state_dict(cfg, synth_state_dict(cfg, 1000, 0), IdsTokenizer(1000), synth_mimi_state_dict(),
                                   device="cuda:0", weight_dtype="bf16")
    gen = torch.Generator().manual_seed(7)
    refs = [tts.prepare_reference(ref_tokens_tq=torch.randint(0, 2048, (38, 32), generator=gen)) for _ in range(3)]
    names = {"anna": refs[1], "ben": refs[2]}
    kw = dict(max_frames=40, min_gen_frames=10 ** 9, max_tokens=64)  # 40 frames = 76,800 samples = 3.2 s per cue
    n_cues = 1000
    lines = ["WEBVTT", ""]
    t = 0.5
    for k in range(n_cues):
        slot = 2.6 if k % 4 == 0 else 3.4  # a quarter need a speed-up of about 1.23
        text = " ".join(str((17 * k + 5 * w) % 997) for w in range(12)) + "."
        v = "" if k % 3 == 0 else f"<v {'anna' if k % 3 == 1 else 'ben'}>"
        lines += [f"{_stamp(t)} --> {_stamp(t + slot)}", v + text, ""]
        t += 3.6
    track = "\n".join(lines)
    cues = parse(track)

    def run_timed():
        return tts.synthesize_timed(track, ref=refs[0], voices=names, seed=1, **kw)

    def run_loop():
        rows, S, off = [], [], []
        for k, c in enumerate(cues):
            voice = refs[0] if c.voice is None else names[c.voice]
            w = tts.synthesize_long(c.text, ref=voice, seed=1 + k, **kw).reshape(-1)
            slot = round(c.end * 24000) - round(c.start * 24000)
            s = 1.0 if w.numel() <= slot else min(1.5, -(-w.numel() * 65536 // slot) / 65536)
            rows.append(w if s == 1.0 else stretch_rows(w.reshape(1, -1), [s]).reshape(-1))
            off.append(round(c.start * 24000))
        N = max(max(round(c.end * 24000), o + r.numel()) for c, o, r in zip(cues, off, rows))
        y = torch.zeros(N, device=dev)
        for o, r in zip(off, rows):
            y[o: o + r.numel()] += r
        return y

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, r

    small = "\n".join(track.split("\n")[: 2 + 3 * 80])  # warm-up: every shape of one group
    tts.synthesize_timed(small, ref=refs[0], voices=names, seed=1, **kw)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    base = torch.cuda.memory_allocated(dev)
    t_timed, (wav, fits) = timed(run_timed)
    peak = torch.cuda.max_memory_allocated(dev) - base
    t_timed2, _ = timed(run_timed)
    t_loop, y = timed(run_loop)
    diff = float((wav.reshape(-1) - y).abs().max()) if wav.numel() == y.numel() else None
    out["one_hour_track"] = {
        "cues": n_cues, "audio_s": wav.shape[-1] / 24000, "stretched_cues": sum(f.rate > 1 for f in fits),
        "synthesize_timed_s": [t_timed, t_timed2], "loop_of_synthesize_long_s": t_loop,
        "speedup": t_loop / min(t_timed, t_timed2), "max_abs_diff_vs_loop": diff,
        "peak_device_bytes_above_start": peak, "timeline_bytes": 4 * wav.shape[-1],
    }
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
