"""Cost of speech markup on the GPU, in one process (synthetic seeded weights; segment lengths forced with
min_gen_frames=10**9, so every round does the same work; nothing is written):
  - CUDA-event time of one `stretch_rows` launch over 64 rows of mixed rates (0.5 .. 2, a quarter of them at rate 1,
    ragged, up to 400 frames = 768,000 samples) against 64 calls of `stretch`, one per row at its rate;
  - `synthesize_ssml` of a 64-segment script (rates, volumes and breaks) against `synthesize_long` of the same text,
    alternating, three rounds each.
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


def main():
    from sopro_b200 import SoproTTS
    from sopro_b200.config import SoproTTSConfig
    from sopro_b200.stretch import stretch, stretch_rows
    from sopro_b200.tokenizer import IdsTokenizer
    from sopro_b200.weights import synth_mimi_state_dict, synth_state_dict

    torch.set_grad_enabled(False)
    dev = torch.device("cuda:0")
    out = {"card": card()}

    # ---- the stretch stage: one launch against a launch per row
    g = np.random.default_rng(1)
    B, L = 64, 768000
    lens = [int(v) for v in g.integers(L // 4, L + 1, B)]
    speeds = [float(v) for v in g.choice([0.5, 0.75, 0.9, 1.0, 1.25, 1.5, 2.0, 1.0], B)]
    x = torch.randn(B, L, generator=torch.Generator().manual_seed(2)).to(dev)
    rows = [x[b, : lens[b]] for b in range(B)]
    y = stretch_rows(x, speeds, lens=lens)
    for b in range(B):  # the timed paths compute the same samples
        want = rows[b] if speeds[b] == 1.0 else stretch(rows[b], speeds[b])
        assert torch.equal(y[b, : want.numel()], want), b
    out["stretch_64_rows"] = {
        "rows": B, "samples_in": sum(lens), "rate_1_rows": speeds.count(1.0),
        "stretch_rows_ms": event_ms(lambda: stretch_rows(x, speeds, lens=lens), 5),
        "per_row_stretch_ms": event_ms(lambda: [stretch(rows[b], speeds[b]) for b in range(B) if speeds[b] != 1.0], 5),
    }

    # ---- synthesize_ssml against synthesize_long of the same text
    cfg = SoproTTSConfig()
    tts = SoproTTS.from_state_dict(cfg, synth_state_dict(cfg, 1000, 0), IdsTokenizer(1000), synth_mimi_state_dict(),
                                   device="cuda:0", weight_dtype="bf16")
    ref = tts.prepare_reference(ref_tokens_tq=torch.randint(0, 2048, (38, 32), generator=torch.Generator().manual_seed(7)))
    kw = dict(max_frames=400, min_gen_frames=10 ** 9)
    sents = [" ".join(str((17 * k + 5 * w) % 997) for w in range(40)) + "." for k in range(64)]
    text = " ".join(sents)
    marks = ['<prosody rate="slow">{}</prosody>', '<prosody rate="fast" volume="-6dB">{}</prosody>', '{}',
             '{}<break time="400ms"/>']
    ssml = "<speak>" + " ".join(marks[k % 4].format(s) for k, s in enumerate(sents)) + "</speak>"

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        w = fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, w

    def run_ssml():
        return tts.synthesize_ssml(ssml, ref=ref, seed=1, **kw)

    def run_long():
        return tts.synthesize_long(text, ref=ref, seed=1, **kw)

    _t, w = timed(run_ssml)
    _t, wl = timed(run_long)
    r = {"segments": 64, "ssml_audio_s": w.shape[-1] / 24000, "long_audio_s": wl.shape[-1] / 24000,
         "synthesize_ssml_ms": [], "synthesize_long_ms": []}
    for _round in range(3):
        r["synthesize_ssml_ms"].append(timed(run_ssml)[0])
        r["synthesize_long_ms"].append(timed(run_long)[0])
    r["median_ratio_ssml_over_long"] = float(np.median(r["synthesize_ssml_ms"]) / np.median(r["synthesize_long_ms"]))
    out["synthesize_ssml_64_segments"] = r
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
