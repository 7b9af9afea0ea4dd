"""Cost of best-of-N synthesis on the GPU, in one process (synthetic seeded weights, bf16 AR weights as in bench.py; the
EOS logit is pushed down by 30 so every take runs the full 401 AR steps and every round does the same work; nothing is
written):
  - `synthesize` wall time (host clock around a call that ends in a device synchronise) at 401 frames for best_of 1, 2,
    4, 8 and 16, five rounds each after one warm-up call, rounds of the different N interleaved;
  - CUDA-event time of one `RefPrepEngine.speaker_vectors` launch over 16 rows of 400 frames (with the cosine).
Prints one JSON object with the card's name, power limit and maximum SM clock."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
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
    from sopro_b200.weights import synth_mimi_state_dict, synth_state_dict

    torch.set_grad_enabled(False)
    out = {"card (name, power limit, max SM clock, SM clock)": card()}
    cfg = SoproTTSConfig()
    sd = synth_state_dict(cfg, 1000, 0)
    sd["ar.head.bias"] = sd["ar.head.bias"].clone()
    sd["ar.head.bias"][int(cfg.codebook_size)] -= 30.0  # EOS never sampled: 401 steps per take
    tts = SoproTTS.from_state_dict(cfg, sd, IdsTokenizer(1000), synth_mimi_state_dict(), device="cuda:0", weight_dtype="bf16")
    ref = tts.prepare_reference(ref_tokens_tq=torch.randint(0, 2048, (38, 32), generator=torch.Generator().manual_seed(7)))
    text = " ".join(str((17 * j + 5) % 997) for j in range(50))  # 52 ids, as in bench.py

    # ---- the scoring launch: 16 rows x 400 frames
    codes = torch.randint(0, 2048, (16, 400, 32), generator=torch.Generator().manual_seed(3)).to("cuda:0", torch.int32)
    rp = tts.model.refprep
    lens = [400] * 16
    sv_ms = event_ms(lambda: rp.speaker_vectors(codes, lens, ref.sv_ref), 50)
    out["speaker_vectors_16x400_ms (incl. the host check's synchronise)"] = sv_ms

    # ---- synthesize at 401 frames
    Ns = (1, 2, 4, 8, 16)

    def call(n):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        w = tts.synthesize(text, ref=ref, max_frames=400, seed=1, best_of=n)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, w

    for n in Ns:
        _t, w = call(n)  # warm-up: sessions, workspaces, JIT-free but first-use allocations
        assert w.shape[-1] == 401 * 1920, w.shape
    res = {str(n): [] for n in Ns}
    for _round in range(5):
        for n in Ns:
            res[str(n)].append(call(n)[0])
    out["synthesize_401_frames_ms"] = {n: {"median": sorted(v)[len(v) // 2], "all": v} for n, v in res.items()}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
