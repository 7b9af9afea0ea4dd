"""Cost of a voice per text on the GPU (bench.py's workload: synthetic seeded checkpoint, bf16 AR weights, EOS logit
pushed down so every utterance runs the full 401 AR steps, 52-id texts; nothing is written):
  - 64 texts in 64 distinct voices: a loop of 64 `synthesize` calls against one `synthesize_batch(ref=[...])`, host
    clock around calls that end in a device synchronise, rounds alternated after one warm-up of each;
  - 64 texts in one voice: `synthesize_batch(ref=r)` of this tree against another build of the project (`--parent DIR`,
    a built checkout of the parent commit), each in its own resident worker process, calls alternated between the
    two, with a digest of every waveform so equal outputs show as equal digests;
  - the prefill alone (PrefillEngine.run, 64 texts, 401 frames), one voice against 64 voices, CUDA events.
Prints one JSON object with the card's name, power limit and SM clocks read in the same run.

  python tools/prof_voices.py [--parent DIR] [--rounds N]"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_TEXTS = 64


def card():
    import torch

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def build_tts(root):
    """bench.py's model from the tree at `root` (its own bench.py and library)."""
    sys.path.insert(0, root)
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


def digest(wavs):
    h = hashlib.sha256()
    for w in wavs:
        h.update(w.detach().cpu().numpy().tobytes())
    return h.hexdigest()[:16]


def worker(root):
    """Resident shared-voice worker: one line on stdin = one timed synthesize_batch of 64 texts; replies with a JSON
    line {ms, digest}."""
    tts, bench = build_tts(root)
    ref = tts.prepare_reference(ref_tokens_tq=bench.bench_ref_tokens())
    texts = bench.bench_texts(0, N_TEXTS)
    seeds = list(range(1234, 1234 + N_TEXTS))

    def call():
        return tts.synthesize_batch(texts, ref=ref, seeds=seeds, max_frames=400, min_gen_frames=10 ** 9)

    call()  # warm-up: sessions, workspaces
    print(json.dumps({"ready": True}), flush=True)
    for _line in sys.stdin:
        ms, wavs = timed(call)
        print(json.dumps({"ms": ms, "digest": digest(wavs)}), flush=True)


def shared_voice(parent, rounds):
    trees = {"this": ROOT, "parent": parent}
    procs = {k: subprocess.Popen([sys.executable, os.path.abspath(__file__), "--worker", v], stdin=subprocess.PIPE,
                                 stdout=subprocess.PIPE, text=True, cwd=v) for k, v in trees.items()}
    try:
        for p in procs.values():
            assert json.loads(p.stdout.readline())["ready"]
        res = {k: {"ms": [], "digests": set()} for k in trees}
        for _ in range(rounds):
            for k in ("parent", "this"):
                procs[k].stdin.write("go\n")
                procs[k].stdin.flush()
                r = json.loads(procs[k].stdout.readline())
                res[k]["ms"].append(r["ms"])
                res[k]["digests"].add(r["digest"])
    finally:
        for p in procs.values():
            p.stdin.close()
            p.wait(timeout=120)
    out = {k: {"median_ms": sorted(v["ms"])[len(v["ms"]) // 2], "all_ms": v["ms"], "digests": sorted(v["digests"])}
           for k, v in res.items()}
    out["outputs_identical"] = out["this"]["digests"] == out["parent"]["digests"] and len(out["this"]["digests"]) == 1
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", default=None, help="a built checkout of the parent commit (shared-voice comparison)")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--worker", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        return worker(args.worker)
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("prof_voices.py measures on a CUDA device; there is none")
    out = {"card (name, power limit, max SM clock, SM clock)": card()}
    tts, bench = build_tts(ROOT)
    g = torch.Generator().manual_seed(5)
    trs = torch.randint(38, 301, (N_TEXTS,), generator=g).tolist()  # 3 to 24 s of reference audio
    refs = [tts.prepare_reference(ref_tokens_tq=torch.randint(0, 2048, (t, 32), generator=g)) for t in trs]
    texts = bench.bench_texts(0, N_TEXTS)
    seeds = list(range(1234, 1234 + N_TEXTS))
    kw = dict(max_frames=400, min_gen_frames=10 ** 9)

    # ---- 64 texts in 64 voices: a loop of synthesize against one synthesize_batch
    def loop():
        return [tts.synthesize(t, ref=r, seed=s, **kw) for t, r, s in zip(texts, refs, seeds)]

    def batch():
        return tts.synthesize_batch(texts, ref=refs, seeds=seeds, **kw)

    _, a = timed(loop)
    _, b = timed(batch)
    same = sum(bool(torch.equal(x, y)) for x, y in zip(a, b))
    res = {"loop_of_synthesize": [], "synthesize_batch": []}
    for _ in range(max(1, args.rounds // 2)):
        res["loop_of_synthesize"].append(timed(loop)[0])
        res["synthesize_batch"].append(timed(batch)[0])
    med = {k: sorted(v)[len(v) // 2] for k, v in res.items()}
    out["64_texts_64_voices_401_frames"] = {
        "reference_frames": {"min": min(trs), "max": max(trs)},
        "median_ms": med, "all_ms": res, "speedup": med["loop_of_synthesize"] / med["synthesize_batch"],
        "rows_equal_to_synthesize": f"{same}/{N_TEXTS}"}

    # ---- the prefill alone: one voice against 64 voices
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

    pre = {"1_voice": [], "64_voices": []}
    for _ in range(3):
        pre["1_voice"].append(event_ms(refs[0]))
        pre["64_voices"].append(event_ms(refs))
    out["prefill_64_texts_401_frames_ms (CUDA events, incl. host copies of the voice table)"] = {
        k: {"median": sorted(v)[len(v) // 2], "all": v} for k, v in pre.items()}
    del tts, refs, pe
    torch.cuda.empty_cache()

    # ---- 64 texts in one voice: this build against the parent's
    if args.parent:
        out["64_texts_1_voice_synthesize_batch (this vs parent, alternated)"] = shared_voice(os.path.abspath(args.parent),
                                                                                              args.rounds)
    else:
        out["64_texts_1_voice_synthesize_batch (this vs parent, alternated)"] = "not measured: no --parent"
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
