"""Cost of preparing reference voices on the GPU, in one process (synthetic seeded weights; the WAV files go to a temporary
directory that is removed at the end):
  (a) today's loop, one `prepare_reference(ref_audio_path=...)` per voice, split into its host preparation (file read,
      energy trim, torchaudio resample, crop: host clock) and its device part (Mimi encode + reference preparation:
      CUDA events);
  (b) one `prepare_references(paths)` call (host clock around a call that ends in a device synchronise; it reads the
      same files), and the same call on the clips already on the device (no file read).
B = 1, 8 and 64 clips of 10 s at 44.1 kHz and at 16 kHz; three rounds after one warm-up, (a) and (b) interleaved within
each round.  Prints one JSON object with the card's name, power limit, maximum SM clock and SM clock."""
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def voice(sr, seed, secs=10.0):
    """speech-like: a gliding tone in syllable-rate bursts over a faint noise floor, 0.6 s of silence at both ends"""
    g = np.random.default_rng(seed)
    t = np.arange(int(sr * secs)) / sr
    f0 = 120 + 60 * np.sin(2 * np.pi * 0.3 * t + seed)
    env = (0.5 + 0.5 * np.sin(2 * np.pi * 4.0 * t)) * ((t > 0.6) & (t < secs - 0.6))
    x = 0.4 * env * np.sin(2 * np.pi * np.cumsum(f0) / sr) + 1e-3 * g.standard_normal(t.size)
    return torch.from_numpy(x.astype(np.float32))


def main():
    from sopro_b200 import SoproTTS
    from sopro_b200.audio import center_crop_audio, load_audio_file, resample, save_audio, trim_silence_energy
    from sopro_b200.config import SoproTTSConfig
    from sopro_b200.tokenizer import IdsTokenizer
    from sopro_b200.weights import synth_mimi_encoder_state_dict, synth_mimi_state_dict, synth_state_dict

    torch.set_grad_enabled(False)
    out = {"card (name, power limit, max SM clock, SM clock)": card()}
    cfg = SoproTTSConfig()
    msd = dict(synth_mimi_state_dict())
    msd.update(synth_mimi_encoder_state_dict())
    tts = SoproTTS.from_state_dict(cfg, synth_state_dict(cfg, 1000, 0), IdsTokenizer(1000), msd, device="cuda:0")
    codec, model = tts.codec, tts.model
    win = 12 * 1920

    def loop(paths):
        """(a): returns (host prep ms, device ms, wall ms)"""
        host = dev = 0.0
        torch.cuda.synchronize()
        t_all = time.perf_counter()
        for p in paths:
            t0 = time.perf_counter()
            w, sr = load_audio_file(p)
            w = center_crop_audio(resample(trim_silence_energy(w, sr), sr, 24000), win)
            host += time.perf_counter() - t0
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            model.prepare_reference(codec.encode_wav(w).long(), device=tts.device)
            b.record()
            b.synchronize()
            dev += a.elapsed_time(b)
        return host * 1e3, dev, (time.perf_counter() - t_all) * 1e3

    def batched(clips, rates):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        refs = tts.prepare_references(clips, sample_rates=rates)
        torch.cuda.synchronize()
        assert len(refs) == len(clips)
        return (time.perf_counter() - t0) * 1e3

    res = {}
    with tempfile.TemporaryDirectory() as tmp:
        cases = []
        for sr in (44100, 16000):
            wavs = [voice(sr, 100 * (sr // 1000) + i) for i in range(64)]
            paths = []
            for i, w in enumerate(wavs):
                paths.append(os.path.join(tmp, f"v{sr}_{i}.wav"))
                save_audio(paths[-1], w, sr)
            dev_wavs = [w.cuda() for w in wavs]
            for B in (1, 8, 64):
                cases.append((f"{B} x 10 s @ {sr} Hz", paths[:B], dev_wavs[:B], sr))
        for name, paths, dw, sr in cases:  # warm-up: workspaces, resamplers, first-use allocations
            loop(paths[:1])
            batched(paths, None)
            batched(dw, [sr] * len(dw))
            res[name] = {"a_host_prep_ms": [], "a_device_ms": [], "a_wall_ms": [], "b_paths_ms": [], "b_device_clips_ms": []}
        for _round in range(3):
            for name, paths, dw, sr in cases:
                h, d, w = loop(paths)
                r = res[name]
                r["a_host_prep_ms"].append(h)
                r["a_device_ms"].append(d)
                r["a_wall_ms"].append(w)
                r["b_paths_ms"].append(batched(paths, None))
                r["b_device_clips_ms"].append(batched(dw, [sr] * len(dw)))
    out["ms (median of 3 rounds)"] = {n: {k: round(sorted(v)[1], 2) for k, v in r.items()} for n, r in res.items()}
    out["ms (all rounds)"] = {n: {k: [round(x, 2) for x in v] for k, v in r.items()} for n, r in res.items()}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
