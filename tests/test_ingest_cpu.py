"""Voice ingestion without a GPU: the float64 oracle of the trim and crop against the unmodified reference's fixture and
against sopro_b200.audio.trim_silence_energy at every common rate, and the argument refusals of prepare_references,
which happen before any clip is read or any device work."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import ingest_oracle as O
from sopro_b200 import ingest
from sopro_b200.audio import trim_silence_energy
from tests.golden.make_audio_golden import CASES, signal

HERE = os.path.dirname(os.path.abspath(__file__))
RATES = [8000, 16000, 22050, 24000, 44100, 48000]


def test_oracle_reproduces_the_reference_fixture():
    with open(os.path.join(HERE, "golden", "audio_prep.json")) as f:
        gold = json.load(f)
    assert sorted(gold) == sorted(c[0] for c in CASES)
    for i, (name, sr, n, lo, hi, floor) in enumerate(CASES):
        x = signal(sr, n, lo, hi, floor, i)[0].numpy()
        s, e = O.trim_extent(x, sr)
        t = x[s:e]
        o, m = O.crop_plan(t.size, 12 * 1920)
        c = t[o:o + m]
        g = gold[name]
        assert (t.size, float(t[0]), float(t[-1])) == (g["trim_len"], g["trim_first"], g["trim_last"]), name
        assert (c.size, float(c[0])) == (g["crop_len"], g["crop_first"]), name
        assert t.astype(np.float64).sum() == pytest.approx(g["trim_sum"], rel=1e-12, abs=1e-12), name
        assert c.astype(np.float64).sum() == pytest.approx(g["crop_sum"], rel=1e-12, abs=1e-12), name


def seeded_clip(sr: int, seed: int) -> np.ndarray:
    """A tone burst with a random span, level and noise floor, 0.05 to 4 s long."""
    rng = np.random.default_rng(seed)
    n = int(rng.integers(int(0.05 * sr), 4 * sr))
    floor = float(rng.choice([0.0, 1e-4, 1e-3, 3e-2]))
    x = rng.standard_normal(n) * floor
    lo, hi = int(rng.uniform(0.0, 0.45) * n), n - int(rng.uniform(0.0, 0.45) * n)
    t = np.arange(hi - lo) / sr
    x[lo:hi] += float(rng.uniform(0.05, 0.8)) * np.sin(2 * np.pi * float(rng.uniform(80, 900)) * t)
    x[lo:hi] += rng.standard_normal(hi - lo) * 0.02
    return x.astype(np.float32)


def near_tie(x: np.ndarray, sr: int, tol_db: float = 1e-4) -> bool:
    d = O.trim_detail(x, sr)
    return d["db"] is not None and bool((np.abs(d["db"] - d["thr"]) <= tol_db).any())


@pytest.mark.parametrize("sr", RATES)
def test_oracle_matches_the_host_trim(sr):
    kept = 0
    for seed in range(12):
        x = seeded_clip(sr, 1000 * sr + seed)
        s, e = O.trim_extent(x, sr)
        got = trim_silence_energy(torch.from_numpy(x).unsqueeze(0), sr)[0]
        if got.numel() == e - s and torch.equal(got, torch.from_numpy(x[s:e])):
            kept += int((s, e) != (0, x.size))
            continue
        assert near_tie(x, sr), (sr, seed, (s, e), got.numel())
    assert kept >= 3, kept  # the clips exercise the trim, not only its untouched cases


def test_crop_window_and_plan():
    assert ingest.crop_samples(None) == O.crop_window(None) == 0
    assert ingest.crop_samples(0) == ingest.crop_samples(-1.0) == 0
    for s in (0.01, 1.0, 3.3, 12.0, 12.04, 30):
        assert ingest.crop_samples(s) == O.crop_window(s) == max(1, round(s * 12.5)) * 1920
    for n, w in ((100, 0), (100, 100), (101, 100), (5000, 1920), (1, 1920)):
        assert ingest.crop_plan(n, w) == O.crop_plan(n, w)
    assert O.crop_plan(5001, 1920) == ((5001 - 1920) // 2, 1920)


def _stub():
    from sopro_b200.model import SoproTTS

    return SoproTTS.__new__(SoproTTS)  # no codec, no model, no device: a refusal must come first


@pytest.mark.parametrize("clips,rates,exc", [
    ([], None, ValueError),
    ("voice.wav", None, TypeError),
    ([torch.zeros(0)], [16000], ValueError),
    ([torch.zeros(2, 0)], [16000], ValueError),
    ([torch.zeros(100, dtype=torch.int16)], [16000], TypeError),
    ([torch.zeros(100, dtype=torch.bool)], [16000], TypeError),
    ([torch.zeros(100)], [44099], ValueError),
    ([torch.zeros(100)], None, ValueError),
    ([torch.zeros(100)], [16000, 16000], ValueError),
    ([torch.zeros(100), 3], [16000, None], TypeError),
    ([torch.zeros(1).expand(24000 * 600 + 1)], [24000], ValueError),
    ([torch.zeros(1).expand(8000 * 600 + 1)], [8000], ValueError),
    ([torch.zeros(1, 1, 100)], [16000], ValueError),
])
def test_refusals_before_anything_is_loaded(clips, rates, exc):
    # a path listed first would raise FileNotFoundError if it were read before the tensors are checked
    if isinstance(clips, list) and clips:
        clips = ["/nonexistent/voice.wav"] + clips
        rates = None if rates is None else [None] + list(rates)
    with pytest.raises(exc):
        _stub().prepare_references(clips, sample_rates=rates)
    with pytest.raises(TypeError):
        _stub().prepare_references([torch.zeros(100)], sample_rates=[16000], ref_seconds="12")


def test_a_long_clip_at_the_bound_is_accepted():
    wavs, rates = ingest.load_clips([torch.zeros(1).expand(8000 * 600)], 8000)
    assert rates == [8000] and wavs[0].shape == (8000 * 600,)
