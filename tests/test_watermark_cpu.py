"""CPU: the watermark's host side (sopro_b200/watermark.py, csrc/watermark.cu) -- the library's pattern against the
float64 oracle, the constants against include/sopro_b200.h, refused keys, workspace sizes -- and the robustness and
null behaviour of the definition itself, through the float64 oracle (oracle/watermark_oracle.py) the GPU tests judge
the kernels by."""
import ctypes as C
import inspect
import os
import re
from fractions import Fraction

import numpy as np
import pytest
import torch
from scipy.signal import resample_poly

from oracle import flac_oracle as FO
from oracle import watermark_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REFUSED = (-1, 1 << 32, 2 ** 40, True, False, np.bool_(True), 1.0, 3.5, "7", [7], float("nan"))
SR = 24000
# the shortest crop the robustness test promises detection on: at the fixed -30 dB level, 3 s crops of these rows
# scored as low as 6.3 (a Mimi row, its peak one lag off) and 6.8 (a speech-like row), 4 s crops 7.8 at the lowest
MIN_CROP = 4 * SR


def speech_like(n: int, seed: int) -> np.ndarray:
    """A voiced, speech-like row at 24 kHz: a gliding f0 of 100 to 245 Hz, harmonics falling 6 dB per octave under three
    formants, a 3 to 5 Hz syllable envelope with silences, and a -60 dB noise floor; 0.3 peak."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / SR
    f0 = 100 + 120 * rng.random() + 25 * np.sin(2 * np.pi * (0.3 + 0.5 * rng.random()) * t + 6 * rng.random())
    ph = 2 * np.pi * np.cumsum(f0) / SR
    formants = [(400 + 400 * rng.random(), 1.0), (1200 + 800 * rng.random(), 0.5), (2400 + 600 * rng.random(), 0.3)]
    x = np.zeros(n)
    for h in range(1, 60):
        fh = h * f0
        env = sum(a * np.exp(-((fh - f) / 150.0) ** 2) for f, a in formants) + 0.02
        x += env / h * np.sin(h * ph + 6 * rng.random()) * (fh < 0.45 * SR)
    syl = np.clip(np.sin(2 * np.pi * (3 + 2 * rng.random()) * t + 6 * rng.random()), 0, None) ** 0.7
    x = x * syl + 0.001 * rng.standard_normal(n)
    return 0.3 * x / np.abs(x).max()


_MIMI = {}


def mimi_rows(k: int, n: int) -> list:
    """k rows of a real Mimi decode (synthetic checkpoint, seeded codes) on the CPU oracle, each n samples, 0.5 peak."""
    if "w" not in _MIMI:
        from oracle import mimi_oracle as MO

        codes = torch.randint(0, 2048, (1, 32, 50), generator=torch.Generator().manual_seed(7))
        w = MO.mimi_decode(MO.synth_mimi_state_dict(), codes).reshape(-1).double().numpy()
        _MIMI["w"] = 0.5 * w / np.abs(w).max()
    w = _MIMI["w"]
    return [np.roll(np.tile(w, n // len(w) + 1), -9973 * i)[:n] for i in range(k)]


def round_trip(x: np.ndarray, sr: int) -> np.ndarray:
    f = Fraction(sr, SR)
    return resample_poly(resample_poly(x, f.numerator, f.denominator), f.denominator, f.numerator)[: len(x)]


def pcm16(x: np.ndarray) -> np.ndarray:
    return FO.to_pcm16(x.astype(np.float32)).astype(np.float64) / 32767.0


CONDITIONS = {
    "none": lambda x: x,
    "8k": lambda x: round_trip(x, 8000),
    "16k": lambda x: round_trip(x, 16000),
    "22.05k": lambda x: round_trip(x, 22050),
    "44.1k": lambda x: round_trip(x, 44100),
    "48k": lambda x: round_trip(x, 48000),
    "gain-20dB": lambda x: x * 10 ** (-20 / 20),
    "limit-1dBFS": lambda x: np.clip(x * (1.0 / np.abs(x).max()), -10 ** (-1 / 20), 10 ** (-1 / 20)),
    "pcm16": pcm16,
    "flac": lambda x: FO.decode(FO.encode(x.astype(np.float32), SR))[1].astype(np.float64) / 32767.0,
}


def _header_defines():
    hdr = open(os.path.join(ROOT, "include", "sopro_b200.h")).read()
    return {k: float(v) for k, v in re.findall(r"#define SOPRO_WATERMARK_([A-Z_]+) \(?(-?[0-9.]+)\)?", hdr)}


def test_constants_agree_with_the_header():
    from sopro_b200 import watermark as W

    d = _header_defines()
    assert (d["PERIOD"], d["BLOCK"], d["THRESHOLD"]) == (W.PERIOD, W.BLOCK, W.THRESHOLD)
    assert (d["PERIOD"], d["BLOCK"], d["THRESHOLD"]) == (O.P, O.BLOCK, O.THRESHOLD)
    assert (d["LO_HZ"], d["HI_HZ"]) == (O.LO_HZ, O.HI_HZ)
    assert O.LEVEL == 10 ** (d["LEVEL_DB"] / 20) and O.FLOOR == 10 ** (d["FLOOR_DB"] / 20)
    assert (O.bins()[0], O.bins()[-1]) == (342, 1194)


@pytest.mark.parametrize("key", (0, 1, 12345, 2 ** 32 - 1))
def test_pattern_equals_the_oracle_rounded_once_in_band_with_unit_rms(key):
    from sopro_b200.watermark import watermark_pattern

    got = watermark_pattern(key)
    want = O.pattern(key)
    assert got.dtype == np.float32 and got.shape == (O.P,)
    # the library sums in a different order; both round the same double to fp32 (at most one ulp apart at a tie)
    ulp = np.spacing(np.abs(want).astype(np.float32))
    assert (np.abs(got.astype(np.float64) - want) <= ulp).all()
    spec = np.abs(np.fft.rfft(got.astype(np.float64)))
    band = np.zeros(len(spec), dtype=bool)
    band[O.bins()] = True
    assert spec[~band].max() <= 1e-4 * spec[band].min()
    assert abs(np.sqrt(np.mean(got.astype(np.float64) ** 2)) - 1.0) <= 1e-6


def test_keys_give_unrelated_patterns():
    from sopro_b200.watermark import watermark_pattern

    a, b = watermark_pattern(5).astype(np.float64), watermark_pattern(6).astype(np.float64)
    assert np.abs(O.correlate(a, b)).max() / O.P < 0.1


@pytest.mark.parametrize("key", REFUSED)
def test_refused_keys_raise_value_error(key):
    from sopro_b200.watermark import check_watermark, watermark_pattern

    with pytest.raises(ValueError):
        check_watermark(key)
    with pytest.raises(ValueError):
        watermark_pattern(key)


def test_the_library_refuses_keys_and_geometry():
    from sopro_b200 import _lib

    lib = _lib.load()
    out = np.full(O.P, 7.0, dtype=np.float32)
    for key in (-1, 1 << 32):
        assert lib.sopro_watermark_pattern(key, out.ctypes.data) == -1 and (out == 7.0).all()
    e, d = C.c_int64(), C.c_int64()
    assert lib.sopro_watermark_sizes(0, 100, C.byref(e), C.byref(d)) == -1
    assert lib.sopro_watermark_sizes(1, -1, C.byref(e), C.byref(d)) == -1
    assert lib.sopro_watermark_sizes(3, 1000, C.byref(e), C.byref(d)) == 0
    assert e.value >= 3 * 5 * 8 and d.value >= e.value + 2 * 3 * O.P * 4


def test_the_public_api_takes_a_watermark_key():
    from sopro_b200 import detect_watermark
    from sopro_b200.model import SoproTTS
    from sopro_b200.streaming import stream

    for fn in (SoproTTS.synthesize, SoproTTS.synthesize_batch, SoproTTS.synthesize_long, SoproTTS.stream,
               stream):
        p = inspect.signature(fn).parameters["watermark"]
        assert p.default is None and p.kind is inspect.Parameter.KEYWORD_ONLY
    assert list(inspect.signature(detect_watermark).parameters) == ["wav", "sample_rate", "key", "lens"]


class _FakeTTS:
    def _resampler(self, sample_rate):
        from sopro_b200.resample import check_rates

        if sample_rate is not None:
            check_rates(24000, sample_rate)
        return None


def test_output_chain_checks_the_key_after_loudness_and_before_any_draw():
    from sopro_b200.output import OutputChain

    tts = _FakeTTS()
    before = torch.get_rng_state()
    with pytest.raises(ValueError, match="loudness"):
        OutputChain(tts, None, None, 5.0, -1)  # a refused target is reported first
    with pytest.raises(ValueError, match="speed"):
        OutputChain(tts, None, 9.0, None, True)
    for key in REFUSED:
        with pytest.raises(ValueError, match="watermark"):
            OutputChain(tts, None, None, -16.0, key)
    assert torch.equal(before, torch.get_rng_state())
    assert OutputChain(tts, None, None, None, 2 ** 32 - 1).key == 2 ** 32 - 1
    assert OutputChain(tts).key is None


def _rows():
    """20 speech-like rows and 4 Mimi rows, 5 s each."""
    n = 5 * SR
    return [speech_like(n, s) for s in range(20)] + mimi_rows(4, n)


def test_oracle_mark_survives_every_condition_and_crop():
    """Every row marked with its own key, every condition, a random crop of MIN_CROP up to the whole row: score >=
    THRESHOLD and the offset is the crop's start modulo P."""
    rng = np.random.default_rng(11)
    worst = {}
    for i, x in enumerate(_rows()):
        key = 1000 + 17 * i
        p = O.pattern(key)
        y = O.embed(x, p)
        for name, f in CONDITIONS.items():
            z = f(y)
            m = int(rng.integers(MIN_CROP, len(z) + 1))
            s = int(rng.integers(0, len(z) - m + 1))
            score, off = O.detect(z[s: s + m], p)
            assert score >= O.THRESHOLD and off == s % O.P, (i, name, score, off, s % O.P)
            worst[name] = min(worst.get(name, np.inf), score)
    print("lowest score per condition:", {k: round(v, 2) for k, v in worst.items()})


def test_oracle_null_never_reaches_the_threshold():
    """2000 unmarked rows (speech-like, Mimi, white noise), and marked rows under a wrong key: no score reaches THRESHOLD."""
    rng = np.random.default_rng(5)
    base = [speech_like(4 * SR, 100 + s) for s in range(12)] + mimi_rows(4, 4 * SR)
    scores = []
    for i in range(2000):
        key = int(rng.integers(0, 2 ** 32))
        p = O.pattern(key) if i < 40 else _cached_pattern(i % 40, rng)
        kind = i % 3
        if kind == 0:
            x = base[i % len(base)]
        elif kind == 1:
            x = 0.1 * rng.standard_normal(3 * SR)
        else:  # marked with another key
            x = O.embed(base[i % len(base)], _cached_pattern((i + 7) % 40, rng))
        m = int(rng.integers(SR, len(x) + 1))
        s = int(rng.integers(0, len(x) - m + 1))
        scores.append(O.detect(x[s: s + m], p)[0])
    print(f"null: max score {max(scores):.2f}, 99th percentile {np.percentile(scores, 99):.2f} over {len(scores)} rows")
    assert max(scores) < O.THRESHOLD


_PATTERNS = {}


def _cached_pattern(j, rng):
    if j not in _PATTERNS:
        _PATTERNS[j] = O.pattern(50_000 + 7919 * j)
    return _PATTERNS[j]
