"""CPU: the live leveller's float64 oracle (oracle/loudness_live_oracle.py) against the one-shot meter's definition
(oracle/loudness_oracle.py) -- M_k of every prefix, the boost cap, the ceiling, short rows and the tail, convergence on
stationary noise and on the one-shot gain -- and the public API's refusals and signatures."""
import inspect
import math

import numpy as np
import pytest
import torch

from oracle import loudness_live_oracle as LO
from oracle import loudness_oracle as O

CEIL32 = float(np.float32(O.CEILING))


def _noise(n, amp, seed=0):
    return (amp * np.random.default_rng(seed).standard_normal(n)).astype(np.float32)


def _gated(n, seed=1):
    """loud noise, 20 dB quieter noise, silence, loud again: both gates act on some prefix"""
    x = _noise(n, 0.3, seed)
    x[n // 4: n // 2] *= 0.1
    x[n // 2: 3 * n // 4] = 0
    return x


@pytest.mark.parametrize("sr", (8000, 22050, 48000))
def test_meter_is_the_integrated_loudness_of_each_prefix(sr):
    s = O.sub_block(sr)
    x = _gated(23 * s + 17)
    M = LO.meters(x, sr)
    assert np.isnan(M[:3]).all()
    for k in range(3, M.size):
        want = O.integrated(x[: (k + 1) * s], sr)
        assert (M[k] == want) or abs(M[k] - want) < 1e-9, (k, M[k], want)
    assert M[-1] == O.integrated(x, sr)


def test_silence_meters_minus_inf_and_keeps_gain_one():
    sr = 16000
    x = np.zeros(9 * O.sub_block(sr) + 5, dtype=np.float32)
    y, a, M = LO.level_live(x, sr, -16.0)
    assert np.isneginf(M[3:]).all() and (a[3:] == 1.0).all()
    assert (y == 0).all()


def test_boost_cap():
    sr = 24000
    x = _noise(30 * O.sub_block(sr), 10 ** (-62 / 20) * 3, seed=3)  # about -60 LUFS: 44 dB under -16
    y, a, M = LO.level_live(x, sr, -16.0)
    assert np.isfinite(M[3:]).all()
    assert (-16.0 - M[3:] > LO.MAX_BOOST_DB).all()
    assert (a[3:] == LO.MAX_BOOST).all()
    # the released gain never exceeds the cap
    assert np.abs(y.astype(np.float64)).max() <= LO.MAX_BOOST * np.abs(x.astype(np.float64)).max()


@pytest.mark.parametrize("sr", (8000, 24000, 96000))
def test_ceiling_holds_in_fp32_on_hot_signals(sr):
    s = O.sub_block(sr)
    g = np.random.default_rng(5)
    for amp, T in ((0.99, 0.0), (0.5, -5.0), (0.05, 0.0)):
        x = (amp * np.clip(g.standard_normal(13 * s + 101), -3, 3) / 3).astype(np.float32)
        x[s // 2] = amp  # a peak
        y, a, _M = LO.level_live(x, sr, T)
        assert np.abs(y).max() <= CEIL32, (amp, T, np.abs(y).max())


@pytest.mark.parametrize("m", (0, 1, 3))
def test_rows_under_four_sub_blocks_go_out_at_unity_under_the_ceiling(m):
    sr = 8000
    s = O.sub_block(sr)
    x = _noise(m * s + 37, 1.5, seed=m)
    y, a, M = LO.level_live(x, sr, -10.0)
    assert a.size == m and np.isnan(M).all()
    for q in range(m + 1):
        seg = x[q * s: min((q + 1) * s, x.size)]
        c = O.CEILING / float(np.abs(seg).max())
        g = np.float32(min(1.0, c))
        if float(g) > min(1.0, c):
            g = np.nextafter(g, np.float32(0))
        assert np.array_equal(y[q * s: q * s + seg.size], (np.float64(g) * seg.astype(np.float64)).astype(np.float32))
    assert np.abs(y).max() <= CEIL32


def test_tail_goes_out_at_the_last_gain():
    sr = 16000
    s = O.sub_block(sr)
    x = _noise(9 * s + 300, 0.01, seed=2)
    y, a, _M = LO.level_live(x, sr, -20.0)
    tail = x[9 * s:].astype(np.float64)
    want = np.float32(a[8])
    if float(want) > a[8]:
        want = np.nextafter(want, np.float32(0))
    assert np.array_equal(y[9 * s:], (np.float64(want) * tail).astype(np.float32))


def test_ramp_between_sub_blocks():
    sr = 8000
    s = O.sub_block(sr)
    x = _gated(12 * s, seed=4) * np.float32(0.05)
    y, a, _M = LO.level_live(x, sr, -23.0)
    k = 6
    i = np.arange(s, dtype=np.float64)
    r = a[k - 1] + (a[k] - a[k - 1]) * ((i + 1) / s)
    g = LO._rz32(r)  # the ceiling does not bind at this level
    assert np.array_equal(y[k * s: (k + 1) * s], (g.astype(np.float64) * x[k * s: (k + 1) * s]).astype(np.float32))


# Stationary noise, 20 s: the meter settles within the first seconds, so the passage's integrated loudness after
# levelling is within 0.1 LU of the target (measured: about 0.01).
@pytest.mark.parametrize("sr,T", ((24000, -16.0), (48000, -23.0), (16000, -30.0)))
def test_stationary_noise_converges_on_the_target(sr, T):
    x = _noise(20 * sr, 0.02, seed=sr % 97)
    y, a, _M = LO.level_live(x, sr, T)
    assert abs(O.integrated(y, sr) - T) < 0.1


@pytest.mark.parametrize("sr", (22050, 24000))
def test_last_gain_is_the_one_shot_gain_when_nothing_binds(sr):
    x = _gated(7 * sr + 11, seed=6) * np.float32(0.1)
    T = -20.0
    _y, a, M = LO.level_live(x, sr, T)
    L = O.integrated(x, sr)
    want = 10 ** ((T - L) / 20)
    assert want < LO.MAX_BOOST and want < O.CEILING / float(np.abs(x).max())
    assert M[-1] == L
    assert math.isclose(a[-1], want, rel_tol=1e-15)


def test_refusals_before_any_device_work():
    from sopro_b200 import _lib
    from sopro_b200.loudness import LiveLeveller, level_live, level_stream, level_stream_batch

    x = torch.zeros(4800)
    for bad in (None, -61.0, 0.5, float("nan"), float("inf"), True, "loud"):
        with pytest.raises(ValueError):
            level_live(x, 24000, bad)
        with pytest.raises(ValueError):
            LiveLeveller(24000, bad, device="cpu")
        with pytest.raises(ValueError):
            level_stream(iter(()), 24000, target=bad)
        with pytest.raises(ValueError):
            level_stream_batch(iter(()), 24000, target=bad)
    for sr in (3999, 192001, 24000.5, "24000"):
        with pytest.raises(ValueError):
            level_live(x, sr, -16.0)
        with pytest.raises(ValueError):
            LiveLeveller(sr, -16.0, device="cpu")
        with pytest.raises(ValueError):
            level_stream(iter(()), sr, target=-16.0)
    with pytest.raises(_lib.SoproError):
        level_live(x, 24000, -16.0)  # a CPU tensor: no CPU path
    with pytest.raises(_lib.SoproError):
        LiveLeveller(24000, -16.0, device="cpu")
    assert list(level_stream(iter(()), 24000, target=-16.0)) == []
    assert list(level_stream_batch(iter(()), 24000, target=-16.0)) == []


def test_public_signatures():
    import sopro_b200
    from sopro_b200 import loudness

    for name in ("level_live", "LiveLeveller", "level_stream", "level_stream_batch"):
        assert name in sopro_b200.__all__ and getattr(sopro_b200, name) is getattr(loudness, name)
    p = inspect.signature(loudness.level_live).parameters
    assert list(p)[:4] == ["wav", "sample_rate", "target", "lens"] and p["lens"].default is None
    p = inspect.signature(loudness.LiveLeveller).parameters
    assert list(p) == ["sample_rate", "target", "device"] and p["device"].default is None
    for f in (loudness.level_stream, loudness.level_stream_batch):
        p = inspect.signature(f).parameters
        assert list(p) == ["items", "sample_rate", "target"]
        assert p["sample_rate"].default == 24000 and p["target"].kind is inspect.Parameter.KEYWORD_ONLY
    from sopro_b200.model import SoproTTS

    for name in ("stream", "stream_batch", "stream_long", "stream_dialogue"):
        assert "loudness" not in inspect.signature(getattr(SoproTTS, name)).parameters


def test_header_states_the_boost_cap():
    import os

    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "sopro_b200.h")).read()
    assert "B = 30 dB" in hdr and LO.MAX_BOOST_DB == 30.0
