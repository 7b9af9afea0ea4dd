"""CPU: the loudness meter's host side (sopro_b200/loudness.py, csrc/loudness.cu) -- K-weighting coefficients, refused
targets and rates, workspace sizes, the `loudness` keyword of the public API -- and known answers of the float64 oracle
(oracle/loudness_oracle.py) the GPU tests judge the kernels by."""
import inspect
import math

import numpy as np
import pytest
import torch

from oracle import loudness_oracle as O

RATES = (8000, 11025, 16000, 22050, 24000, 44100, 48000, 96000, 192000, 12345)
REFUSED = (float("nan"), float("inf"), -float("inf"), -60.5, 0.5, True, False, "-16", [-16.0], np.bool_(True))


def test_coefficients_at_48k_match_the_bs1770_table():
    from sopro_b200.loudness import loudness_filter

    b1, a1, b2, a2 = loudness_filter(48000)
    assert np.abs(b1 - [1.53512485958697, -2.69169618940638, 1.19839281085285]).max() <= 1e-12
    assert np.abs(a1 - [1.0, -1.69065929318241, 0.73248077421585]).max() <= 1e-12
    assert np.array_equal(b2, [1.0, -2.0, 1.0])
    assert np.abs(a2 - [1.0, -1.99004745483398, 0.99007225036621]).max() <= 1e-12


@pytest.mark.parametrize("sr", RATES)
def test_coefficients_equal_the_oracle_bit_for_bit(sr):
    from sopro_b200.loudness import loudness_filter

    for got, want in zip(loudness_filter(sr), O.filter_coeffs(sr)):
        assert got.dtype == np.float64 and np.array_equal(got.view(np.uint64), want.view(np.uint64)), sr


def test_refused_rates():
    import ctypes as C

    from sopro_b200 import _lib
    from sopro_b200.loudness import loudness_filter, workspace_bytes

    lib = _lib.load()
    c = (C.c_double * 10)(*([7.0] * 10))
    for sr in (0, 3999, 192001, -48000):
        assert lib.sopro_loudness_filter(sr, C.cast(c, C.c_void_p)) == -1 and list(c) == [7.0] * 10
        assert lib.sopro_loudness_workspace(1, 100, sr) < 0
        with pytest.raises(ValueError):
            loudness_filter(sr)
        with pytest.raises(ValueError):
            workspace_bytes(1, 100, sr)
    for sr in (4000, 192000):
        loudness_filter(sr)
    with pytest.raises(ValueError):
        loudness_filter(44100.5)


@pytest.mark.parametrize("target", REFUSED)
def test_refused_targets_raise_value_error(target):
    from sopro_b200.loudness import check_loudness

    with pytest.raises(ValueError):
        check_loudness(target)


def test_accepted_targets():
    from sopro_b200 import _lib
    from sopro_b200.loudness import check_loudness

    assert check_loudness(None) is None
    for t in (-60, -60.0, -23, -16.5, -14, 0, 0.0, np.float32(-24.0), np.float64(-1.0)):
        assert check_loudness(t) == float(t)
    lib = _lib.load()
    for t in (float("nan"), float("inf"), -float("inf"), -60.000001, 1e-9):
        assert lib.sopro_loudness_target(t) == -1


def test_workspace_is_host_arithmetic():
    """Sizes come from (rows, length, rate) alone; they grow with both, and zero-length rows still have their L and g."""
    from sopro_b200.loudness import workspace_bytes

    w = {(B, n): workspace_bytes(B, n, 48000) for B in (1, 3, 64) for n in (0, 1, 8192, 8193, 19_200_000)}
    assert all(v > 0 for v in w.values())
    for B in (1, 3, 64):
        assert w[(B, 0)] <= w[(B, 1)] <= w[(B, 8192)] < w[(B, 8193)] < w[(B, 19_200_000)]
    for n in (1, 8193, 19_200_000):
        assert w[(1, n)] < w[(3, n)] < w[(64, n)]
    assert w[(1, 19_200_000)] < 4 * 19_200_000  # a few bytes per sample
    for bad in ((0, 100), (-1, 100), (1, -1)):
        with pytest.raises(ValueError):
            workspace_bytes(*bad, 48000)


def test_loudness_keyword_defaults_to_none_and_stream_has_none():
    from sopro_b200 import SoproTTS
    from sopro_b200.streaming import stream

    for f in (SoproTTS.synthesize, SoproTTS.synthesize_batch):
        p = inspect.signature(f).parameters["loudness"]
        assert p.default is None and p.kind == inspect.Parameter.KEYWORD_ONLY, f
    for f in (SoproTTS.stream, stream):
        assert "loudness" not in inspect.signature(f).parameters, f


def test_refused_target_raises_before_any_work():
    """The target is checked next to the output rate and the speed, before the text, the reference, the prefill or a
    random draw: these objects have no model at all."""
    from sopro_b200.model import SoproTTS

    tts = SoproTTS.__new__(SoproTTS)
    tts._resamplers = {}
    before = torch.get_rng_state()
    for target in (float("nan"), 3.0, -61, True, "-16"):
        with pytest.raises(ValueError):
            tts.synthesize("1 2", loudness=target)
        with pytest.raises(ValueError):
            tts.synthesize_batch(["1 2"], ref=None, loudness=target)
    assert torch.equal(before, torch.get_rng_state())


# ---- the float64 oracle's known answers

def _sine(f, n, sr, amp):
    return amp * np.sin(2 * np.pi * f * np.arange(n) / sr)


@pytest.mark.parametrize("amp", (1.0, 0.5, 0.1, 0.01))
def test_oracle_997_hz_sine(amp):
    """BS.1770: a 997 Hz sine at 48 kHz reads 20 log10(A) - 3.01 LUFS (the K-weighting is ~0 dB there)."""
    L = O.integrated(_sine(997.0, 5 * 48000, 48000, amp), 48000)
    assert abs(L - (20 * math.log10(amp) - 3.01)) <= 0.01, L


def test_oracle_relative_gate():
    """A loud segment next to one more than 10 LU quieter reads as the loud segment alone (up to the three blocks that
    straddle the join: 20 s segments keep them under 0.05 LU)."""
    sr = 16000
    loud = _sine(997.0, 20 * sr, sr, 0.5)
    quiet = _sine(997.0, 20 * sr, sr, 0.5 * 10 ** (-15 / 20))
    alone = O.integrated(loud, sr)
    both = O.integrated(np.concatenate([loud, quiet]), sr)
    assert abs(both - alone) <= 0.05, (both, alone)
    # without the relative gate the quiet blocks would pull the mean down by ~3 LU
    z = O.block_energies(np.concatenate([loud, quiet]), sr)
    ungated = -0.691 + 10 * math.log10(z[z > O.ABS_GATE_E].mean())
    assert both - ungated > 2.0, (both, ungated)


def test_oracle_absolute_gate():
    """A -71 LUFS segment is ignored next to a -65 LUFS one, although it is within 10 LU of it: the relative gate alone
    would keep it."""
    sr = 24000
    main = _sine(997.0, 20 * sr, sr, 10 ** ((-65 + 3.01) / 20))
    faint = _sine(997.0, 20 * sr, sr, 10 ** ((-71 + 3.01) / 20))
    assert O.integrated(faint, sr) == -math.inf
    alone = O.integrated(main, sr)
    assert abs(alone + 65) <= 0.05
    assert abs(O.integrated(np.concatenate([main, faint]), sr) - alone) <= 0.05
    z = O.block_energies(np.concatenate([main, faint]), sr)
    no_abs = -0.691 + 10 * math.log10(z[z > z.mean() * O.REL_FACTOR].mean())
    assert alone - no_abs > 2.0, (alone, no_abs)


@pytest.mark.parametrize("sr", (8000, 11025, 24000, 48000))
def test_oracle_short_rows_and_silence_read_minus_inf(sr):
    s = O.sub_block(sr)
    x = _sine(997.0, 4 * s, sr, 0.5)
    assert O.integrated(x[: 4 * s - 1], sr) == -math.inf
    assert math.isfinite(O.integrated(x, sr))
    assert O.integrated(np.zeros(10 * s), sr) == -math.inf
    assert O.integrated(np.zeros(0), sr) == -math.inf
    assert O.gain(-math.inf, 0.0, -16.0) == 1.0
