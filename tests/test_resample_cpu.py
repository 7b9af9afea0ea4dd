"""CPU: the output resampler's host side (sopro_b200/resample.py, csrc/resample.cu) -- the filter taps and output lengths
against torchaudio's float64 resampler, refused rates, and the `sample_rate` keyword of the public API."""
import inspect
import math

import numpy as np
import pytest
import torch

TA_RATES = (8000, 11025, 16000, 22050, 32000, 44100, 48000, 96000, 12345)


def _ta_kernel(sr):
    """torchaudio's own kernel for 24 kHz -> sr in float64 (the oracle), [n, 2 * width + o], and width."""
    F = pytest.importorskip("torchaudio.functional.functional")
    k, width = F._get_sinc_resample_kernel(24000, sr, math.gcd(24000, sr), dtype=torch.float64)
    return k[:, 0].numpy(), int(width)


@pytest.mark.parametrize("sr", TA_RATES)
def test_taps_are_torchaudio_float64_rounded_once_with_zeros_trimmed(sr):
    from sopro_b200.resample import filter_taps

    k64, width = _ta_kernel(sr)
    o, n, w, first, span, taps = filter_taps(24000, sr)
    g = math.gcd(24000, sr)
    assert (o, n, w) == (24000 // g, sr // g, width) and k64.shape == (n, 2 * w + o)
    k32 = k64.astype(np.float32)
    assert taps.shape == (n, int(span.max()))
    for p in range(n):
        nz = np.nonzero(k32[p])[0]
        assert (first[p], span[p]) == (nz[0], nz[-1] - nz[0] + 1), p  # exactly the nonzero fp32 span
        ref = k32[p, first[p]: first[p] + span[p]]
        ulp = np.spacing(np.abs(ref)).astype(np.float64)
        assert np.all(np.abs(taps[p, : span[p]].astype(np.float64) - ref) <= ulp), p
        assert not np.any(taps[p, span[p]:])
        assert not np.any(k32[p, : first[p]]) and not np.any(k32[p, first[p] + span[p]:])


@pytest.mark.parametrize("sr", TA_RATES)
def test_output_length_is_torchaudios(sr):
    AF = pytest.importorskip("torchaudio.functional")
    from sopro_b200.resample import resampled_length

    g = math.gcd(24000, sr)
    o = 24000 // g
    for N in sorted({1, max(1, o - 1), o, o + 1, 1920, 7 * 1920, 41 * 1920}):
        want = AF.resample(torch.zeros(1, N, dtype=torch.float64), 24000, sr).shape[-1]
        assert resampled_length(24000, sr, N) == want, N
    assert resampled_length(24000, sr, 0) == 0


@pytest.mark.parametrize("sr", [0, -1, 3999, 192001, 44099, 24000.5, "48000", True])
def test_refused_rates_raise_value_error(sr):
    from sopro_b200.resample import check_rates, filter_taps, resampled_length

    for f in (lambda: check_rates(24000, sr), lambda: filter_taps(24000, sr), lambda: resampled_length(24000, sr, 100)):
        with pytest.raises(ValueError):
            f()


def test_identical_rates_and_bad_lengths_are_refused():
    from sopro_b200 import _lib
    from sopro_b200.resample import check_rates

    with pytest.raises(ValueError):
        check_rates(24000, 24000)
    assert check_rates(24000, 48000.0) == (24000, 48000)
    assert _lib.load().sopro_resampled_length(24000, 48000, -1) < 0


def test_sample_rate_keyword_defaults_to_none():
    from sopro_b200 import SoproTTS
    from sopro_b200.streaming import stream

    for f in (SoproTTS.synthesize, SoproTTS.synthesize_batch, SoproTTS.stream, stream):
        p = inspect.signature(f).parameters["sample_rate"]
        assert p.default is None and p.kind == inspect.Parameter.KEYWORD_ONLY, f
    assert inspect.signature(SoproTTS.save_wav).parameters["sample_rate"].default == 24000


def test_refused_rate_raises_before_any_work():
    """SoproTTS._resampler is the first thing every synthesis entry point calls: it refuses a rate on the host without a
    model, a device or a random draw (the object below has no model at all)."""
    from sopro_b200.model import SoproTTS

    tts = SoproTTS.__new__(SoproTTS)
    tts._resamplers = {}
    before = torch.get_rng_state()
    assert tts._resampler(None) is None and tts._resampler(24000) is None
    for sr in (44099, 3999, 24000.5):
        with pytest.raises(ValueError):
            tts._resampler(sr)
    assert tts._resamplers == {} and torch.equal(before, torch.get_rng_state())
