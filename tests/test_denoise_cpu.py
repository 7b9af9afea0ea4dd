"""Reference-voice denoising without a GPU: the float64 oracle's round trip, its pass-through cases and its noise
reduction on seeded signals, the argument refusals of the denoise= switch (before any file read or device work), and
the host-side checks of the C-ABI."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import denoise_oracle as O

N = 6 * O.SR


def _clean():
    return O.voiced()


def test_unit_gain_round_trip():
    for n in (512, 513, 24000, 24000 * 3 + 77):
        x = O.white(n, n)
        assert np.abs(O.round_trip(x) - x).max() <= 1e-12, n


def test_short_rows_come_back_unchanged():
    for n in (1, 2, 100, 511):
        x = O.white(n, 7)
        d = O.denoise_detail(x)
        assert d["sel"] is None and np.array_equal(d["y"], x)


def test_non_finite_rows_come_back_unchanged():
    for bad in (np.nan, np.inf, -np.inf):
        x = O.white(5000, 8)
        x[2345] = bad
        d = O.denoise_detail(x)
        assert d["sel"] is None and np.array_equal(d["y"], x, equal_nan=True)


def test_digital_silence_gaps_pass_through():
    """The quietest frames are exact zeros, so lambda = 0 in every bin and G = 1: the round trip."""
    s = _clean()
    d = O.denoise_detail(s)
    assert d["sel"] is not None and not d["lam"].any() and (d["G"] == 1.0).all()
    assert np.abs(d["y"] - s).max() <= 1e-12


def test_geometry():
    assert O.n_frames(512) == 3 and O.candidates(512) == 1 and O.n_noise(512) == 1
    assert O.n_frames(513) == 4 and O.candidates(24000) == 92 and O.n_noise(24000) == 9
    x = O.white(24000, 9)
    d = O.denoise_detail(x)
    E = d["E"]
    assert E.size == O.n_frames(24000) and d["sel"].size == 9
    worst = max(E[m] for m in d["sel"])
    assert all(E[m] >= worst for m in range(1, 93) if m not in d["sel"])


def test_noise_frame_ties_go_to_the_lower_frame():
    x = np.zeros(256 * 40)
    x[256 * 20:] = O.white(256 * 20, 10)  # frames 1 .. 19 are exact zeros: the tie
    d = O.denoise_detail(x)
    assert d["sel"].tolist() == [1, 2, 3]


@pytest.mark.parametrize("snr,want", [(0, 7.0), (10, 15.0)])
def test_white_noise_is_reduced(snr, want):
    s = _clean()
    y = O.denoise(s + O.at_snr(s, O.white(N, 1), snr))
    assert O.snr_db(s, y) >= want


def test_pink_noise_is_reduced():
    s = _clean()
    assert O.snr_db(s, O.denoise(s + O.at_snr(s, O.pink(N, 2), 10))) >= 11.0


def test_pure_noise_is_attenuated():
    w = 0.1 * O.white(N, 3)
    y = O.denoise(w)
    assert 10 * np.log10(np.sum(y * y) / np.sum(w * w)) <= -18.0


def test_a_clean_signal_over_a_low_floor_is_not_harmed():
    s = _clean()
    assert O.snr_db(s, O.denoise(s + O.at_snr(s, O.white(N, 4), 60))) >= 55.0


def test_a_clip_without_pauses_loses_stationary_content():
    """The stated limit: a harmonic signal that never drops below 30 % gains little, and may lose, at 10 dB."""
    u = O.voiced(gated=False)
    assert O.snr_db(u, O.denoise(u + O.at_snr(u, O.white(N, 5), 10))) < 10.0


# ---- the switch

def _stub():
    from sopro_b200.model import SoproTTS

    return SoproTTS.__new__(SoproTTS)  # no codec, no model, no device: a refusal must come first


@pytest.mark.parametrize("flag", [1, 0, None, "yes", np.bool_(True), 1.0])
def test_denoise_must_be_a_bool(flag):
    # a missing file listed first would raise FileNotFoundError if it were read before the flag is checked
    with pytest.raises(TypeError):
        _stub().prepare_references(["/nonexistent/voice.wav"], denoise=flag)
    with pytest.raises(TypeError):
        _stub().prepare_references([torch.zeros(100)], sample_rates=[44099], denoise=flag)  # before the rate check


def test_prepare_reference_keeps_the_reference_signature():
    """A denoised voice from one file is prepare_references([path], denoise=True)[0]; prepare_reference has no switch."""
    import inspect

    from sopro_b200.model import SoproTTS

    assert "denoise" not in inspect.signature(SoproTTS.prepare_reference).parameters
    assert inspect.signature(SoproTTS.prepare_references).parameters["denoise"].default is False


# ---- the C-ABI on the host

def test_symbols_resolve():
    from sopro_b200 import _lib

    lib = _lib.load()
    assert lib.sopro_denoise_sizes and lib.sopro_denoise


def test_workspace_sizes_and_refusals():
    from sopro_b200 import _lib
    from sopro_b200.denoising import workspace_bytes

    lib = _lib.load()
    n = C.c_int64()
    assert lib.sopro_denoise_sizes(1, 240000, C.byref(n)) == 0 and n.value > 0
    small = n.value
    assert lib.sopro_denoise_sizes(8, 240000, C.byref(n)) == 0 and n.value >= 8 * (small - 1024)
    assert workspace_bytes(2, 0) >= 1
    assert lib.sopro_denoise_sizes(0, 100, C.byref(n)) == -1
    assert lib.sopro_denoise_sizes(1, -1, C.byref(n)) == -1
    assert lib.sopro_denoise_sizes(1, (1 << 36) + 1, C.byref(n)) == -1
    assert lib.sopro_denoise_sizes(1, 100, None) == -1
    with pytest.raises(ValueError):
        workspace_bytes(0, 100)


def test_denoise_refuses_before_any_launch():
    """Every refusal returns before the first CUDA call, so it holds on a machine without a device."""
    from sopro_b200 import _lib

    f = _lib.load().sopro_denoise
    p = 4096  # never dereferenced: each call is refused on its arguments
    lens = (C.c_int64 * 2)(1000, 2000)
    assert f(p, 0, 2000, lens, p, p, 2000, None) == -1          # B < 1
    assert f(p, 2, 1999, lens, p, p, 1999, None) == -1          # a row longer than the stride
    assert f(p, 2, 2000, (C.c_int64 * 2)(-1, 5), p, p, 2000, None) == -1
    assert f(None, 2, 2000, lens, p, p, 2000, None) == -1       # null x
    assert f(p, 2, 2000, lens, None, p, 2000, None) == -1       # null workspace
    assert f(p, 2, 2000, lens, p, None, 2000, None) == -1       # null y
    assert f(p, 2, 2000, lens, p, p, 1999, None) == -1          # y rows overlap
    assert f(p, 1, (1 << 36) + 1, None, p, p, 0, None) == -1    # longer than the bound
    with pytest.raises(_lib.SoproError):
        from sopro_b200.denoising import denoise

        denoise(torch.zeros(1000))  # a CPU tensor: there is no CPU path
