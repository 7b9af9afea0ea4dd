"""CPU: the time-stretch's host side (sopro_b200/stretch.py, csrc/stretch.cu) -- window taps, speed quantisation, output
lengths and frame positions, refused speeds, the `speed` keyword of the public API -- and known answers of the float64
oracle (oracle/stretch_oracle.py) the GPU tests judge the kernels by."""
import inspect
import math

import numpy as np
import pytest
import torch

from oracle import stretch_oracle as O

SPEEDS = (0.25, 0.5, 0.8, 1.0737, 1.25, 2.0, 3.7, 4.0)
REFUSED = (float("nan"), float("inf"), -float("inf"), 0, 0.0, -1.25, 0.2499, 4.0001, 100, True, False, "1.25", [1.0],
           np.bool_(True))


def test_window_is_periodic_hann_rounded_once():
    from sopro_b200.stretch import stretch_window

    w = stretch_window()
    n = np.arange(480, dtype=np.float64)
    want = (np.sin(np.pi * n / 480) ** 2).astype(np.float32)
    assert w.dtype == np.float32 and w.shape == (480,)
    assert np.array_equal(w.view(np.uint32), want.view(np.uint32))
    assert np.array_equal(w, O.window().astype(np.float32))
    # 50 % overlap: the windows sum to 1, off by at most half an fp32 ulp at 1 (2^-25 = 3.0e-8: the two roundings,
    # of a value in [0.5, 1) and one in [0, 0.5], partly cancel)
    s = w[:240].astype(np.float64) + w[240:].astype(np.float64)
    assert np.abs(s - 1.0).max() <= 2.0 ** -25


def test_speed_quantisation():
    from sopro_b200.stretch import check_speed, quantise

    for s in SPEEDS + (1.0, 0.25 + 0.5 / 65536, 0.25 + 1.5 / 65536, 1 + 0.4 / 65536, 1 - 0.5 / 65536, np.float32(1.5),
                       np.float64(2.5), 3):
        assert quantise(s) == round(float(s) * 65536) == O.quantise(s), s
    assert quantise(0.25 + 0.5 / 65536) == 16384 and quantise(0.25 + 1.5 / 65536) == 16386  # halves to even
    assert check_speed(None) is None and check_speed(1.0) is None and check_speed(1) is None
    assert check_speed(1 + 0.4 / 65536) is None  # S = 65536: a bypass
    assert check_speed(1.25) == 81920 and check_speed(0.25) == 16384 and check_speed(4) == 262144


@pytest.mark.parametrize("speed", REFUSED)
def test_refused_speeds_raise_value_error(speed):
    from sopro_b200.stretch import check_speed, quantise, stretched_length

    for f in (lambda: check_speed(speed), lambda: quantise(speed), lambda: stretched_length(speed, 100)):
        with pytest.raises(ValueError):
            f()


def test_refused_at_the_c_abi():
    import ctypes as C

    from sopro_b200 import _lib

    lib = _lib.load()
    S = C.c_int32(7)
    for v in (float("nan"), float("inf"), 0.0, -1.0, 0.24, 4.01):
        assert lib.sopro_stretch_speed(v, C.byref(S)) == -1 and S.value == 7
    for bad_S in (0, 16383, 262145, -65536):
        assert lib.sopro_stretched_length(bad_S, 100) < 0 and lib.sopro_stretch_positions(bad_S, 100, None) < 0
    assert lib.sopro_stretched_length(65536, -1) < 0


@pytest.mark.parametrize("speed", SPEEDS + (1.0,))
def test_lengths_and_positions_follow_the_formulas(speed):
    from sopro_b200.stretch import frame_positions, n_frames, stretched_length

    S = round(speed * 65536)
    for L in (0, 1, 2, 239, 240, 241, 479, 480, 1919, 1920, 7 * 1920 + 13, 41 * 1920, 400 * 1920, 4095 * 1920):
        M = -(-L * 65536 // S)
        assert stretched_length(speed, L) == M == O.out_len(S, L), L
        K = 0 if M == 0 else -(-M // 240) + 1
        assert n_frames(M) == K == O.n_frames(M)
        a = frame_positions(speed, L)
        k = np.arange(K, dtype=np.int64)
        assert a.shape == (K,) and np.array_equal(a, (k * 240 * S + 32768) // 65536), L
        if K:
            assert int(a[-1]) == O.pos_a(K - 1, S)


def test_largest_api_size():
    """max_frames 4095 x 1920 samples at speed 0.25: 31.4 M outputs, 131,041 frames, positions exact in int64."""
    from sopro_b200.stretch import frame_positions, stretched_length

    L = 4095 * 1920
    assert stretched_length(0.25, L) == 4 * L
    a = frame_positions(0.25, L)
    assert a.size == 4 * L // 240 + 1 == 131041
    assert np.array_equal(a, np.arange(a.size, dtype=np.int64) * 60)
    a = frame_positions(3.7, L)
    S = round(3.7 * 65536)
    assert a.size == -(-(-(-L * 65536 // S)) // 240) + 1
    big = [(int(k) * 240 * S + 32768) // 65536 for k in (a.size - 2, a.size - 1)]
    assert a[-2:].tolist() == big


def test_speed_keyword_defaults_to_none():
    from sopro_b200 import SoproTTS
    from sopro_b200.streaming import stream

    for f in (SoproTTS.synthesize, SoproTTS.synthesize_batch, SoproTTS.stream, stream):
        p = inspect.signature(f).parameters["speed"]
        assert p.default is None and p.kind == inspect.Parameter.KEYWORD_ONLY, f


def test_refused_speed_raises_before_any_work():
    """The speed is checked next to the output rate, before the text, the reference, the prefill or a random draw:
    these objects have no model at all."""
    from sopro_b200.model import SoproTTS
    from sopro_b200.streaming import stream

    tts = SoproTTS.__new__(SoproTTS)
    tts._resamplers = {}
    before = torch.get_rng_state()
    for speed in (0, float("nan"), 5.0, True, "2"):
        with pytest.raises(ValueError):
            tts.synthesize("1 2", speed=speed)
        with pytest.raises(ValueError):
            tts.synthesize_batch(["1 2"], ref=None, speed=speed)
        with pytest.raises(ValueError):
            stream(tts, "1 2", speed=speed)
    assert torch.equal(before, torch.get_rng_state())


# ---- the float64 oracle's known answers

def _sine(f, L, amp=0.5):
    return amp * np.sin(2 * np.pi * f * np.arange(L) / 24000.0)


def _block_rms_error(y, x_rms, L, S):
    """max |RMS - x_rms| / x_rms over the 960-sample output blocks clear of the input's edges: from the second block
    (at speed 0.25 every in-phase candidate of frame 1 overlaps the zeros before sample 0, and block 0 is 1.9 % off)
    to the last block whose frames read no sample past the input's end."""
    clean = int((L - 400) * 65536 / S) - 2 * 240
    nb = clean // 960
    assert nb >= 3
    r = np.sqrt((y[: nb * 960].reshape(nb, 960)[1:] ** 2).mean(axis=1))
    return float(np.abs(r - x_rms).max() / x_rms)


def test_oracle_identity_replay_at_speed_one():
    x = np.random.default_rng(3).standard_normal(24013) * 0.3
    r = O.stretch(x, 65536, offsets=np.zeros(O.n_frames(x.size), dtype=np.int64))
    assert r.y.size == x.size and np.abs(r.y - x).max() <= 1e-7


@pytest.mark.parametrize("speed", SPEEDS)
def test_oracle_sines_keep_their_block_rms(speed):
    S = O.quantise(speed)
    L = 24000
    for f in (200.0, 150.0):  # periods of 120 and 160 samples: both divide the 960-sample block
        x = _sine(f, L)
        r = O.stretch(x, S)
        assert r.y.size == O.out_len(S, L) == math.ceil(L * 65536 / S)
        assert r.deltas.size == O.n_frames(r.y.size) and r.deltas[0] == 0 and np.abs(r.deltas).max() <= 160
        assert _block_rms_error(r.y, 0.5 / math.sqrt(2), L, S) <= 1e-3, (f, speed)


@pytest.mark.parametrize("speed", (0.8, 1.25))
def test_oracle_without_the_search_fails_the_rms_check(speed):
    S = O.quantise(speed)
    x = _sine(200.0, 24000)
    r = O.stretch(x, S, offsets=np.zeros(O.n_frames(O.out_len(S, x.size)), dtype=np.int64))
    assert _block_rms_error(r.y, 0.5 / math.sqrt(2), x.size, S) > 0.1


def test_oracle_tie_rule():
    c = np.zeros(321)
    c[160 + 7] = c[160 - 7] = c[160 + 30] = 2.0
    assert O.best_delta(c) == -7
    c[160 + 3] = 2.0
    assert O.best_delta(c) == 3
    c[160] = 2.0
    assert O.best_delta(c) == 0
