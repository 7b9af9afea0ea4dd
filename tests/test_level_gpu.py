"""GPU: the live leveller (csrc/level.cu through sopro_b200/loudness.py) -- push schedules against the one-shot
level_live bit for bit, the float64 oracle (oracle/loudness_live_oracle.py) per rate, the meter against
measure_loudness, the ceiling, ragged batches, the stream contract, and level_stream / level_stream_batch around every
streaming entry point of the synthetic checkpoint."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import loudness_live_oracle as LO
from oracle import loudness_oracle as O

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
RATES = (8000, 16000, 22050, 24000, 44100, 48000, 96000)
CEIL32 = float(np.float32(O.CEILING))


def _signal(n, sr, seed=0, amp=0.05):
    """noise with a quieter stretch, a silent one and a hot burst: both gates, the ramp and the ceiling all act"""
    g = np.random.default_rng(seed)
    x = (amp * g.standard_normal(n)).astype(np.float32)
    x[n // 5: 2 * n // 5] *= 0.1
    x[2 * n // 5: n // 2] = 0
    b = 3 * n // 4
    k = min(sr // 20, n - b)
    x[b: b + k] = (0.9 * np.sign(g.standard_normal(k))).astype(np.float32)
    return torch.from_numpy(x).cuda()


def _push_all(x, sr, T, sizes):
    from sopro_b200.loudness import LiveLeveller

    lev = LiveLeveller(sr, T, device=x.device)
    out, a = [], 0
    for n in sizes:
        out.append(lev.push(x[a: a + n]))
        a += n
    assert a == x.numel()
    out.append(lev.finish())
    assert all(o.dim() == 2 and o.shape[0] == 1 for o in out)
    return torch.cat(out, dim=1).reshape(-1)


def _sizes(n, step):
    return [min(step, n - a) for a in range(0, n, step)]


def _ragged(n, seed):
    g = np.random.default_rng(seed)
    out, a = [], 0
    while a < n:
        k = int(min(n - a, g.choice([0, 1, 7, 300, 2401, 5000, 17000])))
        out.append(k)
        a += k
    return out


@pytest.mark.parametrize("sr,n", ((8000, 7 * 800 + 123), (24000, 3 * 24000 + 1111)))
def test_every_push_schedule_equals_level_live(sr, n):
    from sopro_b200.loudness import level_live

    s = O.sub_block(sr)
    x = _signal(n, sr, seed=sr)
    want = level_live(x, sr, -18.0)
    schedules = [_sizes(n, s - 1), _sizes(n, s), _sizes(n, s + 1), _sizes(n, 11520), _ragged(n, 1), _ragged(n, 2), [n]]
    if n < 10000:
        schedules.append([1] * n)
    for sizes in schedules:
        got = _push_all(x, sr, -18.0, sizes)
        assert got.shape == want.shape and torch.equal(got, want), sizes[:4]


@pytest.mark.parametrize("sr", RATES)
def test_matches_the_float64_oracle(sr):
    from sopro_b200.loudness import level_live, measure_loudness

    x = _signal(3 * sr + 77, sr, seed=3)
    T = -20.0
    y, a, M = level_live(x, sr, T, return_gains=True)
    xn = x.cpu().numpy()
    wy, wa, wM = LO.level_live(xn, sr, T)
    M, a = M.cpu().numpy(), a.cpu().numpy()
    assert np.isnan(M[:3]).all() and np.isnan(a[:3]).all()
    # fp64 filter, sums and pow in another order: stated tolerances 1e-9 LU and 1e-10 relative on the gain
    fin = np.isfinite(wM[3:])
    assert np.array_equal(np.isfinite(M[3:]), fin)
    assert np.abs(M[3:][fin] - wM[3:][fin]).max() < 1e-9
    assert np.abs(a[3:] / wa[3:] - 1).max() < 1e-10
    # the release rules, given the kernel's own gains, are exact
    ry, _, _ = LO.level_live(xn, sr, T, a=a)
    assert np.array_equal(y.cpu().numpy(), ry)
    # with the oracle's gains every sample is within a few fp32 ulps
    assert np.abs(y.cpu().numpy() - wy).max() <= 4 * np.spacing(np.float32(CEIL32))
    # the last M is the one-shot meter of the row
    L = float(measure_loudness(x, sr))
    assert abs(M[-1] - L) < 1e-6
    assert float(y.abs().max()) <= CEIL32


def test_ceiling_on_hot_rows():
    from sopro_b200.loudness import level_live

    for sr in (16000, 48000):
        g = torch.Generator().manual_seed(sr)
        x = (torch.rand(5 * sr + 13, generator=g) * 2 - 1).cuda()
        for T in (0.0, -3.0):
            y = level_live(x, sr, T)
            assert float(y.abs().max()) <= CEIL32


def test_a_ragged_batch_row_equals_the_row_alone():
    from sopro_b200.loudness import level_live

    sr = 24000
    lens = [0, 100, 4 * 2400 - 1, 4 * 2400, 7 * 2400 + 5, 2 * sr + 3333, 50000]
    L = max(lens)
    x = torch.stack([_signal(L, sr, seed=i, amp=0.02 * (i + 1)) for i in range(len(lens))])
    x_nan = x.clone()
    for b, n in enumerate(lens):
        x_nan[b, n:] = float("nan")  # never read
    y = level_live(x_nan, sr, -16.0, lens=lens)
    for b, n in enumerate(lens):
        alone = level_live(x[b, :n], sr, -16.0)
        assert torch.equal(y[b, :n], alone) and (y[b, n:] == 0).all()


def _raw_state(max_chunk, sr):
    from sopro_b200 import _lib

    lib = _lib.load()
    h = C.c_void_p()
    _lib.check_arg(lib.sopro_level_stream_create(max_chunk, sr, 0, C.byref(h)))
    return lib, h


def test_stream_contract():
    from sopro_b200 import _lib
    from sopro_b200.loudness import level_live

    sr, mc = 8000, 1000
    s = O.sub_block(sr)
    x = _signal(9 * s + 33, sr, seed=9)
    lib, h = _raw_state(mc, sr)
    sp = _lib.stream_ptr(x.device)
    try:
        assert lib.sopro_level_stream_ready(h, 10, 0) < 0  # before the first reset
        with pytest.raises(_lib.SoproError):
            _lib.check_arg(lib.sopro_level_push(h, x.data_ptr(), 10, None, sp))
        with pytest.raises(ValueError):
            _lib.check_arg(lib.sopro_level_stream_reset(h, 1.0))
        _lib.check_arg(lib.sopro_level_stream_reset(h, -40.0))

        def run(T, row):
            out, a = [], 0
            while a < row.numel():
                n = min(mc, row.numel() - a)
                k = lib.sopro_level_stream_ready(h, n, 0)
                y = torch.full((max(k, 1),), float("nan"), device=x.device)
                if a == mc:  # an oversized push: refused, nothing launched, the state unchanged
                    y_big = torch.full((8 * s,), float("nan"), device=x.device)
                    with pytest.raises(ValueError):
                        _lib.check_arg(lib.sopro_level_push(h, row.data_ptr(), mc + 1, y_big.data_ptr(), sp))
                    assert torch.isnan(y_big).all()
                _lib.check_arg(lib.sopro_level_push(h, row[a:].data_ptr(), n, y.data_ptr(), sp))
                out.append(y[:k])
                a += n
            k = lib.sopro_level_stream_ready(h, 0, 1)
            y = torch.empty(max(k, 1), device=x.device)
            _lib.check_arg(lib.sopro_level_finish(h, y.data_ptr(), sp))
            out.append(y[:k])
            return torch.cat(out)

        # reset mid-row: half a row at one target, then a whole row at another
        _lib.check_arg(lib.sopro_level_push(h, x.data_ptr(), 700, torch.empty(1, device=x.device).data_ptr(), sp))
        _lib.check_arg(lib.sopro_level_stream_reset(h, -20.0))
        x2 = x.clone()
        x2[::7] *= 0.5
        assert torch.equal(run(-20.0, x2), level_live(x2, sr, -20.0))
        # after finish: SOPRO_ERR_STATE for a push and a finish, ready < 0, until a reset
        assert lib.sopro_level_stream_ready(h, 0, 1) < 0
        with pytest.raises(_lib.SoproError):
            _lib.check_arg(lib.sopro_level_push(h, x.data_ptr(), 10, None, sp))
        with pytest.raises(_lib.SoproError):
            _lib.check_arg(lib.sopro_level_finish(h, None, sp))
        _lib.check_arg(lib.sopro_level_stream_reset(h, -30.0))
        assert torch.equal(run(-30.0, x), level_live(x, sr, -30.0))
    finally:
        lib.sopro_level_stream_destroy(h)


def test_leveller_refusals_on_the_device():
    from sopro_b200 import _lib
    from sopro_b200.loudness import LiveLeveller

    lev = LiveLeveller(24000, -16.0)
    with pytest.raises(_lib.SoproError):
        lev.push(torch.zeros(100))  # a CPU chunk
    if torch.cuda.device_count() > 1:
        with pytest.raises(ValueError):
            lev.push(torch.zeros(100, device="cuda:1"))
    lev.finish()
    with pytest.raises(_lib.SoproError):
        lev.push(torch.zeros(100, device=lev.device))
    lev.reset(-20.0)
    assert lev.push(torch.zeros(100, device=lev.device)).shape == (1, 0)


def test_store_growth_keeps_the_stream_exact():
    """A stream longer than the store's first capacity (6000 sub-blocks, ten minutes) grows it mid-stream."""
    from sopro_b200.loudness import level_live

    sr = 4000
    s = O.sub_block(sr)
    n = 6100 * s + 17
    x = _signal(n, sr, seed=12, amp=0.01)
    got = _push_all(x, sr, -16.0, _sizes(n, 50 * s + 3))
    assert torch.equal(got, level_live(x, sr, -16.0))


# ---- end to end on the synthetic checkpoint -------------------------------------------------------------------------

TEXT = "3 7 11 15 5 9 13 17 21 4 8"
KW = dict(max_frames=40, min_gen_frames=3)


def _api():
    from tests.test_stream_batch_gpu import _tts

    return _tts()


def _tee(items, seen):
    for it in items:
        seen.append(it)
        yield it


def _same(a, b):
    return len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("chain", (dict(), dict(speed=1.25), dict(sample_rate=16000), dict(watermark=0xC0FFEE)))
def test_level_stream_of_stream(chain):
    from sopro_b200.loudness import level_live, level_stream

    tts, refs = _api()
    sr = chain.get("sample_rate", 24000)
    plain = [c.clone() for c in tts.stream(TEXT, ref=refs[0], seed=5, **KW, **chain)]
    seen = []
    got = list(level_stream(_tee(tts.stream(TEXT, ref=refs[0], seed=5, **KW, **chain), seen), sr, target=-18.0))
    assert _same(seen, plain)
    assert all(g.dim() == 2 and g.shape[0] == 1 and g.shape[1] > 0 for g in got)
    want = level_live(torch.cat(plain, dim=1), sr, -18.0)
    assert torch.equal(torch.cat(got, dim=1), want)


def test_level_stream_keeps_the_words():
    from sopro_b200.loudness import level_live, level_stream

    tts, refs = _api()
    plain = list(tts.stream(TEXT, ref=refs[1], seed=6, word_timestamps=True, **KW))
    got = list(level_stream(tts.stream(TEXT, ref=refs[1], seed=6, word_timestamps=True, **KW), target=-16.0))
    assert [w for _c, ws in got for w in ws] == [w for _c, ws in plain for w in ws]
    want = level_live(torch.cat([c for c, _ws in plain], dim=1), 24000, -16.0)
    assert torch.equal(torch.cat([c for c, _ws in got], dim=1), want)


@pytest.mark.parametrize("words", (False, True))
def test_level_stream_batch_per_row(words):
    from sopro_b200.loudness import level_live, level_stream_batch

    tts, refs = _api()
    texts = [TEXT, "2 4 6", "1 3 5 7 9 11 13 15 17 19 21 23"]
    kw = dict(ref=refs[2], seeds=[11, 12, 13], word_timestamps=words, **KW)
    plain = [tuple(v.clone() if isinstance(v, torch.Tensor) else v for v in it) for it in tts.stream_batch(texts, **kw)]
    seen = []
    got = list(level_stream_batch(_tee(tts.stream_batch(texts, **kw), seen), target=-20.0))
    assert len(seen) == len(plain) and all(_same([a[1]], [b[1]]) and a[0] == b[0] and a[2] == b[2] for a, b in zip(seen, plain))
    for i in range(len(texts)):
        rows = [it for it in got if it[0] == i]
        assert rows and rows[-1][2] and not any(it[2] for it in rows[:-1])
        assert all(len(it) == (4 if words else 3) for it in rows)
        want = level_live(torch.cat([it[1] for it in plain if it[0] == i], dim=1), 24000, -20.0)
        assert torch.equal(torch.cat([it[1] for it in rows], dim=1), want)
        if words:
            assert [w for it in rows for w in it[3]] == [w for it in plain if it[0] == i for w in it[3]]


def test_level_stream_of_stream_long_and_stream_dialogue():
    from sopro_b200.loudness import level_live, level_stream

    tts, refs = _api()
    text = "3 7 11 15. 5 9 13 17 21! 4 8?\n\n6 2 10 12 14 16 18 20 22 24, 26 28 30. 1"
    script = [(refs[0], "3 7 11 15. 5 9 13 17 21!"), (refs[1], "4 8? 6 2 10 12 14."), (refs[2], "16 18 20.")]
    for make, sr in ((lambda: tts.stream_long(text, ref=refs[0], seed=40, max_tokens=7, **KW), 24000),
                     (lambda: tts.stream_dialogue(script, seed=41, max_tokens=7, sample_rate=48000, **KW), 48000)):
        plain = [c.clone() for c in make()]
        seen = []
        got = list(level_stream(_tee(make(), seen), sr, target=-16.0))
        assert _same(seen, plain)
        want = level_live(torch.cat(plain, dim=1), sr, -16.0)
        assert torch.equal(torch.cat(got, dim=1), want)
