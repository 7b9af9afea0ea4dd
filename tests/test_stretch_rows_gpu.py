"""GPU: the time-stretch with a speed per row (sopro_stretch_rows) -- every row equals stretch of that row alone bit
for bit (offsets included), a row at speed 1 is its input, ragged lengths down to 0 and 1 and under one window, speeds
0.25 and 4, and a row alone against the same row inside a 64-row batch."""
import numpy as np
import pytest
import torch

from sopro_b200.stretch import stretch, stretch_rows, stretched_length

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)


def _bits(t):
    return t.reshape(-1).cpu().numpy().view(np.uint32)


def _signal(B, L, seed):
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(L, dtype=torch.float64) / 24000
    f = 120 + 300 * torch.rand(B, 1, generator=g, dtype=torch.float64)
    x = torch.sin(2 * torch.pi * f * t) * (0.3 + 0.2 * torch.sin(2 * torch.pi * 3 * t)) + 0.05 * torch.randn(B, L, generator=g, dtype=torch.float64)
    return x.to(torch.float32).cuda()


def _check(x, speeds, lens):
    y, offs = stretch_rows(x, speeds, lens=lens, return_offsets=True)
    assert y.shape == (x.shape[0], max(stretched_length(s, n) for s, n in zip(speeds, lens)))
    for b, (s, n) in enumerate(zip(speeds, lens)):
        M = stretched_length(s, n)
        assert not y[b, M:].any(), b  # zeros past the row's outputs
        if round(s * 65536) == 65536:
            assert M == n and torch.equal(y[b, :n], x[b, :n]), b  # copied through, not stretched
            assert not offs[b].any()
            continue
        want, w_offs = stretch(x[b, :n], s, return_offsets=True)
        assert np.array_equal(_bits(y[b, :M]), _bits(want)), (b, s, n)
        k = w_offs.shape[-1]
        assert torch.equal(offs[b, :k], w_offs.reshape(-1)) and not offs[b, k:].any(), b


def test_every_row_equals_its_own_stretch():
    lens = [0, 1, 2, 239, 240, 479, 480, 481, 1000, 4801, 24000, 37123, 0, 12345, 9999, 7]
    speeds = [1.0, 0.25, 4.0, 0.5, 1.0, 2.0, 0.25, 4.0, 1.0, 1.37, 0.8, 0.25, 3.0, 1.0, 4.0, 1.25]
    x = _signal(len(lens), max(lens), 1)
    _check(x, speeds, lens)


def test_speeds_that_quantise_to_one_are_copied():
    x = _signal(3, 5000, 2)
    y = stretch_rows(x, [1.0, 1.0 + 2 ** -18, 0.75], lens=[5000, 4000, 3000])
    assert torch.equal(y[0, :5000], x[0]) and torch.equal(y[1, :4000], x[1, :4000]) and not y[1, 4000:].any()


def test_one_row_alone_equals_the_row_in_a_64_row_batch():
    g = np.random.default_rng(7)
    lens = [int(v) for v in g.integers(0, 48000, 64)]
    lens[5], lens[17], lens[40] = 0, 1, 300
    choices = np.array([0.25, 0.5, 0.75, 1.0, 1.25, 1.5, 2.0, 4.0, 0.9, 1.1])
    speeds = [float(v) for v in g.choice(choices, 64)]
    speeds[3], speeds[9] = 0.25, 4.0
    x = _signal(64, max(lens), 3)
    y = stretch_rows(x, speeds, lens=lens)
    for b in range(64):
        alone = stretch_rows(x[b: b + 1, : lens[b]], [speeds[b]])
        M = stretched_length(speeds[b], lens[b])
        assert alone.shape == (1, M) and np.array_equal(_bits(y[b, :M]), _bits(alone)), b
    _check(x, speeds, lens)


def test_shapes_and_refusals():
    x = _signal(2, 100, 4)
    assert stretch_rows(x, [1.0, 0.5]).shape == (2, 200)
    assert stretch_rows(x.reshape(2, 1, 100), [2.0, 2.0]).shape == (2, 1, 50)
    assert stretch_rows(x, [0.5, 0.5], lens=[0, 0]).shape == (2, 0)
    for bad in ([1.0], [1.0, 1.0, 1.0], [1.0, 5.0], [0.1, 1.0], [1.0, float("nan")]):
        with pytest.raises(ValueError):
            stretch_rows(x, bad)
    with pytest.raises(ValueError):
        stretch_rows(x, [1.0, 1.0], lens=[101, 3])
