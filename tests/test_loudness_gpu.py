"""GPU: the loudness meter and gain (csrc/loudness.cu through sopro_b200/loudness.py) against the float64 oracle
(oracle/loudness_oracle.py) -- L per rate, signal and length, ragged batches, determinism, the gain and its ceiling, graph
capture -- and `loudness=` through the public API."""
import math

import numpy as np
import pytest
import torch

from oracle import loudness_oracle as O
from oracle import mimi_oracle as MO

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
RATES = (8000, 16000, 22050, 24000, 44100, 48000, 96000)
KINDS = ("noise", "sweep", "sine200", "sine997", "mimi", "gated")
HOP = 1920
_CACHE = {}


def _mimi_wav():
    """A real Mimi decode (synthetic checkpoint, seeded codes): 41 frames = 78,720 samples, scaled to a 0.5 peak."""
    if "mimi" not in _CACHE:
        from sopro_b200.codec import MimiEngine

        codes = torch.randint(0, 2048, (1, 32, 41), generator=torch.Generator().manual_seed(7))
        eng = MimiEngine(MO.synth_mimi_state_dict(), 0, 32)
        w = eng.decode(codes).reshape(-1).double()
        _CACHE["mimi"] = (0.5 * w / w.abs().max()).float().cuda()
    return _CACHE["mimi"]


def _signal(kind, N, sr, seed=0):
    """fp32 [N] on the device.  "gated": loud noise, then the same 20 dB quieter, then silence, in thirds -- the quiet
    third fails the relative gate and the silent one (apart from the filter's ringing) the absolute gate."""
    g = torch.Generator().manual_seed(1000 * seed + N % 997)
    t = torch.arange(N, dtype=torch.float64) / sr
    if kind == "noise":
        return (0.3 * torch.randn(N, generator=g)).float().cuda()
    if kind == "sweep":  # log sweep 20 Hz -> 0.45 sr
        T = max(N, 2) / sr
        k = math.log(0.45 * sr / 20.0)
        return (0.6 * torch.sin(2 * math.pi * 20.0 * T / k * (torch.exp(t / T * k) - 1))).float().cuda()
    if kind.startswith("sine"):
        return (0.5 * torch.sin(2 * math.pi * float(kind[4:]) * t)).float().cuda()
    if kind == "gated":
        x = 0.3 * torch.randn(N, generator=g)
        x[N // 3: 2 * N // 3] *= 0.1
        x[2 * N // 3:] = 0
        return x.float().cuda()
    w = _mimi_wav()
    return w[:N].clone() if N <= w.numel() else w.repeat(N // w.numel() + 1)[:N].contiguous()


def _lengths(sr):
    s = O.sub_block(sr)
    return [4 * s - 1, 4 * s, 4 * s + 1, 7 * s + 4321, 2 * (3 * 8192) + 77, 2 * (sr * 5 // 2) + 1]


def _oracle_L(x, sr):
    return O.integrated(x.double().cpu().numpy(), sr)


def _close(got, want, tol):
    if math.isinf(want) or math.isinf(got):
        return got == want
    return abs(got - want) <= tol


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("sr", RATES)
def test_measure_matches_the_float64_oracle(sr, kind):
    """L within 1e-6 LU of the oracle, every row of a ragged batch (NaN padding), lengths 4s - 1, 4s, 4s + 1 and odd."""
    from sopro_b200.loudness import measure_loudness

    lens = _lengths(sr)
    x = torch.full((len(lens), max(lens)), float("nan"), device="cuda")
    for b, n in enumerate(lens):
        x[b, :n] = _signal(kind, n, sr, seed=b)
    got = measure_loudness(x, sr, lens=lens).cpu().numpy()
    worst = 0.0
    for b, n in enumerate(lens):
        want = _oracle_L(x[b, :n], sr)
        assert _close(float(got[b]), want, 1e-6), (n, float(got[b]), want)
        if math.isfinite(want):
            worst = max(worst, abs(float(got[b]) - want))
    assert got[0] == -math.inf and math.isfinite(got[1])
    print(f"sr {sr} {kind}: L {np.round(got, 3).tolist()}, worst |L - oracle| {worst:.2e} LU")


def test_full_length_waveform():
    """The 10k-frame length once: 19.2 M samples at 24 kHz, a level that changes every 2 s (both gates at work)."""
    from sopro_b200.loudness import measure_loudness, normalize_loudness

    N = 10000 * HOP
    g = torch.Generator().manual_seed(3)
    env = torch.tensor([1.0, 0.3, 0.02, 0.0, 0.5, 0.004, 1.0, 0.1])[(torch.arange(N) // 48000) % 8]
    x = (0.3 * torch.randn(N, generator=g) * env).float().cuda()
    L = float(measure_loudness(x, 24000))
    want = _oracle_L(x, 24000)
    print(f"19.2 M samples: L {L:.6f}, oracle {want:.6f}, |diff| {abs(L - want):.2e} LU")
    assert _close(L, want, 1e-6)
    y, gain = normalize_loudness(x, 24000, -23.0, return_gain=True)
    assert torch.equal(y, x * gain)


def _batch(sr, lens, kinds):
    x = torch.full((len(lens), max(lens)), float("nan"), device="cuda")
    for b, (n, k) in enumerate(zip(lens, kinds)):
        x[b, :n] = _signal(k, n, sr, seed=b)
    return x


@pytest.mark.parametrize("sr", (16000, 24000, 48000))
def test_ragged_rows_equal_single_rows_and_runs_repeat(sr):
    """Each row of a ragged batch with NaN padding gives the L, g and y bits of that row alone; two runs give the same
    bits; outputs past lens[b] are zero.  Also a batch of 130 rows (two launches)."""
    from sopro_b200.loudness import measure_loudness, normalize_loudness

    s = O.sub_block(sr)
    lens = [5 * sr + 3, 4 * s - 1, 0, 3 * 8192 + 1, 4 * s, 9 * s + 11]
    x = _batch(sr, lens, ("noise", "sweep", "noise", "mimi", "sine997", "gated"))
    y, g = normalize_loudness(x, sr, -16.0, lens=lens, return_gain=True)
    L = measure_loudness(x, sr, lens=lens)
    y2, g2 = normalize_loudness(x, sr, -16.0, lens=lens, return_gain=True)
    assert torch.equal(y, y2) and torch.equal(g, g2) and torch.equal(L, measure_loudness(x, sr, lens=lens))
    assert bool(torch.isfinite(y).all())
    for b, n in enumerate(lens):
        row = x[b, :n].clone()
        yb, gb = normalize_loudness(row, sr, -16.0, return_gain=True)
        assert torch.equal(y[b, :n], yb) and torch.equal(g[b], gb), b
        assert torch.equal(L[b], measure_loudness(row, sr)), b
        assert not bool(y[b, n:].any())
    lens = [int(v) for v in torch.randint(1, 6 * s, (130,), generator=torch.Generator().manual_seed(sr)).tolist()]
    x = _batch(sr, lens, ["noise"] * 130)
    y, g = normalize_loudness(x, sr, -20.0, lens=lens, return_gain=True)
    for b in (0, 64, 127, 128, 129):
        yb, gb = normalize_loudness(x[b, : lens[b]].clone(), sr, -20.0, return_gain=True)
        assert torch.equal(y[b, : lens[b]], yb) and torch.equal(g[b], gb), b
    with pytest.raises(ValueError):
        normalize_loudness(x, sr, -20.0, lens=lens[:-1] + [x.shape[1] + 1])


@pytest.mark.parametrize("sr", (8000, 24000, 44100, 96000))
@pytest.mark.parametrize("target", (-40.0, -23.0, -16.0, -1.0))
def test_gain_and_its_ceiling(sr, target):
    """y = x * g bit for bit; g within 1 fp32 ulp of fp32(g64) from the GPU's own L and max|x|; without the ceiling the
    oracle re-measures y at the target within 1e-4 LU; with it, max|y| <= fp32(10^(-1/20))."""
    from sopro_b200.loudness import measure_loudness, normalize_loudness

    kinds = ("noise", "sweep", "sine200", "sine997", "mimi")
    lens = [3 * sr + 2 * b + 1 for b in range(len(kinds))]
    x = _batch(sr, lens, kinds)
    x[2] *= 0.01  # a quiet row
    y, g = normalize_loudness(x, sr, target, lens=lens, return_gain=True)
    L = measure_loudness(x, sr, lens=lens).cpu().numpy()
    ceil32 = float(np.float32(O.CEILING))
    bound = 0
    for b, n in enumerate(lens):
        xb = x[b, :n]
        assert torch.equal(y[b, :n], xb * g[b])
        peak = float(xb.abs().max())
        g64 = O.gain(float(L[b]), peak, target)
        g32 = np.float32(g64)
        assert abs(float(g[b]) - float(g32)) <= float(np.spacing(g32)), (b, float(g[b]), g64)
        if 10.0 ** ((target - float(L[b])) / 20.0) < O.CEILING / peak:
            got = _oracle_L(y[b, :n], sr)
            assert abs(got - target) <= 1e-4, (b, got, target)
        else:
            bound += 1
            assert float(y[b, :n].abs().max()) <= ceil32, b
    print(f"sr {sr} target {target}: {bound} of {len(lens)} rows at the ceiling")


def test_minus_inf_rows_come_back_bit_equal():
    from sopro_b200.loudness import measure_loudness, normalize_loudness

    sr = 24000
    s = O.sub_block(sr)
    lens = [4 * s - 1, 50000, 0, 30000]
    x = _batch(sr, lens, ("noise", "noise", "noise", "noise"))
    x[1, :50000] = 0
    x[3, :30000] *= 1e-5  # about -100 LUFS: no block passes the absolute gate
    y, g = normalize_loudness(x, sr, -14.0, lens=lens, return_gain=True)
    assert bool((measure_loudness(x, sr, lens=lens) == -math.inf).all())
    assert bool((g == 1).all())
    for b, n in enumerate(lens):
        assert torch.equal(y[b, :n].view(torch.int32), x[b, :n].view(torch.int32)), b


def test_graph_capture_replays_the_same_bits():
    """One row (no lens): nothing in the call synchronises, so it captures into a CUDA graph."""
    from sopro_b200.loudness import normalize_loudness

    x = _signal("mimi", 400 * HOP // 10, 24000)
    want, want_g = normalize_loudness(x, 24000, -16.0, return_gain=True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        normalize_loudness(x, 24000, -16.0)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y, g = normalize_loudness(x, 24000, -16.0, return_gain=True)
    for _ in range(2):
        y.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(y, want) and torch.equal(g, want_g)


def test_refused_calls_launch_nothing():
    from sopro_b200.loudness import measure_loudness, normalize_loudness

    x = _signal("noise", 10000, 24000)
    for bad in (float("nan"), 0.5, -61.0, True):
        with pytest.raises(ValueError):
            normalize_loudness(x, 24000, bad)
    for sr in (3999, 192001):
        with pytest.raises(ValueError):
            measure_loudness(x, sr)
    with pytest.raises(ValueError):
        measure_loudness(x, 24000, lens=[10001])


# ---- through the public API (the e2e fixture of test_e2e_gpu.py)

def _api():
    from tests.cases import e2e_inputs
    from tests.test_e2e_gpu import TEXT, _tts

    tts, _ = _tts()
    _cfg, _sd, inp = e2e_inputs()
    return tts, tts.prepare_reference(ref_tokens_tq=inp["ref_tokens_tq"]), TEXT


@pytest.mark.parametrize("mode", ("fp32", "bf16_tc"))
@pytest.mark.parametrize("target,speed,sr", ((-16.0, None, None), (-23.0, 1.25, None), (-14.0, None, 48000),
                                             (-30.0, 0.8, 16000)))
def test_synthesize_loudness_equals_normalize_of_synthesize(mode, target, speed, sr):
    from sopro_b200.loudness import measure_loudness, normalize_loudness

    tts, ref, text = _api()
    eng = tts.codec.engine
    kw = dict(ref=ref, max_frames=20, seed=4, min_gen_frames=10 ** 9, speed=speed, sample_rate=sr)
    eng.set_precision(mode)
    try:
        base = tts.synthesize(text, **kw)
        got = tts.synthesize(text, loudness=target, **kw)
        texts = [text, " ".join(str(i) for i in range(3, 40, 3)), "5 9"]
        bkw = dict(ref=ref, max_frames=16, min_gen_frames=10 ** 9, speed=speed, sample_rate=sr, loudness=target)
        wavs = tts.synthesize_batch(texts, seeds=[1, 2, 3], **bkw)
        singles = [tts.synthesize(t, seed=s, **bkw) for t, s in zip(texts, [1, 2, 3])]
    finally:
        eng.set_precision("bf16_tc")
    rate = sr or 24000
    assert torch.equal(got, normalize_loudness(base, rate, target))
    print(f"{mode} target {target}: L {float(measure_loudness(base, rate)):.3f} -> {float(measure_loudness(got, rate)):.3f}")
    for w, s in zip(wavs, singles):
        assert torch.equal(w, s)


def test_no_loudness_makes_no_launch_in_the_chain(monkeypatch):
    import sopro_b200.output as output_mod

    tts, ref, text = _api()
    kw = dict(ref=ref, max_frames=16, min_gen_frames=10 ** 9)
    texts = [text, "5 9"]
    base = tts.synthesize(text, seed=3, **kw)
    base_b = tts.synthesize_batch(texts, seeds=[1, 2], **kw)

    def boom(*a, **k):
        raise AssertionError("the loudness stage ran without a target")

    monkeypatch.setattr(output_mod, "normalize_loudness", boom)
    assert torch.equal(tts.synthesize(text, seed=3, loudness=None, **kw), base)
    assert all(torch.equal(a, b) for a, b in zip(tts.synthesize_batch(texts, seeds=[1, 2], loudness=None, **kw), base_b))
    with pytest.raises(AssertionError):
        tts.synthesize(text, seed=3, loudness=-16.0, **kw)


def test_refused_loudness_raises_before_the_rng_moves():
    tts, ref, text = _api()
    for target in (float("nan"), float("inf"), -float("inf"), -60.5, 0.5, True, "-16"):
        before = torch.get_rng_state()
        with pytest.raises(ValueError):
            tts.synthesize(text, ref=ref, max_frames=8, loudness=target)
        with pytest.raises(ValueError):
            tts.synthesize_batch([text], ref=ref, max_frames=8, loudness=target)
        assert torch.equal(before, torch.get_rng_state())
