"""GPU: the output resampler (csrc/resample.cu through sopro_b200/resample.py) against torchaudio's float64 resampler, the
ragged batch, the stream under several chunk schedules, and `sample_rate=` through the public API."""
import math

import numpy as np
import pytest
import torch

from oracle import mimi_oracle as M

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
RATES = (8000, 11025, 16000, 22050, 32000, 44100, 48000, 96000, 12345)
HOP = 1920
_CACHE = {}


def _taf():
    return pytest.importorskip("torchaudio.functional.functional")


def _rs(sr):
    from sopro_b200.resample import Resampler

    if sr not in _CACHE:
        _CACHE[sr] = Resampler(24000, sr, "cuda:0")
    return _CACHE[sr]


def _mimi_wav():
    """A real Mimi decode (synthetic checkpoint, seeded codes): 41 frames = 78,720 samples."""
    if "mimi" not in _CACHE:
        from sopro_b200.codec import MimiEngine

        codes = torch.randint(0, 2048, (1, 32, 41), generator=torch.Generator().manual_seed(7))
        eng = MimiEngine(M.synth_mimi_state_dict(), 0, 32)
        _CACHE["mimi"] = eng.decode(codes).reshape(-1).clone()
    return _CACHE["mimi"]


def _signal(kind, N):
    g = torch.Generator().manual_seed(1000 + N)
    if kind == "noise":
        return (0.3 * torch.randn(N, generator=g)).cuda()
    if kind == "sweep":  # 20 Hz -> 12 kHz linear chirp at 24 kHz
        t = torch.arange(N, dtype=torch.float64) / 24000.0
        T = max(N, 2) / 24000.0
        return (0.8 * torch.sin(2 * math.pi * (20 * t + (12000 - 20) / (2 * T) * t * t))).float().cuda()
    w = _mimi_wav()
    return w[:N].clone() if N <= w.numel() else w.repeat(N // w.numel() + 1)[:N].contiguous()


def _oracle(x, sr):
    """(y64, bound): torchaudio's resample in float64 and, per element, (S + 2) 2^-24 sum|k64 x| with S the phase's taps."""
    from sopro_b200.resample import filter_taps

    F = _taf()
    g = math.gcd(24000, sr)
    k64, width = F._get_sinc_resample_kernel(24000, sr, g, device=x.device, dtype=torch.float64)
    x64 = x.double().reshape(1, -1)
    y64 = F._apply_sinc_resample_kernel(x64, 24000, sr, g, k64, width)[0]
    mag = F._apply_sinc_resample_kernel(x64.abs(), 24000, sr, g, k64.abs(), width)[0]
    _o, n, _w, _f, span, _t = filter_taps(24000, sr)
    S = torch.as_tensor(span, device=x.device, dtype=torch.float64)[torch.arange(y64.numel(), device=x.device) % n]
    return y64, (S + 2) * 2.0 ** -24 * mag


@pytest.mark.parametrize("sr", RATES)
def test_one_shot_matches_float64_torchaudio(sr):
    AF = pytest.importorskip("torchaudio.functional")
    rs = _rs(sr)
    o = 24000 // math.gcd(24000, sr)
    worst, worst_ta = 0.0, 0.0
    for N in sorted({1, 2, max(1, o - 1), o, o + 1, 41 * HOP}):
        for kind in ("noise", "sweep", "mimi"):
            x = _signal(kind, N)
            y = rs(x)
            assert y.shape == (rs.length(N),) == (AF.resample(torch.zeros(N, dtype=torch.float64), 24000, sr).numel(),)
            y64, bound = _oracle(x, sr)
            err = (y.double() - y64).abs()
            assert bool((err <= bound).all()), (N, kind, float((err - bound).max()))
            worst = max(worst, float((err / bound.clamp_min(1e-300)).max()))
            ta32 = AF.resample(x.reshape(1, -1), 24000, sr)[0]
            worst_ta = max(worst_ta, float((y - ta32).abs().max()))
    print(f"24000 -> {sr}: worst error / bound {worst:.3f}; max |ours - torchaudio fp32 CUDA| {worst_ta:.3e}")


def test_one_shot_full_bench_waveform():
    """The bench's 10k-frame length once: 19.2 M samples -> 38.4 M at 48 kHz."""
    rs = _rs(48000)
    x = _signal("noise", 10000 * HOP)
    y = rs(x)
    y64, bound = _oracle(x, 48000)
    assert y.numel() == 2 * x.numel() and bool(((y.double() - y64).abs() <= bound).all())


@pytest.mark.parametrize("sr", (8000, 11025, 44100, 12345))
def test_ragged_batch_rows_equal_single_rows(sr):
    rs = _rs(sr)
    lens = [41 * HOP, 7 * HOP + 13, 1]
    x = torch.full((3, max(lens)), float("nan"), device="cuda")
    for b, L in enumerate(lens):
        x[b, :L] = _signal(("noise", "sweep", "mimi")[b], L)
    y = rs(x, lens=lens)
    assert y.shape == (3, rs.length(max(lens))) and bool(torch.isfinite(y).all())
    for b, L in enumerate(lens):
        single = rs(x[b, :L].clone())
        assert torch.equal(y[b, : single.numel()], single), b
        assert not bool(y[b, single.numel():].any())
    with pytest.raises(ValueError):
        rs(x, lens=[1, 2, max(lens) + 1])


def _schedule(name, N):
    if name == "single":
        return [N]
    if name == "6x1920":
        return [6 * HOP] * (N // (6 * HOP)) + ([N % (6 * HOP)] if N % (6 * HOP) else [])
    if name == "ragged":
        out, pat, i = [], (1, 7, 1919, 3841, 2, 5000, 1920), 0
        while sum(out) < N:
            out.append(min(pat[i % len(pat)], N - sum(out)))
            i += 1
        return out
    return [1] * N


def _run_stream(st, x, sizes, o, n, width):
    outs, seen, emitted = [], 0, 0
    for m in sizes:
        assert st.ready(m) == n * max(0, (seen + m - width) // o) - emitted
        y = st.push(x[seen: seen + m])
        seen += m
        emitted += y.numel()
        assert emitted == n * max(0, (seen - width) // o), (seen, emitted)  # every block whose window has arrived
        outs.append(y)
    tail = st.finish()
    assert emitted + tail.numel() == -(-n * seen // o)
    return torch.cat(outs + [tail])


@pytest.mark.parametrize("sr", RATES)
@pytest.mark.parametrize("schedule", ("single", "6x1920", "ragged", "ones"))
def test_stream_equals_one_shot_bit_for_bit(sr, schedule):
    from sopro_b200.resample import filter_taps

    rs = _rs(sr)
    o, n, width, *_ = filter_taps(24000, sr)
    N = 2000 if schedule == "ones" else 41 * HOP
    x = _signal("mimi", N)
    want = rs(x)
    sizes = _schedule(schedule, N)
    st = rs.stream(max(sizes))
    assert torch.equal(_run_stream(st, x, sizes, o, n, width), want)
    st.reset()  # reuse after a reset == a fresh stream
    assert torch.equal(_run_stream(st, x, sizes, o, n, width), want)


@pytest.mark.parametrize("sr", (11025, 48000))
def test_stream_errors_leave_the_state_intact(sr):
    from sopro_b200 import _lib
    from sopro_b200.resample import filter_taps

    rs = _rs(sr)
    o, n, width, *_ = filter_taps(24000, sr)
    x = _signal("sweep", 5 * HOP)
    st = rs.stream(HOP)
    a = st.push(x[:HOP])
    with pytest.raises(ValueError):  # larger than max_chunk: refused before any launch
        st.push(x[HOP: 3 * HOP + 1])
    b = [st.push(x[i: i + HOP]) for i in range(HOP, 5 * HOP, HOP)]
    tail = st.finish()
    for bad in (lambda: st.push(x[:10]), st.finish):
        with pytest.raises(_lib.SoproError):
            bad()
    assert torch.equal(torch.cat([a] + b + [tail]), rs(x))
    st.reset()
    assert torch.equal(_run_stream(st, x, [HOP] * 5, o, n, width), rs(x))


# ---- through the public API (the e2e fixture of test_e2e_gpu.py)

def _api():
    from tests.cases import e2e_inputs
    from tests.test_e2e_gpu import TEXT, _tts

    tts, _ = _tts()
    _cfg, _sd, inp = e2e_inputs()
    return tts, tts.prepare_reference(ref_tokens_tq=inp["ref_tokens_tq"]), TEXT


@pytest.mark.parametrize("sr", (8000, 16000, 44100, 48000))
def test_synthesize_sample_rate_equals_resampler_on_24k(sr):
    tts, ref, text = _api()
    kw = dict(ref=ref, max_frames=20, seed=4, min_gen_frames=10 ** 9)
    base = tts.synthesize(text, **kw)
    got = tts.synthesize(text, sample_rate=sr, **kw)
    assert got.shape == (1, 1, -(-base.shape[-1] * sr // 24000))
    assert torch.equal(got, _rs(sr)(base))
    assert torch.equal(tts.synthesize(text, sample_rate=None, **kw), base)
    assert torch.equal(tts.synthesize(text, sample_rate=24000, **kw), base)


@pytest.mark.parametrize("sr", (16000, 44100))
def test_synthesize_batch_sample_rate_equals_single(sr):
    tts, ref, text = _api()
    texts = [text, " ".join(str(i) for i in range(3, 40, 3)), "5 9"]
    wavs = tts.synthesize_batch(texts, ref=ref, max_frames=16, seeds=[1, 2, 3], min_gen_frames=10 ** 9, sample_rate=sr)
    for t, s, w in zip(texts, [1, 2, 3], wavs):
        assert torch.equal(w, tts.synthesize(t, ref=ref, max_frames=16, seed=s, min_gen_frames=10 ** 9, sample_rate=sr))
    plain = tts.synthesize_batch(texts, ref=ref, max_frames=16, seeds=[1, 2, 3], min_gen_frames=10 ** 9, sample_rate=24000)
    assert all(torch.equal(a, b) for a, b in zip(plain, tts.synthesize_batch(texts, ref=ref, max_frames=16, seeds=[1, 2, 3],
                                                                             min_gen_frames=10 ** 9)))


@pytest.mark.parametrize("sr", (8000, 44100))
def test_stream_sample_rate(sr):
    """One chunk: stream == synthesize at the same rate.  Six-frame chunks, both Mimi modes: the chunks concatenate to the
    one-shot resample of the 24 kHz stream, and each chunk but the last carries every output its audio completes."""
    from sopro_b200.resample import filter_taps

    tts, ref, text = _api()
    o, n, width, *_ = filter_taps(24000, sr)
    kw = dict(ref=ref, max_frames=25, seed=9, min_gen_frames=10 ** 9)
    eng = tts.codec.engine
    eng.set_precision("fp32")
    try:
        one = list(tts.stream(text, chunk_frames=64, sample_rate=sr, **kw))
        assert len(one) == 1 and torch.equal(one[0].reshape(-1), tts.synthesize(text, sample_rate=sr, **kw).reshape(-1))
    finally:
        eng.set_precision("bf16_tc")
    for mode in ("fp32", "bf16_tc"):
        eng.set_precision(mode)
        try:
            c24 = list(tts.stream(text, chunk_frames=6, **kw))
            cr = list(tts.stream(text, chunk_frames=6, sample_rate=sr, **kw))
        finally:
            eng.set_precision("bf16_tc")
        assert torch.equal(torch.cat(cr, dim=1), _rs(sr)(torch.cat(c24, dim=1)))
        assert len(cr) in (len(c24), len(c24) + 1)  # + 1 only when the last 24 kHz step had no audio left to carry the tail
        seen = 0
        for a, b in zip(c24[:-1], cr):
            prev = n * max(0, (seen - width) // o)
            seen += a.shape[1]
            assert b.shape == (1, n * max(0, (seen - width) // o) - prev)


def test_interleaved_and_abandoned_resampled_streams():
    tts, ref, text = _api()
    t2 = " ".join(str(5 * i + 1) for i in range(20))
    kw = dict(ref=ref, max_frames=18, min_gen_frames=10 ** 9, sample_rate=44100)
    solo_a = list(tts.stream(text, seed=21, **kw))
    solo_b = list(tts.stream(t2, seed=22, **kw))
    ga, gb = tts.stream(text, seed=21, **kw), tts.stream(t2, seed=22, **kw)
    mixa, mixb = [], []
    for _ in range(max(len(solo_a), len(solo_b))):
        for g, out in ((ga, mixa), (gb, mixb)):
            c = next(g, None)
            if c is not None:
                out.append(c)
    assert len(mixa) == len(solo_a) and all(torch.equal(x, y) for x, y in zip(mixa, solo_a))
    assert len(mixb) == len(solo_b) and all(torch.equal(x, y) for x, y in zip(mixb, solo_b))
    g = tts.stream(t2, seed=22, **kw)
    next(g)
    g.close()  # abandoned after one chunk: its resampler state goes back to the pool mid-utterance
    again = list(tts.stream(text, seed=21, **kw))
    assert len(again) == len(solo_a) and all(torch.equal(x, y) for x, y in zip(again, solo_a))


def test_refused_rate_raises_before_the_rng_moves():
    tts, ref, text = _api()
    for sr in (44099, 3999, 24000.5):
        before = torch.get_rng_state()
        with pytest.raises(ValueError):
            tts.synthesize(text, ref=ref, max_frames=8, sample_rate=sr)
        with pytest.raises(ValueError):
            tts.synthesize_batch([text], ref=ref, max_frames=8, sample_rate=sr)
        with pytest.raises(ValueError):
            tts.stream(text, ref=ref, max_frames=8, sample_rate=sr)
        assert torch.equal(before, torch.get_rng_state())
