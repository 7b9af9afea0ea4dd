"""GPU: the time-stretch (csrc/stretch.cu through sopro_b200/stretch.py) against the float64 oracle
(oracle/stretch_oracle.py) frame by frame, content checks on sines, the ragged batch, the stream under several push
schedules, and `speed=` through the public API."""
import math

import numpy as np
import pytest
import torch

from oracle import mimi_oracle as MO
from oracle import stretch_oracle as O

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
SPEEDS = (0.25, 0.5, 0.8, 1.0737, 1.25, 2.0, 3.7, 4.0)
KINDS = ("noise", "sweep", "sine200", "sine150", "mimi")
HOP = 1920
U = 2.0 ** -24
_CACHE = {}


def _gamma(n):
    return n * U / (1 - n * U)


def _mimi_wav():
    """A real Mimi decode (synthetic checkpoint, seeded codes): 41 frames = 78,720 samples."""
    if "mimi" not in _CACHE:
        from sopro_b200.codec import MimiEngine

        codes = torch.randint(0, 2048, (1, 32, 41), generator=torch.Generator().manual_seed(7))
        eng = MimiEngine(MO.synth_mimi_state_dict(), 0, 32)
        _CACHE["mimi"] = eng.decode(codes).reshape(-1).clone()
    return _CACHE["mimi"]


def _signal(kind, N):
    g = torch.Generator().manual_seed(2000 + N)
    t = torch.arange(N, dtype=torch.float64) / 24000.0
    if kind == "noise":
        return (0.3 * torch.randn(N, generator=g)).cuda()
    if kind == "sweep":  # 20 Hz -> 12 kHz linear chirp
        T = max(N, 2) / 24000.0
        return (0.8 * torch.sin(2 * math.pi * (20 * t + (12000 - 20) / (2 * T) * t * t))).float().cuda()
    if kind.startswith("sine"):
        return (0.5 * torch.sin(2 * math.pi * float(kind[4:]) * t)).float().cuda()
    w = _mimi_wav()
    return w[:N].clone() if N <= w.numel() else w.repeat(N // w.numel() + 1)[:N].contiguous()


def _gpu(kind, speed, N=41 * HOP):
    from sopro_b200.stretch import stretch

    key = (kind, speed, N)
    if key not in _CACHE:
        x = _signal(kind, N)
        y, offs = stretch(x, speed, return_offsets=True)
        _CACHE[key] = (x, y, offs[0].cpu().numpy().astype(np.int64))
    return _CACHE[key]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("speed", SPEEDS)
def test_offsets_are_within_the_fp32_bound_of_the_float64_argmax(speed, kind):
    """Every frame, scored in float64 given the GPU's own d_{k-1}: the GPU's d_k is within 2 gamma_N max sum|t x| of the
    float64 maximum; where the float64 margin exceeds that bound, it is the float64 argmax (>= 95 % of noise frames)."""
    S = O.quantise(speed)
    x, _y, d = _gpu(kind, speed)
    r = O.stretch(x.double().cpu().numpy(), S, offsets=d)
    K = d.size
    assert K == O.n_frames(O.out_len(S, x.numel())) and d[0] == 0 and np.abs(d).max() <= 160
    worst, clear, exact = 0.0, 0, 0
    for k in range(1, K):
        c = r.scores[k]
        bound = 2 * _gamma(480) * r.score_mag[k]
        gap = c.max() - c[d[k] + 160]
        assert gap <= bound, (k, gap, bound)
        if bound > 0:
            worst = max(worst, gap / bound)
        srt = np.sort(c)
        if srt[-1] - srt[-2] > bound:
            clear += 1
            assert d[k] == O.best_delta(c), k
    if kind == "noise":
        assert clear >= 0.95 * (K - 1), (clear, K - 1)
    print(f"speed {speed} {kind}: {K} frames, worst gap / bound {worst:.3f}, {clear} frames with a clear float64 argmax")


@pytest.mark.parametrize("speed", SPEEDS)
def test_exact_scores_follow_the_tie_rule(speed):
    """Small-integer inputs make every fp32 score exact (integer partial sums below 2^24), so the GPU must pick the
    float64 argmax at every frame, ties included: a period-97 pattern ties candidates 97 apart, and silence ties all
    321 (the tie rule then picks d = 0)."""
    from sopro_b200.stretch import stretch

    S = O.quantise(speed)
    pat = torch.randint(-2, 3, (97,), generator=torch.Generator().manual_seed(5)).float()
    for x in (pat.repeat(200)[: 12000].cuda(), torch.zeros(6000, device="cuda")):
        _y, offs = stretch(x, speed, return_offsets=True)
        d = offs[0].cpu().numpy().astype(np.int64)
        r = O.stretch(x.double().cpu().numpy(), S)
        ties = sum(int((r.scores[k] == r.scores[k].max()).sum() > 1) for k in range(1, d.size))
        assert np.array_equal(d, r.deltas), (speed, np.flatnonzero(d != r.deltas)[:5])
        assert ties > 0.5 * (d.size - 1)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("speed", SPEEDS)
def test_samples_match_the_replay_of_the_gpu_path(speed, kind):
    """Given the GPU's d path, every output is within 3 * 2^-24 * sum|w x| of the float64 replay (the kernel does one
    product and one fma per output: 2 roundings)."""
    S = O.quantise(speed)
    x, y, d = _gpu(kind, speed)
    r = O.stretch(x.double().cpu().numpy(), S, offsets=d)
    assert y.numel() == r.y.size == O.out_len(S, x.numel())
    err = np.abs(y.double().cpu().numpy() - r.y)
    bound = 3 * U * r.y_mag
    assert bool((err <= bound).all()), float((err - bound).max())
    print(f"speed {speed} {kind}: worst sample error / bound {float((err / np.maximum(bound, 1e-300)).max()):.3f}")


@pytest.mark.parametrize("speed", SPEEDS)
def test_sines_keep_their_rms_and_pitch(speed):
    S = O.quantise(speed)
    L = 41 * HOP
    for f in (200, 150):
        x, y, _d = _gpu(f"sine{f}", speed)
        assert y.numel() == O.out_len(S, L)
        clean = int((L - 400) * 65536 / S) - 480
        nb = clean // 960
        yb = y[960: nb * 960].double().cpu().numpy()  # clear of both edges (test_stretch_cpu._block_rms_error)
        rms = np.sqrt((yb.reshape(nb - 1, 960) ** 2).mean(axis=1))
        want = 0.5 / math.sqrt(2)
        assert float(np.abs(rms - want).max()) <= 1e-3 * want, (f, speed)
        spec = np.abs(np.fft.rfft(yb))
        assert abs(int(np.argmax(spec)) - f * yb.size / 24000.0) <= 1.0, (f, speed)


@pytest.mark.parametrize("speed", (0.25, 1.0737, 4.0))
def test_ragged_batch_rows_equal_single_rows(speed):
    from sopro_b200.stretch import stretch, stretched_length

    lens = [41 * HOP, 7 * HOP + 13, 1, 500, 0]
    x = torch.full((len(lens), max(lens)), float("nan"), device="cuda")
    for b, L in enumerate(lens):
        x[b, :L] = _signal(("noise", "sweep", "mimi", "sine200", "noise")[b], L)
    y = stretch(x, speed, lens=lens)
    assert y.shape == (len(lens), stretched_length(speed, max(lens))) and bool(torch.isfinite(y).all())
    for b, L in enumerate(lens):
        single = stretch(x[b, :L].clone(), speed)
        assert single.numel() == stretched_length(speed, L)
        assert torch.equal(y[b, : single.numel()], single), b
        assert not bool(y[b, single.numel():].any())
    with pytest.raises(ValueError):
        stretch(x, speed, lens=[1, 2, 3, 4, max(lens) + 1])


def _schedule(name, N):
    if name == "single":
        return [N]
    if name == "6x1920":
        return [6 * HOP] * (N // (6 * HOP)) + ([N % (6 * HOP)] if N % (6 * HOP) else [])
    if name == "ragged":
        rng, out = np.random.default_rng(11), []
        while sum(out) < N:
            out.append(min(int(rng.integers(1, 5000)), N - sum(out)))
        return out
    return [1] * N


def _frames_ready(S, n_seen, k=0):
    """The stream rule in host arithmetic: frame k is ready once max(a_k + 400, a_{k-1} + 640) samples have arrived."""
    while max(O.pos_a(k, S) + 400, O.pos_a(k - 1, S) + 640 if k else 0) <= n_seen:
        k += 1
    return k


def _run_stream(st, x, sizes, S):
    outs, seen, emitted, k = [], 0, 0, 0
    for m in sizes:
        want = st.ready(m)
        y = st.push(x[seen: seen + m])
        seen += m
        k = _frames_ready(S, seen, k)
        assert y.numel() == want == max(0, k - 1) * 240 - emitted, (seen, y.numel(), want)
        emitted += y.numel()
        outs.append(y)
    assert st.ready(0, final=True) == O.out_len(S, seen) - emitted
    tail = st.finish()
    assert emitted + tail.numel() == O.out_len(S, seen)
    return torch.cat(outs + [tail])


@pytest.mark.parametrize("schedule", ("single", "6x1920", "ragged", "ones"))
def test_stream_equals_one_shot_bit_for_bit(schedule):
    """One state serves every speed through reset(speed), and the chunks equal the one-shot result bit for bit."""
    from sopro_b200.stretch import StretchStream, stretch

    N = 2000 if schedule == "ones" else 41 * HOP
    x = _signal("mimi", N)
    sizes = _schedule(schedule, N)
    st = StretchStream(max(sizes), 0)
    for speed in SPEEDS:
        st.reset(speed)
        want = stretch(x, speed)
        assert torch.equal(_run_stream(st, x, sizes, O.quantise(speed)), want), speed
    st.close()


@pytest.mark.parametrize("speed", (0.5, 1.25, 4.0))
def test_stream_errors_leave_the_state_intact(speed):
    from sopro_b200 import _lib
    from sopro_b200.stretch import StretchStream, stretch

    x = _signal("sweep", 5 * HOP)
    st = StretchStream(HOP, 0)
    with pytest.raises(_lib.SoproError):  # no speed yet
        st.push(x[:10])
    st.reset(speed)
    a = st.push(x[:HOP])
    with pytest.raises(ValueError):  # larger than max_chunk: refused before any launch
        st.push(x[HOP: 3 * HOP + 1])
    b = [st.push(x[i: i + HOP]) for i in range(HOP, 5 * HOP, HOP)]
    tail = st.finish()
    for bad in (lambda: st.push(x[:10]), st.finish):
        with pytest.raises(_lib.SoproError):
            bad()
    assert torch.equal(torch.cat([a] + b + [tail]), stretch(x, speed))
    with pytest.raises(ValueError):
        st.reset(0.0)
    st.reset(speed)
    assert torch.equal(_run_stream(st, x, [HOP] * 5, O.quantise(speed)), stretch(x, speed))


# ---- through the public API (the e2e fixture of test_e2e_gpu.py)

def _api():
    from tests.cases import e2e_inputs
    from tests.test_e2e_gpu import TEXT, _tts

    tts, _ = _tts()
    _cfg, _sd, inp = e2e_inputs()
    return tts, tts.prepare_reference(ref_tokens_tq=inp["ref_tokens_tq"]), TEXT


def _resampled(wav, sr):
    if sr is None:
        return wav
    from sopro_b200.resample import Resampler

    return Resampler(24000, sr, wav.device)(wav)


@pytest.mark.parametrize("mode", ("fp32", "bf16_tc"))
@pytest.mark.parametrize("speed,sr", ((0.5, None), (1.25, None), (3.7, 16000), (0.8, 44100)))
def test_synthesize_speed_equals_stretch_of_24k(mode, speed, sr):
    from sopro_b200.stretch import stretch

    tts, ref, text = _api()
    eng = tts.codec.engine
    kw = dict(ref=ref, max_frames=20, seed=4, min_gen_frames=10 ** 9)
    eng.set_precision(mode)
    try:
        base = tts.synthesize(text, **kw)
        got = tts.synthesize(text, speed=speed, sample_rate=sr, **kw)
        texts = [text, " ".join(str(i) for i in range(3, 40, 3)), "5 9"]
        wavs = tts.synthesize_batch(texts, ref=ref, max_frames=16, seeds=[1, 2, 3], min_gen_frames=10 ** 9, speed=speed,
                                    sample_rate=sr)
        singles = [tts.synthesize(t, ref=ref, max_frames=16, seed=s, min_gen_frames=10 ** 9, speed=speed, sample_rate=sr)
                   for t, s in zip(texts, [1, 2, 3])]
    finally:
        eng.set_precision("bf16_tc")
    assert torch.equal(got, _resampled(stretch(base, speed), sr))
    for w, s in zip(wavs, singles):
        assert torch.equal(w, s)


@pytest.mark.parametrize("speed,sr", ((0.5, None), (1.25, 8000), (3.7, None)))
def test_stream_speed(speed, sr):
    """One chunk: stream == synthesize.  Six-frame chunks, both Mimi modes: the chunks concatenate to the one-shot
    stretch (then resample) of the concatenated 24 kHz stream."""
    from sopro_b200.stretch import stretch

    tts, ref, text = _api()
    kw = dict(ref=ref, max_frames=25, seed=9, min_gen_frames=10 ** 9)
    eng = tts.codec.engine
    eng.set_precision("fp32")
    try:
        one = list(tts.stream(text, chunk_frames=64, speed=speed, sample_rate=sr, **kw))
        assert len(one) == 1
        assert torch.equal(one[0].reshape(-1), tts.synthesize(text, speed=speed, sample_rate=sr, **kw).reshape(-1))
    finally:
        eng.set_precision("bf16_tc")
    for mode in ("fp32", "bf16_tc"):
        eng.set_precision(mode)
        try:
            c24 = list(tts.stream(text, chunk_frames=6, **kw))
            cs = list(tts.stream(text, chunk_frames=6, speed=speed, sample_rate=sr, **kw))
        finally:
            eng.set_precision("bf16_tc")
        assert torch.equal(torch.cat(cs, dim=1), _resampled(stretch(torch.cat(c24, dim=1), speed), sr))
        assert len(cs) in (len(c24), len(c24) + 1)


def test_interleaved_and_abandoned_stretched_streams():
    tts, ref, text = _api()
    t2 = " ".join(str(5 * i + 1) for i in range(20))
    kw = dict(ref=ref, max_frames=18, min_gen_frames=10 ** 9)
    solo_a = list(tts.stream(text, seed=21, speed=1.25, **kw))
    solo_b = list(tts.stream(t2, seed=22, speed=0.5, sample_rate=44100, **kw))
    ga, gb = tts.stream(text, seed=21, speed=1.25, **kw), tts.stream(t2, seed=22, speed=0.5, sample_rate=44100, **kw)
    mixa, mixb = [], []
    for _ in range(max(len(solo_a), len(solo_b))):
        for g, out in ((ga, mixa), (gb, mixb)):
            c = next(g, None)
            if c is not None:
                out.append(c)
    assert len(mixa) == len(solo_a) and all(torch.equal(x, y) for x, y in zip(mixa, solo_a))
    assert len(mixb) == len(solo_b) and all(torch.equal(x, y) for x, y in zip(mixb, solo_b))
    g = tts.stream(t2, seed=22, speed=0.5, **kw)
    next(g)
    g.close()  # abandoned after one chunk: its stretch state goes back to the pool mid-utterance
    again = list(tts.stream(text, seed=21, speed=1.25, **kw))
    assert len(again) == len(solo_a) and all(torch.equal(x, y) for x, y in zip(again, solo_a))


def test_bypass_speeds_return_todays_outputs_without_a_stretch_in_the_chain(monkeypatch):
    import sopro_b200.output as output_mod

    tts, ref, text = _api()
    kw = dict(ref=ref, max_frames=16, min_gen_frames=10 ** 9)
    texts = [text, "5 9"]
    base = tts.synthesize(text, seed=3, **kw)
    base_b = tts.synthesize_batch(texts, seeds=[1, 2], **kw)
    base_s = list(tts.stream(text, seed=3, **kw))

    def boom(*a, **k):
        raise AssertionError("the time-stretch ran on a bypass speed")

    monkeypatch.setattr(output_mod, "stretch", boom)
    monkeypatch.setattr(tts._stretch_pool, "checkout", boom)
    for speed in (None, 1.0, 1, 1 + 0.4 / 65536):
        assert torch.equal(tts.synthesize(text, seed=3, speed=speed, **kw), base)
        assert all(torch.equal(a, b) for a, b in zip(tts.synthesize_batch(texts, seeds=[1, 2], speed=speed, **kw), base_b))
        got = list(tts.stream(text, seed=3, speed=speed, **kw))
        assert len(got) == len(base_s) and all(torch.equal(a, b) for a, b in zip(got, base_s))


def test_refused_speed_raises_before_the_rng_moves():
    tts, ref, text = _api()
    for speed in (0.0, -1.0, float("nan"), float("inf"), 4.5, True, "1.5"):
        before = torch.get_rng_state()
        with pytest.raises(ValueError):
            tts.synthesize(text, ref=ref, max_frames=8, speed=speed)
        with pytest.raises(ValueError):
            tts.synthesize_batch([text], ref=ref, max_frames=8, speed=speed)
        with pytest.raises(ValueError):
            tts.stream(text, ref=ref, max_frames=8, speed=speed)
        assert torch.equal(before, torch.get_rng_state())
