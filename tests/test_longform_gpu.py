"""GPU: long-form synthesis -- the speech-extents kernel against the float64 oracle (oracle/longform_oracle.py), the join
against the oracle's fp32 replay bit for bit, and `synthesize_long` against its parts: split_text, synthesize_batch /
synthesize per segment, the join, and the existing stretch / resample / loudness chain."""
import numpy as np
import pytest
import torch

from oracle import longform_oracle as O
from oracle import mimi_oracle as MO

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
_CACHE = {}


def _mimi_wav():
    """A real Mimi decode (synthetic checkpoint, seeded codes): 41 frames = 78,720 samples."""
    if "mimi" not in _CACHE:
        from sopro_b200.codec import MimiEngine

        codes = torch.randint(0, 2048, (1, 32, 41), generator=torch.Generator().manual_seed(7))
        _CACHE["mimi"] = MimiEngine(MO.synth_mimi_state_dict(), 0, 32).decode(codes).reshape(-1).float().cpu().numpy()
    return _CACHE["mimi"]


def _rows():
    """(name, fp32 numpy row) pairs: the audio_prep.json recipes at 24 kHz, noise, silence, a Mimi decode, a loud +
    quiet + silent row, bursts between silences, and rows at the edges of the length rules."""
    from tests.golden.make_audio_golden import CASES, signal

    g = np.random.default_rng(11)
    out = [(name, signal(24000, n, lo, hi, floor, i)[0].numpy()) for i, (name, _sr, n, lo, hi, floor) in enumerate(CASES)]
    out.append(("noise", (0.3 * g.standard_normal(50000)).astype(np.float32)))
    out.append(("silence", np.zeros(40000, dtype=np.float32)))
    m = _mimi_wav()
    out.append(("mimi", m))
    pad = np.zeros(30000, dtype=np.float32)
    out.append(("mimi_padded", np.concatenate([pad, m, pad])))
    x = (0.9 * g.standard_normal(90000)).astype(np.float32)
    x[30000:60000] *= 0.03
    x[60000:] = 0
    out.append(("loud_quiet_silent", x))
    for n in (599, 600, 2399, 2400, 11999, 12000, 12001, 30000):
        y = np.zeros(n, dtype=np.float32)
        k = n // 4
        y[n // 3: n // 3 + k] = (0.5 * g.standard_normal(k)).astype(np.float32)
        out.append((f"burst_{n}", y))
    return out


def _agrees(got, x):
    """The GPU's extent equals the oracle's, or differs only through a frame within 1e-9 dB of the threshold."""
    d = O.extent_detail(x)
    if tuple(got) == (d["start"], d["end"]):
        return True
    assert d["db"] is not None and np.abs(d["db"] - d["thr"]).min() <= 1e-9, (tuple(got), d["start"], d["end"])
    return False


def _batch(rows):
    lens = [r.size for r in rows]
    x = torch.full((len(rows), max(lens)), float("nan"), device="cuda")
    for b, r in enumerate(rows):
        x[b, : r.size] = torch.from_numpy(r).cuda()
    return x, lens


def test_extents_match_the_float64_oracle_alone_and_in_ragged_batches():
    from sopro_b200.longform import speech_extents

    named = _rows()
    rows = [r for _n, r in named]
    exact = 0
    alone = []
    for name, r in named:
        e = speech_extents(torch.from_numpy(r).cuda()).cpu().numpy()
        assert e.shape == (1, 2), name
        exact += _agrees(e[0], r)
        alone.append(e[0])
    alone = np.stack(alone)
    x, lens = _batch(rows)  # NaN padding: a read past lens[b] would show
    got = speech_extents(x, lens=lens).cpu().numpy()
    assert np.array_equal(got, alone)
    perm = list(reversed(range(len(rows))))
    x2, lens2 = _batch([rows[i] for i in perm])
    assert np.array_equal(speech_extents(x2.unsqueeze(1), lens=lens2).cpu().numpy(), alone[perm])
    # 130 rows: two launches
    many = [rows[i % len(rows)] for i in range(130)]
    x3, lens3 = _batch(many)
    assert np.array_equal(speech_extents(x3, lens=lens3).cpu().numpy(), alone[[i % len(rows) for i in range(130)]])
    print(f"{exact} of {len(rows)} extents equal to the oracle's; the rest within 1e-9 dB of the threshold")
    d = dict(zip([n for n, _ in named], alone.tolist()))
    assert d["silence"] == [0, 40000] and d["burst_599"] == [0, 599] and d["burst_2399"] == [0, 2399]
    assert 0 < d["mimi_padded"][0] < 30000 and 30000 + 78720 < d["mimi_padded"][1] < 30000 * 2 + 78720
    assert d["loud_quiet_silent"][0] == 0 and 60000 < d["loud_quiet_silent"][1] <= 61320


def test_extents_refusals():
    from sopro_b200.longform import speech_extents

    x = torch.zeros(2, 100, device="cuda")
    for lens in ([101, 5], [-1, 5]):
        with pytest.raises(ValueError):
            speech_extents(x, lens=lens)
    with pytest.raises(ValueError):
        speech_extents(x, lens=[5])


@pytest.mark.parametrize("pause_ms", (0, 250, 2000, 0.1))
def test_join_replays_the_oracle_bit_for_bit(pause_ms):
    """Rows read in place from several padded chunks and single rows; extents from the GPU plus crafted ones: a span
    shorter than 2F, a span of 1, empty extents (skipped), a segment of no samples."""
    from sopro_b200.longform import join_segments, pause_samples, speech_extents

    g = torch.Generator().manual_seed(3)
    chunk_a = torch.randn(3, 1, 40000, generator=g).cuda()
    chunk_b = torch.randn(2, 1, 25000, generator=g).cuda()
    single = torch.randn(1, 1, 31000, generator=g).cuda()
    empty = torch.zeros(1, 1, 0, device="cuda")
    parts = [chunk_a, chunk_b, single, empty]
    rows = [chunk_a[i, 0] for i in range(3)] + [chunk_b[i, 0] for i in range(2)] + [single[0, 0], empty[0, 0]]
    ext = torch.cat([speech_extents(chunk_a), speech_extents(chunk_b), speech_extents(single),
                     torch.zeros(1, 2, dtype=torch.int64, device="cuda")]).cpu()
    ext[1] = torch.tensor([100, 400])    # 300 samples: F = 150
    ext[3] = torch.tensor([7, 7])        # empty: skipped
    ext[4] = torch.tensor([9, 10])       # one sample: F = 0
    want = O.join([r.cpu().numpy() for r in rows], ext.numpy().tolist(), pause_samples(pause_ms))
    for src in (parts, rows):
        got = join_segments(src, ext.cuda(), pause_ms)
        assert got.shape == (1, 1, want.size) and got.dtype == torch.float32
        assert np.array_equal(got.reshape(-1).cpu().numpy().view(np.uint32), want.view(np.uint32))
    # more than one launch's worth of segments (64), and all-empty extents
    many = [chunk_a[i % 3, 0] for i in range(70)]
    e = torch.tensor([[i * 10, i * 10 + 500 + i] for i in range(70)])
    want = O.join([r.cpu().numpy() for r in many], e.numpy().tolist(), pause_samples(pause_ms))
    got = join_segments(many, e, pause_ms)
    assert np.array_equal(got.reshape(-1).cpu().numpy().view(np.uint32), want.view(np.uint32))
    assert join_segments(rows[:2], torch.zeros(2, 2, dtype=torch.int64), pause_ms).shape == (1, 1, 0)


def test_join_refusals():
    from sopro_b200.longform import join_segments

    rows = [torch.zeros(100, device="cuda"), torch.zeros(50, device="cuda")]
    for ext in ([[0, 101], [0, 5]], [[5, 4], [0, 5]], [[-1, 4], [0, 5]], [[0, 5], [0, 51]]):
        with pytest.raises(ValueError):
            join_segments(rows, ext, 250)
    with pytest.raises(ValueError):
        join_segments(rows, [[0, 5]], 250)
    for bad in (-1, 2001, float("nan"), True):
        with pytest.raises(ValueError):
            join_segments(rows, [[0, 5], [0, 5]], bad)


# ---- through the public API (the e2e fixture of test_e2e_gpu.py)

TEXT = "3 7 11 15. 5 9 13 17 21! 4 8?\n\n6 2 10 12 14 16 18 20 22 24, 26 28 30. 1"
KW = dict(max_frames=16, min_gen_frames=10 ** 9)


def _api():
    from tests.cases import e2e_inputs
    from tests.test_e2e_gpu import _tts

    tts, _ = _tts()
    _cfg, _sd, inp = e2e_inputs()
    return tts, tts.prepare_reference(ref_tokens_tq=inp["ref_tokens_tq"])


def _parts(tts, ref, segs, seeds, pause_ms=250):
    """The join of synthesize_batch's waveforms at 24 kHz, with their extents found one row at a time."""
    from sopro_b200.longform import join_segments, speech_extents

    wavs = tts.synthesize_batch(segs, ref=ref, seeds=seeds, **KW)
    ext = torch.cat([speech_extents(w) if w.numel() else torch.zeros(1, 2, dtype=torch.int64, device="cuda") for w in wavs])
    return wavs, ext, join_segments(wavs, ext, pause_ms)


@pytest.mark.parametrize("mode", ("fp32", "bf16_tc"))
def test_synthesize_long_equals_its_parts(mode):
    from sopro_b200.longform import pause_samples, split_text

    tts, ref = _api()
    eng = tts.codec.engine
    segs = split_text(TEXT, tts.tokenizer, 7)
    assert len(segs) >= 5
    eng.set_precision(mode)
    try:
        got = tts.synthesize_long(TEXT, ref=ref, max_tokens=7, seed=40, **KW)
        wavs, ext, want = _parts(tts, ref, segs, [40 + i for i in range(len(segs))])
        singles = [tts.synthesize(s, ref=ref, seed=40 + i, **KW) for i, s in enumerate(segs)]
        got2 = tts.synthesize_long(TEXT, ref=ref, max_tokens=7, seed=40, pause_ms=0, **KW)
    finally:
        eng.set_precision("bf16_tc")
    assert torch.equal(got, want)
    for w, s in zip(wavs, singles):
        assert torch.equal(w, s)
    e = ext.cpu().numpy()
    replay = O.join([w.reshape(-1).cpu().numpy() for w in wavs], e.tolist(), pause_samples(250))
    assert np.array_equal(got.reshape(-1).cpu().numpy().view(np.uint32), replay.view(np.uint32))
    assert got2.shape[-1] == got.shape[-1] - (len(segs) - 1) * 6000
    print(f"{mode}: {len(segs)} segments, extents {e.tolist()}, {got.shape[-1]} samples")


def test_grouping_does_not_change_the_result(monkeypatch):
    import sopro_b200.longform as LF

    tts, ref = _api()
    base = tts.synthesize_long(TEXT, ref=ref, max_tokens=7, seed=3, **KW)
    for group in (1, 2, 4):
        monkeypatch.setattr(LF, "SEGMENT_GROUP", group)
        assert torch.equal(tts.synthesize_long(TEXT, ref=ref, max_tokens=7, seed=3, **KW), base), group


def test_global_generator_is_consumed_like_synthesize_batch(monkeypatch):
    import sopro_b200.longform as LF

    tts, ref = _api()
    segs = LF.split_text(TEXT, tts.tokenizer, 7)
    monkeypatch.setattr(LF, "SEGMENT_GROUP", 2)  # across groups
    torch.manual_seed(17)
    got = tts.synthesize_long(TEXT, ref=ref, max_tokens=7, **KW)
    after = torch.get_rng_state()
    torch.manual_seed(17)
    _wavs, _ext, want = _parts(tts, ref, segs, None)
    assert torch.equal(got, want)
    assert torch.equal(after, torch.get_rng_state())


@pytest.mark.parametrize("speed,sr,target", ((1.25, None, None), (None, 48000, None), (None, None, -16.0),
                                             (0.8, 16000, -23.0)))
def test_post_chain_is_the_existing_chain_on_the_joined_row(speed, sr, target):
    from sopro_b200.loudness import normalize_loudness
    from sopro_b200.resample import Resampler
    from sopro_b200.stretch import stretch

    tts, ref = _api()
    base = tts.synthesize_long(TEXT, ref=ref, max_tokens=7, seed=8, **KW)
    got = tts.synthesize_long(TEXT, ref=ref, max_tokens=7, seed=8, speed=speed, sample_rate=sr, loudness=target, **KW)
    want = base
    if speed is not None:
        want = stretch(want, speed)
    if sr is not None:
        want = Resampler(24000, sr, want.device)(want)
    if target is not None:
        want = normalize_loudness(want, sr or 24000, target)
    assert torch.equal(got, want)


def test_refused_arguments_raise_before_the_rng_moves():
    tts, ref = _api()
    bad = (dict(pause_ms=-1), dict(pause_ms=2500), dict(pause_ms=float("nan")), dict(pause_ms=True), dict(max_tokens=3),
           dict(max_tokens=10 ** 6), dict(max_tokens=8.0), dict(speed=0.1), dict(sample_rate=1000), dict(loudness=3.0))
    for kw in bad:
        before = torch.get_rng_state()
        with pytest.raises(ValueError):
            tts.synthesize_long(TEXT, ref=ref, **KW, **kw)
        assert torch.equal(before, torch.get_rng_state()), kw
    for text in ("", " \n\n  "):
        before = torch.get_rng_state()
        with pytest.raises(ValueError):
            tts.synthesize_long(text, ref=ref, **KW)
        assert torch.equal(before, torch.get_rng_state())
