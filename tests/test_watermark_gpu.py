"""GPU: the watermark kernels (csrc/watermark.cu through sopro_b200/watermark.py) against the float64 oracle
(oracle/watermark_oracle.py) -- embed within a derived fp32 bound, silent blocks bit-equal, ragged batches and stream
chunkings bit-equal to the rows alone, detection scores and offsets -- and `watermark=` through the public API."""
import numpy as np
import pytest
import torch

from oracle import watermark_oracle as O
from tests.test_watermark_cpu import mimi_rows, speech_like

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
KEY = 0xC0FFEE
SR = 24000


def _signal(n, seed):
    """fp32 [n] on the device: speech-like, with one silent stretch (the blocks there and beside it get g = 0)."""
    if n == 0:
        return torch.zeros(0, device="cuda")
    x = speech_like(n, seed) if seed % 3 else mimi_rows(1, n)[0] * (0.2 + 0.1 * (seed % 5))
    if n > 3000:
        x[n // 3: n // 3 + 1000] = 0.0
    return torch.tensor(x, dtype=torch.float32, device="cuda")


LENGTHS = (0, 1, 239, 240, 241, 480, 8191, 8193, 24000 * 3 + 17, 24000 * 10)


def test_embed_matches_the_float64_oracle_within_the_fp32_bound_and_silent_blocks_are_bit_equal():
    """|y - y64| <= 2^-24 (|y64| + 3 |g p|) per sample: the fma rounds once, g and p are each rounded once to fp32, the
    block sums differ from the oracle's only in double rounding.  Where g = 0 the input comes back bit for bit."""
    from sopro_b200.watermark import embed_watermark, watermark_pattern

    p32 = watermark_pattern(KEY).astype(np.float64)
    for i, n in enumerate(LENGTHS):
        x = _signal(n, i)
        y = embed_watermark(x, KEY).cpu().numpy().astype(np.float64)
        xn = x.cpu().numpy().astype(np.float64)
        want = O.embed(xn, p32)
        gp = np.repeat(O.gains(xn), O.BLOCK)[:n] * p32[np.arange(n) % O.P]
        assert (np.abs(y - want) <= 2.0 ** -24 * (np.abs(want) + 3 * np.abs(gp)) + 1e-30).all(), n
        silent = np.repeat(O.gains(xn) == 0, O.BLOCK)[:n]
        assert np.array_equal(y[silent].view(np.uint64), xn[silent].view(np.uint64)), n
        if n > 240:
            assert silent[:240].all() and not silent.all()


@pytest.mark.parametrize("B", (1, 7, 64))
def test_ragged_batch_equals_the_rows_alone(B):
    from sopro_b200.watermark import embed_watermark

    rng = np.random.default_rng(B)
    lens = [int(v) for v in rng.integers(0, 5 * SR, B)]
    lens[0] = 5 * SR
    x = torch.full((B, max(lens)), float("nan"), device="cuda")
    for b, n in enumerate(lens):
        x[b, :n] = _signal(n, b)
    y = embed_watermark(x, KEY, lens=lens)
    for b, n in enumerate(lens):
        assert torch.equal(y[b, :n], embed_watermark(x[b, :n].clone(), KEY)), b
        assert not y[b, n:].any()
    if B == 7:  # the same rows as a [B, 1, L] batch without lens
        full = torch.stack([_signal(5 * SR, b) for b in range(B)]).unsqueeze(1)
        yf = embed_watermark(full, KEY)
        assert yf.shape == full.shape
        assert all(torch.equal(yf[b, 0], embed_watermark(full[b, 0], KEY)) for b in range(B))


@pytest.mark.parametrize("push", (1, 239, 240, 241, 11520, "random"))
def test_stream_chunks_concatenate_to_the_one_shot_result(push):
    from sopro_b200.watermark import WatermarkStream, embed_watermark

    rng = np.random.default_rng(3)
    for n in (0, 239, 240, 9 * 240 + 5, 24000 * 2 + 123):
        x = _signal(n, n % 7)
        want = embed_watermark(x, KEY)
        st = WatermarkStream(1 << 16, 0, KEY)
        parts, i = [], 0
        while i < n:
            k = int(rng.integers(1, 3000)) if push == "random" else push
            if push == "random" and rng.random() < 0.1:
                k = 0
            parts.append(st.push(x[i: i + k]))
            i += k
        parts.append(st.finish())
        assert all(p.numel() % 240 == 0 for p in parts[:-1]) and parts[-1].numel() < 240
        assert torch.equal(torch.cat(parts), want), (push, n)
        st.reset(KEY + 1)  # one state serves the next utterance with another key
        got = torch.cat([st.push(x[: n // 2]), st.push(x[n // 2:]), st.finish()])
        assert torch.equal(got, embed_watermark(x, KEY + 1))
        st.close()


def test_stream_refuses_oversized_pushes_and_pushes_after_finish():
    from sopro_b200 import _lib
    from sopro_b200.watermark import WatermarkStream

    st = WatermarkStream(480, 0)
    with pytest.raises(_lib.SoproError):
        st.ready(1)  # no key yet
    st.reset(1)
    with pytest.raises(ValueError):
        st.push(torch.zeros(481, device="cuda"))
    assert st.push(torch.ones(300, device="cuda")).numel() == 240
    assert st.finish().numel() == 60
    with pytest.raises(_lib.SoproError):
        st.push(torch.ones(3, device="cuda"))
    st.close()


def test_detect_matches_the_float64_oracle_and_ragged_equals_alone():
    from sopro_b200.watermark import THRESHOLD, detect_watermark, embed_watermark, watermark_pattern

    p32 = watermark_pattern(KEY).astype(np.float64)
    rng = np.random.default_rng(9)
    lens, rows = [], []
    for i in range(12):
        n = int(rng.integers(3 * SR, 8 * SR))
        x = _signal(n + 30000, i)
        y = embed_watermark(x, KEY) if i % 2 == 0 else x  # every other row unmarked
        s = int(rng.integers(0, 30000))
        rows.append(y[s: s + n])
        lens.append(n)
    lens.append(0)
    rows.append(torch.zeros(0, device="cuda"))
    X = torch.zeros((len(rows), max(lens)), device="cuda")
    for b, r in enumerate(rows):
        X[b, : lens[b]] = r
    det = detect_watermark(X, SR, KEY, lens=lens)
    for b, r in enumerate(rows):
        want_s, want_o = O.detect(r.cpu().numpy().astype(np.float64), p32)
        got_s, got_o = float(det.score[b]), int(det.offset[b])
        assert abs(got_s - want_s) <= 1e-4 * max(abs(want_s), 1e-3), (b, got_s, want_s)
        assert bool(det.detected[b]) == (got_s >= THRESHOLD)
        if b % 2 == 0 and lens[b]:
            assert got_o == want_o and got_s >= THRESHOLD, (b, got_s)
        one = detect_watermark(r, SR, KEY)
        assert torch.equal(one.score, det.score[b]) and torch.equal(one.offset, det.offset[b])


def test_detect_at_other_rates_resamples_first():
    from sopro_b200.resample import Resampler
    from sopro_b200.watermark import detect_watermark, embed_watermark

    y = embed_watermark(_signal(5 * SR, 4), KEY)
    for sr in (8000, 16000, 22050, 44100, 48000):
        z = Resampler(SR, sr, 0)(y)
        d = detect_watermark(z, sr, KEY)
        assert bool(d.detected) and int(d.offset) == 0, (sr, float(d.score))
        assert not bool(detect_watermark(z, sr, KEY + 1).detected)


# ---- through the public API (the e2e fixture of test_e2e_gpu.py)

def _api():
    from tests.cases import e2e_inputs
    from tests.test_e2e_gpu import TEXT, _tts

    tts, _ = _tts()
    _cfg, _sd, inp = e2e_inputs()
    return tts, tts.prepare_reference(ref_tokens_tq=inp["ref_tokens_tq"]), TEXT


KW = dict(max_frames=60, min_gen_frames=10 ** 9)


def test_no_watermark_runs_nothing_on_every_entry_point(monkeypatch):
    import sopro_b200.output as output_mod

    tts, ref, text = _api()
    texts = [text, "5 9"]
    base = tts.synthesize(text, ref=ref, seed=3, **KW)
    base_b = tts.synthesize_batch(texts, ref=ref, seeds=[1, 2], **KW)
    base_l = tts.synthesize_long(text, ref=ref, max_tokens=7, seed=4, max_frames=20, min_gen_frames=10 ** 9)
    base_s = torch.cat(list(tts.stream(text, ref=ref, seed=5, chunk_frames=6, **KW)), dim=1)

    def boom(*a, **k):
        raise AssertionError("the watermark stage ran without a key")

    monkeypatch.setattr(output_mod, "embed_watermark", boom)
    monkeypatch.setattr(tts._watermark_pool, "checkout", boom)
    assert torch.equal(tts.synthesize(text, ref=ref, seed=3, watermark=None, **KW), base)
    assert all(torch.equal(a, b) for a, b in zip(tts.synthesize_batch(texts, ref=ref, seeds=[1, 2], watermark=None, **KW),
                                                 base_b))
    assert torch.equal(tts.synthesize_long(text, ref=ref, max_tokens=7, seed=4, max_frames=20, min_gen_frames=10 ** 9,
                                           watermark=None), base_l)
    assert torch.equal(torch.cat(list(tts.stream(text, ref=ref, seed=5, chunk_frames=6, watermark=None, **KW)), dim=1),
                       base_s)
    with pytest.raises(AssertionError):
        tts.synthesize(text, ref=ref, seed=3, watermark=1, **KW)


def test_refused_keys_raise_before_the_rng_moves():
    tts, ref, text = _api()
    for key in (-1, 2 ** 32, True, 1.0, "7"):
        before = torch.get_rng_state()
        for call in (lambda: tts.synthesize(text, ref=ref, max_frames=8, watermark=key),
                     lambda: tts.synthesize_batch([text], ref=ref, max_frames=8, watermark=key),
                     lambda: tts.synthesize_long(text, ref=ref, max_frames=8, watermark=key),
                     lambda: tts.stream(text, ref=ref, max_frames=8, watermark=key)):
            with pytest.raises(ValueError):
                call()
        assert torch.equal(before, torch.get_rng_state())


@pytest.mark.parametrize("sr", (8000, 24000, 48000))
def test_synthesize_is_detected_with_its_key_only(sr):
    from sopro_b200 import detect_watermark

    tts, ref, text = _api()
    for extra in ({}, {"speed": 1.25}, {"loudness": -16.0}):
        wav = tts.synthesize(text, ref=ref, seed=7, sample_rate=sr, watermark=KEY, **extra, **KW)
        d = detect_watermark(wav.reshape(-1), sr, KEY)
        wrong = detect_watermark(wav.reshape(-1), sr, KEY + 1)
        plain = detect_watermark(tts.synthesize(text, ref=ref, seed=7, sample_rate=sr, **extra, **KW).reshape(-1), sr, KEY)
        print(f"{sr} Hz {extra}: score {float(d.score):.2f}, wrong key {float(wrong.score):.2f}, "
              f"unmarked {float(plain.score):.2f}")
        assert bool(d.detected) and int(d.offset) == 0
        assert not bool(wrong.detected) and not bool(plain.detected)


def test_synthesize_batch_rows_equal_synthesize():
    tts, ref, text = _api()
    texts = [text, " ".join(str(i) for i in range(3, 40, 3)), "5 9"]
    kw = dict(ref=ref, watermark=KEY, speed=1.1, sample_rate=16000, **KW)
    wavs = tts.synthesize_batch(texts, seeds=[1, 2, 3], **kw)
    for t, s, w in zip(texts, [1, 2, 3], wavs):
        assert torch.equal(w, tts.synthesize(t, seed=s, **kw))


def test_synthesize_long_and_best_of_are_detected_and_keep_their_word_timings():
    from sopro_b200 import detect_watermark

    tts, ref, text = _api()
    kw = dict(ref=ref, word_timestamps=True, min_gen_frames=10 ** 9)
    for call in (lambda **k: tts.synthesize_long(text, max_tokens=7, seed=2, max_frames=30, **kw, **k),
                 lambda **k: tts.synthesize(text, seed=2, best_of=4, max_frames=60, **kw, **k)):
        wav, words = call(watermark=KEY)
        _wav0, words0 = call()
        assert words == words0
        d = detect_watermark(wav.reshape(-1), SR, KEY)
        assert bool(d.detected), float(d.score)


def test_stream_concatenates_to_synthesize():
    """One chunk covering the utterance: stream() == synthesize() with the mark, bit for bit.  Chunked: the mark is the
    one-shot embed of the unmarked stream's 24 kHz audio, bit for bit."""
    from sopro_b200.watermark import embed_watermark

    tts, ref, text = _api()
    kw = dict(ref=ref, seed=9, max_frames=25, min_gen_frames=10 ** 9)
    tts.codec.engine.set_precision("fp32")  # the mode in which the stream decoder equals the one-shot decode
    try:
        full = tts.synthesize(text, watermark=KEY, **kw)
        one = torch.cat(list(tts.stream(text, chunk_frames=64, watermark=KEY, **kw)), dim=1)
        assert torch.equal(one.reshape(-1), full.reshape(-1))
        fast = torch.cat(list(tts.stream(text, chunk_frames=64, watermark=KEY, speed=1.25, sample_rate=48000, **kw)), dim=1)
        want = tts.synthesize(text, watermark=KEY, speed=1.25, sample_rate=48000, **kw)
        assert torch.equal(fast.reshape(-1), want.reshape(-1))
    finally:
        tts.codec.engine.set_precision("bf16_tc")
    plain = torch.cat(list(tts.stream(text, chunk_frames=6, **kw)), dim=1)
    chunks = list(tts.stream(text, chunk_frames=6, watermark=KEY, **kw))
    assert torch.equal(torch.cat(chunks, dim=1).reshape(-1), embed_watermark(plain.reshape(-1), KEY))


def test_null_over_unmarked_synthesize_batch_rows():
    """512 unmarked rows of synthesize_batch (8 batches of 64), each scored against 4 keys: no detection."""
    from sopro_b200 import detect_watermark

    tts, ref, _text = _api()
    rng = np.random.default_rng(1)
    texts = [" ".join(str(int(v)) for v in rng.integers(1, 999, int(rng.integers(3, 25)))) for _ in range(512)]
    wavs = []
    for b0 in range(0, len(texts), 64):
        wavs += tts.synthesize_batch(texts[b0: b0 + 64], ref=ref, seeds=list(range(b0, b0 + 64)), max_frames=60,
                                     min_gen_frames=30)
    lens = [int(w.shape[-1]) for w in wavs]
    X = torch.zeros((len(wavs), max(lens)), device="cuda")
    for b, w in enumerate(wavs):
        X[b, : lens[b]] = w.reshape(-1)
    top = 0.0
    for key in (0, 1, KEY, 2 ** 32 - 1):
        d = detect_watermark(X, SR, key, lens=lens)
        top = max(top, float(d.score.max()))
        assert not bool(d.detected.any())
    print(f"null over {len(wavs)} rows x 4 keys: max score {top:.2f}")
