"""GPU: dialogue synthesis -- the join with a pause per gap and a gain per span against its fp32 replay
(oracle/dialogue_oracle.py) bit for bit; synthesize_dialogue against synthesize_long for one turn and against its
segments for a script of several voices; per-turn levelling against normalize_loudness of each turn's own join; and
stream_dialogue against the dialogue join of stream_batch's rows."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import dialogue_oracle as DO
from oracle import longform_oracle as O

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)


def _bits(t):
    return t.reshape(-1).cpu().numpy().view(np.uint32)


def _c_join(rows, ext, P):
    """sopro_longform_join itself, through the C-ABI."""
    from sopro_b200 import _lib

    ext = np.ascontiguousarray(np.asarray(ext, dtype=np.int64).reshape(-1, 2))
    N = O.join([np.zeros(int(r.numel()), np.float32) for r in rows], ext.tolist(), P).size
    y = torch.empty(N, dtype=torch.float32, device="cuda")
    n = len(rows)
    src = (C.c_void_p * n)(*[r.data_ptr() if r.numel() else None for r in rows])
    lens = (C.c_int64 * n)(*[int(r.numel()) for r in rows])
    _lib.check_arg(_lib.load().sopro_longform_join(src, n, lens, ext.ctypes.data, P, y.data_ptr() if N else None, N,
                                                   _lib.stream_ptr(y.device)))
    return y


def test_join_gaps_replays_the_oracle_bit_for_bit():
    from sopro_b200.longform import gap_pauses, join_gaps

    g = torch.Generator().manual_seed(4)
    lens = [40000, 25000, 0, 31000, 900, 333, 12, 1, 5000, 7000, 2]
    rows = [torch.randn(n, generator=g).cuda() for n in lens]
    ext = np.array([(100, 39000), (0, 25000), (0, 0), (7, 7), (0, 900), (20, 300), (0, 12), (0, 1), (4000, 4479),
                    (10, 6000), (0, 2)])
    turn_of = [0, 0, 0, 1, 1, 1, 2, 2, 3, 3, 3]
    host = [r.cpu().numpy() for r in rows]
    gains = torch.tensor([0.5, 1.0, 3.0, 2.0, 1e-4, 7.3e-4, 1.0, 0.25, 1.5, 9.9e-4, 1.0], device="cuda")
    for P, TP in ((0, 0), (6000, 12000), (48000, 0), (0, 48000), (1, 48000)):
        pauses = gap_pauses(ext, P, turn_of, TP)
        assert pauses == DO.gaps(ext.tolist(), turn_of, P, TP)
        for gain in (None, gains):
            got = join_gaps(rows, ext, pauses, gain)
            want = DO.join(host, ext.tolist(), pauses, None if gain is None else gain.cpu().numpy())
            assert got.shape == (1, 1, want.size) and np.array_equal(_bits(got), want.view(np.uint32)), (P, TP)
        # uniform pauses and no gain: sopro_longform_join bit for bit
        uni = join_gaps(rows, ext, gap_pauses(ext, P), None)
        assert np.array_equal(_bits(uni), _bits(_c_join(rows, ext, P)))
    # more than one launch of 64 segments, pauses that vary gap by gap, every gain distinct
    many = [rows[i % 2] for i in range(150)]
    e = np.array([(i * 10, i * 10 + 400 + 3 * i) for i in range(150)])
    pauses = [(37 * m) % 48001 for m in range(149)]
    gm = torch.rand(150, generator=g).cuda()
    want = DO.join([r.cpu().numpy() for r in many], e.tolist(), pauses, gm.cpu().numpy())
    assert np.array_equal(_bits(join_gaps(many, e, pauses, gm)), want.view(np.uint32))
    # nothing to join, and refusals before any launch
    assert join_gaps(rows[:2], np.zeros((2, 2), np.int64), []).shape == (1, 1, 0)
    for bad in ([48001], [-1], [1, 2], []):  # two spans: one pause in [0, 48000]
        with pytest.raises(ValueError):
            join_gaps(rows[:2], ext[:2], bad)
    with pytest.raises(ValueError):
        join_gaps(rows[:2], ext[:2], [5], torch.ones(3, device="cuda"))


# ---- through the public API (tests/test_stream_batch_gpu.py's checkpoint: ragged lengths, three voices)

TEXT = "3 7 11 15. 5 9 13 17 21! 4 8?\n\n6 2 10 12 14 16 18 20 22 24, 26 28 30. 1"
FRAMES = 40
KW = dict(max_frames=FRAMES, min_gen_frames=3, max_tokens=7)


def _api():
    from tests.test_stream_batch_gpu import _tts

    return _tts()


def _script(refs):
    a, b, c = refs
    return [(a, "3 7 11 15. 5 9 13 17 21!"), (b, "4 8? 6 2 10 12 14."), (c, "16 18 20."),
            (c, "22 24, 26 28 30. 1 5"), (a, "9 13."), (b, "2 4 6 8 10 12 14 16 18.")]


@pytest.mark.parametrize("chain", (dict(), dict(speed=1.25), dict(sample_rate=16000), dict(watermark=0xC0FFEE),
                                   dict(speed=0.8, sample_rate=48000, watermark=7)))
def test_one_turn_equals_synthesize_long(chain):
    tts, refs = _api()
    got = tts.synthesize_dialogue([(refs[0], TEXT)], seed=40, **KW, **chain)
    want = tts.synthesize_long(TEXT, ref=refs[0], seed=40, **KW, **chain)
    assert got.shape == want.shape and torch.equal(got, want)


def test_one_turn_levelled_and_with_words_equals_synthesize_long():
    tts, refs = _api()
    got = tts.synthesize_dialogue([(refs[1], TEXT)], seed=9, loudness=-16.0, **KW)
    want = tts.synthesize_long(TEXT, ref=refs[1], seed=9, loudness=-16.0, **KW)
    assert got.shape == want.shape and torch.equal(got, want)
    for chain in (dict(), dict(speed=1.25)):
        wav, words = tts.synthesize_dialogue([(refs[1], TEXT)], seed=9, word_timestamps=True, **KW, **chain)
        wl, wwords = tts.synthesize_long(TEXT, ref=refs[1], seed=9, word_timestamps=True, **KW, **chain)
        assert torch.equal(wav, wl) and len(words) == 1 and words[0] == wwords


def _segment_audio(tts, voice, seg, seed):
    """synthesize(segment) trimmed to its extent and faded, as the join places it."""
    from sopro_b200.longform import speech_extents

    w = tts.synthesize(seg, ref=voice, seed=seed, max_frames=FRAMES, min_gen_frames=3)
    if w.numel() == 0:
        return np.zeros(0, np.float32)
    e = speech_extents(w).cpu().numpy()[0]
    return O.join([w.reshape(-1).cpu().numpy()], [tuple(e)], 0)


def test_script_of_three_voices_is_its_segments_joined_with_the_planned_gaps():
    from sopro_b200 import dialogue as D
    from sopro_b200.longform import pause_samples

    tts, refs = _api()
    script = _script(refs)
    assert script[2][0] is script[3][0]  # consecutive turns by the same voice object
    seed, P, TP = 100, pause_samples(200), pause_samples(700)
    wav, words = tts.synthesize_dialogue(script, seed=seed, pause_ms=200, turn_pause_ms=700, word_timestamps=True, **KW)
    y = wav.reshape(-1).cpu().numpy()
    segs, turn_of, voice_of = D.plan(script, tts.tokenizer, KW["max_tokens"])
    assert len(set(turn_of)) == 6 and len(segs) > 6
    parts = [_segment_audio(tts, voice_of[k], s, seed + k) for k, s in enumerate(segs)]
    o, prev, placed = 0, None, 0
    starts = {}
    for k, p in enumerate(parts):
        if p.size == 0:
            continue
        if prev is not None:
            gap = TP if turn_of[k] != prev else P
            assert not y[o: o + gap].any(), k  # the planned zeros
            o += gap
        starts.setdefault(turn_of[k], o)
        assert np.array_equal(y[o: o + p.size].view(np.uint32), p.view(np.uint32)), k
        o, prev, placed = o + p.size, turn_of[k], placed + 1
    assert o == y.size and placed >= 6
    # each turn's words are synthesize_long's for that turn alone, shifted by the turn's start
    k0 = 0
    for j, (voice, text) in enumerate(script):
        n = turn_of.count(j)
        _w, solo = tts.synthesize_long(text, ref=voice, seed=seed + k0, pause_ms=200, word_timestamps=True, **KW)
        k0 += n
        assert len(words[j]) == len(solo)
        last_empty = parts[k0 - 1].size == 0  # then the trailing words sit at the next turn's start instead
        for a, b in zip(words[j], solo):
            assert (a.word, a.char_start, a.char_end) == (b.word, b.char_start, b.char_end)
            if not last_empty:
                assert abs(a.start - (b.start + starts[j] / 24000)) < 1e-9 and abs(a.end - (b.end + starts[j] / 24000)) < 1e-9
    print(f"{len(segs)} segments, {placed} spans, {y.size} samples")


def test_levelling_brings_each_turn_to_the_target():
    from sopro_b200 import dialogue as D
    from sopro_b200.loudness import measure_loudness, normalize_loudness
    from sopro_b200.longform import gap_pauses, join_gaps, pause_samples

    tts, refs = _api()
    script = _script(refs)
    T, seed = -16.0, 5
    got = tts.synthesize_dialogue(script, seed=seed, loudness=T, **KW).reshape(-1)
    raw = tts.synthesize_dialogue(script, seed=seed, **KW).reshape(-1)
    assert got.shape == raw.shape
    segs, turn_of, voice_of = D.plan(script, tts.tokenizer, KW["max_tokens"])
    # the turns' own joins, from the same segments (synthesize equals the batch rows, seeds seed + k)
    from sopro_b200.longform import speech_extents

    rows = [tts.synthesize(s, ref=voice_of[k], seed=seed + k, max_frames=FRAMES, min_gen_frames=3).reshape(-1)
            for k, s in enumerate(segs)]
    ext = np.stack([speech_extents(r).cpu().numpy()[0] if r.numel() else np.zeros(2, np.int64) for r in rows])
    P, TP = pause_samples(250), pause_samples(500)
    pauses = gap_pauses(ext, P, turn_of, TP)
    starts, _after = D.turn_placement(ext, turn_of, len(script), pauses)
    ceiling = np.float32(10 ** (-1 / 20))
    levels = []
    for j, idx in enumerate(D.turn_segments(turn_of, len(script))):
        solo = join_gaps([rows[k] for k in idx], ext[idx], gap_pauses(ext[idx], P))
        n = solo.numel()
        region = got[starts[j]: starts[j] + n]
        want, g = normalize_loudness(solo, 24000, T, return_gain=True)
        assert torch.equal(region, want.reshape(-1)), j
        assert torch.equal(raw[starts[j]: starts[j] + n], solo.reshape(-1)), j
        L0 = float(measure_loudness(solo, 24000))
        levels.append(L0)
        peak = float(solo.abs().max())
        if 10 ** ((T - L0) / 20) * peak < float(ceiling) * (1 - 1e-6):
            assert abs(float(measure_loudness(region, 24000)) - T) < 1e-4, j
        else:
            assert float(region.abs().max()) <= ceiling, j
    print("raw turn levels (LUFS):", [round(v, 2) for v in levels])


def _streamed_rows(tts, segs, voice_of, seed, chunk_frames):
    rows = [[] for _ in segs]
    for i, w, _last in tts.stream_batch(segs, ref=list(voice_of), seeds=[seed + k for k in range(len(segs))],
                                        chunk_frames=chunk_frames, max_frames=FRAMES, min_gen_frames=3):
        rows[i].append(w)
    return [torch.cat(r, dim=1).reshape(-1) for r in rows]


@pytest.mark.parametrize("chain", (dict(), dict(speed=1.25), dict(sample_rate=16000)))
def test_stream_dialogue_equals_the_dialogue_join_of_stream_batch_rows(monkeypatch, chain):
    import sopro_b200.longform as LF
    from sopro_b200 import dialogue as D
    from sopro_b200.output import OutputChain

    tts, refs = _api()
    monkeypatch.setattr(LF, "SEGMENT_GROUP", 2)  # several groups, two slots reused
    script = _script(refs)
    items = list(tts.stream_dialogue(script, seed=40, chunk_frames=6, pause_ms=100, turn_pause_ms=600, **KW, **chain))
    for y in items:
        assert y.dim() == 2 and y.shape[0] == 1 and y.shape[1] > 0
    got = torch.cat(items, dim=1)
    segs, turn_of, voice_of = D.plan(script, tts.tokenizer, KW["max_tokens"])
    rows = _streamed_rows(tts, segs, voice_of, 40, 6)
    for r in rows:  # stream_long's condition, so that the comparison is not vacuous
        if r.numel() >= O.FRAME:
            assert O.frame_db(r.cpu().numpy()).max() <= 0.0
    ext = torch.cat([LF.speech_extents(r) if r.numel() else torch.zeros(1, 2, dtype=torch.int64, device="cuda")
                     for r in rows]).cpu().numpy()
    want = LF.join_gaps(rows, ext, LF.gap_pauses(ext, LF.pause_samples(100), turn_of, LF.pause_samples(600)))
    want, _ = OutputChain(tts, chain.get("sample_rate"), chain.get("speed"))(want)
    assert got.shape[1] == want.shape[-1] and torch.equal(got.reshape(-1), want.reshape(-1))


def test_closing_stream_dialogue_early_releases_its_state(monkeypatch):
    import sopro_b200.longform as LF

    tts, refs = _api()
    monkeypatch.setattr(LF, "SEGMENT_GROUP", 2)
    script = _script(refs)
    fresh = torch.cat(list(tts.stream_dialogue(script, seed=3, speed=1.25, **KW)), dim=1)
    gen = tts.stream_dialogue(script, seed=3, speed=1.25, **KW)
    next(gen)
    gen.close()
    assert not tts.model._sessions_busy
    assert tts._join_pool._idle
    again = torch.cat(list(tts.stream_dialogue(script, seed=3, speed=1.25, **KW)), dim=1)
    assert torch.equal(again, fresh)


def test_refusals_leave_the_generator_untouched():
    tts, refs = _api()
    before = torch.get_rng_state()
    for turns, kw in (([(refs[0], "1 2.")], dict(turn_pause_ms=-5)), ([], {}), ([(refs[0], " ")], {}),
                      ([(refs[0], "1 2.")], dict(loudness=5.0))):
        with pytest.raises((ValueError, TypeError)):
            tts.synthesize_dialogue(turns, **KW, **kw)
    assert torch.equal(before, torch.get_rng_state())


@pytest.mark.parametrize("chain", (dict(speed=0.8), dict(speed=1.25), dict(sample_rate=16000), dict(sample_rate=48000)))
def test_levelling_happens_before_the_chain(chain):
    """The chain runs on the levelled 24 kHz passage, with no loudness stage of its own, so a stretch or a resample
    moves the measured level; the shifts are printed (DESIGN.md §5r records them)."""
    from sopro_b200.loudness import measure_loudness
    from sopro_b200.output import OutputChain

    tts, refs = _api()
    T = -16.0
    base = tts.synthesize_dialogue([(refs[0], TEXT)], seed=40, loudness=T, **KW)
    got = tts.synthesize_dialogue([(refs[0], TEXT)], seed=40, loudness=T, **KW, **chain)
    want, _ = OutputChain(tts, chain.get("sample_rate"), chain.get("speed"))(base)
    assert torch.equal(got, want)
    L0 = float(measure_loudness(base, 24000))
    L = float(measure_loudness(got, chain.get("sample_rate", 24000)))
    print(f"{chain}: {L0:.4f} LUFS at 24 kHz, {L:.4f} LUFS after the chain, shift {L - L0:+.4f} LU")
    assert abs(L0 - T) < 1e-4
