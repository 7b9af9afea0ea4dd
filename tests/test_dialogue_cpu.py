"""CPU: dialogue synthesis's host side (sopro_b200/dialogue.py) -- the script's segment plan and seeds, the gap plan
against its definition (oracle/dialogue_oracle.py), where each turn sits in the passage, the word-timing mapping with
a pause per span, every refusal before any random draw -- and the join oracle's operation order."""
import inspect
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import dialogue_oracle as DO
from oracle import longform_oracle as O
from sopro_b200 import dialogue as D
from sopro_b200 import longform as LF
from sopro_b200 import timestamps as TS
from sopro_b200 import voices
from sopro_b200.config import SoproTTSConfig
from sopro_b200.prefill import PreparedReference
from sopro_b200.tokenizer import IdsTokenizer

IDS = IdsTokenizer(1000)
CFG = SoproTTSConfig()


def _voice(Tr=5, layers=None):
    g = voices.geometry(CFG)
    shape = (1, g["heads"], Tr, g["head_dim"])
    caches = [{"k": torch.zeros(shape), "v": torch.zeros(shape), "key_padding_mask": None}
              for _ in range(g["layers"] if layers is None else layers)]
    return PreparedReference(ref_tokens_btq=torch.zeros((1, Tr, 32), dtype=torch.long), sv_ref=torch.zeros((1, g["sv_dim"])),
                             ref_seq=torch.zeros((1, Tr, g["heads"] * g["head_dim"])), ref_kv_caches=caches)


A, B, C_ = _voice(5), _voice(7), _voice(9)
SCRIPT = [(A, "1 2 3. 4 5 6 7. 8"), (B, "  "), (A, "9 10. 11 12 13 14 15 16."), (A, "17"), (C_, "18 19.\n\n20 21 22.")]


def test_segment_plan_flattens_the_turns_in_order():
    segs, turn_of, voice_of = D.plan(SCRIPT, IDS, 6)
    per_turn = [LF.split_text(t, IDS, 6) for _v, t in SCRIPT]
    assert segs == [s for p in per_turn for s in p]
    assert turn_of == [j for j, p in enumerate(per_turn) for _ in p]
    assert all(voice_of[k] is SCRIPT[turn_of[k]][0] for k in range(len(segs)))
    assert 1 not in turn_of  # the whitespace-only turn speaks nothing
    for j, (_v, text) in enumerate(SCRIPT):
        mine = [s for s, t in zip(segs, turn_of) if t == j]
        pars = [" ".join(p.split()) for p in LF._PARAGRAPH.split(text) if p.split()]
        assert " ".join(mine) == " ".join(pars), j
    assert D.turn_segments(turn_of, len(SCRIPT))[1] == []
    # one voice object for every segment takes synthesize_long's one-voice path; several take the per-segment list
    assert D.segment_voices([A, A, A]) is A
    assert D.segment_voices(voice_of) == voice_of and isinstance(D.segment_voices(voice_of), list)


def _stub_tts(calls):
    """A SoproTTS with no engines: _best_codes records each group and returns no frames, so nothing is decoded."""
    from sopro_b200.model import SoproTTS

    tts = SoproTTS.__new__(SoproTTS)
    tts.device = torch.device("cpu")
    tts._resamplers = {}
    tts.tokenizer = IDS
    tts.cfg = CFG
    tts.model = SimpleNamespace(prefill=SimpleNamespace(max_text_len=2056), device=torch.device("cpu"))

    def best_codes(texts, ref, best_of, *, seeds, trace_out=None, **kw):
        calls.append((list(texts), ref, seeds))
        return [0] * len(texts), None

    tts._best_codes = best_codes
    return tts


@pytest.mark.parametrize("group", (64, 2, 3))
def test_segments_are_seeded_and_voiced_in_script_order(monkeypatch, group):
    calls = []
    tts = _stub_tts(calls)
    monkeypatch.setattr(LF, "SEGMENT_GROUP", group)
    segs, turn_of, voice_of = D.plan(SCRIPT, IDS, 6)
    rows, ext, _f, _T = tts._speak_segments(segs, D.segment_voices(voice_of), 1, seed=100, word_timestamps=False,
                                            max_frames=16)
    assert len(rows) == len(segs) and tuple(ext.shape) == (len(segs), 2)
    assert [t for c in calls for t in c[0]] == segs
    assert [s for c in calls for s in c[2]] == [100 + k for k in range(len(segs))]
    got_voices = [v for c in calls for v in c[1]]
    assert len(got_voices) == len(segs) and all(a is b for a, b in zip(got_voices, voice_of))
    assert all(len(c[0]) <= group for c in calls)
    calls.clear()
    tts._speak_segments(segs[:3], A, 1, seed=None, word_timestamps=False, max_frames=16)
    assert calls[0][1] is A and calls[0][2] is None  # one voice, no seed: synthesize_long's groups exactly


def test_gap_plan_follows_the_turns_of_the_non_empty_spans():
    P, TP = 6000, 12000
    cases = [
        # (extents, turn of each segment)
        ([(0, 9), (0, 9), (0, 9)], [0, 0, 0]),
        ([(0, 9), (0, 9), (0, 9), (0, 9)], [0, 0, 1, 1]),
        # empty segments at a turn's edges: the gap goes to the next non-empty span, by its turn
        ([(3, 3), (0, 9), (0, 0), (0, 9), (4, 4)], [0, 0, 0, 1, 1]),
        ([(0, 9), (5, 5), (0, 0), (0, 9)], [0, 0, 1, 2]),  # turn 1 produces nothing: turn 0 to turn 2 is a turn gap
        ([(0, 9), (0, 0)], [0, 1]),
        ([(0, 0), (0, 0)], [0, 1]),
        ([(0, 9), (0, 9), (0, 9)], [0, 2, 2]),
    ]
    for ext, turns in cases:
        got = LF.gap_pauses(np.array(ext), P, turns, TP)
        assert got == DO.gaps(ext, turns, P, TP), (ext, turns)
    assert LF.gap_pauses(np.array([(0, 9), (0, 9), (0, 9), (0, 9)]), P, [0, 0, 1, 1], TP) == [P, TP, P]
    assert LF.gap_pauses(np.array([(3, 3), (0, 9), (0, 0), (0, 9), (4, 4)]), P, [0, 0, 0, 1, 1], TP) == [TP]
    assert LF.gap_pauses(np.array([(0, 9), (5, 5), (0, 0), (0, 9)]), P, [0, 0, 1, 2], TP) == [TP]
    assert LF.gap_pauses(np.array([(0, 9), (0, 9)]), P) == [P]  # one turn: synthesize_long's uniform pause
    # consecutive turns by the same voice object are still two turns
    script = [(A, "1 2."), (A, "3 4."), (B, "5 6.")]
    _segs, turn_of, _v = D.plan(script, IDS, 64)
    assert LF.gap_pauses(np.array([(0, 9)] * 3), P, turn_of, TP) == [TP, TP]


def test_turn_placement():
    P, TP = 10, 100
    ext = np.array([(0, 50), (5, 5), (0, 30), (0, 0), (10, 30), (0, 40)])
    turn_of = [0, 0, 0, 2, 2, 3]  # turn 1 has no segments, turn 2 starts with an empty one
    pauses = LF.gap_pauses(ext, P, turn_of, TP)
    assert pauses == [P, TP, TP]
    starts, after = D.turn_placement(ext, turn_of, 4, pauses)
    # turn 0: [0, 50) + 10 + [60, 90); + 100 -> turn 2 at 190: [190, 210); + 100 -> turn 3 at 310
    assert starts == [0, 190, 190, 310]
    assert after == [[P, TP], [], [TP], [0]]
    assert sum(int(e - s) for s, e in ext) + sum(pauses) == 310 + 40


def test_long_timings_with_a_pause_per_span_and_a_start():
    """A hand-computed case: two segments of two words, hop 100; spans (100, 700) and (0, 400) after a 50-sample
    start, 30 zeros after the first span; the words follow their first frames."""
    text = "1 2 3 4"
    segs = ["1 2", "3 4"]
    spans = [IDS.encode_with_offsets(s)[1] for s in segs]
    assert [len(s) for s in spans] == [4, 4]  # BOS, two words, EOS
    firsts = [np.array([0, 2, 4, 6]), np.array([0, 1, 3, 4])]
    Ts = [7, 5]
    ext = [(100, 700), (0, 400)]
    got = TS.long_timings(text, segs, spans, firsts, Ts, 100, ext, [30, 999], None, start=50)
    # segment 0: word "1" = frames [2, 4) -> samples [200, 400) - 100 + 50 = [150, 350); "2" = [4, 6) -> [350, 550)
    # segment 1 starts at 50 + 600 + 30 = 680: "3" = frames [1, 3) -> [780, 980); "4" = [3, 4) -> [980, 1080)
    want = [("1", 150, 350, 0, 1), ("2", 350, 550, 2, 3), ("3", 780, 980, 4, 5), ("4", 980, 1080, 6, 7)]
    assert [(w.word, w.start, w.end, w.char_start, w.char_end) for w in got] == \
        [(a, b / 24000, c / 24000, d, e) for a, b, c, d, e in want]
    # an int pause is every span's, and start 0 is synthesize_long's mapping
    u = TS.long_timings(text, segs, spans, firsts, Ts, 100, ext, 30, None)
    assert [(w.start, w.end) for w in u] == [((b - 50) / 24000, (c - 50) / 24000) for _a, b, c, _d, _e in want]
    # a segment with an empty extent sits where the audio continues: after span 0 and its pause
    e2 = TS.long_timings(text, segs, spans, firsts, Ts, 100, [(100, 700), (3, 3)], [77], None, start=50)
    assert [(w.start, w.end) for w in e2[2:]] == [(727 / 24000, 727 / 24000)] * 2
    with pytest.raises(ValueError):
        TS.long_timings(text, segs, spans, firsts, Ts, 100, ext, [30], None)


def _bare_tts():
    """A SoproTTS with no engines at all: a call that got past its checks would fail on the first device step."""
    from sopro_b200.model import SoproTTS

    tts = SoproTTS.__new__(SoproTTS)
    tts._resamplers = {}
    tts.tokenizer = IDS
    tts.cfg = CFG
    tts.model = SimpleNamespace(prefill=SimpleNamespace(max_text_len=2056))
    return tts


def test_refusals_happen_before_any_random_draw():
    tts = _bare_tts()
    good = [(A, "1 2 3."), (B, "4 5.")]
    bad_voice = _voice(layers=1)
    cases = [
        (TypeError, "1 2 3", {}), (TypeError, None, {}), (TypeError, [A, "1 2"], {}), (TypeError, [(A, 5)], {}),
        (TypeError, [("1 2", A)], {}), (TypeError, [(A, "1", "2")], {}), (ValueError, [], {}),
        (ValueError, [(A, ""), (B, "  \n\n ")], {}),
        (ValueError, [(A, "1 2."), (bad_voice, "3.")], {}), (ValueError, [(_voice(Tr=5000), "1.")], {}),
        (ValueError, good, dict(pause_ms=-1)), (ValueError, good, dict(pause_ms=2001)),
        (ValueError, good, dict(turn_pause_ms=float("nan"))), (ValueError, good, dict(turn_pause_ms=True)),
        (ValueError, good, dict(turn_pause_ms=2500)), (ValueError, good, dict(max_tokens=3)),
        (ValueError, good, dict(max_tokens=10 ** 6)), (ValueError, good, dict(sample_rate=3999)),
        (ValueError, good, dict(speed=5.0)), (ValueError, good, dict(watermark=-1)),
    ]
    before = torch.get_rng_state()
    for exc, turns, kw in cases:
        with pytest.raises(exc):
            tts.synthesize_dialogue(turns, **kw)
        with pytest.raises(exc):
            tts.stream_dialogue(turns, **kw)
    for kw in (dict(loudness=1.0), dict(loudness=float("nan")), dict(best_of=0), dict(word_timestamps=1)):
        with pytest.raises((ValueError, TypeError)):
            tts.synthesize_dialogue(good, **kw)
    for kw in (dict(chunk_frames=0), dict(chunk_frames=257)):
        with pytest.raises(ValueError):
            tts.stream_dialogue(good, **kw)
    with pytest.raises(TypeError):
        tts.stream_dialogue(good, chunk_frames=6.0)
    for kw in (dict(loudness=-16.0), dict(best_of=2), dict(word_timestamps=True)):
        with pytest.raises(TypeError):  # not stream_dialogue's arguments
            tts.stream_dialogue(good, **kw)
    assert torch.equal(before, torch.get_rng_state())


def test_signatures():
    from sopro_b200 import SoproTTS

    want = dict(seed=None, pause_ms=250, turn_pause_ms=500, max_frames=400, max_tokens=64, top_p=0.9, temperature=1.05,
                anti_loop=True, style_strength=None, min_gen_frames=None, sample_rate=None, speed=None, watermark=None)
    for fn, extra in ((SoproTTS.synthesize_dialogue, dict(loudness=None, word_timestamps=False, best_of=1)),
                      (SoproTTS.stream_dialogue, dict(chunk_frames=6, nar_context_frames=None))):
        p = inspect.signature(fn).parameters
        for k, v in {**want, **extra}.items():
            assert p[k].default == v and p[k].kind == inspect.Parameter.KEYWORD_ONLY, (fn.__name__, k)
        assert list(p)[1] == "turns" and p["turns"].kind == inspect.Parameter.POSITIONAL_OR_KEYWORD


# ---- the join oracle

def test_join_oracle_is_the_long_form_join_with_uniform_pauses_and_no_gain():
    g = np.random.default_rng(5)
    rows = [g.standard_normal(n).astype(np.float32) for n in (3000, 500, 0, 900, 17)]
    ext = [(100, 2900), (10, 490), (0, 0), (300, 300), (0, 17)]
    for P in (0, 1, 6000, 48000):
        pauses = DO.gaps(ext, [0] * 5, P, 0)
        assert pauses == [P, P]
        assert np.array_equal(DO.join(rows, ext, pauses).view(np.uint32), O.join(rows, ext, P).view(np.uint32))


def test_join_oracle_applies_the_gain_to_the_rounded_faded_sample():
    g = np.random.default_rng(6)
    rows = [g.standard_normal(n).astype(np.float32) for n in (2000, 700, 1500)]
    ext = [(0, 2000), (100, 400), (20, 1500)]
    gains = [np.float32(0.3), np.float32(1.0), np.float32(7.5e-4)]
    got = DO.join(rows, ext, [11, 0], gains)
    # span by span: fp32(g * fp32(x * f)), as normalize_loudness scales an already-joined row
    o = 0
    for i, (s, e) in enumerate(ext):
        solo = O.join([rows[i]], [(s, e)], 0)
        assert np.array_equal(got[o: o + e - s].view(np.uint32), (gains[i] * solo).astype(np.float32).view(np.uint32))
        o += e - s + ([11, 0] + [0])[i]
    assert got.size == 2000 + 300 + 1480 + 11
    assert not got[2000: 2011].any()
    # a run of spans with one gain is the run's own join scaled by it
    same = DO.join(rows, ext, [11, 0], [np.float32(0.3)] * 3)
    assert np.array_equal(same.view(np.uint32), (np.float32(0.3) * DO.join(rows, ext, [11, 0])).view(np.uint32))
    # the order matters: rounding the fade's product first differs from x * (f * g) somewhere
    f = O.fade(240)
    x = rows[0][:240]
    assert not np.array_equal((np.float32(0.3) * (x * f)).view(np.uint32), (x * (f * np.float32(0.3))).view(np.uint32))
