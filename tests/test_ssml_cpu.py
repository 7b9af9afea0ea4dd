"""CPU: the speech-markup plan (sopro_b200/ssml.py) -- every element, nesting, breaks at the edges and stacked, <p>
versus <s> gaps, voice switches inside a sentence, the merge rule for silent segments -- against its restatement in
oracle/ssml_oracle.py; every refusal before any random draw; synthesize_ssml's signature."""
import inspect
import math

import numpy as np
import pytest
import torch

from oracle import ssml_oracle as SO
from sopro_b200 import longform as LF
from sopro_b200 import ssml as M
from sopro_b200.tokenizer import IdsTokenizer
from tests.test_dialogue_cpu import _bare_tts, _voice

IDS = IdsTokenizer(1000)
A, B, C_ = _voice(5), _voice(7), _voice(9)
VOICES = {"a": A, "b": B}
P, PP = 6000, 12000


def _plan(ssml, **kw):
    args = dict(pause_ms=250, paragraph_pause_ms=500, speed=None, max_tokens=6)
    args.update(kw)
    return M.parse(ssml, VOICES, C_, args["pause_ms"], args["paragraph_pause_ms"], args["speed"], args["max_tokens"], IDS)


def _summary(p):
    return [(s.text, s.voice, s.rate, s.db) for s in p.segments], p.gaps, p.lead, p.trail


# (markup, segments as (text, voice, rate, dB), gaps, lead, trail)
TABLE = [
    ("1 2 3. 4 5 6. 7 8", [("1 2 3.", C_, 1.0, 0.0), ("4 5 6.", C_, 1.0, 0.0), ("7 8", C_, 1.0, 0.0)], [P, P], 0, 0),
    ("<speak>1 2.\n\n3 4.</speak>", [("1 2.", C_, 1.0, 0.0), ("3 4.", C_, 1.0, 0.0)], [P], 0, 0),
    ('<speak xmlns="http://www.w3.org/2001/10/synthesis" version="1.0" xml:lang="en-US"><p>1.</p><p>2.</p></speak>',
     [("1.", C_, 1.0, 0.0), ("2.", C_, 1.0, 0.0)], [PP], 0, 0),
    ("<p><s>1 2</s><s>3</s></p><p>4</p>", [("1 2", C_, 1.0, 0.0), ("3", C_, 1.0, 0.0), ("4", C_, 1.0, 0.0)], [P, PP], 0, 0),
    ("1 <p>2</p> 3", [("1", C_, 1.0, 0.0), ("2", C_, 1.0, 0.0), ("3", C_, 1.0, 0.0)], [PP, PP], 0, 0),
    # breaks: replace the default, stack, sit at the edges
    ('1 <break time="350ms"/> 2', [("1", C_, 1.0, 0.0), ("2", C_, 1.0, 0.0)], [8400], 0, 0),
    ('1. <break time="1.5s"/><break strength="weak"/> 2', [("1.", C_, 1.0, 0.0), ("2", C_, 1.0, 0.0)], [36000 + 3600], 0, 0),
    ('<p>1.</p><break strength="none"/><p>2.</p>', [("1.", C_, 1.0, 0.0), ("2.", C_, 1.0, 0.0)], [0], 0, 0),
    ('<break/><break strength="x-strong"/>1 2<break time="10s"/>', [("1 2", C_, 1.0, 0.0)], [], P + 24000, 240000),
    ('1<break strength="x-weak"/>2<break strength="strong"/>3<break strength="medium"/>4',
     [("1", C_, 1.0, 0.0), ("2", C_, 1.0, 0.0), ("3", C_, 1.0, 0.0), ("4", C_, 1.0, 0.0)], [1200, 12000, P], 0, 0),
    # voice switches: a split inside a sentence is 0, after a sentence P
    ('1 2 <voice name="a">3 4</voice> 5.', [("1 2", C_, 1.0, 0.0), ("3 4", A, 1.0, 0.0), ("5.", C_, 1.0, 0.0)], [0, 0], 0, 0),
    ('<voice name="a">1 2.</voice> <voice name="b">3 4.</voice>', [("1 2.", A, 1.0, 0.0), ("3 4.", B, 1.0, 0.0)], [P], 0, 0),
    ('<voice name="a">1 <voice name="a">2</voice></voice>', [("1 2", A, 1.0, 0.0)], [], 0, 0),  # no change, no cut
    # prosody nesting: rates multiply, dB add, silent is sticky
    ('<prosody rate="slow">1 <prosody rate="200%">2 <prosody rate="x-fast">3</prosody></prosody></prosody>',
     [("1", C_, 0.75, 0.0), ("2", C_, 1.5, 0.0), ("3", C_, 2.25, 0.0)], [0, 0], 0, 0),
    ('<prosody rate="0.8" volume="x-soft">1 <prosody volume="+3dB" rate="fast">2</prosody></prosody>',
     [("1", C_, 0.8, -12.0), ("2", C_, 0.8 * 1.25, -9.0)], [0], 0, 0),
    ('1 <prosody volume="silent">2 <prosody volume="x-loud">3</prosody></prosody>',
     [("1", C_, 1.0, 0.0), ("2 3", C_, 1.0, -math.inf)], [0], 0, 0),
    ('<prosody volume="loud">1</prosody><prosody volume="-6dB">2</prosody><prosody volume="medium" rate="medium">3</prosody>',
     [("1", C_, 1.0, 6.0), ("2", C_, 1.0, -6.0), ("3", C_, 1.0, 0.0)], [0, 0], 0, 0),
    # sub speaks the alias inside the surrounding run
    ('1 <sub alias="2 3">x</sub> 4.', [("1 2 3 4.", C_, 1.0, 0.0)], [], 0, 0),
    # split_text cuts inside a styled run
    ('<voice name="b">1 2 3. 4 5 6.</voice>', [("1 2 3.", B, 1.0, 0.0), ("4 5 6.", B, 1.0, 0.0)], [P], 0, 0),
    # whitespace-only runs between boundaries speak nothing and do not separate the boundaries
    ('1.<voice name="a"> </voice><break time="20ms"/> <p> </p>2', [("1.", C_, 1.0, 0.0), ("2", C_, 1.0, 0.0)], [480], 0, 0),
]


@pytest.mark.parametrize("case", range(len(TABLE)))
def test_markup_to_plan(case):
    ssml, segs, gaps, lead, trail = TABLE[case]
    got = _plan(ssml)
    g_segs, g_gaps, g_lead, g_trail = _summary(got)
    assert [(t, r, d) for t, _v, r, d in g_segs] == [(t, r, d) for t, _v, r, d in segs]
    assert all(a[1] is b[1] for a, b in zip(g_segs, segs))
    assert (g_gaps, g_lead, g_trail) == (gaps, lead, trail)
    # the restatement agrees
    o_segs, o_gaps, o_lead, o_trail = SO.plan(ssml, VOICES, C_, 250, 500, None, lambda t: LF.split_text(t, IDS, 6))
    assert [(t, r, d) for t, _v, r, d in o_segs] == [(t, r, d) for t, _v, r, d in g_segs]
    assert all(a[1] is b[1] for a, b in zip(o_segs, g_segs))
    assert (o_gaps, o_lead, o_trail) == (g_gaps, g_lead, g_trail)


def test_plain_text_is_synthesize_long_and_pauses_are_the_arguments():
    text = "1 2 3. 4 5. 6 7 8 9 10 11, 12 13.\n\n14 15."
    p = _plan(f"<speak>{text}</speak>", pause_ms=120, max_tokens=6)
    assert [s.text for s in p.segments] == LF.split_text(text, IDS, 6)
    assert p.gaps == [LF.pause_samples(120)] * (len(p.segments) - 1) and p.lead == p.trail == 0
    assert all(s.gain == 1.0 and s.rate == 1.0 for s in p.segments)
    q = _plan("<p>1.</p><p>2.</p><s>3.</s><s>4.</s>", pause_ms=0, paragraph_pause_ms=2000)
    assert q.gaps == [48000, 48000, 0]
    # pause_ms larger than paragraph_pause_ms: a <p> edge still takes the paragraph pause
    assert _plan("<p>1.</p><p>2.</p>", pause_ms=800, paragraph_pause_ms=100).gaps == [2400]


def test_speed_multiplies_every_rate_but_not_the_breaks():
    ssml = '1 <break time="1s"/> <prosody rate="x-slow">2</prosody>'
    p = _plan(ssml, speed=2)
    assert [s.rate for s in p.segments] == [2.0, 1.0] and p.gaps == [24000]
    assert SO.plan(ssml, VOICES, C_, 250, 500, 2, lambda t: LF.split_text(t, IDS, 6))[0][1][2] == 1.0
    assert _plan('<prosody rate="x-fast">1</prosody>', speed=2.5).segments[0].rate == 3.75
    with pytest.raises(ValueError, match="effective rate"):
        _plan('<prosody rate="x-fast">1</prosody>', speed=3)
    with pytest.raises(ValueError, match="effective rate"):
        _plan('<prosody rate="x-slow">1</prosody>', speed=0.25)


def test_gains_are_one_double_evaluation_rounded_once():
    for db in (-60.0, -12.0, -9.0, -6.0, 0.0, 3.0, 6.0, 12.0, -0.1):
        s = M.Segment("1", A, 1.0, db)
        assert s.gain == float(np.float32(10.0 ** (db / 20.0))) == float(SO.gain(db))
    assert M.Segment("1", A, 1.0, -math.inf).gain == 0.0 and SO.gain(-math.inf) == 0.0
    assert M.Segment("1", A, 1.0, 0.0).gain == 1.0


def test_empty_segments_merge_their_gaps_into_the_larger():
    p = M.Plan([M.Segment(str(k), A, 1.0, 0.0) for k in range(6)], [10, 50, 20, 30, 5], 7, 9)
    cases = [
        ([True] * 6, [10, 50, 20, 30, 5]),
        ([True, False, True, True, True, True], [50, 20, 30, 5]),
        ([True, False, False, True, True, True], [50, 30, 5]),
        ([True, True, True, False, True, False], [10, 50, 30]),
        ([False, True, True, True, True, True], [50, 20, 30, 5]),  # the gap to the edge goes with the segment
        ([False, False, True, False, False, True], [30]),
        ([False] * 6, []),
        ([False, False, True, False, False, False], []),
    ]
    for spoken, want in cases:
        assert p.pauses(spoken) == want, spoken
        assert SO.merged_pauses(p.gaps, spoken) == want, spoken
    with pytest.raises(ValueError):
        p.pauses([True] * 5)


def test_assembly_oracle_places_the_edges_and_the_gains():
    g = np.random.default_rng(3)
    rows = [g.standard_normal(n).astype(np.float32) for n in (900, 0, 500, 40)]
    out = SO.assemble(rows, [5, 70, 3], [0.0, 6.0, -math.inf, -6.0], 11, 13)
    body = 900 + 70 + 500 + 3 + 40
    assert out.size == 11 + body + 13
    assert not out[:11].any() and not out[-13:].any()
    assert not out[11 + 900 + 70: 11 + 900 + 70 + 500].any()  # the silent span keeps its length, at gain 0
    tail = out[11 + body - 40: 11 + body]
    want = SO.join([rows[3]], [(0, 40)], [], [np.float32(10.0 ** (-6.0 / 20.0))])
    assert np.array_equal(tail.view(np.uint32), want.view(np.uint32))


REFUSALS = [
    ("<emphasis>1</emphasis>", "emphasis"), ('<say-as interpret-as="digits">1</say-as>', "say-as"),
    ('<phoneme ph="x">1</phoneme>', "phoneme"), ('<audio src="x.wav"/>1', "audio"), ('1 <mark name="m"/>', "mark"),
    ('<prosody pitch="+2st">1</prosody>', "pitch"), ('<prosody rate="fast" pitch="low">1</prosody>', "pitch"),
    ('<prosody contour="(0%,+20Hz)">1</prosody>', "contour"), ('<voice gender="female">1</voice>', "gender"),
    ('<break time="2s" strength="weak" foo="1"/>1', "foo"), ('<p xml:lang="fr">1</p>', "xml:lang"),
    ("<speak>1", "well-formed"), ("1 & 2", "well-formed"), ("<speak><p>1</speak>", "well-formed"),
    ("<speak><speak>1</speak></speak>", "speak"), ('<voice name="zed">1</voice>', "zed"), ("<voice>1</voice>", "None"),
    ('<prosody rate="x-slow"><prosody rate="40%">1</prosody></prosody>', "rate"), ('<prosody rate="5">1</prosody>', "rate"),
    ('<prosody rate="-1">1</prosody>', "rate"), ('<prosody rate="quick">1</prosody>', "rate"),
    ('<prosody volume="+13dB">1</prosody>', "volume"), ('<prosody volume="x-soft"><prosody volume="-49dB">1</prosody></prosody>', "volume"),
    ('<prosody volume="loud">1</prosody><prosody volume="+12dB"><prosody volume="+1dB">2</prosody></prosody>', "volume"),
    ('<prosody volume="quiet">1</prosody>', "volume"), ('<break time="10.5s"/>1', "break"), ('<break time="-1s"/>1', "break"),
    ('<break time="5min"/>1', "break"), ('<break strength="huge"/>1', "break"), ("<sub>1</sub>", "alias"),
    ("", "nothing"), ("  <speak> <p> </p> <break/> </speak>", "nothing"), ('<sub alias=" ">1</sub>', "nothing"),
]


@pytest.mark.parametrize("ssml,what", REFUSALS)
def test_parse_refusals_name_what_is_refused(ssml, what):
    with pytest.raises(ValueError, match=what):
        _plan(ssml)


def test_refusals_happen_before_any_random_draw():
    tts = _bare_tts()
    before = torch.get_rng_state()
    for ssml, _what in REFUSALS:
        with pytest.raises(ValueError):
            tts.synthesize_ssml(ssml, ref=A, voices=VOICES)
    good = '<voice name="b">1 2.</voice> 3.'
    for kw in (dict(pause_ms=-1), dict(pause_ms=2001), dict(paragraph_pause_ms=float("nan")), dict(paragraph_pause_ms=True),
               dict(max_tokens=3), dict(max_tokens=10 ** 6), dict(sample_rate=3999), dict(speed=5.0), dict(speed=0.2),
               dict(speed=True), dict(loudness=1.0), dict(watermark=-1), dict(best_of=0),
               dict(voices={"b": _voice(layers=1)}), dict(voices={"b": _voice(Tr=5000)})):
        with pytest.raises(ValueError):
            tts.synthesize_ssml(good, **{"ref": A, "voices": VOICES, **kw})
    with pytest.raises(TypeError):
        tts.synthesize_ssml(good, ref=A, voices={"b": "not a voice"})
    with pytest.raises(TypeError):
        tts.synthesize_ssml(good, ref=A, voices=[B])
    with pytest.raises(TypeError):
        tts.synthesize_ssml(b"1 2.", ref=A)
    assert torch.equal(before, torch.get_rng_state())


def test_signature():
    from sopro_b200 import SoproTTS

    want = dict(ref=inspect.Parameter.empty, voices=None, seed=None, pause_ms=250, paragraph_pause_ms=500,
                max_frames=400, max_tokens=64, top_p=0.9, temperature=1.05, anti_loop=True, style_strength=None,
                min_gen_frames=None, sample_rate=None, speed=None, loudness=None, watermark=None, best_of=1)
    p = inspect.signature(SoproTTS.synthesize_ssml).parameters
    assert list(p) == ["self", "ssml", *want]
    assert p["ssml"].kind == inspect.Parameter.POSITIONAL_OR_KEYWORD
    for k, v in want.items():
        assert p[k].default == v and p[k].kind == inspect.Parameter.KEYWORD_ONLY, k
    assert list(inspect.signature(M.parse).parameters) == ["ssml", "voices", "default_voice", "pause_ms",
                                                           "paragraph_pause_ms", "speed", "max_tokens", "tokenizer"]
