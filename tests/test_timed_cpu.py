"""CPU: timed synthesis's host side -- the SRT and WebVTT reader (sopro_b200/cues.py) against its restatement in
oracle/timed_oracle.py, with every tag, block, entity and refusal (each refusal's line number); the millisecond to
sample identity over 4 h; the fit rule at its boundaries; the host refusals of sopro_timeline_mix (placeholder device
pointers are never dereferenced); synthesize_timed's refusals before any random draw, and its signature."""
import ctypes as C
import dataclasses
import inspect
import os

import numpy as np
import pytest
import torch

from oracle import timed_oracle as TO
from sopro_b200 import _lib
from sopro_b200 import cues as CU
from sopro_b200.stretch import stretched_length
from tests.test_dialogue_cpu import _bare_tts, _voice

A, B = _voice(5), _voice(7)
FAKE = 0x1000  # a non-null pointer no refused call may touch

SRT = ("1\r\n00:00:01,000 --> 00:00:02,500\r\n<i>Hello</i> <b>there</b>,\r\n<font color=\"#ff0\">general</font> {\\an8}Kenobi.\r\n"
       "\r\n2\r\n00:00:02.400 --> 00:00:04,000 X1:40 X2:600\r\n<U>two</U>\r\n\r\n"
       "00:01:00,000 --> 01:00:00,001\r\n  no   index  \r\n\r\n\r\n4\r\n00:02:00,000 --> 00:02:01,000\r\n<i></i>\r\n")

VTT = "\ufeff" + """WEBVTT - a title
Kind: captions

NOTE a comment
that spans lines

STYLE
::cue { color: red }

REGION
id:r1

intro
00:01.000 --> 00:02.500 align:start position:10%
<v Roger Bingham>We are in New York City</v>

00:00:02.000 --> 00:00:04.000
<v.loud Neil>Hi &amp; bye &lt;3 &gt; x&nbsp;y&lrm;z&rlm;</v>
<c.yellow>second</c> <lang en-GB>line</lang> <00:00:03.000><i>timed</i> <b>b</b> <u>u</u>

3
01:00:00.000 --> 01:00:01.000
<ruby>漢<rt>kan</rt>字<rt>ji</rt></ruby> and <v Neil>more <v Neil>same</v>

00:10.000 --> 00:11.000
<b></b>
"""


def test_srt_reads_blocks_tags_and_line_ends():
    got = CU.parse(SRT)
    assert got == [CU.Cue(1.0, 2.5, "Hello there, general Kenobi."), CU.Cue(2.4, 4.0, "two"),
                   CU.Cue(60.0, 3600.001, "no   index"), CU.Cue(120.0, 121.0, "")]
    assert [(c.start, c.end, c.text, c.voice) for c in got] == TO.parse(SRT)


def test_webvtt_reads_voices_tags_entities_and_skips_blocks():
    got = CU.parse(VTT)
    assert got == [CU.Cue(1.0, 2.5, "We are in New York City", "Roger Bingham"),
                   CU.Cue(2.0, 4.0, "Hi & bye <3 > x yz second line timed b u", "Neil"),
                   CU.Cue(3600.0, 3601.0, "漢字 and more same", "Neil"),
                   CU.Cue(10.0, 11.0, "")]
    assert [(c.start, c.end, c.text, c.voice) for c in got] == TO.parse(VTT)
    # an entity decodes once: "&amp;lt;" is the text "&lt;"
    assert CU.parse("WEBVTT\n\n00:00.000 --> 00:01.000\n&amp;lt;")[0].text == "&lt;"
    # a text that does not start with WEBVTT is SRT, even with a BOM
    assert CU.parse("\ufeff00:00:00,000 --> 00:00:01,000\nx") == [CU.Cue(0.0, 1.0, "x")]


REFUSALS = [
    ("1\n00:00:01,000 -> 00:00:02,000\nx\n", 2, "timing"),
    ("1\n00:00:01,000 --> 00:00:02,000\nx\n\n2\n0:01:00 --> 0:02:00\ny\n", 6, "timing"),
    ("00:00:01,000 --> 00:00:02,000\nx\n\njust text\n", 4, "timing"),
    ("00:00:02,000 --> 00:00:02,000\nx\n", 1, "not after"),
    ("\n\n00:00:03,000 --> 00:00:02,000\nx\n", 3, "not after"),
    ("00:00:01,000 --> 00:61:02,000\nx\n", 1, "below 60"),
    ("00:00:01,000 --> 04:00:00,001\nx\n", 1, "past 4 h"),
    ("03:59:59,000 --> 04:00:00,000\nx\n\n04:00:00,000 --> 04:00:01,000\ny", 4, "past 4 h"),
    ("", 1, "no cue"),
    ("\r\n\r\n  \r\n", 4, "no cue"),
    ("WEBVTT\n\nNOTE only\n", 4, "no cue"),
    ("WEBVTT\n\n00:01.000 --> 00:02.000\n<v A>x\n<v B>y\n", 5, "two voices"),
    ("WEBVTT\n\n00:01,000 --> 00:02.000\nx\n", 3, "timing"),
    ("WEBVTT\n\n00:01.000-->00:02.000\nx\n", 3, "timing"),
    ("WEBVTT\n\nan id\nnot a timing\n", 4, "timing"),
    ("WEBVTT\n\nlonely id\n", 3, "timing"),
    ("WEBVTT\n\n00:02.000 --> 00:01.000\nx\n", 3, "not after"),
    ("WEBVTT\n\n04:00:00.000 --> 04:00:00.001\nx\n", 3, "past 4 h"),
]


@pytest.mark.parametrize("text,line,what", REFUSALS)
def test_parse_refusals_name_their_line(text, line, what):
    with pytest.raises(ValueError, match=f"line {line}: .*{what}"):
        CU.parse(text)


def test_cue_records_check_themselves():
    for bad in ((1.0, 1.0), (2.0, 1.0), (-0.5, 1.0), (0.0, CU.MAX_SECONDS + 0.001), (float("nan"), 1.0),
                (0.0, float("inf")), (True, 2.0)):
        with pytest.raises(ValueError):
            CU.Cue(bad[0], bad[1], "x")
    with pytest.raises(TypeError):
        CU.Cue(0.0, 1.0, b"x")
    with pytest.raises(TypeError):
        CU.Cue(0.0, 1.0, "x", voice=3)
    c = CU.Cue(0, 1, "x")
    with pytest.raises(dataclasses.FrozenInstanceError):
        c.start = 2.0
    with pytest.raises(TypeError):
        CU.parse(b"00:00:00,000 --> 00:00:01,000\nx")


def test_every_millisecond_maps_to_24_samples_over_4_hours():
    ms = np.arange(0, 4 * 3600 * 1000 + 1, dtype=np.int64)
    t = ms / 1000  # the reader's seconds
    assert np.array_equal(np.rint(t * 24000).astype(np.int64), ms * 24)
    assert list(map(CU.to_samples, t.tolist())) == (ms * 24).tolist()
    # and through the reader, at the range's ends
    got = CU.parse("00:00:00,001 --> 03:59:59,999\nx\n\n03:59:59.999 --> 04:00:00,000\ny")
    assert [(CU.to_samples(c.start), CU.to_samples(c.end)) for c in got] == [(24, 345599976), (345599976, 345600000)]


def test_fit_rule_at_its_boundaries():
    slot = 48000
    cap = CU.check_max_rate(1.5)
    assert cap == 98304 and CU.check_max_rate(1) == 65536 and CU.check_max_rate(4.0) == 262144
    cases = [(0, 65536), (1, 65536), (slot, 65536), (slot + 1, 65538), (slot * 3 // 2, 98304), (slot * 3 // 2 + 1, 98304),
             (slot * 5, 98304)]
    for n, S in cases:
        assert CU.fit_speed(n, slot, cap) == S, n
        oS, oM, over, offs, N = TO.fit([n], [1.0], [3.0], 1.5)
        assert oS == [S] and oM == [stretched_length(S / 65536, n)]
        M = oM[0]
        assert (M <= slot) == (n <= slot * 3 // 2)  # it fits unless the cap bit
        assert over == [max(0, M - slot)] and offs == [24000] and N == max(72000, 24000 + M)
    # n = slot + 1 needs the least S with ceil(n * 65536 / S) <= slot
    S = CU.fit_speed(slot + 1, slot, cap)
    assert stretched_length(S / 65536, slot + 1) <= slot < stretched_length((S - 1) / 65536, slot + 1)
    # a track: the cap, an overrun and the track's length
    S, M, over, offs, N = TO.fit([1000, 96000, 0], [0.0, 1.0, 1.5], [1.0, 2.0, 9.0], 2.0)
    assert S == [65536, 131072, 65536] and M == [1000, 48000, 0] and over == [0, 24000, 0] and N == 216000


def test_max_rate_and_group_refusals():
    for bad in (0.99, 4.01, float("nan"), True, "2", None):
        with pytest.raises(ValueError):
            CU.check_max_rate(bad)
    assert CU.groups([3, 0, 2, 5, 0, 9, 1], 5) == [(0, 3), (3, 5), (5, 6), (6, 7)]
    assert CU.groups([0, 0], 64) == [(0, 2)]


def _mix(n_items, lens, offs, y_len, src=True, y=FAKE, null_item=None):
    lib = _lib.load()
    n = max(len(offs if lens is None else lens), 1)
    sp = (C.c_void_p * n)(*[None if i == null_item else FAKE for i in range(n_items)]) if src else None
    lp = (C.c_int64 * n)(*lens) if lens is not None else None
    op = (C.c_int64 * n)(*offs) if offs is not None else None
    return lib.sopro_timeline_mix(sp, n_items, lp, op, y, y_len, None)


def test_mix_symbol_is_exported_with_its_binding():
    lib = _lib.load()
    assert "sopro_timeline_mix" in _lib.SYMBOLS
    fn = lib.sopro_timeline_mix
    assert fn.restype is C.c_int and len(fn.argtypes) == 7
    with open(os.path.join(os.path.dirname(__file__), "..", "include", "sopro_b200.h")) as f:
        assert "int sopro_timeline_mix(" in f.read()


@pytest.mark.parametrize("args", [
    dict(n_items=-1, lens=[], offs=[], y_len=10),
    dict(n_items=2, lens=[5, 5], offs=[0, 1], y_len=10, src=False),
    dict(n_items=2, lens=None, offs=[0, 1], y_len=10),
    dict(n_items=2, lens=[5, 5], offs=None, y_len=10),
    dict(n_items=2, lens=[5, 5], offs=[0, 1], y_len=10, null_item=1),   # a null source for a non-empty item
    dict(n_items=2, lens=[5, -1], offs=[0, 1], y_len=10),
    dict(n_items=2, lens=[5, 5], offs=[0, -1], y_len=10),
    dict(n_items=2, lens=[5, 5], offs=[0, 6], y_len=10),                # ends past y_len
    dict(n_items=1, lens=[11], offs=[0], y_len=10),
    dict(n_items=1, lens=[0], offs=[11], y_len=10),                     # an empty item past the end too
    dict(n_items=1, lens=[1], offs=[0], y_len=(1 << 40) + 1),
    dict(n_items=0, lens=[], offs=[], y_len=-1),
    dict(n_items=1, lens=[5], offs=[0], y_len=10, y=None),
])
def test_mix_refusals_happen_before_any_launch(args):
    assert _mix(**args) == -1  # SOPRO_ERR_INVALID, on a machine with or without a GPU
    assert _lib.load().sopro_last_error()


def test_mix_of_nothing_is_not_an_error():
    assert _mix(n_items=0, lens=[], offs=[], y_len=0, src=False, y=None) == 0
    assert _mix(n_items=2, lens=[0, 0], offs=[0, 0], y_len=0, y=None, null_item=0) == 0


def test_mix_oracle_is_a_sequential_fp32_sum():
    g = np.random.default_rng(0)
    rows = [g.standard_normal(n).astype(np.float32) for n in (10, 7, 0, 12)]
    y = TO.mix(rows, [0, 5, 3, 8], 25)
    want = np.zeros(25, np.float32)
    for t in range(25):
        acc = None
        for r, o in zip(rows, [0, 5, 3, 8]):
            if o <= t < o + r.size:
                acc = r[t - o] if acc is None else np.float32(acc + r[t - o])
        want[t] = 0.0 if acc is None else acc
    assert np.array_equal(y.view(np.uint32), want.view(np.uint32))
    z = TO.mix([np.array([-0.0], np.float32)], [1], 2)  # a single cover keeps its sign bit
    assert z.view(np.uint32).tolist() == [0, 0x80000000]


GOOD = "1\n00:00:01,000 --> 00:00:02,000\n1 2 3.\n\n2\n00:00:02,000 --> 00:00:03,000\n4 5.\n"


def test_refusals_happen_before_any_random_draw():
    tts = _bare_tts()
    before = torch.get_rng_state()
    for text, _line, _what in REFUSALS:
        with pytest.raises(ValueError):
            tts.synthesize_timed(text, ref=A)
    vtt = "WEBVTT\n\n00:01.000 --> 00:02.000\n<v b>1 2.\n\n00:02.000 --> 00:03.000\n<v zed>3.\n"
    cases = [
        (ValueError, vtt, dict(voices={"b": B})),                            # an unknown voice name
        (ValueError, GOOD, dict(voices={"b": B}, ref=_voice(layers=1))),   # a voice of the wrong geometry
        (ValueError, "WEBVTT\n\n00:01.000 --> 00:02.000\n<v b>1 2.\n", dict(voices={"b": _voice(Tr=5000)})),
        (TypeError, "WEBVTT\n\n00:01.000 --> 00:02.000\n<v b>1 2.\n", dict(voices={"b": "not a voice"})),
        (TypeError, GOOD, dict(voices=[B])),
        (TypeError, [CU.Cue(0, 1, "1"), (0, 1, "2")], {}),
        (TypeError, 5, {}),
        (ValueError, [], {}),
        (ValueError, [CU.Cue(1.0, 1.00001, "1 2.")], {}),                  # start and end round to one sample
        (ValueError, "00:00:00,000 --> 00:00:01,000\n<i> </i>\n\n00:00:01,000 --> 00:00:02,000\n{\\an8}", {}),
        (ValueError, [CU.Cue(0, 1, ""), CU.Cue(1, 2, "  ")], {}),
    ] + [(ValueError, GOOD, kw) for kw in (
        dict(max_rate=0.5), dict(max_rate=4.5), dict(max_rate=float("nan")), dict(max_rate=True),
        dict(pause_ms=-1), dict(pause_ms=2001), dict(max_tokens=3), dict(max_tokens=10 ** 6),
        dict(sample_rate=3999), dict(loudness=1.0), dict(watermark=-1), dict(best_of=0))]
    for exc, cues, kw in cases:
        with pytest.raises(exc):
            tts.synthesize_timed(cues, **{"ref": A, **kw})
    assert torch.equal(before, torch.get_rng_state())


def test_signature_and_exports():
    import sopro_b200
    from sopro_b200 import SoproTTS

    want = dict(ref=inspect.Parameter.empty, voices=None, seed=None, max_rate=1.5, pause_ms=250, max_frames=400,
                max_tokens=64, top_p=0.9, temperature=1.05, anti_loop=True, style_strength=None, min_gen_frames=None,
                sample_rate=None, loudness=None, watermark=None, best_of=1)
    p = inspect.signature(SoproTTS.synthesize_timed).parameters
    assert list(p) == ["self", "cues", *want]
    for k, v in want.items():
        assert p[k].default == v and p[k].kind == inspect.Parameter.KEYWORD_ONLY, k
    assert sopro_b200.Cue is CU.Cue and sopro_b200.CueFit is CU.CueFit and sopro_b200.parse_cues is CU.parse
    assert {"Cue", "CueFit", "parse_cues"} <= set(sopro_b200.__all__)
    assert [f.name for f in dataclasses.fields(CU.CueFit)] == ["index", "rate", "spoken", "overrun"]
