"""CPU: long-form synthesis's host side (sopro_b200/longform.py) -- the text segmenter's rules and invariant, the fade
window, lengths, refused arguments -- and the float64 extents oracle (oracle/longform_oracle.py) against the project's
energy trim, sopro_b200.audio.trim_silence_energy, which tests/golden/audio_prep.json pins to the reference."""
import inspect
import math

import numpy as np
import pytest
import torch

from oracle import longform_oracle as O
from sopro_b200 import longform as LF
from sopro_b200.tokenizer import IdsTokenizer


class Words:
    """A stand-in tokenizer: one token per whitespace-separated word, plus BOS and EOS."""

    def encode(self, text):
        return [0] + [1] * len(text.split()) + [2]


IDS = IdsTokenizer(1000)


def _normalised(par):
    return " ".join(par.split())


def _check_invariant(text, segs, tok, budget):
    pars = [_normalised(p) for p in LF._PARAGRAPH.split(text)]
    pars = [p for p in pars if p]
    assert all(s and s == s.strip() for s in segs)
    # every segment fits, except a single whitespace-free run
    for s in segs:
        assert len(tok.encode(s)) <= budget or " " not in s, s
    # the segments, in order, rebuild each paragraph
    i = 0
    for p in pars:
        got = []
        while i < len(segs) and len(" ".join(got + [segs[i]])) <= len(p) and p.startswith(" ".join(got + [segs[i]])):
            got.append(segs[i])
            i += 1
            if " ".join(got) == p:
                break
        assert " ".join(got) == p, (p, got)
    assert i == len(segs)


def test_sentence_boundaries():
    f = LF._sentences
    assert f("One. Two! Three? Four… Five") == ["One.", "Two!", "Three?", "Four…", "Five"]
    assert f("Wait...?! Yes.") == ["Wait...?!", "Yes."]
    assert f('He said "stop." Then (he left.) And [so.] ‘Right.’ “Quite!” Done.') == \
        ['He said "stop."', "Then (he left.)", "And [so.]", "‘Right.’", "“Quite!”", "Done."]
    assert f("Use e.g. this one. And approx. five more.") == ["Use e.g. this one.", "And approx. five more."]
    assert f("Dr. Smith is here.") == ["Dr.", "Smith is here."]  # no abbreviation list
    assert f("Pi is 3.14 today. Ok") == ["Pi is 3.14 today.", "Ok"]
    assert f("No terminator here") == ["No terminator here"]
    assert f("A.B. C") == ["A.B.", "C"]
    assert f("Fine!") == ["Fine!"]


@pytest.mark.parametrize("tok", (Words(), IDS), ids=("words", "ids"))
def test_packing_and_paragraphs(tok):
    text = "  One two.   Three four five!\n\n\n  \n Six seven? Eight.\nNine ten\n \n\nEleven. "
    segs = LF.split_text(text, tok, 8)
    # 7 tokens fit, so one paragraph's sentences merge; a segment never spans a blank line
    assert segs == ["One two. Three four five!", "Six seven? Eight. Nine ten", "Eleven."]
    _check_invariant(text, segs, tok, 8)
    assert LF.split_text(text, tok, 5) == ["One two.", "Three four five!", "Six seven? Eight.", "Nine ten", "Eleven."]
    assert LF.split_text(text, tok, 4) == ["One two.", "Three four", "five!", "Six seven?", "Eight.", "Nine ten", "Eleven."]
    for budget in (4, 5, 6, 7, 9, 64):
        _check_invariant(text, LF.split_text(text, tok, budget), tok, budget)
    assert LF.split_text("", tok, 8) == [] and LF.split_text(" \n\n \t\n", tok, 8) == []


def test_over_long_sentences_are_cut_at_clause_marks_then_whitespace():
    tok = Words()
    s = "a b c, d e f; g h: i j — k l – m n o p q r s t"
    # budget 6 = 4 words: the last clause mark whose left piece fits
    assert LF.split_text(s, tok, 6) == ["a b c,", "d e f;", "g h:", "i j —", "k l –", "m n o p", "q r s t"]
    # a mark not followed by whitespace is not a clause mark
    assert LF.split_text("a,b,c,d e f g h", tok, 4) == ["a,b,c,d e", "f g", "h"]
    # a single whitespace-free run over the budget is a segment of its own
    long_word = "x" * 50
    ids_tok = type("Chars", (), {"encode": lambda self, t: [0] * (len(t) // 5 + 2)})()
    segs = LF.split_text(f"Short one. {long_word} tail words here.", ids_tok, 6)
    assert long_word in segs
    _check_invariant(f"Short one. {long_word} tail words here.", segs, ids_tok, 6)
    for budget in (4, 5, 6, 7, 8, 13):
        _check_invariant(s, LF.split_text(s, tok, budget), tok, budget)


def test_segments_counted_with_the_ids_tokenizer():
    text = " ".join(str(i) for i in range(200)) + ". " + ", ".join(str(i) for i in range(40)) + ". Done."
    for budget in (4, 10, 32, 64):
        segs = LF.split_text(text, IDS, budget)
        _check_invariant(text, segs, IDS, budget)
        assert all(len(IDS.encode(s)) <= budget for s in segs)
    segs = LF.split_text(text, IDS, 64)
    assert len(IDS.encode(segs[0])) == 64 and segs[-1].endswith("Done.")


def test_fade_window_bits_and_refusals():
    for F in (1, 2, 3, 7, 100, 239, 240):
        got = LF.fade_window(F)
        assert got.dtype == np.float32 and np.array_equal(got.view(np.uint32), O.fade(F).view(np.uint32)), F
        want = np.array([np.float32(0.5 - 0.5 * math.cos(math.pi * (i + 0.5) / F)) for i in range(F)])
        assert np.array_equal(got, want)
        assert np.all(got > 0) and np.all(got < 1) and np.all(np.diff(got) > 0)
        assert np.abs(got.astype(np.float64) + got[::-1] - 1.0).max() <= 2 ** -24  # complementary up to rounding
    assert LF.fade_window(0).size == 0
    for F in (-1, 241):
        with pytest.raises(ValueError):
            LF.fade_window(F)


def test_lengths():
    assert [LF.fade_length(s) for s in (0, 1, 2, 3, 479, 480, 481, 10 ** 6)] == [0, 0, 1, 1, 239, 240, 240, 240]
    assert LF.pause_samples(250) == 6000 and LF.pause_samples(0) == 0 and LF.pause_samples(2000) == 48000
    assert LF.pause_samples(0.1) == 2 and LF.pause_samples(1 / 48) == 0  # round half to even at 0.5 samples
    ext = [(0, 100), (5, 5), (10, 30), (0, 0), (7, 8)]
    assert LF.joined_length(ext, 6) == 100 + 20 + 1 + 2 * 6
    assert LF.joined_length([(3, 3)], 6) == 0 and LF.joined_length([(0, 9)], 6) == 9
    rows = [np.ones(200, dtype=np.float32)] * 5
    assert O.join(rows, ext, 6).size == LF.joined_length(ext, 6)


@pytest.mark.parametrize("bad", (float("nan"), float("inf"), -1, -0.001, 2000.5, True, "250", None, [250]))
def test_refused_pauses(bad):
    with pytest.raises(ValueError):
        LF.check_pause(bad)


def test_accepted_pauses_and_budgets():
    for p in (0, 0.0, 250, 1999.9, 2000, np.float32(10.0), np.int64(5)):
        assert LF.check_pause(p) == float(p)
    for m in (4, 64, 2056, np.int64(10)):
        assert LF.check_max_tokens(m, 2056) == int(m)
    for bad in (3, 0, -5, 2057, 64.0, True, "64", None, float("nan")):
        with pytest.raises(ValueError):
            LF.check_max_tokens(bad, 2056)


def test_synthesize_long_signature():
    from sopro_b200 import SoproTTS

    p = inspect.signature(SoproTTS.synthesize_long).parameters
    want = dict(max_frames=400, max_tokens=64, pause_ms=250, top_p=0.9, temperature=1.05, anti_loop=True,
                style_strength=None, min_gen_frames=None, seed=None, sample_rate=None, speed=None, loudness=None)
    for k, v in want.items():
        assert p[k].default == v and p[k].kind == inspect.Parameter.KEYWORD_ONLY, k
    assert p["ref"].kind == inspect.Parameter.KEYWORD_ONLY and p["ref"].default is inspect.Parameter.empty


def test_refused_arguments_raise_before_any_work():
    """Rate, speed, loudness, pause, budget and an empty text are refused before the prefill or a random draw: this
    object has no engines at all."""
    from types import SimpleNamespace

    from sopro_b200.model import SoproTTS

    tts = SoproTTS.__new__(SoproTTS)
    tts._resamplers = {}
    tts.tokenizer = IDS
    tts.model = SimpleNamespace(prefill=SimpleNamespace(max_text_len=2056))
    before = torch.get_rng_state()
    bad = (dict(sample_rate=3999), dict(speed=5.0), dict(loudness=1.0), dict(pause_ms=-1), dict(pause_ms=float("nan")),
           dict(max_tokens=3), dict(max_tokens=True), dict(max_tokens=5000))
    for kw in bad:
        with pytest.raises(ValueError):
            tts.synthesize_long("1 2. 3 4.", ref=None, **kw)
    for text in ("", "   ", "\n\n \t \n"):
        with pytest.raises(ValueError):
            tts.synthesize_long(text, ref=None)
    assert torch.equal(before, torch.get_rng_state())


# ---- the extents oracle against the energy trim

def _trim_extent(x: np.ndarray):
    """(start, end) that sopro_b200.audio.trim_silence_energy keeps of a 24 kHz row (its result is a view of the input),
    and its fp32 frame dB and threshold."""
    from sopro_b200.audio import trim_silence_energy

    w = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).unsqueeze(0)
    t = trim_silence_energy(w, 24000)
    start = t.storage_offset() - w.storage_offset()
    n = x.size
    db32 = thr32 = None
    if n >= O.FRAME:
        db32 = (10.0 * torch.log10(w.unfold(-1, 600, 240).pow(2).mean(dim=-1).squeeze(0) + 1e-10)).numpy()
        thr32 = max(float(db32.max()) - 40.0, -40.0)
    return (start, start + int(t.shape[-1])), db32, thr32


def _agree(x):
    """The oracle's extent equals the trim's; a differing first or last voiced frame is accepted only when the trim's
    fp32 dB of the frame either side chose lies within 1e-3 dB of its threshold."""
    got = O.extent_detail(x)
    (s, e), db32, thr32 = _trim_extent(x)
    if (got["start"], got["end"]) == (s, e):
        return True
    near = [k for k in range(len(db32)) if abs(float(db32[k]) - thr32) <= 1e-3]
    assert near, (got["start"], got["end"], s, e)
    return False


def _recipes():
    from tests.golden.make_audio_golden import CASES, signal

    for i, (name, _sr, n, lo, hi, floor) in enumerate(CASES):
        yield name, signal(24000, n, lo, hi, floor, i)[0].numpy()


def test_oracle_extents_equal_the_energy_trim_on_the_fixture_signals():
    for name, x in _recipes():
        assert _agree(x), name
        d = O.extent_detail(x)
        if name == "margins_24k":
            assert 0 < d["start"] < 20000 < 50000 < d["end"] < 72000
        if name in ("short_burst_24k", "tiny_24k", "silent_24k"):
            assert (d["start"], d["end"]) == (0, x.size)


def test_oracle_extents_on_loud_quiet_silent_rows():
    g = np.random.default_rng(5)
    n = 3 * 30000
    x = (0.9 * g.standard_normal(n)).astype(np.float32)
    x[30000:60000] *= 0.03   # about 30 dB down, at -31 dB: voiced (the floor is 40 dB under the loudest frame)
    x[60000:] = 0
    assert _agree(x)
    d = O.extent_detail(x)
    assert d["start"] == 0 and 60000 < d["end"] <= 60000 + 600 + 720
    y = x.copy()
    y[30000:60000] *= 0.01   # now 70 dB down: trimmed away
    assert _agree(y)
    d = O.extent_detail(y)
    assert d["start"] == 0 and 30000 <= d["end"] <= 30000 + 600 + 720
    for n in (599, 600, 2399, 2400, 11999, 12000, 12001):
        z = (0.1 * g.standard_normal(n)).astype(np.float32)
        assert _agree(z), n
        assert O.extent(z) == (0, n), n  # too short to be trimmed below 12,000 samples, or all voiced
