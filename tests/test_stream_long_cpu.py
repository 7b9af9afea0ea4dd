"""Host-side: the causal restatement of stream_long's trim (oracle/longform_stream_oracle.py: stream_extent, stream_join)
against the one-shot extent and join, its certain-prefix bounds, and the refusals of SoproTTS.stream_long, which come
before any device work or random draw."""
import inspect

import numpy as np
import pytest
import torch

from oracle import longform_oracle as O
from oracle import longform_stream_oracle as S
from sopro_b200.tokenizer import IdsTokenizer

SCHEDULES = (1, 239, 240, 601, 11520, None)  # None: the whole row in one push


def _rows():
    """(name, fp32 row) pairs, every frame at most 0 dB: the audio_prep.json recipes at 24 kHz, noise, silence, a loud +
    quiet + silent row, speech-like bursts padded with silence, and bursts at the edges of the length rules."""
    from tests.golden.make_audio_golden import CASES, signal

    g = np.random.default_rng(11)
    out = [(name, signal(24000, n, lo, hi, floor, i)[0].numpy()) for i, (name, _sr, n, lo, hi, floor) in enumerate(CASES)]
    out.append(("noise", (0.3 * g.standard_normal(50000)).astype(np.float32)))
    out.append(("silence", np.zeros(40000, dtype=np.float32)))
    x = (0.9 * g.standard_normal(90000)).astype(np.float32)
    x[30000:60000] *= 0.03
    x[60000:] = 0
    out.append(("loud_quiet_silent", x))
    y = np.zeros(70000, dtype=np.float32)
    for a in (15000, 31000, 44000):
        y[a: a + 6000] = (0.2 * g.standard_normal(6000)).astype(np.float32)
    out.append(("bursts", y))
    for n in (599, 600, 2399, 2400, 11999, 12000, 12001, 30000):
        z = np.zeros(n, dtype=np.float32)
        k = n // 4
        z[n // 3: n // 3 + k] = (0.5 * g.standard_normal(k)).astype(np.float32)
        out.append((f"burst_{n}", z))
    return out


def _max_db(x):
    return float(O.frame_db(x).max()) if x.size >= O.FRAME else -np.inf


def test_rows_meet_the_precondition():
    for name, x in _rows():
        assert _max_db(x) <= 0.0, name


@pytest.mark.parametrize("schedule", SCHEDULES)
def test_causal_oracle_equals_the_one_shot_extent_and_join(schedule):
    named = _rows()
    rows = [x for _n, x in named]
    for name, x in named:
        d = S.stream_extent(x, schedule if schedule is not None else x.size)
        assert (d["start"], d["end"]) == O.extent(x), (name, schedule)
    sched = schedule if schedule is not None else [[x.size] for x in rows]
    for P in (0, 6000):
        got, _det = S.stream_join(rows, sched, P)
        want = O.join(rows, [O.extent(x) for x in rows], P)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (schedule, P)


def _causal_by_hand(x):
    """The causal rule written out frame by frame, independently of stream_extent's bookkeeping."""
    db = O.frame_db(x)
    voiced = []
    for k in range(db.size):
        thr = max(db[: k + 1].max() - 40.0, -40.0)
        if db[k] > thr:
            voiced.append(k)
    n = x.size
    s, e = max(0, voiced[0] * 240 - 720), min(n, voiced[-1] * 240 + 1320)
    return (s, e) if e - s >= 12000 else (0, n)


def test_a_row_above_full_scale_takes_the_causal_rule():
    """Quiet speech at about -33 dB, then a burst at about +6 dB: one-shot, the threshold is -34 dB and the quiet part
    keeps only its loudest frames; causally, the quiet part was classified against -40 dB before the burst came."""
    g = np.random.default_rng(3)
    x = np.zeros(80000, dtype=np.float32)
    x[10000:40000] = (0.022 * g.standard_normal(30000)).astype(np.float32)
    x[50000:60000] = (2.0 * g.standard_normal(10000)).astype(np.float32)
    assert _max_db(x) > 0.0
    want = _causal_by_hand(x)
    for schedule in SCHEDULES:
        d = S.stream_extent(x, schedule if schedule is not None else x.size)
        assert (d["start"], d["end"]) == want, schedule
    assert want != O.extent(x)
    assert want[0] < O.extent(x)[0]


@pytest.mark.parametrize("schedule", (1, 240, 601, 11520))
def test_bounds_follow_the_certain_prefix(schedule):
    for name, x in _rows():
        st = S.stream_extent(x, schedule)["status"]
        db = O.frame_db(x) if x.size >= O.FRAME else np.zeros(0)
        prev = None
        for i, (n, decided, start, avail, final) in enumerate(st):
            assert final == (i == len(st) - 1)
            K = (n - 600) // 240 + 1 if n >= 600 else 0
            M = -np.inf
            voiced = []
            for k in range(K):
                M = max(M, db[k])
                if db[k] > max(M - 40, -40):
                    voiced.append(k)
            if final:
                assert decided and (start, avail) == O.extent(x), name
                continue
            if voiced:
                s, e = max(0, voiced[0] * 240 - 720), min(n, voiced[-1] * 240 + 1320)
                if e - s >= 12000:
                    assert (decided, start, avail) == (1, s, e - 240), (name, n)
                    if prev is not None and prev[1]:
                        assert start == prev[2] and avail >= prev[3]  # the start is fixed, the bound only grows
                    prev = (n, decided, start, avail)
                    continue
            assert (decided, start, avail) == (0, 0, 0), (name, n)  # nothing before end_p - start >= 12000
            assert prev is None or not prev[1]
            prev = (n, decided, start, avail)


def test_whole_row_cases_are_released_only_at_the_end():
    g = np.random.default_rng(9)
    cases = {"short": (0.3 * g.standard_normal(2399)).astype(np.float32), "silent": np.zeros(30000, dtype=np.float32),
             "narrow": np.zeros(30000, dtype=np.float32)}
    cases["narrow"][10000:12000] = 0.3  # voiced span under 12000 samples
    for name, x in cases.items():
        for schedule in (1, 240, 11520):
            st = S.stream_extent(x, schedule)["status"]
            assert all(s[1] == 0 for s in st[:-1]), name
            assert st[-1] == (x.size, 1, 0, x.size, 1), name


def test_pauses_only_ahead_of_a_later_span():
    """Zero-sample and whole-silence rows: the pause goes between non-empty spans only, never before the first or after
    the last (the join's layout)."""
    g = np.random.default_rng(4)
    a = (0.3 * g.standard_normal(20000)).astype(np.float32)
    empty = np.zeros(0, dtype=np.float32)
    rows = [empty, a, empty, a[:5000], empty]
    got, det = S.stream_join(rows, 601, 1000)
    assert got.size == 20000 + 1000 + 5000
    assert np.all(got[20000:21000] == 0)
    assert [(d["start"], d["end"]) for d in det] == [(0, 0), (0, 20000), (0, 0), (0, 5000), (0, 0)]


# ---- SoproTTS.stream_long's signature and refusals

def test_stream_long_signature():
    from sopro_b200 import SoproTTS

    p = inspect.signature(SoproTTS.stream_long).parameters
    want = dict(seed=None, max_frames=400, max_tokens=64, pause_ms=250, top_p=0.9, temperature=1.05, anti_loop=True,
                style_strength=None, min_gen_frames=None, chunk_frames=6, nar_context_frames=None, sample_rate=None,
                speed=None, watermark=None)
    for k, v in want.items():
        assert p[k].default == v and p[k].kind == inspect.Parameter.KEYWORD_ONLY, k
    assert p["ref"].kind == inspect.Parameter.KEYWORD_ONLY and p["ref"].default is inspect.Parameter.empty
    for k in ("loudness", "best_of", "word_timestamps"):
        assert k not in p


@pytest.mark.parametrize("kw,err", [(dict(pause_ms=-1), ValueError), (dict(pause_ms=2500), ValueError),
                                    (dict(pause_ms=float("nan")), ValueError), (dict(pause_ms=True), ValueError),
                                    (dict(max_tokens=3), ValueError), (dict(max_tokens=5000), ValueError),
                                    (dict(max_tokens=8.0), ValueError), (dict(chunk_frames=0), ValueError),
                                    (dict(chunk_frames=257), ValueError), (dict(chunk_frames=6.0), TypeError),
                                    (dict(sample_rate=3999), ValueError), (dict(speed=5.0), ValueError),
                                    (dict(watermark=-1), ValueError), (dict(text=""), ValueError),
                                    (dict(text=" \n\n \t"), ValueError)])
def test_refused_arguments_raise_at_the_call_before_any_work(kw, err):
    """This object has no engines, no codec and no device: any work past the checks would fail differently."""
    from types import SimpleNamespace

    from sopro_b200.model import SoproTTS

    tts = SoproTTS.__new__(SoproTTS)
    tts._resamplers = {}
    tts.tokenizer = IdsTokenizer(1000)
    tts.model = SimpleNamespace(prefill=SimpleNamespace(max_text_len=2056))
    kw = dict(kw)
    text = kw.pop("text", "1 2. 3 4.")
    torch.manual_seed(5)
    before = torch.get_rng_state()
    with pytest.raises(err):
        tts.stream_long(text, ref=None, **kw)
    assert torch.equal(before, torch.get_rng_state())
