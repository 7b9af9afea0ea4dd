"""Host-side control flow of SoproTTS.stream_batch WITHOUT a GPU, through the oracle-backed fakes of
test_host_pipeline_cpu.py: rows against stream(), the shared NAR windows, the refusals, the one-row case and the global
generator.  The Mimi fake gains a row dimension: each row is decoded by the oracle over its own code history."""
import pytest
import torch

from sopro_b200.streaming import MAX_STREAM_ROWS
from tests.test_host_pipeline_cpu import _FakeMimiEngine, _FakeMimiStream, tts  # noqa: F401  (the fixture)

torch.set_grad_enabled(False)

TEXTS = ["3 14 15 92 65 35", " ".join(str(7 * i + 1) for i in range(15)), "27 18 28 18"]
SEEDS = [2, 5, 9]
KW = dict(max_frames=20, min_gen_frames=3, chunk_frames=4)


class _RowsMimiStream:
    """MimiStream of `rows` rows: row b's samples are the oracle decode of row b's code history.  The frames of code 0
    a row is fed after its end are left out of that decode (their samples are zeros): the CUDA decoder is causal bit
    for bit, the oracle's CPU convolutions over a longer sequence are not."""

    def __init__(self, eng, rows):
        self.eng, self.rows, self.hist = eng, rows, None

    def reset(self):
        self.hist = None

    def step(self, codes, trusted=False):
        assert codes.dim() == 3 and codes.shape[0] == self.rows
        self.hist = codes if self.hist is None else torch.cat([self.hist, codes], dim=2)
        T = self.hist.shape[2]
        wav = torch.zeros(self.rows, T * 1920)
        for b in range(self.rows):
            live = self.hist[b].ne(0).any(dim=0).nonzero()
            n = int(live[-1]) + 1 if live.numel() else 0
            if n:
                wav[b, : n * 1920] = self.eng.decode(self.hist[b: b + 1, :, :n]).reshape(-1)
        return wav[:, (self.hist.shape[2] - codes.shape[2]) * 1920:]


class _RowsMimiEngine(_FakeMimiEngine):
    def stream(self, max_chunk_frames=16, rows=1):
        return _FakeMimiStream(self) if rows == 1 else _RowsMimiStream(self, rows)


@pytest.fixture(scope="module")
def btts(tts):  # noqa: F811
    tts.codec.engine = _RowsMimiEngine(tts.codec.engine.msd)
    tts.__dict__.pop("_stream_decoder", None)
    return tts


def _rows(items, n):
    """stream_batch items -> per row (the wavs in order, the flags in order); checks the row order within a cycle"""
    wavs, flags = [[] for _ in range(n)], [[] for _ in range(n)]
    for i, w, last in items:
        assert w.dim() == 2 and w.shape[0] == 1
        assert last or w.shape[1] > 0, "only a row's last item may be empty"
        wavs[i].append(w)
        flags[i].append(last)
    for f in flags:
        assert f and f[-1] and not any(f[:-1]), "each row ends with exactly one last item"
    return wavs


def _same_as_stream(row_wavs, solo):
    """a row's items against list(stream(...)): the last item is the stream's final chunk, or empty"""
    got = row_wavs if row_wavs[-1].shape[1] > 0 else row_wavs[:-1]
    assert len(got) == len(solo), ([w.shape for w in got], [w.shape for w in solo])
    for a, b in zip(got, solo):
        assert torch.equal(a, b)


def test_rows_equal_stream(btts):
    items = list(btts.stream_batch(TEXTS, ref=btts.ref, seeds=SEEDS, **KW))
    rows = _rows(items, len(TEXTS))
    lens = []
    for i, (text, seed) in enumerate(zip(TEXTS, SEEDS)):
        solo = list(btts.stream(text, ref=btts.ref, seed=seed, **KW))
        _same_as_stream(rows[i], solo)
        lens.append(sum(w.shape[1] for w in solo))
    assert len(set(lens)) >= 2, f"the case must produce ragged rows, got {lens}"
    # within a chunk cycle the rows come in index order
    cycle, prev = [], -1
    for i, _w, _l in items:
        if i <= prev:
            cycle = []
        cycle.append(i)
        prev = i
        assert cycle == sorted(cycle)


def test_nar_windows_follow_the_reference(btts, monkeypatch):
    """Every row's NAR windows are those of its solo stream (reference streaming.py:80-104); the live rows of a chunk
    share one call, in row order, each with its own length."""
    cf, ctx = KW["chunk_frames"], 3
    want = []
    for text, seed in zip(TEXTS, SEEDS):
        prep = btts.model.prepare_conditioning(btts.encode_text(text), btts.ref, max_frames=KW["max_frames"],
                                               style_strength=btts.cfg.style_strength)
        toks = []
        for _t, tok, is_eos in btts.model.ar_stream(prep, seed=seed, max_frames=KW["max_frames"],
                                                    min_gen_frames=KW["min_gen_frames"]):
            if is_eos:
                break
            toks.append(tok)
        T = len(toks)
        ends = list(range(cf, T + 1, cf)) + ([T] if T % cf else [])
        wins, emitted = [], 0
        for e in ends:
            lo = max(0, emitted - ctx)
            wins.append(toks[lo:e])
            emitted = e
        want.append(wins)
    seen = []
    real = btts.model.nar_refine

    def spy(cond, rvq1, lens=None):
        n = [int(rvq1.shape[1])] * int(rvq1.shape[0]) if lens is None else [int(x) for x in lens]
        assert int(cond.shape[1]) == int(rvq1.shape[1]) == max(n)
        seen.append([rvq1[j, : n[j]].tolist() for j in range(int(rvq1.shape[0]))])
        return real(cond, rvq1, lens)

    monkeypatch.setattr(btts.model, "nar_refine", spy)
    list(btts.stream_batch(TEXTS, ref=btts.ref, seeds=SEEDS, nar_context_frames=ctx, **KW))
    calls = [[w[k] for w in want if k < len(w)] for k in range(max(len(w) for w in want))]
    assert seen == calls


@pytest.mark.parametrize("case", ["empty", "seeds", "ref_len", "ref_type", "chunk_low", "chunk_high", "rate", "speed",
                                  "watermark", "rows"])
def test_refusals_leave_the_generator_untouched(btts, case):
    r = btts.ref
    kw = dict(ref=r, max_frames=20)
    texts = TEXTS
    err = ValueError
    if case == "empty":
        texts = []
    elif case == "seeds":
        kw["seeds"] = [1, 2]
    elif case == "ref_len":
        kw["ref"] = [r, r]
    elif case == "ref_type":
        kw["ref"], err = [r, "voice.wav", r], TypeError
    elif case == "chunk_low":
        kw["chunk_frames"] = 0
    elif case == "chunk_high":
        kw["chunk_frames"] = 257
    elif case == "rate":
        kw["sample_rate"] = 7
    elif case == "speed":
        kw["speed"] = 9.0
    elif case == "watermark":
        kw["watermark"] = -1
    elif case == "rows":
        texts = ["1 2"] * (MAX_STREAM_ROWS + 1)
    torch.manual_seed(123)
    before = torch.get_rng_state()
    with pytest.raises(err):
        btts.stream_batch(texts, **kw)
    assert torch.equal(torch.get_rng_state(), before)


def test_batch_of_one_is_stream_including_the_generator(btts):
    torch.manual_seed(31)
    solo = list(btts.stream(TEXTS[1], ref=btts.ref, **KW))
    after_solo = torch.get_rng_state()
    torch.manual_seed(31)
    rows = _rows(btts.stream_batch([TEXTS[1]], ref=btts.ref, **KW), 1)
    assert torch.equal(torch.get_rng_state(), after_solo)
    _same_as_stream(rows[0], solo)
    # seeded: the generator is not touched at all
    before = torch.get_rng_state()
    rows = _rows(btts.stream_batch([TEXTS[0]], ref=btts.ref, seeds=[4], **KW), 1)
    assert torch.equal(torch.get_rng_state(), before)
    _same_as_stream(rows[0], list(btts.stream(TEXTS[0], ref=btts.ref, seed=4, **KW)))


def test_unseeded_rows_draw_as_synthesize_batch(btts):
    torch.manual_seed(77)
    btts.synthesize_batch(TEXTS, ref=btts.ref, max_frames=KW["max_frames"], min_gen_frames=KW["min_gen_frames"])
    want = torch.get_rng_state()
    torch.manual_seed(77)
    _rows(btts.stream_batch(TEXTS, ref=btts.ref, **KW), len(TEXTS))
    assert torch.equal(torch.get_rng_state(), want)


def test_closing_early_releases_everything(btts):
    gen = btts.stream_batch(TEXTS, ref=btts.ref, seeds=SEEDS, **KW)
    next(gen)
    gen.close()
    assert not btts.model._sessions_busy
    rows = _rows(btts.stream_batch(TEXTS, ref=btts.ref, seeds=SEEDS, **KW), len(TEXTS))
    _same_as_stream(rows[0], list(btts.stream(TEXTS[0], ref=btts.ref, seed=SEEDS[0], **KW)))
