"""GPU: stream_long's streaming trim stage (sopro_b200/longform.py::StreamJoin) against the causal oracle
(oracle/longform_stream_oracle.py::stream_extent) push by push and against the one-shot extents + join bit for bit, and
SoproTTS.stream_long against the join of stream_batch's rows through the output chain."""
import numpy as np
import pytest
import torch

from oracle import longform_oracle as O
from oracle import longform_stream_oracle as S
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
    """test_longform_gpu.py's row families: the audio_prep.json recipes at 24 kHz, noise, silence, a Mimi decode
    alone and padded with silence, bursts between silences, a loud + quiet + silent row, and the length edges."""
    from tests.golden.make_audio_golden import CASES, signal

    g = np.random.default_rng(11)
    out = [signal(24000, n, lo, hi, floor, i)[0].numpy() for i, (_name, _sr, n, lo, hi, floor) in enumerate(CASES)]
    out.append((0.3 * g.standard_normal(50000)).astype(np.float32))
    out.append(np.zeros(40000, dtype=np.float32))
    m = _mimi_wav()
    pad = np.zeros(30000, dtype=np.float32)
    out += [m, np.concatenate([pad, m, pad])]
    y = np.zeros(70000, dtype=np.float32)
    for a in (15000, 31000, 44000):
        y[a: a + 6000] = (0.2 * g.standard_normal(6000)).astype(np.float32)
    out.append(y)
    x = (0.9 * g.standard_normal(90000)).astype(np.float32)
    x[30000:60000] *= 0.03
    x[60000:] = 0
    out.append(x)
    for n in (599, 600, 2399, 2400, 11999, 12000, 12001, 30000):
        z = np.zeros(n, dtype=np.float32)
        k = n // 4
        z[n // 3: n // 3 + k] = (0.5 * g.standard_normal(k)).astype(np.float32)
        out.append(z)
    out.append(np.zeros(0, dtype=np.float32))
    return out


def _schedule(n, kind, b):
    """Row b's pushes over n samples: fixed sizes, sizes that vary by row, and sizes with empty pushes between."""
    if kind == "fixed":
        sizes = [min(11520, n - a) for a in range(0, n, 11520)]
    elif kind == "ragged":
        step = (601, 239, 1920 * 3, 240, 7000)[b % 5]
        sizes = [min(step, n - a) for a in range(0, n, step)]
    else:  # "gaps"
        sizes = []
        for a in range(0, n, 3840):
            sizes += [min(3840, n - a)] + [0] * ((a // 3840 + b) % 3)
    return sizes or [0]


def _near_threshold(x, status):
    """Whether a frame of x lies within 1e-9 dB of a threshold the causal rule used (then a last-bit difference between
    the device's and numpy's dB may decide it either way; test_longform_gpu._agrees's allowance)."""
    if x.size < O.FRAME:
        return False
    db = O.frame_db(x)
    thr = np.maximum(np.maximum.accumulate(db) - 40.0, -40.0)
    return bool(np.abs(db - thr).min() <= 1e-9)


def _drive(rows, kind, P, limit=11520):
    """Push the rows as one ragged batch per launch (row b's schedule, 0 once it has ended) and take what is certain
    after every push -> (the passage, the status after every push per row, the oracle's)."""
    from sopro_b200.longform import StreamJoin

    B = len(rows)
    sched = [_schedule(r.size, kind, b) for b, r in enumerate(rows)]
    T = max(len(s) for s in sched)
    join = StreamJoin(B, max(max(r.size for r in rows), 1), "cuda:0")
    join.begin(B, P, B)
    join.start_group(0, B)
    dev = [torch.from_numpy(r).cuda() for r in rows]
    pos = [0] * B
    got, seen = [], [[] for _ in range(B)]
    for t in range(T):
        counts = [sched[b][t] if t < len(sched[b]) else 0 for b in range(B)]
        final = [t == len(sched[b]) - 1 for b in range(B)]
        w = max(max(counts), 1)
        x = torch.full((B, w), float("nan"), device="cuda")
        for b in range(B):
            if counts[b]:
                x[b, : counts[b]] = dev[b][pos[b]: pos[b] + counts[b]]
                pos[b] += counts[b]
        join.push(x, counts, final)
        torch.cuda.synchronize()
        for b in range(B):
            if t < len(sched[b]):
                seen[b].append(join.status(b))
        while True:
            y = join.take(limit)
            if y is None:
                break
            assert 0 < y.shape[1] <= limit
            got.append(y)
    assert join.done()
    join.close()
    passage = torch.cat(got, dim=1).reshape(-1) if got else torch.zeros(0, device="cuda")
    want = [S.stream_extent(r, s)["status"] for r, s in zip(rows, sched)]
    return passage, seen, want


@pytest.mark.parametrize("kind", ("fixed", "ragged", "gaps"))
@pytest.mark.parametrize("P", (0, 6000))
def test_stage_equals_the_one_shot_join_and_the_oracle_push_by_push(kind, P):
    from sopro_b200.longform import join_segments, speech_extents

    rows = _rows()
    for r in rows:
        assert r.size < O.FRAME or O.frame_db(r).max() <= 0.0
    passage, seen, want = _drive(rows, kind, P)
    dev = [torch.from_numpy(r).cuda() for r in rows]
    ext = torch.cat([speech_extents(d) if d.numel() else torch.zeros(1, 2, dtype=torch.int64, device="cuda") for d in dev])
    one = join_segments(dev, ext, P / 24.0).reshape(-1)
    assert passage.shape == one.shape and torch.equal(passage.view(torch.int32), one.view(torch.int32))
    exact = 0
    for r, s, w in zip(rows, seen, want):
        if [tuple(v) for v in w] == s:
            exact += 1
        else:
            assert _near_threshold(r, w), (s, w)
    assert exact >= len(rows) - 2, exact


def test_rows_above_full_scale_follow_the_causal_rule():
    """Rows scaled above 0 dB, and quiet speech followed by a loud burst (where the causal extent starts earlier than
    the one-shot one): the extents are the causal oracle's, and the passage is the join of those extents."""
    g = np.random.default_rng(3)
    x = np.zeros(80000, dtype=np.float32)
    x[10000:40000] = (0.022 * g.standard_normal(30000)).astype(np.float32)
    x[50000:60000] = (2.0 * g.standard_normal(10000)).astype(np.float32)
    rows = [x] + [(8.0 * r).astype(np.float32) for r in _rows()[:-1] if r.size >= 12000]
    assert sum(O.frame_db(r).max() > 0.0 for r in rows) >= 3
    for kind in ("fixed", "gaps"):
        passage, seen, want = _drive(rows, kind, 6000)
        ext = []
        for r, s, w in zip(rows, seen, want):
            if [tuple(v) for v in w] != s:
                assert _near_threshold(r, w), (s, w)
            ext.append((s[-1][2], s[-1][3]))
        assert ext[0] == (want[0][-1][2], want[0][-1][3]) and ext[0] != O.extent(x)
        replay = O.join(rows, ext, 6000)
        assert np.array_equal(passage.cpu().numpy().view(np.uint32), replay.view(np.uint32))


def test_stage_refusals():
    from sopro_b200.longform import StreamJoin

    j = StreamJoin(2, 1000, "cuda:0")
    j.begin(2, 0, 2)
    j.start_group(0, 2)
    x = torch.zeros(2, 800, device="cuda")
    j.push(x, [800, 1], [False, False])
    with pytest.raises(ValueError):
        j.push(x, [800, 0], [False, False])  # 1600 samples > the capacity of 1000
    j.push(x[:, :10].contiguous(), [10, 10], [True, False])
    with pytest.raises(ValueError):
        j.push(x[:, :10], [1, 0], [False, False])  # a final row takes no more samples
    with pytest.raises(ValueError):
        j.push(x[:, :10], [0, 1], [False])
    j.close()


# ---- through the public API

TEXT = "3 7 11 15. 5 9 13 17 21! 4 8?\n\n6 2 10 12 14 16 18 20 22 24, 26 28 30. 1 5 9."
FRAMES = 40
KW = dict(max_frames=FRAMES, min_gen_frames=3, max_tokens=7)


def _api():
    from tests.test_stream_batch_gpu import _tts

    tts, refs = _tts()
    return tts, refs[0]


def _want(tts, ref, seed, chunk_frames, pause_ms=250, sample_rate=None, speed=None, watermark=None):
    """The chain applied to the join of stream_batch's rows (row i with seed + i), and those rows."""
    from sopro_b200.longform import join_segments, speech_extents, split_text
    from sopro_b200.output import OutputChain

    segs = split_text(TEXT, tts.tokenizer, KW["max_tokens"])
    rows = [[] for _ in segs]
    for i, w, _last in tts.stream_batch(segs, ref=ref, seeds=[seed + i for i in range(len(segs))],
                                        chunk_frames=chunk_frames, max_frames=FRAMES, min_gen_frames=3):
        rows[i].append(w)
    rows = [torch.cat(r, dim=1).reshape(-1) for r in rows]
    ext = torch.cat([speech_extents(r) if r.numel() else torch.zeros(1, 2, dtype=torch.int64, device="cuda") for r in rows])
    wav = join_segments(rows, ext, pause_ms)
    if wav.shape[-1]:
        wav, _ = OutputChain(tts, sample_rate, speed, watermark=watermark)(wav)
    return wav.reshape(1, -1), rows


def _check_rows(rows):
    """The contract's precondition, so that the comparison is not vacuous: rows of several lengths, no frame above
    0 dB."""
    lens = [int(r.numel()) for r in rows]
    assert len(rows) >= 5 and len(set(lens)) >= 3, lens
    for r in rows:
        if r.numel() >= O.FRAME:
            assert O.frame_db(r.cpu().numpy()).max() <= 0.0


def _got(tts, ref, seed, chunk_frames, **kw):
    items = list(tts.stream_long(TEXT, ref=ref, seed=seed, chunk_frames=chunk_frames, **KW, **kw))
    for y in items:
        assert y.dim() == 2 and y.shape[0] == 1 and y.shape[1] > 0 and y.device.type == "cuda"
    return torch.cat(items, dim=1) if items else torch.zeros(1, 0, device="cuda"), items


@pytest.mark.parametrize("mode", ("fp32", "bf16_tc"))
@pytest.mark.parametrize("chunk_frames", (1, 6, 16))
def test_stream_long_equals_the_join_of_stream_batch_rows(monkeypatch, mode, chunk_frames):
    import sopro_b200.longform as LF

    tts, ref = _api()
    monkeypatch.setattr(LF, "SEGMENT_GROUP", 2)  # several groups, two slots reused
    tts.codec.engine.set_precision(mode)
    try:
        got, items = _got(tts, ref, 40, chunk_frames)
        want, rows = _want(tts, ref, 40, chunk_frames)
    finally:
        tts.codec.engine.set_precision("bf16_tc")
    _check_rows(rows)
    assert max(y.shape[1] for y in items) <= chunk_frames * 1920
    assert got.shape == want.shape and torch.equal(got, want)


@pytest.mark.parametrize("chain", (dict(sample_rate=16000), dict(speed=1.25), dict(watermark=0xC0FFEE)))
def test_output_chain_runs_on_the_joined_passage(monkeypatch, chain):
    import sopro_b200.longform as LF

    tts, ref = _api()
    monkeypatch.setattr(LF, "SEGMENT_GROUP", 2)
    got, _ = _got(tts, ref, 7, 6, pause_ms=100, **chain)
    want, rows = _want(tts, ref, 7, 6, pause_ms=100, **chain)
    _check_rows(rows)
    assert got.shape == want.shape and torch.equal(got, want)


def test_one_chunk_in_fp32_equals_synthesize_long():
    tts, ref = _api()
    tts.codec.engine.set_precision("fp32")
    try:
        got, _ = _got(tts, ref, 11, 64)
        want = tts.synthesize_long(TEXT, ref=ref, seed=11, **KW)
    finally:
        tts.codec.engine.set_precision("bf16_tc")
    assert got.shape[1] == want.shape[-1] and torch.equal(got.reshape(-1), want.reshape(-1))


def test_unseeded_groups_draw_as_stream_batch(monkeypatch):
    import sopro_b200.longform as LF

    tts, ref = _api()
    monkeypatch.setattr(LF, "SEGMENT_GROUP", 3)
    segs = LF.split_text(TEXT, tts.tokenizer, KW["max_tokens"])
    torch.manual_seed(17)
    got, _ = _got(tts, ref, None, 6)
    after = torch.get_rng_state()
    torch.manual_seed(17)
    for g0 in range(0, len(segs), 3):
        list(tts.stream_batch(segs[g0: g0 + 3], ref=ref, chunk_frames=6, max_frames=FRAMES, min_gen_frames=3))
    assert torch.equal(after, torch.get_rng_state())
    assert got.shape[1] > 0


def test_closing_early_leaves_the_pools_able_to_serve(monkeypatch):
    import sopro_b200.longform as LF

    tts, ref = _api()
    monkeypatch.setattr(LF, "SEGMENT_GROUP", 2)
    fresh, _ = _got(tts, ref, 40, 6)
    gen = tts.stream_long(TEXT, ref=ref, seed=40, chunk_frames=6, **KW)
    next(gen)
    gen.close()
    assert not tts.model._sessions_busy
    assert tts._join_pool._idle
    again, _ = _got(tts, ref, 40, 6)
    assert torch.equal(again, fresh)
