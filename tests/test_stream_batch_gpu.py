"""GPU: SoproTTS.stream_batch and the batched Mimi stream step.  Every row must equal its own one-row run bit for bit:
the Mimi rows against a one-row stream (and, in fp32, the one-shot decode), the stream_batch rows against stream()."""
import pytest
import torch

from oracle import mimi_oracle as M

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
_TTS = {}
MODES = ["fp32", "bf16_tc"]


def _tts():
    """A synthetic checkpoint whose EOS is a few times more likely than a code, so lengths are ragged."""
    if "t" not in _TTS:
        from sopro_b200 import SoproTTS
        from sopro_b200.config import SoproTTSConfig
        from sopro_b200.tokenizer import IdsTokenizer
        from sopro_b200.weights import synth_state_dict

        cfg = SoproTTSConfig()
        sd = synth_state_dict(cfg, text_vocab=1000, seed=0)
        sd["ar.head.bias"] = sd["ar.head.bias"].clone()
        sd["ar.head.bias"][int(cfg.codebook_size)] += 2.5
        t = SoproTTS.from_state_dict(cfg, sd, IdsTokenizer(1000), M.synth_mimi_state_dict(), device="cuda:0")
        _TTS["t"] = t
        _TTS["refs"] = [t.prepare_reference(ref_tokens_tq=torch.randint(0, 2048, (n, 32), generator=torch.Generator().manual_seed(s)))
                        for n, s in ((38, 7), (25, 8), (50, 9))]
    return _TTS["t"], _TTS["refs"]


TEXTS = [" ".join(str((13 * i + 7 * j + 1) % 997) for i in range(n)) for j, n in enumerate((6, 20, 11, 30, 3))]
FRAMES = 40


def _seeds(tts, ref, texts, kw):
    """One seed per text, from a fixed pool, such that one text reaches max_frames and another ends by EOS
    (synthesize_batch gives each row's length; rows do not depend on each other)."""
    n = int(kw["max_frames"]) + 1
    lens = {}
    for s in range(100, 140):
        lens[s] = [int(w.shape[-1]) // 1920 for w in tts.synthesize_batch(texts, ref=ref, seeds=[s] * len(texts), **kw)]
        full = [(s_, i) for s_ in lens for i, x in enumerate(lens[s_]) if x == n]
        eos = [(s_, i) for s_ in lens for i, x in enumerate(lens[s_]) if x < n]
        for sf, i in full:
            for se, j in eos:
                if j != i:
                    seeds = [se] * len(texts)
                    seeds[i] = sf
                    return seeds
    raise AssertionError(f"no seeds with an EOS row and a full row: {lens}")


def _rows(items, n):
    wavs, flags, order = [[] for _ in range(n)], [[] for _ in range(n)], []
    for i, w, last in items:
        assert w.dim() == 2 and w.shape[0] == 1 and w.device.type == "cuda"
        assert last or w.shape[1] > 0, "only a row's last item may be empty"
        wavs[i].append(w)
        flags[i].append(last)
        order.append(i)
    for f in flags:
        assert f and f[-1] and not any(f[:-1]), "each row ends with exactly one last item"
    return wavs


def _same_as_stream(row, solo):
    got = row if row[-1].shape[1] > 0 else row[:-1]
    assert [w.shape for w in got] == [w.shape for w in solo]
    for a, b in zip(got, solo):
        assert torch.equal(a, b)


@pytest.mark.parametrize("mode", MODES)
def test_batched_mimi_step_rows_equal_one_row_streams(mode):
    from sopro_b200.codec import MimiEngine

    if "mimi" not in _TTS:
        _TTS["mimi"] = MimiEngine(M.synth_mimi_state_dict(), 0, 32)
    eng = _TTS["mimi"]
    eng.set_precision(mode)
    R, T = 5, 310
    codes = torch.randint(0, 2048, (R, 32, T), generator=torch.Generator().manual_seed(55)).to(torch.int32).cuda()
    ended = 170  # row 4 ends here and is fed code 0 afterwards
    fed = codes.clone()
    fed[4, :, ended:] = 0
    sizes, pos, i, parts = [1, 6, 1, 16, 3, 40, 6, 1, 64, 6], 0, 0, []
    st = eng.stream(16, rows=R)
    assert st.rows == R and st.state_bytes > 0
    while pos < T:
        n = min(sizes[i % len(sizes)], T - pos)
        parts.append(st.step(fed[:, :, pos:pos + n]))
        pos, i = pos + n, i + 1
    got = torch.cat(parts, dim=1)
    assert got.shape == (R, T * 1920) and st.frames == T
    for b in range(R):
        one = eng.stream(16)
        n = ended if b == 4 else T
        want = torch.cat([one.step(codes[b, :, a:min(a + 7, n)]) for a in range(0, n, 7)], dim=1)
        assert torch.equal(got[b: b + 1, : n * 1920], want), f"row {b}"
        if mode == "fp32":
            assert torch.equal(got[b, : n * 1920], eng.decode(codes[b: b + 1, :, :n]).reshape(-1)), f"row {b} vs decode"
    # one-row input shape of a one-row state is [Q, n], and a many-row state refuses it
    with pytest.raises(ValueError):
        st.step(codes[0, :, :2])


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("chunk_frames", [1, 6, 16])
def test_stream_batch_rows_equal_stream(mode, chunk_frames):
    tts, refs = _tts()
    ref = refs[0]
    kw = dict(max_frames=FRAMES, min_gen_frames=3)
    if "seeds" not in _TTS:
        _TTS["seeds"] = _seeds(tts, ref, TEXTS, kw)
    seeds = _TTS["seeds"]
    tts.codec.engine.set_precision(mode)
    try:
        rows = _rows(tts.stream_batch(TEXTS, ref=ref, seeds=seeds, chunk_frames=chunk_frames, **kw), len(TEXTS))
        lens = []
        for i, (text, seed) in enumerate(zip(TEXTS, seeds)):
            solo = list(tts.stream(text, ref=ref, seed=seed, chunk_frames=chunk_frames, **kw))
            _same_as_stream(rows[i], solo)
            lens.append(sum(int(w.shape[1]) for w in solo) // 1920)
        assert FRAMES + 1 in lens and min(lens) < FRAMES + 1, lens
    finally:
        tts.codec.engine.set_precision("bf16_tc")


def test_a_voice_per_text():
    tts, refs = _tts()
    texts = TEXTS[:4]
    ref = [refs[0], refs[1], refs[2], refs[0]]  # the last text shares the first one's voice object
    seeds = [3, 4, 5, 6]
    kw = dict(max_frames=FRAMES, min_gen_frames=3, chunk_frames=6)
    rows = _rows(tts.stream_batch(texts, ref=ref, seeds=seeds, **kw), len(texts))
    for i in range(len(texts)):
        _same_as_stream(rows[i], list(tts.stream(texts[i], ref=ref[i], seed=seeds[i], **kw)))


def test_output_chain_per_row():
    tts, refs = _tts()
    kw = dict(max_frames=FRAMES, min_gen_frames=3, chunk_frames=6, sample_rate=16000, speed=1.25, watermark=0xC0FFEE)
    seeds = [21, 22, 23]
    rows = _rows(tts.stream_batch(TEXTS[:3], ref=refs[1], seeds=seeds, **kw), 3)
    for i in range(3):
        _same_as_stream(rows[i], list(tts.stream(TEXTS[i], ref=refs[1], seed=seeds[i], **kw)))


def test_a_batch_larger_than_64():
    tts, refs = _tts()
    B = 130
    texts = [TEXTS[i % len(TEXTS)] for i in range(B)]
    seeds = list(range(500, 500 + B))
    kw = dict(max_frames=12, min_gen_frames=3, chunk_frames=6)
    rows = _rows(tts.stream_batch(texts, ref=refs[2], seeds=seeds, **kw), B)
    for i in (0, 63, 64, 97, 129):
        _same_as_stream(rows[i], list(tts.stream(texts[i], ref=refs[2], seed=seeds[i], **kw)))


def test_closing_early_leaves_nothing_behind():
    tts, refs = _tts()
    ref = refs[0]
    kw = dict(max_frames=FRAMES, min_gen_frames=10 ** 9, chunk_frames=6)
    seeds = [31, 32, 33, 34, 35]
    fresh = _rows(tts.stream_batch(TEXTS, ref=ref, seeds=seeds, **kw), len(TEXTS))
    fresh_solo = list(tts.stream(TEXTS[1], ref=ref, seed=7, **kw))
    fresh_syn = tts.synthesize(TEXTS[2], ref=ref, seed=8, max_frames=FRAMES)
    gen = tts.stream_batch(TEXTS, ref=ref, seeds=seeds, **kw)
    first = [next(gen) for _ in TEXTS]  # the first chunk cycle: one chunk per row
    assert [i for i, _w, _l in first] == list(range(len(TEXTS)))
    gen.close()
    assert not tts.model._sessions_busy
    batch = tts.stream_batch(TEXTS, ref=ref, seeds=seeds, **kw)
    solo = tts.stream(TEXTS[1], ref=ref, seed=7, **kw)
    items, solo_chunks, syn = [], [], None
    b_done = s_done = False
    while not (b_done and s_done):
        if not b_done:
            try:
                items.append(next(batch))
            except StopIteration:
                b_done = True
        if not s_done:
            try:
                solo_chunks.append(next(solo))
            except StopIteration:
                s_done = True
        if syn is None:
            syn = tts.synthesize(TEXTS[2], ref=ref, seed=8, max_frames=FRAMES)
    rows = _rows(items, len(TEXTS))
    for i in range(len(TEXTS)):
        assert [w.shape for w in rows[i]] == [w.shape for w in fresh[i]]
        assert all(torch.equal(a, b) for a, b in zip(rows[i], fresh[i]))
    assert len(solo_chunks) == len(fresh_solo) and all(torch.equal(a, b) for a, b in zip(solo_chunks, fresh_solo))
    assert torch.equal(syn, fresh_syn)
