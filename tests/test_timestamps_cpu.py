"""CPU: word timestamps -- the float64 alignment DP (oracle/align_oracle.py) on planted paths, an exact tie and the edge
geometries; tokens to words with both tokenizers; frames to seconds with speed and through synthesize_long's join."""
import numpy as np
import pytest

from oracle import align_oracle as O
from sopro_b200 import timestamps as TS
from sopro_b200.tokenizer import IdsTokenizer


def _probs_from_path(first, T, L, n_attn=2, H=3, ld=None, noise=0.0, seed=0):
    """A trace [T, n_attn, 1, H, ld] whose weights put 1 / (n_attn H) on the planted token of every frame."""
    ld = ld or L
    g = np.random.default_rng(seed)
    p = (noise * g.random((T, n_attn, 1, H, ld))).astype(np.float32)
    bounds = list(first) + [T]
    for l in range(L):
        p[bounds[l]: bounds[l + 1], :, 0, :, l] += np.float32(1.0)
    return p


@pytest.mark.parametrize("seed", range(8))
def test_dp_recovers_planted_paths(seed):
    g = np.random.default_rng(seed)
    L = int(g.integers(1, 30))
    T = L + int(g.integers(0, 60))
    cuts = np.sort(g.choice(np.arange(1, T), size=L - 1, replace=False)) if L > 1 else np.array([], dtype=np.int64)
    first = np.concatenate([[0], cuts]).astype(np.int64)
    p = _probs_from_path(first, T, L, noise=0.2, seed=seed)
    got = O.first_frames(p, [L], [T])[0]
    assert got.tolist() == first.tolist()


def test_dp_exact_tie_takes_the_stay_predecessor():
    """T = 3, L = 2, one layer, one head, dyadic weights (every sum exact):
    A = [[1, 0], [0.5, 0.5], [0.25, 0.25]].  S[0] = [1, -inf]; S[1] = [1.5, 1 + 0.5 = 1.5] (token 1 entered at t = 1);
    S[2][1] = 0.25 + max(S[1][1] = 1.5, S[1][0] = 1.5): a tie, so the path stays on token 1 -> first = [0, 1].
    (Taking the move instead would give [0, 2].)"""
    A = np.array([[1.0, 0.0], [0.5, 0.5], [0.25, 0.25]], dtype=np.float32)
    p = A[:, None, None, None, :]
    assert O.first_frames(p, [2], [3])[0].tolist() == [0, 1]
    assert O.path_from_scores(A.astype(np.float64)).tolist() == [0, 1]


def test_dp_edge_geometries():
    # T == L: the diagonal, whatever the weights
    g = np.random.default_rng(1)
    p = g.random((9, 3, 1, 4, 9)).astype(np.float32)
    assert O.first_frames(p, [9], [9])[0].tolist() == list(range(9))
    # L == 1: the one token owns every frame
    assert O.first_frames(p, [1], [9])[0].tolist() == [0] + [-1] * 8
    # T < L and T == 0: no path, all -1
    assert O.first_frames(p, [5], [4])[0].tolist() == [-1] * 9
    assert O.first_frames(p, [1], [0])[0].tolist() == [-1] * 9


def test_dp_ragged_batch_rows_are_independent():
    g = np.random.default_rng(2)
    p = g.random((40, 3, 4, 4, 12)).astype(np.float32)
    lens, frames = [12, 5, 1, 7], [40, 3, 17, 30]
    got = O.first_frames(p, lens, frames)
    for b in range(4):
        alone = O.first_frames(np.ascontiguousarray(p[:, :, b: b + 1]), [lens[b]], [frames[b]])[0]
        assert got[b].tolist() == alone.tolist()
        if frames[b] >= lens[b]:
            f = got[b, : lens[b]]
            assert f[0] == 0 and np.all(np.diff(f) >= 1) and f[-1] < frames[b]
    assert got[1].tolist() == [-1] * 12


# ---- tokens -> words

def test_ids_tokenizer_offsets_and_words():
    tok = IdsTokenizer(1000)
    text = "  3 7\n\thello  world! "
    ids, spans = tok.encode_with_offsets(text)
    assert ids == tok.encode(text)
    assert spans[0] is None and spans[-1] is None
    assert [text[a:b] for a, b in spans[1:-1]] == ["3", "7", "hello", "world!"]
    ws = TS.words(text)
    assert ws == O.word_spans_regex(text)
    assert TS.token_words(text, spans, ws) == [None, 0, 1, 2, 3, None]


def _fast_tokenizer_dir(tmp_path):
    """A tiny word-piece-free BPE fast tokenizer (subwords, punctuation, BOS/EOS) built offline and saved for
    transformers' AutoTokenizer."""
    from tokenizers import Tokenizer, models, pre_tokenizers
    from transformers import PreTrainedTokenizerFast

    vocab = {"<s>": 0, "</s>": 1, "<pad>": 2, "h": 3, "e": 4, "l": 5, "o": 6, "w": 7, "r": 8, "d": 9, "!": 10, ",": 11,
             "he": 12, "ll": 13, "hell": 14, "hello": 15, "wo": 16, "wor": 17, "world": 18, "x": 19, "y": 20}
    merges = [("h", "e"), ("l", "l"), ("he", "ll"), ("hell", "o"), ("w", "o"), ("wo", "r"), ("wor", "ld")]
    vocab["ld"] = 21
    merges.insert(0, ("l", "d"))
    tk = Tokenizer(models.BPE(vocab=vocab, merges=merges, unk_token=None))
    tk.pre_tokenizer = pre_tokenizers.Sequence([pre_tokenizers.WhitespaceSplit(), pre_tokenizers.Punctuation()])
    fast = PreTrainedTokenizerFast(tokenizer_object=tk, bos_token="<s>", eos_token="</s>", pad_token="<pad>")
    fast.save_pretrained(str(tmp_path))
    return str(tmp_path)


def test_fast_tokenizer_offsets_and_words(tmp_path):
    pytest.importorskip("tokenizers")
    pytest.importorskip("transformers")
    from sopro_b200.tokenizer import TextTokenizer

    tok = TextTokenizer(_fast_tokenizer_dir(tmp_path))
    text = "hello, world!  xy hellx"
    ids, spans = tok.encode_with_offsets(text)
    assert ids == tok.encode(text)
    assert ids[0] == tok.bos_id and ids[-1] == tok.eos_id and spans[0] is None and spans[-1] is None
    pieces = [text[a:b] for a, b in spans[1:-1]]
    assert pieces == ["hello", ",", "world", "!", "x", "y", "hell", "x"]
    ws = TS.words(text)  # hello, | world! | xy | hellx
    owner = TS.token_words(text, spans, ws)
    assert owner == [None, 0, 0, 1, 1, 2, 2, 3, 3, None]
    # frames: BOS 0-1, then one frame per token from 2, EOS last two
    first = [0, 2, 3, 4, 5, 6, 7, 8, 9, 10]
    T = 12
    got = TS.utterance_timings(text, spans, np.array(first), T, 1920, None)
    want = O.words_for(text, spans, first, T, 1920)
    assert [(w.word, w.start, w.end, w.char_start, w.char_end) for w in got] == want
    assert [(w.word, w.start, w.end) for w in got] == [
        ("hello,", 2 * 0.08, 4 * 0.08), ("world!", 4 * 0.08, 6 * 0.08), ("xy", 6 * 0.08, 8 * 0.08),
        ("hellx", 8 * 0.08, 10 * 0.08)]


def test_word_without_tokens_and_whitespace_tokens():
    text = "ab cd ef"
    spans = [None, (0, 2), (2, 3), (6, 8), None]  # a whitespace-only token; "cd" gets no token
    owner = TS.token_words(text, spans, TS.words(text))
    assert owner == [None, 0, None, 2, None]
    fr = TS.word_frames([0, 1, 3, 4, 6], 8, owner, 3)
    assert fr == [(1, 3), (3, 3), (4, 6)]  # the whitespace token owns frame 3 but no word
    got = TS.utterance_timings(text, spans, np.array([0, 1, 3, 4, 6]), 8, 10, None)
    assert [(w.word, w.start, w.end, w.char_start, w.char_end) for w in got] == \
        O.words_for(text, spans, [0, 1, 3, 4, 6], 8, 10)
    assert TS.utterance_timings(text, spans, np.array([-1] * 5), 8, 10, None) == []


# ---- frames -> seconds

@pytest.mark.parametrize("speed", [0.5, 0.8, 1.25, 3.7])
def test_speed_scaling(speed):
    from sopro_b200.stretch import quantise

    S = quantise(speed)
    tok = IdsTokenizer(1000)
    text = "1 2 3 4"
    _ids, spans = tok.encode_with_offsets(text)
    first = np.array([0, 3, 5, 9, 12, 20])
    got = TS.utterance_timings(text, spans, first, 25, 1920, S)
    want = O.words_for(text, spans, first, 25, 1920, S)
    assert [(w.word, w.start, w.end, w.char_start, w.char_end) for w in got] == want
    assert got[0].start == 3 * 1920 * 65536.0 / S / 24000
    assert all(a.end <= b.start for a, b in zip(got, got[1:]))


def test_long_form_offsets_clamping_skips_and_original_text():
    from sopro_b200.longform import split_text

    tok = IdsTokenizer(1000)
    text = "  1 2 3.  4 5\n\n\n6   7 8 9 10 11.\t12  "
    segs = split_text(text, tok, 5)
    assert len(segs) >= 3
    spans = [tok.encode_with_offsets(s)[1] for s in segs]
    hop, pause = 100, 50
    firsts, Ts, ext = [], [], []
    for i, s in enumerate(segs):
        L = len(spans[i])
        T = 3 * L
        firsts.append(np.arange(L) * 3)
        Ts.append(T)
        ext.append((250, T * hop - 120) if i != 1 else (0, 0))  # segment 1 skipped; the others clamped at both ends
    firsts[2] = np.full(len(spans[2]), -1)  # no alignment: zero length at O_2
    got = TS.long_timings(text, segs, spans, firsts, Ts, hop, ext, pause, None)
    want = O.long_words(text, segs, spans, firsts, Ts, hop, ext, pause)
    assert [(w.word, w.start, w.end, w.char_start, w.char_end) for w in got] == want
    assert [text[w.char_start: w.char_end] for w in got] == text.split()
    assert [w.word for w in got] == text.split()
    # segment 0: its first word starts at frame 3 (after BOS), 300 - e0 = 50 samples into the joined row; its EOS
    # frames are past e1, so the last word's end is clamped to the extent's end
    assert got[0].start == 50 / 24000
    n_last0 = len(segs[0].split()) - 1
    assert got[n_last0].end <= (ext[0][1] - ext[0][0]) / 24000
    n0, n1 = len(segs[0].split()), len(segs[1].split())
    O1 = ext[0][1] - ext[0][0] + pause
    for w in got[n0: n0 + n1]:  # skipped segment: zero length at O_1
        assert w.start == w.end == O1 / 24000
    S = 65536 * 5 // 4
    gs = TS.long_timings(text, segs, spans, firsts, Ts, hop, ext, pause, S)
    assert [(w.start, w.end) for w in gs] == [(a, b) for _w, a, b, _c, _d in O.long_words(text, segs, spans, firsts, Ts, hop, ext, pause, S)]
