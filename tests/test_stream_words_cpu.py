"""CPU: the streaming word alignment's float64 definition (oracle/align_stream_oracle.py::StreamAlign) -- its anchor on the
one-shot path, binding commits, the end rule, chunking -- and the host word emitter (timestamps.WordEmitter) against
utterance_timings and the oracle's finality rule.  Also the new C symbols and the argument refusals."""
import numpy as np
import pytest

from oracle import align_oracle as AO
from oracle import align_stream_oracle as SO
from sopro_b200 import timestamps as TS

RNG = np.random.default_rng(20261018)


def _cases(n, T_max=60, L_max=24, D_max=30):
    for _ in range(n):
        T, L, D = int(RNG.integers(0, T_max)), int(RNG.integers(1, L_max)), int(RNG.integers(1, D_max))
        yield T, L, D, RNG.random((T, L))


def test_equals_the_one_shot_path_without_commits():
    n = 0
    for _ in range(400):
        L = int(RNG.integers(1, 30))
        T = int(RNG.integers(L, 70))
        D = int(RNG.integers(T, T + 5))
        A = RNG.random((T, L))
        assert np.array_equal(SO.stream_path(A, D), AO.path_from_scores(A))
        n += 1
    # peaked weights too (ties in S are rare with random A; equal columns force them)
    A = np.ones((12, 4))
    assert np.array_equal(SO.stream_path(A, 12), AO.path_from_scores(A))
    assert n == 400


def test_commits_are_never_revised_and_the_path_is_monotone():
    for T, L, D, A in _cases(300):
        s = SO.StreamAlign(L, D)
        snaps = []
        for t in range(T):
            s.push(A[t: t + 1])
            snaps.append((s.F, s.K, s.first.copy()))
            assert s.F == max(0, t + 1 - D)
        final = s.end()
        if T == 0:
            assert final is None
            continue
        for F, K, fr in snaps:
            assert np.array_equal(fr[:K], final[:K]) and (fr[K:] == -1).all()
            if F:
                assert fr[K - 1] <= F - 1  # the committed token's first frame is committed
        assert final[0] == 0 and (np.diff(final) >= 0).all() and (final <= T).all()
        reached = final < T
        # every token the path reached gets at least one frame; the rest start at T with zero length
        ends = np.append(final[1:], T)
        assert (ends[reached] > final[reached]).all()
        assert (final[~reached] == T).all()
        if T >= L and D >= T:
            assert reached.all()


def test_end_rule_fallbacks():
    # T < L: the end state is the highest finite one, the tokens past it start at T
    A = RNG.random((5, 9))
    f = SO.stream_path(A, 3)
    assert AO.path_from_scores(A) is None
    assert f[0] == 0 and (f[5:] == 5).all() and (f[:5] < 5).all()
    assert np.array_equal(f[:5], np.arange(5))  # five frames can only reach token 4 by moving every frame
    # T = 0: no path
    assert SO.stream_path(np.zeros((0, 4)), 2) is None
    # pruning made (T-1, L-1) -inf: token 0 holds the attention, so early commits keep the path there
    A = np.zeros((3, 3))
    A[:, 0] = 1.0
    f = SO.stream_path(A, 1)
    assert np.array_equal(f, [0, 2, 3])  # frame 1 committed to token 0, so (2, 2) was pruned; token 2 gets no frame
    assert np.array_equal(AO.path_from_scores(A), [0, 1, 2])


def test_any_chunking_gives_the_same_result():
    for T, L, D, A in _cases(120):
        want = SO.stream_path(A, D)
        for _ in range(3):
            s = SO.StreamAlign(L, D)
            t = 0
            while t < T:
                n = int(RNG.integers(0, 8))
                s.push(A[t: t + n])
                t += n
            got = s.end()
            assert (got is None and want is None) or np.array_equal(got, want)


def _text_and_spans(n_words):
    """A text of numbers and spans as a tokenizer makes them: BOS, 1-3 tokens per word (one of them sometimes a
    leading space only), EOS."""
    words = [str(int(RNG.integers(0, 10 ** int(RNG.integers(1, 6))))) for _ in range(n_words)]
    text = " ".join(words)
    spans, pos = [None], 0
    for w in words:
        a = text.index(w, pos)
        if a > 0 and RNG.random() < 0.2:
            spans.append((a - 1, a))  # whitespace only: no word
        k = int(RNG.integers(1, min(3, len(w)) + 1))
        cuts = sorted(RNG.choice(np.arange(1, len(w)), size=k - 1, replace=False).tolist()) if k > 1 else []
        edges = [a] + [a + c for c in cuts] + [a + len(w)]
        spans += [(edges[i], edges[i + 1]) for i in range(k)]
        pos = a + len(w)
    spans.append(None)
    return text, spans


@pytest.mark.parametrize("S", [None, 50000])
def test_word_emitter_equals_utterance_timings(S):
    hop = 1920
    for _ in range(150):
        text, spans = _text_and_spans(int(RNG.integers(1, 12)))
        L = len(spans)
        T, D = int(RNG.integers(0, 3 * L + 10)), int(RNG.integers(1, 20))
        A = RNG.random((T, L))
        s, em = SO.StreamAlign(L, D), TS.WordEmitter(text, spans, hop, S)
        end_tok = SO.word_end_tokens(text, spans)
        got, t, K_prev = [], 0, 0
        while t < T:
            n = int(RNG.integers(1, 7))
            s.push(A[t: t + n])
            t = min(T, t + n)
            new = em.take(s.first, s.K, t, False)
            # exactly the words the oracle's rule makes final now
            assert len(new) == sum(1 for e in end_tok if K_prev <= e < s.K)
            got += new
            K_prev = s.K
        final = s.end()
        got += em.take(s.first, s.K, T, True)
        want = TS.utterance_timings(text, spans, final, T, hop, S)
        assert got == want
        if T > 0:
            assert [w.word for w in got] == text.split()
            assert want == [TS.WordTiming(*w) for w in AO.words_for(text, spans, final, T, hop, S)]
        assert em.take(s.first, s.K, T, True) == []


def test_new_symbols_are_exported():
    from sopro_b200 import _lib

    lib = _lib.load()
    for name in ("sopro_ar_set_attn_trace_ring", "sopro_align_stream_sizes", "sopro_align_stream_create",
                 "sopro_align_stream_begin", "sopro_align_stream_push", "sopro_align_stream_destroy"):
        assert hasattr(lib, name), name


def test_stream_state_geometry_refusals():
    import ctypes as C

    from sopro_b200 import _lib

    lib = _lib.load()
    nb = C.c_int64()
    assert lib.sopro_align_stream_sizes(2, 40, 24, 401, C.byref(nb)) == 0 and nb.value > 0
    for bad in ((0, 40, 24, 401), (257, 40, 24, 401), (2, 0, 24, 401), (2, 40, 0, 401), (2, 40, 24, 0)):
        assert lib.sopro_align_stream_sizes(*bad, C.byref(nb)) != 0, bad


class _Tok:
    def encode_with_offsets(self, text):
        raise AssertionError("tokenised before the flag was checked")


class _TTS:
    tokenizer = _Tok()


def test_word_timestamps_flag_is_checked_first():
    from sopro_b200.streaming import _word_spans

    for bad in (1, "yes", None, np.bool_(True)):
        with pytest.raises(TypeError):
            _word_spans(_TTS(), ["a"], bad)
    assert _word_spans(_TTS(), ["a"], False) is None


def test_a_text_over_2048_tokens_is_refused():
    from sopro_b200.streaming import _word_spans

    class Tok:
        def encode_with_offsets(self, text):
            n = len(text.split())
            return list(range(n)), [(0, 1)] * n

    class T:
        tokenizer = Tok()

    assert len(_word_spans(T(), ["a " * 2048], True)[0]) == 2048
    with pytest.raises(ValueError):
        _word_spans(T(), ["a " * 10, "a " * 2049], True)
    assert TS.STREAM_ALIGN_LAG == 24
