"""GPU: word timestamps for streams -- the AR kernel's ring trace against the full-length trace, the streaming
alignment kernel (sopro_align_stream_*) against oracle/align_stream_oracle.py::StreamAlign bit for bit, and
word_timestamps= on stream / stream_batch against the oracle on the captured trace and against synthesize."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import align_oracle as AO
from oracle import align_stream_oracle as SO
from oracle import ar_oracle as O
from tests.test_timestamps_gpu import KW, TEXT, _api, _engine, _sampling, _trace, _tuples

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)


# ---- the ring trace

@pytest.mark.parametrize("name,B", [("default_fp32", 1), ("default_bf16", 3)])
@pytest.mark.parametrize("ring", [1, 6, 7])
def test_ring_trace_equals_the_full_trace(name, B, ring):
    """Launches of 1, 6 and 7 steps (at most `ring`) into a ring: each launch's rows equal the full-length trace's rows
    of the same steps bit for bit, and the tokens are those of the untraced run."""
    spec, cfg, sd, inp, eng = _engine(name)
    steps = 61
    L = int(inp["txt_seq"].shape[1])
    lens = [L - (b % 3) for b in range(B)]
    tape = O.noise_tape(spec["noise_seed"], steps, cfg.ar_vocab())[:, :50].contiguous()
    cond = inp["cond_ar"][:, :steps].expand(B, -1, -1).contiguous()
    txt = inp["txt_seq"].expand(B, -1, -1).contiguous()
    noise = tape.unsqueeze(0).expand(B, -1, -1).contiguous()
    samp = _sampling(inp["sampling"], cfg, min_gen_frames=2 ** 31 - 1)
    sizes = [s for s in (1, 6, 7) if s <= ring]
    sched, t = [], 0
    while t < steps:
        sched.append(min(sizes[len(sched) % len(sizes)], steps - t))
        t += sched[-1]

    def run(trace, ring_rows):
        ses = eng.session(B, steps, L)
        if trace is not None:
            ses.set_attn_trace(trace, ring_rows)
        ses.begin(cond, txt, lens, noise, samp)
        rows, t = [], 0
        for n in sched:
            ses.run(n)
            if ring_rows:
                rows.append(trace[[(t + i) % ring_rows for i in range(n)]].cpu())
            t += n
        toks, _n, _ = ses.read()
        ses.close()
        return toks, rows

    plain, _ = run(None, None)
    full = _trace(cfg, steps, B, L)
    toks_full, _ = run(full, None)
    ring_buf = _trace(cfg, ring, B, L)
    toks_ring, rows = run(ring_buf, ring)
    assert np.array_equal(toks_full, plain) and np.array_equal(toks_ring, plain)
    got = torch.cat(rows)
    want = full.cpu()
    for b in range(B):  # entries past text_len[b] are not written
        assert torch.equal(got[:, :, b, :, : lens[b]], want[:, :, b, :, : lens[b]])


def test_a_launch_longer_than_the_ring_is_refused():
    from sopro_b200 import _lib

    spec, cfg, sd, inp, eng = _engine("small_fp32")
    steps, L = 20, int(inp["txt_seq"].shape[1])
    ses = eng.session(1, steps, L)
    ses.set_attn_trace(_trace(cfg, 6, 1, L), 6)
    tape = O.noise_tape(spec["noise_seed"], steps, cfg.ar_vocab())[:, :50].contiguous().unsqueeze(0)
    ses.begin(inp["cond_ar"][:, :steps].contiguous(), inp["txt_seq"], [L], tape, _sampling(inp["sampling"], cfg))
    with pytest.raises(_lib.SoproError):
        ses.run(7)
    assert ses.position == 0
    ses.run(6)
    assert ses.position == 6
    with pytest.raises(_lib.SoproError):
        ses.set_attn_trace(_trace(cfg, 6, 1, L), 0)
    ses.close()


# ---- the streaming alignment kernel against the oracle

class _Stream:
    """The raw C-ABI: one state of B rows, a ring of `ring` steps the test fills per row."""

    def __init__(self, lens, ld, lag, max_frames, ring, n_attn, H):
        from sopro_b200 import _lib

        self.lib, self._lib = _lib.load(), _lib
        self.B, self.ld = len(lens), ld
        nb = C.c_int64()
        _lib.check_arg(self.lib.sopro_align_stream_sizes(self.B, ld, lag, max_frames, C.byref(nb)))
        self.state = torch.empty(int(nb.value), dtype=torch.uint8, device="cuda:0")
        h = C.c_void_p()
        _lib.check_arg(self.lib.sopro_align_stream_create(self.B, ld, lag, max_frames, self.state.data_ptr(), C.byref(h)))
        self.h = h
        self.ring = torch.zeros((ring, n_attn, self.B, H, ld), dtype=torch.float32, device="cuda:0")
        _lib.check_arg(self.lib.sopro_align_stream_begin(h, (C.c_int32 * self.B)(*lens), None))
        self.t = [0] * self.B

    def push(self, probs, n, end):
        """probs: the full trace [steps, n_attn, B, H, ld] (device); row b's next n[b] frames go to its ring slots."""
        R = self.ring.shape[0]
        for b in range(self.B):
            for i in range(n[b]):
                t = self.t[b] + i
                self.ring[t % R, :, b] = probs[t, :, b]
        rc = self.lib.sopro_align_stream_push(self.h, self.ring.data_ptr(), R, self.ring.shape[1], self.B, self.ring.shape[3],
                                              self.ld, (C.c_int32 * self.B)(*n), (C.c_int32 * self.B)(*[int(e) for e in end]),
                                              None)
        self._lib.check_arg(rc)
        for b in range(self.B):
            self.t[b] += n[b]
        return self.state[: self.B * (2 + self.ld) * 4].view(torch.int32).view(self.B, 2 + self.ld).cpu().numpy()

    def close(self):
        self.lib.sopro_align_stream_destroy(self.h)


def _check_stream(probs, lens, frames, lag, schedule, ring):
    """Push `schedule(b, k)` frames per row per push (a row ends with its last frames) and compare every push's
    committed state with the oracle's, then the final paths."""
    steps, n_attn, B, H, ld = probs.shape
    p_np = probs.cpu().numpy()
    dev = _Stream(lens, ld, lag, steps, ring, n_attn, H)
    ora = [SO.StreamAlign(lens[b], lag) for b in range(B)]
    A = [AO.accumulate(p_np, b, frames[b], lens[b]) for b in range(B)]
    done = [False] * B
    k = 0
    while not all(done):
        n = [0] * B
        end = [False] * B
        for b in range(B):
            if done[b]:
                continue
            n[b] = min(schedule(b, k), frames[b] - dev.t[b], ring)
            end[b] = dev.t[b] + n[b] == frames[b]
        t0 = list(dev.t)
        out = dev.push(probs, n, end)
        for b in range(B):
            if done[b]:
                continue
            ora[b].push(A[b][t0[b]: t0[b] + n[b]])
            if end[b]:
                ora[b].end()
                done[b] = True
            L = lens[b]
            assert (out[b, 0], out[b, 1]) == (ora[b].F, ora[b].K), (b, k)
            assert np.array_equal(out[b, 2: 2 + L], ora[b].first), (b, k)
        k += 1
    dev.close()
    return out


def _random_probs(steps, B, ld, seed, n_attn=2, H=4):
    g = torch.Generator().manual_seed(seed)
    p = torch.rand((steps, n_attn, B, H, ld), generator=g)
    return (p / p.sum(-1, keepdim=True)).to("cuda:0")


@pytest.mark.parametrize("lag", [1, 6, 24, 80])
@pytest.mark.parametrize("push", ["1", "6", "7", "ragged"])
def test_stream_kernel_matches_the_oracle(lag, push):
    steps, B, ld = 70, 5, 40
    probs = _random_probs(steps, B, ld, seed=lag * 10 + len(push))
    lens = [40, 1, 17, 33, 8]
    frames = [70, 50, 3, 0, 64]  # T >= L, T < L, T = 0
    sched = {"1": lambda b, k: 1, "6": lambda b, k: 6, "7": lambda b, k: 7,
             "ragged": lambda b, k: (3 * b + 5 * k) % 8}[push]
    out = _check_stream(probs, lens, frames, lag, sched, ring=8)
    if lag >= steps:  # no commit: the one-shot path wherever it has one
        from sopro_b200.timestamps import align

        one = align(probs, lens, frames).cpu().numpy()
        for b in range(B):
            if frames[b] >= lens[b] and frames[b] > 0:
                assert np.array_equal(out[b, 2: 2 + lens[b]], one[b, : lens[b]])


def test_stream_kernel_long_text_and_many_rows():
    # L = 2048 (four states per thread), and 130 rows (more than one align launch's 128)
    probs = _random_probs(90, 2, 2048, seed=1, n_attn=1, H=2)
    _check_stream(probs, [2048, 1500], [90, 90], 6, lambda b, k: 6, ring=6)
    B = 130
    probs = _random_probs(40, B, 24, seed=2)
    lens = [1 + (b * 7) % 24 for b in range(B)]
    frames = [(b * 11) % 41 for b in range(B)]
    batch = _check_stream(probs, lens, frames, 6, lambda b, k: 1 + (b + k) % 7, ring=7)
    # each row alone gives what it gives in the batch
    for b in (0, 77, 129):
        alone = _check_stream(probs[:, :, b: b + 1].contiguous(), [lens[b]], [frames[b]], 6, lambda _b, k: 1 + (b + k) % 7,
                              ring=7)
        assert np.array_equal(alone[0, : 2 + lens[b]], batch[b, : 2 + lens[b]])


def test_stream_kernel_on_a_real_ar_trace():
    spec, cfg, sd, inp, eng = _engine("peaked_fp32")
    steps = 61
    L = int(inp["txt_seq"].shape[1])
    B = 3
    lens = [L, L - 2, L - 5]
    tr = _trace(cfg, steps, B, L)
    ses = eng.session(B, steps, L)
    ses.set_attn_trace(tr)
    tape = O.noise_tape(spec["noise_seed"], steps, cfg.ar_vocab())[:, :50].contiguous()
    ses.begin(inp["cond_ar"][:, :steps].expand(B, -1, -1).contiguous(), inp["txt_seq"].expand(B, -1, -1).contiguous(),
              lens, tape.unsqueeze(0).expand(B, -1, -1).contiguous(), _sampling(inp["sampling"], cfg, min_gen_frames=2 ** 31 - 1))
    ses.run()
    ses.read()
    ses.close()
    for lag in (1, 6, 24, 61):
        _check_stream(tr, lens, [61, 40, 12], lag, lambda b, k: 6, ring=6)


def test_stream_push_refusals():
    from sopro_b200 import _lib

    probs = _random_probs(10, 2, 8, seed=3)
    dev = _Stream([8, 4], 8, 3, 10, 4, 2, 4)
    lib, h = dev.lib, dev.h
    P = dev.ring.data_ptr()

    def push(n, e, ring=4, B=2, ld=8):
        return lib.sopro_align_stream_push(h, P, ring, 2, B, 4, ld, (C.c_int32 * 2)(*n), (C.c_int32 * 2)(*e), None)

    assert push([5, 0], [0, 0]) != 0  # more frames than the ring holds
    assert push([1, 0], [0, 0], B=3) != 0  # a trace of another batch
    assert push([1, 0], [0, 0], ld=9) != 0
    assert push([-1, 0], [0, 0]) != 0
    assert push([0, 2], [0, 1]) == 0
    assert push([0, 1], [0, 0]) != 0  # row 1 has ended
    assert push([0, 0], [0, 1]) != 0
    for _ in range(2):
        assert push([4, 0], [0, 0]) == 0
    assert push([3, 0], [0, 0]) != 0  # past max_frames = 10
    torch.cuda.synchronize()
    assert lib.sopro_align_stream_begin(h, (C.c_int32 * 2)(8, 9), None) != 0  # text_len > ld
    dev.close()
    del probs, _lib


# ---- the public API

def _capture(monkeypatch):
    """Records, per StreamAligner push, the ring rows of the launch's new frames (on the stream the push runs on)."""
    from sopro_b200 import timestamps as TS

    log = {"rows": [], "pushes": 0}
    real = TS.StreamAligner.push

    def push(self, frames, ends):
        n = max(frames)
        log["rows"].append((self.ring[:n].clone(), list(frames)))
        log["pushes"] += 1
        return real(self, frames, ends)

    monkeypatch.setattr(TS.StreamAligner, "push", push)
    return log


def _row_trace(log, b):
    """Row b's trace [T, n_attn, 1, H, ld] from the captured pushes (the rows advance in lockstep)."""
    parts = [r[:, :, b: b + 1][: f[b]] for r, f in log["rows"] if f[b] > 0]
    return torch.cat(parts).cpu().numpy() if parts else None


def _oracle_words(text, spans, trace, lag, hop, S):
    L = len(spans)
    T = 0 if trace is None else trace.shape[0]
    s = SO.StreamAlign(L, lag)
    if T:
        s.push(AO.accumulate(trace, 0, T, L))
    first = s.end()
    return AO.words_for(text, spans, first, T, hop, S), first, T


@pytest.mark.parametrize("extra", [{}, dict(speed=1.3), dict(sample_rate=16000, watermark=7)])
def test_stream_words_match_the_oracle(monkeypatch, extra):
    from sopro_b200 import timestamps as TS
    from sopro_b200.stretch import quantise

    tts, ref = _api()
    hop, cf = tts.codec.engine.hop, 6
    plain = list(tts.stream(TEXT, ref=ref, seed=5, chunk_frames=cf, **KW, **extra))
    log = _capture(monkeypatch)
    items, at = [], []
    for wav, words in tts.stream(TEXT, ref=ref, seed=5, chunk_frames=cf, word_timestamps=True, **KW, **extra):
        items.append((wav, words))
        at.append(log["pushes"] - 1)  # the chunk whose push preceded this item
    wavs = [w for w, _ in items if w.shape[1] > 0]
    assert len(wavs) == len(plain) and all(torch.equal(a, b) for a, b in zip(wavs, plain))
    got = [w for _, ws in items for w in ws]
    _ids, spans = tts.tokenizer.encode_with_offsets(TEXT)
    S = quantise(extra["speed"]) if "speed" in extra else None
    want, first, T = _oracle_words(TEXT, spans, _row_trace(log, 0), TS.STREAM_ALIGN_LAG, hop, S)
    assert _tuples(got) == want and len(got) == len(TEXT.split())
    # each word arrives with the first item at or after the chunk that generated frame first[end token] + lag
    end_tok = SO.word_end_tokens(TEXT, spans)
    k = 0
    for i, (_w, ws) in enumerate(items):
        for _ in ws:
            e = end_tok[k]
            f = int(first[e]) + TS.STREAM_ALIGN_LAG if e < len(spans) else T
            if f >= T:
                assert i == len(items) - 1
            else:
                assert at[i] >= f // cf and (i == 0 or at[i - 1] < f // cf)
            k += 1


@pytest.mark.parametrize("speed", [None, 0.8])
def test_stream_words_equal_synthesize_with_a_long_lag(monkeypatch, speed):
    from sopro_b200 import timestamps as TS

    tts, ref = _api()
    monkeypatch.setattr(TS, "STREAM_ALIGN_LAG", KW["max_frames"] + 1)
    _wav, want = tts.synthesize(TEXT, ref=ref, seed=9, word_timestamps=True, speed=speed, **KW)
    got = [w for _wav, ws in tts.stream(TEXT, ref=ref, seed=9, word_timestamps=True, speed=speed, **KW) for w in ws]
    assert want and got == want


def test_stream_words_leave_the_generator_as_without_them():
    tts, ref = _api()
    torch.manual_seed(4)
    a = [w.clone() for w in tts.stream(TEXT, ref=ref, **KW)]
    s1 = torch.get_rng_state()
    torch.manual_seed(4)
    b = [w for w, _ws in tts.stream(TEXT, ref=ref, word_timestamps=True, **KW) if w.shape[1] > 0]
    assert torch.equal(torch.get_rng_state(), s1)
    assert len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b))


def test_stream_batch_words_match_the_oracle_per_row(monkeypatch):
    from sopro_b200 import timestamps as TS
    from tests.test_stream_batch_gpu import FRAMES, TEXTS, _tts

    tts, refs = _tts()
    hop = tts.codec.engine.hop
    kw = dict(max_frames=FRAMES, chunk_frames=6)
    seeds = [41, 42, 43, 44, 45]
    voices = [refs[i % len(refs)] for i in range(len(TEXTS))]
    plain = [(i, w, last) for i, w, last in tts.stream_batch(TEXTS, ref=voices, seeds=seeds, **kw)]
    log = _capture(monkeypatch)
    items = list(tts.stream_batch(TEXTS, ref=voices, seeds=seeds, word_timestamps=True, **kw))
    assert len(items) == len(plain)
    for (i, w, last, _ws), (pi, pw, plast) in zip(items, plain):
        assert (i, last) == (pi, plast) and torch.equal(w, pw)
    ends = set()
    for i, text in enumerate(TEXTS):
        _ids, spans = tts.tokenizer.encode_with_offsets(text)
        got = [x for j, _w, _l, ws in items if j == i for x in ws]
        want, _first, T = _oracle_words(text, spans, _row_trace(log, i), TS.STREAM_ALIGN_LAG, hop, None)
        assert _tuples(got) == want
        ends.add(T)
    assert len(ends) > 1  # ragged rows


def test_stream_batch_closing_early_leaves_nothing_checked_out():
    from tests.test_stream_batch_gpu import FRAMES, TEXTS, _tts

    tts, refs = _tts()
    gen = tts.stream_batch(TEXTS, ref=refs[0], seeds=[1, 2, 3, 4, 5], max_frames=FRAMES, word_timestamps=True)
    first = [next(gen) for _ in TEXTS]
    assert all(len(x) == 4 for x in first)
    gen.close()
    assert not tts.model._sessions_busy
    again = list(tts.stream_batch(TEXTS, ref=refs[0], seeds=[1, 2, 3, 4, 5], max_frames=FRAMES, word_timestamps=True))
    assert sum(1 for x in again if x[2]) == len(TEXTS)


def test_refusals_before_any_work():
    tts, ref = _api()
    torch.manual_seed(0)
    s0 = torch.get_rng_state()
    busy = set(tts.model._sessions_busy)
    with pytest.raises(TypeError):
        tts.stream(TEXT, ref=ref, word_timestamps=1)
    with pytest.raises(TypeError):
        tts.stream_batch([TEXT], ref=ref, word_timestamps="yes")
    long_text = " ".join(["7"] * 2100)
    with pytest.raises(ValueError):
        tts.stream(long_text, ref=ref, word_timestamps=True)
    with pytest.raises(ValueError):
        tts.stream_batch([TEXT, long_text], ref=ref, word_timestamps=True)
    assert torch.equal(torch.get_rng_state(), s0) and tts.model._sessions_busy == busy
