"""GPU: word timestamps -- the AR kernel's exported cross-attention weights against the float64 oracle, tokens unchanged
with the export on, sopro_align against oracle/align_oracle.py bit for bit, and word_timestamps= through the public API."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import align_oracle as AO
from oracle import ar_oracle as O
from tests.cases import AR_CASES, ar_case_inputs

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
_ENG = {}


def _engine(name):
    from sopro_b200.engine import ArEngine

    spec = AR_CASES[name]
    cfg, sd, inp = ar_case_inputs(spec)
    key = (str(sorted(spec["cfg"].items())), spec["head_gain"], spec["bf16"], spec.get("eos_bias", 0.0))
    if key not in _ENG:
        _ENG[key] = ArEngine(cfg, sd, device=0, weight_dtype="bf16" if spec["bf16"] else "fp32")
    return spec, cfg, sd, inp, _ENG[key]


def _sampling(samp, cfg, **over):
    from sopro_b200.engine import Sampling

    mg = samp.min_gen_frames if samp.min_gen_frames is not None else cfg.min_gen_frames
    d = dict(top_p=samp.top_p, temperature=samp.temperature, recovery_top_p=samp.recovery_top_p,
             recovery_temp=samp.recovery_temp, repetition_penalty=samp.repetition_penalty, top_k=samp.top_k,
             anti_loop=samp.anti_loop, loop_streak=samp.loop_streak, min_gen_frames=int(min(mg, 2 ** 31 - 1)))
    d.update(over)
    return Sampling(**d)


def _trace(cfg, steps, B, ld):
    from sopro_b200.timestamps import trace_buffer

    return trace_buffer(cfg, steps, B, ld, "cuda:0")


@pytest.mark.parametrize("name", ["default_fp32", "default_bf16", "peaked_fp32", "small_fp32"])
def test_exported_weights_match_the_float64_oracle(name):
    """Teacher-forced on the oracle's own tokens: every exported weight of the first 48 steps is within 5e-5 of the
    float64 softmax of the oracle's fp32 q and K.  Bound: the device computes q . k in fp32 (Dh products, a different
    order than torch), the scores carry ~1e-6 relative error, the logits feed exp; a weight w moves by about
    w * |d score| <= 1e-5 on these O(1) scores, and the logits themselves are held to 3e-5 of their peak by
    test_teacher_forced_logits_and_blocks.  Each row sums to 1 within fp32 round-off."""
    spec, cfg, sd, inp, eng = _engine(name)
    steps = min(48, inp["max_frames"] + 1)
    L = int(inp["txt_seq"].shape[1])
    tape = O.noise_tape(spec["noise_seed"], steps, cfg.ar_vocab())
    toks = O.ar_generate(sd, cfg, inp["cond_ar"][:, :steps], inp["txt_seq"], inp["text_mask"], max_frames=steps - 1,
                         sampling=inp["sampling"], noise_tv=tape)
    forced = torch.zeros(1, steps, dtype=torch.int32)
    forced[0, : len(toks)] = torch.tensor(toks, dtype=torch.int32)
    # oracle weights along the forced tokens
    st = O.ar_init_state(sd, cfg, inp["txt_seq"], inp["text_mask"], batch=1)
    emb = sd["cb_embed.emb.weight"]
    bos = int(cfg.num_codebooks) * int(cfg.codebook_size)
    want = []
    for t in range(len(toks)):
        row = bos if t == 0 else toks[t - 1]
        _lg, pr = AO.ar_step_attn_probs(sd, cfg, inp["cond_ar"][:, t: t + 1] + emb[row].view(1, 1, -1), st)
        want.append(pr.numpy())
    want = np.stack(want)  # [T, n_attn, 1, H, L]
    tr = _trace(cfg, steps, 1, L + 3)
    ses = eng.session(1, steps, L)
    ses.set_forced(forced)
    ses.set_attn_trace(tr)
    ses.begin(inp["cond_ar"][:, :steps].contiguous(), inp["txt_seq"], [L], tape[:, :50].contiguous().unsqueeze(0),
              _sampling(inp["sampling"], cfg, min_gen_frames=2 ** 31 - 1))
    ses.run()
    ses.read()
    ses.set_attn_trace(None)
    got = tr.cpu().numpy()
    T = len(toks)
    err = np.abs(got[:T, :, :, :, :L] - want).max()
    assert err <= 5e-5, err
    assert np.all(got[:, :, :, :, L:] == 0)  # entries past the text are not written
    sums = got[:T, :, :, :, :L].astype(np.float64).sum(-1)
    assert np.abs(sums - 1).max() <= L * 2 ** -23 * 4
    print(f"{name}: max |w - w64| = {err:.2e} over {T} steps")


def _generate(eng, inp, cfg, spec, B, steps, L_list, trace, team=0, chunks=None, txt=None):
    ses = eng.session(B, steps, max(L_list))
    if team:
        ses.set_team(team)
    tape = O.noise_tape(spec["noise_seed"], steps, cfg.ar_vocab())[:, :50].contiguous()
    cond = inp["cond_ar"][:, :steps].expand(B, -1, -1).contiguous()
    txt = inp["txt_seq"].expand(B, -1, -1).contiguous() if txt is None else txt
    if trace is not None:
        ses.set_attn_trace(trace)
    ses.begin(cond, txt, L_list, tape.unsqueeze(0).expand(B, -1, -1).contiguous(), _sampling(inp["sampling"], cfg))
    if chunks:
        for c in chunks:
            ses.run(c)
    else:
        ses.run()
    toks, n, _ = ses.read()
    ses.set_attn_trace(None)
    ses.close()
    return toks, n


@pytest.mark.parametrize("name,B,team", [
    ("default_fp32", 1, 0), ("default_bf16", 1, 0), ("default_fp32", 64, 0), ("default_bf16", 64, 0),
    ("default_bf16", 64, 8), ("default_fp32", 16, 16), ("default_bf16", 16, 8)])
def test_tokens_unchanged_with_the_export_on(name, B, team):
    spec, cfg, sd, inp, eng = _engine(name)
    steps = 121
    L = int(inp["txt_seq"].shape[1])
    lens = [L - (b % 5) for b in range(B)]
    off, _ = _generate(eng, inp, cfg, spec, B, steps, lens, None, team)
    tr = _trace(cfg, steps, B, L)
    on, _ = _generate(eng, inp, cfg, spec, B, steps, lens, tr, team)
    assert np.array_equal(on, off)
    w = tr.cpu().numpy()
    for b in (0, B - 1):
        s = w[:8, :, b, :, : lens[b]].astype(np.float64).sum(-1)
        assert np.abs(s - 1).max() < 1e-5


def test_long_text_and_resumed_chunks():
    """A text of 300 keys (over 128: several score rounds) -- tokens unchanged -- and a launch resumed in chunks writes
    the same trace as one launch."""
    spec, cfg, sd, inp, eng = _engine("default_fp32")
    from tests.cases import _unit

    D, L, B, steps = int(cfg.d_model), 300, 4, 61
    txt = _unit(B * L * D, 4242).view(B, L, D)
    lens = [300, 129, 250, 7]
    off, _ = _generate(eng, inp, cfg, spec, B, steps, lens, None, txt=txt)
    tr1 = _trace(cfg, steps, B, L)
    on, _ = _generate(eng, inp, cfg, spec, B, steps, lens, tr1, txt=txt)
    assert np.array_equal(on, off)
    tr2 = _trace(cfg, steps, B, L)
    on2, _ = _generate(eng, inp, cfg, spec, B, steps, lens, tr2, txt=txt, chunks=[7, 20, 34])
    assert np.array_equal(on2, off)
    assert torch.equal(tr1, tr2)


def test_refusals():
    from sopro_b200 import _lib

    spec, cfg, sd, inp, eng = _engine("small_fp32")
    lib = _lib.load()
    L = int(inp["txt_seq"].shape[1])
    ses = eng.session(1, 8, L)
    tr = _trace(cfg, 8, 1, L - 1)
    assert lib.sopro_ar_set_attn_trace(ses._h, tr.data_ptr(), 0) == -1
    ses.set_attn_trace(tr)
    tape = O.noise_tape(3, 8, cfg.ar_vocab())[:, :50].contiguous().unsqueeze(0)
    with pytest.raises(_lib.SoproError):
        ses.begin(inp["cond_ar"][:, :8].contiguous(), inp["txt_seq"], [L], tape, _sampling(inp["sampling"], cfg))
    ses.close()
    ws = C.c_int64()
    assert lib.sopro_align_sizes(0, 5, 5, C.byref(ws)) == -1
    assert lib.sopro_align_sizes(2, 5, 5, C.byref(ws)) == 0
    p = torch.zeros(5, 1, 2, 1, 5, device="cuda")
    first = torch.zeros(2, 5, dtype=torch.int32, device="cuda")
    buf = torch.zeros(int(ws.value), dtype=torch.uint8, device="cuda")
    I = C.c_int32 * 2
    for lens, frames in (([0, 1], [5, 5]), ([6, 1], [5, 5]), ([1, 1], [6, 0]), ([1, 1], [-1, 0])):
        assert lib.sopro_align(p.data_ptr(), 5, 1, 2, 1, 5, I(*lens), I(*frames), buf.data_ptr(), first.data_ptr(), None) == -1
    assert lib.sopro_align(p.data_ptr(), 5, 1, 2, 1, 5, I(1, 1), I(5, 5), None, first.data_ptr(), None) == -1
    assert lib.sopro_align(p.data_ptr(), 5, 1, 2, 1, 2049, I(2049, 1), I(5, 5), buf.data_ptr(), first.data_ptr(), None) == -1
    torch.cuda.synchronize()
    assert int(first.abs().sum()) == 0  # nothing launched


def _check_align(p, lens, frames):
    from sopro_b200.timestamps import align

    got = align(torch.from_numpy(p).cuda(), lens, frames).cpu().numpy()
    want = AO.first_frames(p, lens, frames)
    assert np.array_equal(got, want)
    return got


def test_align_matches_the_oracle():
    g = np.random.default_rng(5)
    # random rows, ragged
    p = g.random((90, 3, 7, 4, 70)).astype(np.float32)
    _check_align(p, [70, 1, 33, 64, 65, 2, 50], [90, 90, 40, 64, 63, 0, 89])
    # planted paths and exact ties (dyadic values)
    T, L = 50, 20
    q = np.zeros((T, 1, 2, 2, L), dtype=np.float32)
    cuts = np.sort(g.choice(np.arange(1, T), size=L - 1, replace=False))
    bounds = [0] + cuts.tolist() + [T]
    for l in range(L):
        q[bounds[l]: bounds[l + 1], 0, 0, :, l] = 0.5
    q[:, 0, 1] = 0.25  # every cell equal: ties everywhere
    got = _check_align(q, [L, L], [T, T])
    assert got[0, :L].tolist() == bounds[:-1]
    # 130 utterances: two launches
    r = g.random((12, 1, 130, 2, 9)).astype(np.float32)
    _check_align(r, [1 + b % 9 for b in range(130)], [b % 13 for b in range(130)])


def test_align_long_text():
    """L = 2048 at 401 steps (only the texts of <= 401 tokens have a path), then 2048-token texts over 2100 frames."""
    g = np.random.default_rng(6)
    p = g.random((401, 3, 8, 4, 2048)).astype(np.float32)
    _check_align(p, [2048, 2048, 1000, 401, 402, 1, 2047, 64], [401] * 8)
    del p
    q = g.random((2100, 1, 3, 2, 2048)).astype(np.float32)
    got = _check_align(q, [2048, 2047, 1500], [2100, 2048, 2100])
    f = got[1, :2047]  # 2047 tokens in 2048 frames: one token holds two frames, every other one
    assert f[0] == 0 and np.all(np.diff(f) >= 1) and f[-1] <= 2047 and np.sum(np.diff(f) == 2) + (f[-1] == 2046) == 1


# ---- the public API (the e2e fixture)

TEXT = " ".join(str(7 * i + 3) for i in range(20))
KW = dict(max_frames=40, min_gen_frames=10 ** 9)


def _api():
    from tests.cases import e2e_inputs
    from tests.test_e2e_gpu import _tts

    tts, _ = _tts()
    _cfg, _sd, inp = e2e_inputs()
    return tts, tts.prepare_reference(ref_tokens_tq=inp["ref_tokens_tq"])


def _tuples(ws):
    return [(w.word, w.start, w.end, w.char_start, w.char_end) for w in ws]


def test_synthesize_word_timestamps():
    from sopro_b200.stretch import quantise

    tts, ref = _api()
    hop = tts.codec.engine.hop
    for extra in ({}, dict(speed=1.3), dict(sample_rate=16000, loudness=-20.0)):
        plain = tts.synthesize(TEXT, ref=ref, seed=5, **KW, **extra)
        captured = {}
        real = tts._batch_codes

        def spy(*a, **k):
            out = real(*a, **k)
            captured["trace"], captured["T"] = k["trace_out"]["probs"].clone(), int(out[0][0])
            return out

        tts._batch_codes = spy
        try:
            wav, words = tts.synthesize(TEXT, ref=ref, seed=5, word_timestamps=True, **KW, **extra)
        finally:
            tts._batch_codes = real
        assert torch.equal(wav, plain)
        _ids, spans = tts.tokenizer.encode_with_offsets(TEXT)
        p = captured["trace"].cpu().numpy()
        first = AO.first_frames(p, [len(spans)], [captured["T"]])[0]
        S = quantise(extra["speed"]) if "speed" in extra else None
        assert _tuples(words) == AO.words_for(TEXT, spans, first, captured["T"], hop, S)
        assert [w.word for w in words] == TEXT.split()
        sr = extra.get("sample_rate", 24000)
        dur = wav.shape[-1] / sr
        assert all(0 <= w.start <= w.end <= dur + 1e-9 for w in words)
        assert all(a.end <= b.start for a, b in zip(words, words[1:]))
    # the global generator: same state after the call with and without the flag
    torch.manual_seed(3)
    tts.synthesize(TEXT, ref=ref, **KW)
    s1 = torch.get_rng_state()
    torch.manual_seed(3)
    tts.synthesize(TEXT, ref=ref, word_timestamps=True, **KW)
    assert torch.equal(torch.get_rng_state(), s1)


def test_synthesize_batch_word_timestamps():
    tts, ref = _api()
    hop = tts.codec.engine.hop
    texts = [TEXT, "1 2 3", " ".join(str(i) for i in range(40, 70)), "5"]
    seeds = [11, 12, 13, 14]
    captured = {}
    real = tts._batch_codes

    def spy(*a, **k):
        out = real(*a, **k)
        if k.get("trace_out") is not None:
            captured["probs"] = k["trace_out"]["probs"].clone()
            captured["lens"] = list(k["trace_out"]["lens"])
            captured["Ts"] = list(out[0])
        return out

    tts._batch_codes = spy
    try:
        wavs, words = tts.synthesize_batch(texts, ref=ref, seeds=seeds, word_timestamps=True, **KW)
    finally:
        tts._batch_codes = real
    plain = tts.synthesize_batch(texts, ref=ref, seeds=seeds, **KW)
    assert all(torch.equal(a, b) for a, b in zip(wavs, plain))
    p = captured["probs"].cpu().numpy()
    first = AO.first_frames(p, captured["lens"], captured["Ts"])
    identical = 0
    for i, t in enumerate(texts):
        spans = tts.tokenizer.encode_with_offsets(t)[1]
        assert _tuples(words[i]) == AO.words_for(t, spans, first[i], captured["Ts"][i], hop)
        single, sw = tts.synthesize(t, ref=ref, seed=seeds[i], word_timestamps=True, **KW)
        assert torch.equal(single, wavs[i])
        if captured["Ts"][i] >= len(spans):
            assert len(words[i]) == len(t.split())
    # the batch trace against a single call's trace (team geometry may reorder fp32 sums)
    one = {}

    def spy1(*a, **k):
        out = real(*a, **k)
        one["trace"] = k["trace_out"]["probs"].clone()
        return out

    tts._batch_codes = spy1
    try:
        tts.synthesize(texts[0], ref=ref, seed=seeds[0], word_timestamps=True, **KW)
    finally:
        tts._batch_codes = real
    a = one["trace"][:, :, 0].cpu()
    L0 = captured["lens"][0]
    b = captured["probs"][:, :, 0, :, :L0].cpu()
    T0 = captured["Ts"][0]
    err = float((a[:T0, ..., :L0] - b[:T0]).abs().max())
    assert err <= 5e-5, err
    identical = bool(torch.equal(a[:T0, ..., :L0], b[:T0]))
    print(f"batch vs single trace: max diff {err:.2e}, bit-identical: {identical}")
    # the device alignment of a real trace against the oracle
    _check_align(p, captured["lens"], captured["Ts"])


def test_synthesize_long_word_timestamps():
    from sopro_b200 import longform as LF

    tts, ref = _api()
    text = "3 7 11 15. 5 9 13 17 21! 4 8?\n\n6 2   10 12 14 16 18 20 22 24, 26 28 30. 1"
    kw = dict(max_frames=16, min_gen_frames=10 ** 9)
    plain = tts.synthesize_long(text, ref=ref, max_tokens=7, seed=40, **kw)
    captured = {"probs": [], "lens": [], "Ts": []}
    real = tts._batch_codes
    real_join = LF.join_segments

    def spy(*a, **k):
        out = real(*a, **k)
        captured["probs"].append(k["trace_out"]["probs"].clone())
        captured["lens"].append(list(k["trace_out"]["lens"]))
        captured["Ts"].append(list(out[0]))
        return out

    def spy_join(rows, ext, pause_ms):
        captured["ext"] = ext.cpu().numpy().copy()
        return real_join(rows, ext, pause_ms)

    tts._batch_codes = spy
    LF.join_segments = spy_join
    try:
        wav, words = tts.synthesize_long(text, ref=ref, max_tokens=7, seed=40, word_timestamps=True, **kw)
    finally:
        tts._batch_codes = real
        LF.join_segments = real_join
    assert torch.equal(wav, plain)
    segs = LF.split_text(text, tts.tokenizer, 7)
    firsts, Ts = [], []
    for p, lens, ts in zip(captured["probs"], captured["lens"], captured["Ts"]):
        f = AO.first_frames(p.cpu().numpy(), lens, ts)
        firsts.extend(f[i] for i in range(len(lens)))
        Ts.extend(ts)
    spans = [tts.tokenizer.encode_with_offsets(s)[1] for s in segs]
    want = AO.long_words(text, segs, spans, firsts, Ts, tts.codec.engine.hop, captured["ext"], LF.pause_samples(250))
    assert _tuples(words) == want
    assert [text[w.char_start: w.char_end] for w in words] == text.split()
    dur = wav.shape[-1] / 24000
    assert all(0 <= w.start <= w.end <= dur + 1e-9 for w in words)
