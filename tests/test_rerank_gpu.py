"""GPU: best-of-N synthesis.  The batched Token2SV (sopro_refprep_speaker_vectors) against the float64 restatement
oracle/speaker_oracle.py and, bit for bit, against sopro_refprep_run row by row; then synthesize / synthesize_batch /
synthesize_long with best_of against their own picked single takes."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import speaker_oracle as SO
from tests.cases import e2e_inputs

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
_S = {}
TEXT = " ".join(str(7 * i + 3) for i in range(12))
KW = dict(max_frames=48)
U = 2.0 ** -24  # fp32 unit round-off


def _refprep():
    from sopro_b200.prefill_cuda import RefPrepEngine

    if "rp" not in _S:
        cfg, sd, _ = e2e_inputs()
        _S["rp"] = RefPrepEngine(cfg, sd, 0)
    return _S["rp"]


def _api():
    from tests.test_e2e_gpu import _tts

    tts, _ = _tts()
    _cfg, _sd, inp = e2e_inputs()
    if "ref" not in _S:
        _S["ref"] = tts.prepare_reference(ref_tokens_tq=inp["ref_tokens_tq"])
    return tts, _S["ref"]


def _codes(lens, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 2048, (len(lens), max(lens), 32), generator=g)


def _tol(T: int) -> float:
    """Bound on |sv_fp32 - sv_f64| per component for a T-frame row.  The longest fp32 chains are the pooling sums over
    the T frames (mu, then the variance around it): a recursive fp32 sum of n terms errs by at most n*u times the sum
    of their magnitudes (Higham, gamma_n), and the softmax weights sum to 1, so mu and std carry <= 2*T*u relative error
    each.  The mixes (32 terms), the convolutions (7 taps), the 192-term pooling projection and the 384-term output
    projection add <= (32 + 2*7 + 192 + 384)*u, and the normalisation of a unit vector a few u.  With a margin of 4 for
    the gain of the projection onto a unit vector: 4 * (2T + 650) * u."""
    return 4.0 * (2 * T + 650) * U


@pytest.mark.parametrize("lens", [[1, 2, 6, 7, 37, 400, 4096], [23], "16", "64"])
def test_speaker_vectors_match_the_float64_oracle_and_run_row_by_row(lens):
    rp = _refprep()
    cfg, sd, _ = e2e_inputs()
    if isinstance(lens, str):
        n = int(lens)
        lens = torch.randint(1, 130, (n,), generator=torch.Generator().manual_seed(n)).tolist()
        lens[0] = 17  # just above the skinny kernel's 16 rows
        lens[1] = 16
    codes = _codes(lens, len(lens))
    ref_sv = torch.nn.functional.normalize(torch.randn(192, generator=torch.Generator().manual_seed(2)), dim=0)
    sv, cos = rp.speaker_vectors(codes, lens, ref_sv)
    assert sv.shape == (len(lens), 192) and cos.shape == (len(lens),)
    want, wcos = SO.speaker_vectors(sd, 2048, codes, lens, ref_sv)
    got = sv.cpu().double()
    worst = 0.0
    for b, T in enumerate(lens):
        err = float((got[b] - want[b]).abs().max())
        worst = max(worst, err / _tol(T))
        assert err <= _tol(T), (b, T, err, _tol(T))
        # cos is the dot of the returned sv with ref_sv: 192 fp32 products of unit vectors, <= 192 u
        assert abs(float(cos[b]) - float(got[b] @ ref_sv.double())) <= 192 * U
        assert abs(float(cos[b]) - float(wcos[b])) <= _tol(T) * 192 ** 0.5
    print(f"speaker_vectors vs float64: worst error {worst:.3f} of the bound")
    # every row equals the B = 1 path of sopro_refprep_run on its own codes, bit for bit
    for b, T in enumerate(lens):
        alone = rp.run(codes[b, :T])[0]
        assert torch.equal(alone[0], sv[b]), (b, T)
    sv2, none = rp.speaker_vectors(codes, lens)
    assert none is None and torch.equal(sv2, sv)


def test_speaker_vectors_b1_path_keeps_the_fixture_sv_ref():
    import os

    rp = _refprep()
    _, _, inp = e2e_inputs()
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "e2e_prefill.npz"))
    tok = inp["ref_tokens_tq"]
    sv, _ = rp.speaker_vectors(tok.unsqueeze(0), [int(tok.shape[0])])
    np.testing.assert_allclose(sv.cpu().numpy(), g["sv_ref"], rtol=0, atol=2e-6)
    assert torch.equal(sv, rp.run(tok)[0])


def test_speaker_vectors_refusals():
    from sopro_b200 import _lib

    rp = _refprep()
    codes = _codes([5, 9], 1)
    for bad in ([0, 9], [5, 10], [5], [-1, 3]):
        with pytest.raises(ValueError):
            rp.speaker_vectors(codes, bad)
    with pytest.raises(ValueError):
        rp.speaker_vectors(torch.zeros((1, 4097, 32), dtype=torch.long), [4097])
    with pytest.raises(ValueError):
        rp.speaker_vectors(torch.zeros((0, 4, 32), dtype=torch.long), [])
    # through the C ABI: B < 1, and ref_sv without cos
    lib = _lib.load()
    tok = codes.to("cuda", torch.int32).contiguous()
    ln = (C.c_int32 * 2)(5, 9)
    sv = torch.empty((2, 192), device="cuda")
    ref = torch.zeros(192, device="cuda")
    st = _lib.stream_ptr(tok.device)
    assert lib.sopro_refprep_speaker_vectors(rp._h, tok.data_ptr(), 0, 9, ln, sv.data_ptr(), None, None, st) == -1
    assert lib.sopro_refprep_speaker_vectors(rp._h, tok.data_ptr(), 2, 9, ln, sv.data_ptr(), ref.data_ptr(), None, st) == -1
    # out-of-range codes trip sopro_refprep_check, which clears the flag
    bad = codes.clone()
    bad[1, 8, 3] = 2048
    with pytest.raises(IndexError):
        rp.speaker_vectors(bad, [5, 9])
    rp.speaker_vectors(codes, [5, 9])
    bad[1, 8, 3] = 5
    bad[0, 7, 3] = 5000  # past row 0's 5 frames: never read
    rp.speaker_vectors(bad, [5, 9])


def _pick(tts, ref, text, seeds, **kw):
    """k* computed independently: every candidate alone with best_of=1, scored by speaker_vectors, then choose."""
    from sopro_b200 import rerank

    ids = tts.encode_text(text)
    Ts, stopped, cos = [], [], []
    st = float(tts.cfg.style_strength)
    for s in seeds:
        tok = tts.model.generate_tokens(ids, ref, style_strength=st, seed=s, **kw)
        T = int(tok.shape[0])
        Ts.append(T)
        stopped.append(T < int(kw["max_frames"]) + 1)
        cos.append(float(tts.model.refprep.speaker_vectors(tok.unsqueeze(0), [T], ref.sv_ref)[1][0]) if T else 0.0)
    return rerank.choose(Ts, stopped, int(ids.numel()), cos), Ts


def _tuples(ws):
    return [(w.word, w.start, w.end, w.char_start, w.char_end) for w in ws]


@pytest.mark.parametrize("N", [2, 8])
def test_synthesize_best_of_equals_the_picked_take(N):
    tts, ref = _api()
    s = 21
    k, Ts = _pick(tts, ref, TEXT, [s + k for k in range(N)], **KW)
    print(f"best_of={N}: frames {Ts}, picked {k}")
    got = tts.synthesize(TEXT, ref=ref, seed=s, best_of=N, **KW)
    assert torch.equal(got, tts.synthesize(TEXT, ref=ref, seed=s + k, **KW))
    for extra in (dict(speed=1.3), dict(sample_rate=16000, loudness=-20.0)):
        got = tts.synthesize(TEXT, ref=ref, seed=s, best_of=N, **KW, **extra)
        assert torch.equal(got, tts.synthesize(TEXT, ref=ref, seed=s + k, **KW, **extra)), extra
    wav, words = tts.synthesize(TEXT, ref=ref, seed=s, best_of=N, word_timestamps=True, speed=1.3, **KW)
    wav1, words1 = tts.synthesize(TEXT, ref=ref, seed=s + k, word_timestamps=True, speed=1.3, **KW)
    assert torch.equal(wav, wav1) and _tuples(words) == _tuples(words1)


def test_synthesize_batch_best_of_equals_each_picked_take():
    tts, ref = _api()
    texts, seeds, N = [TEXT, "1 2 3", " ".join(str(i) for i in range(40, 70))], [5, 50, 500], 4
    wavs, words = tts.synthesize_batch(texts, ref=ref, seeds=seeds, best_of=N, word_timestamps=True, **KW)
    for i, t in enumerate(texts):
        k, _ = _pick(tts, ref, t, [seeds[i] + k for k in range(N)], **KW)
        w1, ws1 = tts.synthesize(t, ref=ref, seed=seeds[i] + k, word_timestamps=True, **KW)
        assert torch.equal(wavs[i], w1), i
        assert _tuples(words[i]) == _tuples(ws1), i


def test_synthesize_long_best_of_joins_the_picked_takes():
    from sopro_b200 import longform as LF

    tts, ref = _api()
    text = "3 7 11 15. 5 9 13 17 21! 4 8?\n\n6 2   10 12 14 16 18 20 22 24, 26 28 30. 1"
    kw, seed, N = dict(max_frames=24), 40, 3
    segs = LF.split_text(text, tts.tokenizer, 7)
    picks = [_pick(tts, ref, sg, [seed + i + k for k in range(N)], **kw)[0] for i, sg in enumerate(segs)]
    wav, words = tts.synthesize_long(text, ref=ref, max_tokens=7, seed=seed, best_of=N, word_timestamps=True, **kw)
    # the same passage with best_of=1 and each segment's picked seed
    real = tts._batch_codes

    def picked(part, ref_, *, seeds, **k):
        return real(part, ref_, seeds=[s + picks[s - seed] for s in seeds], **k)

    tts._batch_codes = picked
    try:
        want, wwords = tts.synthesize_long(text, ref=ref, max_tokens=7, seed=seed, word_timestamps=True, **kw)
    finally:
        tts._batch_codes = real
    assert torch.equal(wav, want)
    assert _tuples(words) == _tuples(wwords)


def test_default_is_unchanged_and_only_picked_rows_are_decoded():
    tts, ref = _api()
    assert torch.equal(tts.synthesize(TEXT, ref=ref, seed=3, best_of=1, **KW), tts.synthesize(TEXT, ref=ref, seed=3, **KW))
    torch.manual_seed(4)
    a = tts.synthesize(TEXT, ref=ref, **KW)
    sa = torch.get_rng_state()
    torch.manual_seed(4)
    b = tts.synthesize(TEXT, ref=ref, best_of=1, **KW)
    assert torch.equal(a, b) and torch.equal(torch.get_rng_state(), sa)
    eng = tts.codec.engine
    real = eng.decode
    rows = []

    def count(codes_bqt, *a, **k):
        rows.append(int(codes_bqt.shape[0]))
        return real(codes_bqt, *a, **k)

    eng.decode = count
    try:
        tts.synthesize(TEXT, ref=ref, seed=3, best_of=8, **KW)
        assert sum(rows) == 1, rows
        rows.clear()
        texts = [TEXT, "1 2 3", "9 8 7 6"]
        out = tts.synthesize_batch(texts, ref=ref, seeds=[1, 2, 3], best_of=4, **KW)
        assert sum(rows) == sum(1 for w in out if w.shape[-1] > 0), rows
    finally:
        eng.decode = real
