"""GPU: voice blends.  The blended prefill (sopro_prefill_run_blends) against the float64 oracle
(oracle/blend_oracle.py) and, bit for bit, against run_voices and one-voice launches; blend_voices through every entry
point that takes a voice; the C-ABI's refusals."""
import ctypes as C

import pytest
import torch

from tests.cases import e2e_inputs

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
_S = {}
F = 40


def _engines():
    from sopro_b200 import prefill as P
    from sopro_b200.prefill_cuda import PrefillEngine, RefPrepEngine

    if "e" not in _S:
        cfg, sd, _ = e2e_inputs()
        tpos = P.sinusoid_table(int(cfg.max_text_len) + 8, int(cfg.d_model), "cpu")
        fpos = P.sinusoid_table(int(cfg.pos_emb_max) + 8, int(cfg.d_model), "cpu")
        _S["e"] = PrefillEngine(cfg, sd, 0, tpos, fpos)
        _S["rp"] = RefPrepEngine(cfg, sd, 0)
        _S["pos"] = (tpos, fpos)
    return _S["e"], _S["rp"], _S["pos"]


def _device_voice(Tr, seed):
    from sopro_b200.prefill import PreparedReference

    _, rp, _ = _engines()
    tok = torch.randint(0, 2048, (Tr, 32), generator=torch.Generator().manual_seed(seed))
    sv, seq, caches = rp.run(tok)
    return PreparedReference(ref_tokens_btq=tok.unsqueeze(0), sv_ref=sv, ref_seq=seq, ref_kv_caches=caches)


def _blend(vs, ws=None):
    from sopro_b200 import voices

    return voices.blend(vs, ws, device="cuda:0", **voices.geometry(e2e_inputs()[0]))


def _texts(B, seed=11):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 1000, (int(n),), generator=g) for n in torch.randint(1, 61, (B,), generator=g)]


# segment lengths: 2, 3 and 16 segments, lengths of 1, totals up to the 4096-frame limit
CASES = [((1, 150), (1.0, 1.0)), ((38, 1, 7), (0.2, 0.5, 0.3)), ((150, 2048), (3.0, 1.0)), ((4095, 1), (1.0, 1.0)),
         ((2048, 2048), (1.0, 2.0)), (tuple(1 + 17 * i for i in range(16)), tuple(1.0 + i for i in range(16)))]


@pytest.mark.parametrize("segs,ws", CASES, ids=[f"{len(s)}seg_{sum(s)}fr" for s, _ in CASES])
def test_blended_rows_match_the_float64_oracle(segs, ws):
    from oracle import blend_oracle as BO

    eng, _, (tpos, fpos) = _engines()
    cfg, sd, _ = e2e_inputs()
    m = _blend([_device_voice(n, 500 + i) for i, n in enumerate(segs)], list(ws))
    assert m.segments == segs
    texts = _texts(3)
    txt, lens, pool, cond = eng.run(texts, m, n_frames=F + 1, style_strength=1.2)
    worst = 0.0
    for b, ids in enumerate(texts):
        want = BO.prepare_conditioning(sd, cfg, ids, m, max_frames=F, style_strength=1.2, text_pos=tpos, frame_pos=fpos)
        err = float((cond[b].cpu().double() - want["cond_ar"][0]).abs().max())
        worst = max(worst, err)
        assert err <= 2e-5, (b, err)
    # the mixture is not any one component's read-out
    one = eng.run(texts, _device_voice(segs[0], 500), n_frames=F + 1, style_strength=1.2)[3]
    assert not torch.equal(one, cond)
    print(f"blend {segs}: max abs err against float64 {worst:.2e}")


def test_one_segment_of_weight_one_equals_run_voices_bit_for_bit():
    """Contract: plain voices (one segment, weight 1) in a run_blends launch give the rows run_voices gives them."""
    eng, _, _ = _engines()
    a, b = _device_voice(38, 1), _device_voice(300, 2)
    m = _blend([_device_voice(5, 3), _device_voice(120, 4)])
    texts = _texts(6)
    plain = eng.run(texts, [a, b, a, b, a, b], n_frames=F + 1, style_strength=1.2)
    mixed = eng.run(texts, [a, m, a, b, m, b], n_frames=F + 1, style_strength=1.2)  # run_blends
    for r in (0, 2, 3, 5):
        assert torch.equal(mixed[3][r], plain[3][r]) and torch.equal(mixed[2][r], plain[2][r]), r
    assert torch.equal(mixed[0], plain[0])
    # blend_voices([a]) is one segment of weight 1 over a's frames, run through run_blends
    solo = eng.run(texts, _blend([a]), n_frames=F + 1, style_strength=1.2)
    ref = eng.run(texts, a, n_frames=F + 1, style_strength=1.2)
    assert all(torch.equal(x, y) for x, y in zip((solo[0], solo[2], solo[3]), (ref[0], ref[2], ref[3])))


def test_a_blended_row_equals_its_row_in_a_launch_of_that_blend_alone():
    eng, _, _ = _engines()
    m1 = _blend([_device_voice(7, 11), _device_voice(1, 12), _device_voice(200, 13)], [1.0, 0.5, 2.0])
    m2 = _blend([_device_voice(64, 14), _device_voice(33, 15)])
    a = _device_voice(90, 16)
    texts = _texts(8)
    of = [m1, m2, a, m1, m2, a, m2, m1]
    _, _, pool, cond = eng.run(texts, of, n_frames=F + 1, style_strength=1.2)
    for v in (m1, m2, a):
        _, _, p1, c1 = eng.run(texts, v, n_frames=F + 1, style_strength=1.2)  # the same texts: every M equal
        for r in range(len(texts)):
            if of[r] is v:
                assert torch.equal(cond[r], c1[r]) and torch.equal(pool[r], p1[r]), r


def test_run_blends_refusals_through_the_c_abi():
    from sopro_b200 import _lib

    eng, _, _ = _engines()
    lib = _lib.load()
    ids = torch.zeros((2, 4), dtype=torch.int32, device="cuda")
    ln = torch.full((2,), 4, dtype=torch.int32, device="cuda")
    sv = torch.zeros((2, 192), device="cuda")
    kv = torch.zeros((2, 8, 192), device="cuda")
    out = [torch.empty((2, 4, 384), device="cuda"), torch.empty((2, 384), device="cuda"), torch.empty((2, 5, 384), device="cuda")]
    kp = (C.c_void_p * 6)(*([kv.data_ptr()] * 6))
    st = _lib.stream_ptr(ids.device)

    def call(nseg, frames, ws, tr=(8, 8)):
        return lib.sopro_prefill_run_blends(eng._h, ids.data_ptr(), ln.data_ptr(), 2, 4, 2, (C.c_int32 * 2)(0, 1), sv.data_ptr(),
                                            (C.c_int32 * 2)(*tr), kp, kp, (C.c_int32 * 2)(*nseg),
                                            (C.c_int32 * len(frames))(*frames), (C.c_float * len(ws))(*ws), 1.0, 5,
                                            *[t.data_ptr() for t in out], st)

    assert call([1, 2], [8, 3, 5], [1.0, 0.5, 0.5]) == 0
    assert call([2, 2], [4, 4, 3, 5], [0.5, 0.5, 0.5, 0.5]) == 0
    assert call([0, 1], [8, 8], [1.0, 1.0]) == -1                       # a voice of no segment
    assert call([17, 1], [1] * 8 + [0] * 9 + [8], [1.0] * 18) == -1     # more than 16 segments
    assert call([1, 2], [8, 3, 4], [1.0, 0.5, 0.5]) == -1               # segments that do not cover tr
    assert call([1, 2], [8, 8, 0], [1.0, 0.5, 0.5]) == -1               # an empty segment
    assert call([1, 2], [8, 3, 5], [1.0, 0.0, 0.5]) == -1               # a zero weight
    assert call([1, 2], [8, 3, 5], [1.0, -0.5, 0.5]) == -1
    assert call([1, 2], [8, 3, 5], [1.0, float("nan"), 0.5]) == -1
    assert call([1, 2], [8, 3, 5], [1.0, float("inf"), 0.5]) == -1
    assert call([1, 1], [8, 4097], [1.0, 1.0], tr=(8, 4097)) == -1      # Tr past the limit (prefill_core's check)
    assert lib.sopro_prefill_run_blends(eng._h, ids.data_ptr(), ln.data_ptr(), 2, 4, 2, (C.c_int32 * 2)(0, 1), sv.data_ptr(),
                                        (C.c_int32 * 2)(8, 8), kp, kp, None, None, None, 1.0, 5,
                                        *[t.data_ptr() for t in out], st) == -1
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------
# the public call
# ---------------------------------------------------------------------------------------------------------------
KW = dict(max_frames=40, min_gen_frames=10 ** 9)
TEXTS = [" ".join(str(7 * i + 3) for i in range(20)), " ".join(str(i) for i in range(3, 40, 3)), "5 9",
         " ".join(str(11 * i + 2) for i in range(30))]


def _tts():
    from tests.test_e2e_gpu import _tts as tts

    return tts()[0]


def _voices(tts, n, seed=0, Trs=(38, 1, 120, 7, 300, 64)):
    return [tts.prepare_reference(ref_tokens_tq=torch.randint(0, 2048, (Trs[i % len(Trs)], 32),
                                                              generator=torch.Generator().manual_seed(seed + i)))
            for i in range(n)]


def test_blend_voices_of_one_voice_speaks_as_that_voice():
    from sopro_b200.prefill import PreparedReference
    from sopro_b200.voices import VoiceBlend

    tts = _tts()
    a, b = _voices(tts, 2, seed=70)
    want = tts.synthesize(TEXTS[0], ref=a, seed=5, **KW)
    for m in (tts.blend_voices([a]), tts.blend_voices([a, a]), tts.blend_voices([a, a], [0.2, 5.0])):
        assert isinstance(m, VoiceBlend) and isinstance(m, PreparedReference) and m.sv_ref.device == tts.device
        assert torch.equal(tts.synthesize(TEXTS[0], ref=m, seed=5, **KW), want)
    mix = tts.blend_voices([a, b], [1.0, 1.0])
    assert not torch.equal(tts.synthesize(TEXTS[0], ref=mix, seed=5, **KW), want)


def test_synthesize_batch_rows_in_blends_equal_synthesize():
    tts = _tts()
    a, b, c = _voices(tts, 3, seed=80)
    m1, m2 = tts.blend_voices([a, b], [1.0, 3.0]), tts.blend_voices([b, c, a])
    seeds = [1, 2, 3, 4]
    for ref in ([m1, a, m2, m1], m2):
        wavs = tts.synthesize_batch(TEXTS, ref=ref, seeds=seeds, **KW)
        for i, (t, s) in enumerate(zip(TEXTS, seeds)):
            r = ref[i] if isinstance(ref, list) else ref
            assert torch.equal(wavs[i], tts.synthesize(t, ref=r, seed=s, **KW)), i
    # synthesize_long over a blend is its segments in that blend
    w = tts.synthesize_long(TEXTS[0] + ". " + TEXTS[1], ref=m1, seed=9, max_frames=40)
    assert w.shape[-1] > 0


def test_stream_batch_rows_with_blends_equal_stream():
    from tests.test_stream_batch_gpu import _rows, _same_as_stream

    tts = _tts()
    a, b = _voices(tts, 2, seed=90)
    m = tts.blend_voices([a, b], [2.0, 1.0])
    refs = [m, a, m]
    seeds = [7, 8, 9]
    kw = dict(max_frames=40)
    rows = _rows(tts.stream_batch(TEXTS[:3], ref=refs, seeds=seeds, **kw), 3)
    for i in range(3):
        _same_as_stream(rows[i], list(tts.stream(TEXTS[i], ref=refs[i], seed=seeds[i], **kw)))


def test_best_of_scores_takes_against_the_blend_speaker_vector():
    from tests.test_rerank_gpu import _pick

    tts = _tts()
    a, b = _voices(tts, 2, seed=100)
    m = tts.blend_voices([a, b], [1.0, 2.0])
    kw = dict(max_frames=40, min_gen_frames=3)
    s, N = 21, 4
    k, _ = _pick(tts, m, TEXTS[0], [s + j for j in range(N)], **kw)  # scored against m.sv_ref
    assert torch.equal(tts.synthesize(TEXTS[0], ref=m, seed=s, best_of=N, **kw), tts.synthesize(TEXTS[0], ref=m, seed=s + k, **kw))


def test_dialogue_and_ssml_with_a_blended_voice():
    tts = _tts()
    a, b = _voices(tts, 2, seed=110)
    m = tts.blend_voices([a, b])
    kw = dict(max_frames=40, min_gen_frames=3, max_tokens=7)
    t1, t2 = "3 7 11 15. 5 9 13!", "4 8? 6 2 10."
    got = tts.synthesize_dialogue([(m, t1), (a, t2)], seed=40, **kw)
    # the plain voice of that dialogue as a one-voice blend: the same audio (a one-segment blend speaks as its voice)
    assert torch.equal(got, tts.synthesize_dialogue([(m, t1), (tts.blend_voices([a]), t2)], seed=40, **kw))
    assert not torch.equal(got, tts.synthesize_dialogue([(a, t1), (a, t2)], seed=40, **kw))
    # one turn in the blend is synthesize_long in the blend
    one = tts.synthesize_dialogue([(m, t1)], seed=40, **kw)
    assert torch.equal(one, tts.synthesize_long(t1, ref=m, seed=40, **kw))
    ssml = f'<speak>{t1} <voice name="mix">{t2}</voice></speak>'
    s1 = tts.synthesize_ssml(ssml, ref=a, voices={"mix": m}, seed=3, **kw)
    assert s1.shape[-1] > 0
    assert torch.equal(s1, tts.synthesize_ssml(ssml, ref=tts.blend_voices([a]), voices={"mix": m}, seed=3, **kw))
    assert not torch.equal(s1, tts.synthesize_ssml(ssml, ref=a, voices={"mix": a}, seed=3, **kw))
