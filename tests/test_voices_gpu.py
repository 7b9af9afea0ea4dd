"""GPU: a voice per text.  The prefill over a voice table (sopro_prefill_run_voices) row for row against one-voice
launches, bit for bit, and against the CPU restatement; Token2SV scored against a vector per row; synthesize_batch with
ref=[...] against synthesize with each text's own voice, with every option of the output chain and best-of-N."""
import numpy as np
import pytest
import torch

from tests.cases import e2e_inputs

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
_S = {}
KW = dict(max_frames=40, min_gen_frames=10 ** 9)


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


def _device_voice(rp, Tr, seed):
    from sopro_b200.prefill import PreparedReference

    tok = torch.randint(0, 2048, (Tr, 32), generator=torch.Generator().manual_seed(seed))
    sv, seq, caches = rp.run(tok)
    return PreparedReference(ref_tokens_btq=tok.unsqueeze(0), sv_ref=sv, ref_seq=seq, ref_kv_caches=caches)


# 18 distinct voices (more than the 16 rows of the skinny kernel, so a FiLM launch over all of them would have taken
# the tile kernel), short and long references
TRS = [1, 2, 37, 150, 300, 5, 9, 16, 17, 64, 100, 200, 250, 33, 70, 120, 180, 260]


def test_prefill_rows_equal_one_voice_launches_bit_for_bit():
    from sopro_b200 import prefill as P

    eng, rp, (tpos, fpos) = _engines()
    cfg, sd, _ = e2e_inputs()
    refs = [_device_voice(rp, Tr, 100 + i) for i, Tr in enumerate(TRS)]
    g = torch.Generator().manual_seed(11)
    B = 24
    texts = [torch.randint(0, 1000, (int(n),), generator=g) for n in torch.randint(1, 61, (B,), generator=g)]
    texts[3] = texts[0].clone()  # the same text in two voices
    of = [b % len(refs) for b in range(B)]  # texts 18.. repeat the objects of voices 0..5
    F = 40
    txt, lens, pool, cond = eng.run(texts, [refs[v] for v in of], n_frames=F + 1, style_strength=1.2)
    assert of[0] != of[3] and not torch.equal(cond[0], cond[3]), "two voices gave the same cond_ar"
    worst = 0.0
    for v, r in enumerate(refs):
        rows = [b for b in range(B) if of[b] == v]
        t1, l1, p1, c1 = eng.run(texts, r, n_frames=F + 1, style_strength=1.2)  # the same texts, every M equal
        assert l1 == lens
        for b in rows:
            assert torch.equal(txt[b, : lens[b]], t1[b, : lens[b]]), (v, b)
            assert torch.equal(pool[b], p1[b]) and torch.equal(cond[b], c1[b]), (v, b)
        b = rows[0]
        want = P.prepare_conditioning(sd, cfg, texts[b], r, max_frames=F, device="cpu", style_strength=1.2, text_pos=tpos,
                                      frame_pos=fpos)
        for got, w in ((txt[b, : lens[b]], want["txt_seq"][0]), (pool[b], want["txt_pool"][0]), (cond[b], want["cond_ar"][0])):
            err = float((got.cpu() - w).abs().max())
            worst = max(worst, err)
            assert err <= 2e-5, (v, b, err)
    print(f"voice-table prefill vs CPU restatement: max abs err {worst:.2e}")
    # a sequence of one object is the one-voice launch
    t2, _, p2, c2 = eng.run(texts, [refs[4]] * B, n_frames=F + 1, style_strength=1.2)
    t3, _, p3, c3 = eng.run(texts, refs[4], n_frames=F + 1, style_strength=1.2)
    assert torch.equal(c2, c3) and torch.equal(p2, p3) and torch.equal(t2, t3)


def test_prefill_voice_table_refusals_through_the_c_abi():
    import ctypes as C

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

    def call(nv, vmap, tr, k=kp):
        return lib.sopro_prefill_run_voices(eng._h, ids.data_ptr(), ln.data_ptr(), 2, 4, nv, (C.c_int32 * 2)(*vmap), sv.data_ptr(),
                                            (C.c_int32 * 2)(*tr), k, k, 1.0, 5, *[t.data_ptr() for t in out], st)

    assert call(2, [0, 1], [8, 8]) == 0
    assert call(3, [0, 1], [8, 8]) == -1      # more voices than texts
    assert call(0, [0, 0], [8, 8]) == -1
    assert call(2, [0, 2], [8, 8]) == -1      # a text with no voice
    assert call(2, [0, -1], [8, 8]) == -1
    assert call(2, [0, 1], [8, 4097]) == -1   # Tr outside [1, 4096]
    assert call(2, [0, 1], [0, 8]) == -1
    assert call(2, [0, 1], [8, 8], (C.c_void_p * 6)(*([kv.data_ptr()] * 5 + [None]))) == -1
    torch.cuda.synchronize()


def test_speaker_vectors_with_a_vector_per_row_equal_the_single_vector_calls():
    _, rp, _ = _engines()
    lens = [1, 2, 6, 17, 37, 400, 16, 90]
    codes = torch.randint(0, 2048, (len(lens), max(lens), 32), generator=torch.Generator().manual_seed(5))
    refs = torch.nn.functional.normalize(torch.randn(len(lens), 192, generator=torch.Generator().manual_seed(6)), dim=1)
    sv, cos = rp.speaker_vectors(codes, lens, refs)
    assert sv.shape == (len(lens), 192) and cos.shape == (len(lens),)
    for b in range(len(lens)):
        sv1, cos1 = rp.speaker_vectors(codes, lens, refs[b])
        assert torch.equal(sv1, sv) and torch.equal(cos1[b], cos[b]), b
    with pytest.raises(ValueError):
        rp.speaker_vectors(codes, lens, refs[:3])
    with pytest.raises(ValueError):
        rp.speaker_vectors(codes, lens, torch.zeros(len(lens), 191))


# ---------------------------------------------------------------------------------------------------------------
# the public call
# ---------------------------------------------------------------------------------------------------------------
def _tts():
    from tests.test_e2e_gpu import _tts as tts

    return tts()[0]


def _voices(tts, n, seed=0, Trs=(38, 1, 120, 7, 300, 64)):
    out = []
    for i in range(n):
        tok = torch.randint(0, 2048, (Trs[i % len(Trs)], 32), generator=torch.Generator().manual_seed(seed + i))
        out.append(tts.prepare_reference(ref_tokens_tq=tok))
    return out


TEXTS = [" ".join(str(7 * i + 3) for i in range(20)), " ".join(str(i) for i in range(3, 40, 3)), "5 9",
         " ".join(str(11 * i + 2) for i in range(30))]
SEEDS = [1, 2, 3, 4]


def _tuples(ws):
    return [(w.word, w.start, w.end, w.char_start, w.char_end) for w in ws]


def test_synthesize_batch_voice_per_text_equals_synthesize():
    tts = _tts()
    refs = _voices(tts, len(TEXTS))
    wavs = tts.synthesize_batch(TEXTS, ref=refs, seeds=SEEDS, **KW)
    for t, r, s, w in zip(TEXTS, refs, SEEDS, wavs):
        assert torch.equal(w, tts.synthesize(t, ref=r, seed=s, **KW))
    # the voice matters: the first text in another voice is other audio
    other = tts.synthesize(TEXTS[0], ref=refs[1], seed=SEEDS[0], **KW)
    assert not torch.equal(other, wavs[0])


def test_synthesize_batch_voice_per_text_with_the_output_chain():
    tts = _tts()
    refs = _voices(tts, len(TEXTS), seed=20)
    opts = dict(speed=1.3, sample_rate=16000, loudness=-20.0, watermark=12345)
    wavs = tts.synthesize_batch(TEXTS, ref=refs, seeds=SEEDS, **opts, **KW)
    for t, r, s, w in zip(TEXTS, refs, SEEDS, wavs):
        assert torch.equal(w, tts.synthesize(t, ref=r, seed=s, **opts, **KW))


def test_synthesize_batch_voice_per_text_word_timestamps():
    tts = _tts()
    refs = _voices(tts, len(TEXTS), seed=40)
    kw = dict(max_frames=60)
    wavs, words = tts.synthesize_batch(TEXTS, ref=refs, seeds=SEEDS, word_timestamps=True, **kw)
    for i, (t, r, s) in enumerate(zip(TEXTS, refs, SEEDS)):
        w1, ws1 = tts.synthesize(t, ref=r, seed=s, word_timestamps=True, **kw)
        assert torch.equal(wavs[i], w1) and _tuples(words[i]) == _tuples(ws1), i


def test_synthesize_batch_voice_per_text_best_of():
    """Text i's three takes run in voice i and are scored against voice i's sv_ref: each result equals synthesize with
    best_of=3 in that voice (whose takes and scores are computed alone)."""
    tts = _tts()
    refs = _voices(tts, 3, seed=60)
    texts, seeds = TEXTS[:3], [5, 50, 500]
    kw = dict(max_frames=48)
    wavs, words = tts.synthesize_batch(texts, ref=refs, seeds=seeds, best_of=3, word_timestamps=True, **kw)
    for i, (t, r, s) in enumerate(zip(texts, refs, seeds)):
        w1, ws1 = tts.synthesize(t, ref=r, seed=s, best_of=3, word_timestamps=True, **kw)
        assert torch.equal(wavs[i], w1) and _tuples(words[i]) == _tuples(ws1), i
    # two texts sharing a voice object and one other
    shared = [refs[0], refs[1], refs[0]]
    wavs = tts.synthesize_batch(texts, ref=shared, seeds=seeds, best_of=3, **kw)
    for t, r, s, w in zip(texts, shared, seeds, wavs):
        assert torch.equal(w, tts.synthesize(t, ref=r, seed=s, best_of=3, **kw))


def test_synthesize_batch_with_voices_from_in_memory_clips():
    from tests.test_ingest_gpu import _tts as tts_with_encoder

    tts = tts_with_encoder()
    g = np.random.default_rng(7)
    clips, rates = [], []
    for i, (sr, f0, sec) in enumerate(((24000, 180.0, 2.0), (16000, 260.0, 3.0), (22050, 120.0, 1.5))):
        t = np.arange(int(sr * sec)) / sr
        clips.append(torch.from_numpy((0.4 * np.sin(2 * np.pi * f0 * t) + 0.02 * g.standard_normal(t.size)).astype(np.float32)))
        rates.append(sr)
    refs = tts.prepare_references(clips, sample_rates=rates)
    wavs = tts.synthesize_batch(TEXTS[:3], ref=refs, seeds=SEEDS[:3], **KW)
    for t, r, s, w in zip(TEXTS, refs, SEEDS, wavs):
        assert torch.equal(w, tts.synthesize(t, ref=r, seed=s, **KW))


def test_repeated_object_equals_the_shared_reference():
    tts = _tts()
    r = _voices(tts, 1, seed=80)[0]
    a = tts.synthesize_batch(TEXTS, ref=[r] * len(TEXTS), seeds=SEEDS, **KW)
    b = tts.synthesize_batch(TEXTS, ref=r, seeds=SEEDS, **KW)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    a = tts.synthesize_batch(TEXTS[:2], ref=(r, r), seeds=SEEDS[:2], best_of=2, **KW)
    b = tts.synthesize_batch(TEXTS[:2], ref=r, seeds=SEEDS[:2], best_of=2, **KW)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_refusals_through_the_public_call_draw_nothing():
    import dataclasses

    tts = _tts()
    r = _voices(tts, 1, seed=90)[0]
    padded = dataclasses.replace(r, ref_kv_caches=[dict(c) for c in r.ref_kv_caches])
    padded.ref_kv_caches[0]["key_padding_mask"] = torch.zeros((1, int(r.ref_kv_caches[0]["k"].shape[2])), dtype=torch.bool)
    long_kv = [{"k": c["k"].new_zeros((1, 2, 4097, 192)), "v": c["v"].new_zeros((1, 2, 4097, 192)), "key_padding_mask": None}
               for c in r.ref_kv_caches]
    small_sv = dataclasses.replace(r, sv_ref=r.sv_ref[:, :128])
    cases = [([r], ValueError), ([r, r, r], ValueError), ([r, "voice.wav"], TypeError), ([r, None], TypeError),
             ([r, dataclasses.replace(r, ref_kv_caches=r.ref_kv_caches[:2])], ValueError), ([r, small_sv], ValueError),
             ([dataclasses.replace(r, ref_kv_caches=long_kv), r], ValueError), ([r, padded], NotImplementedError)]
    for ref, exc in cases:
        torch.manual_seed(3)
        before = torch.get_rng_state()
        with pytest.raises(exc):
            tts.synthesize_batch(TEXTS[:2], ref=ref, max_frames=8)  # no seeds: a draw would move the generator
        assert torch.equal(torch.get_rng_state(), before), (ref, exc)


def test_sixty_four_texts_in_sixty_four_voices_at_full_length():
    """The size a service runs: 64 texts, 64 voices, 401 frames each; a sample of rows against synthesize."""
    tts = _tts()
    refs = _voices(tts, 64, seed=1000, Trs=(38, 150, 12, 300, 75, 1, 220, 9))
    texts = [" ".join(str((13 * i + 5 * j) % 997) for j in range(8 + i % 40)) for i in range(64)]
    seeds = [7000 + i for i in range(64)]
    kw = dict(max_frames=400, min_gen_frames=10 ** 9)
    wavs = tts.synthesize_batch(texts, ref=refs, seeds=seeds, **kw)
    assert len(wavs) == 64
    print(f"64 voices: {sum(int(w.shape[-1]) for w in wavs) // 1920} frames decoded")
    for i in (0, 17, 41, 63):
        assert torch.equal(wavs[i], tts.synthesize(texts[i], ref=refs[i], seed=seeds[i], **kw)), i
