"""GPU: the public API end to end (prefill -> persistent AR kernel -> NAR -> CUDA Mimi) against the oracles."""
import io

import pytest
import torch

from oracle import ar_oracle as O
from oracle import mimi_oracle as M
from tests.cases import e2e_inputs

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
_TTS = {}


def _tts():
    if "t" not in _TTS:
        from sopro_b200 import SoproTTS
        from sopro_b200.tokenizer import IdsTokenizer

        cfg, sd, inp = e2e_inputs()
        _TTS["mimi_sd"] = M.synth_mimi_state_dict()
        _TTS["t"] = SoproTTS.from_state_dict(cfg, sd, IdsTokenizer(1000), _TTS["mimi_sd"], device="cuda:0")
    return _TTS["t"], _TTS["mimi_sd"]


TEXT = " ".join(str(7 * i + 3) for i in range(20))


def test_synthesize_matches_oracle_pipeline():
    tts, mimi_sd = _tts()
    cfg, sd, inp = e2e_inputs()
    ref = tts.prepare_reference(ref_tokens_tq=inp["ref_tokens_tq"])
    F = 40
    # --- product
    wav = tts.synthesize(TEXT, ref=ref, max_frames=F, seed=11, min_gen_frames=10 ** 9)
    assert wav.shape == (1, 1, (F + 1) * 1920) and wav.dtype == torch.float32 and wav.device.type == "cuda"
    # --- oracle, fed the device-computed conditioning (cond_ar / txt_seq are the kernel's INPUTS)
    prep = tts.model.prepare_conditioning(tts.encode_text(TEXT), ref, max_frames=F, style_strength=cfg.style_strength)
    tape = O.noise_tape(11, F + 1, cfg.ar_vocab())
    want = O.ar_generate(sd, cfg, prep["cond_ar"].cpu(), prep["txt_seq"].cpu(), torch.ones(1, prep["txt_seq"].size(1), dtype=torch.bool),
                         max_frames=F, sampling=O.ArSampling(min_gen_frames=10 ** 9), noise_tv=tape)
    toks = tts.model.generate_tokens(tts.encode_text(TEXT), ref, max_frames=F, style_strength=cfg.style_strength, seed=11,
                                     min_gen_frames=10 ** 9)
    assert toks.shape == (F + 1, 32)
    assert toks[:, 0].tolist() == want  # AR ids bit-identical
    # NAR (CUDA kernels): ids identical to the CPU oracle (pinned to the reference's tokens); a difference is accepted
    # only at an id whose two best logits are within 1e-5 (relative) of a tie in the oracle, checked teacher-forced
    from oracle import nar_oracle as N

    nar_cpu, margin = N.nar_refine({k: v.cpu() for k, v in sd.items()}, cfg, prep["cond_ar"][:, : F + 1].cpu(), torch.tensor(want).unsqueeze(0))
    if not torch.equal(nar_cpu[0], toks.cpu()):
        tts.model.nar.set_forced(nar_cpu)
        try:
            tf = tts.model.nar_refine(prep["cond_ar"][:, : F + 1], torch.tensor(want, device=tts.device).unsqueeze(0)).cpu()
        finally:
            tts.model.nar.set_forced(None)
        bad = [(tuple(i), float(margin[tuple(i)])) for i in (tf != nar_cpu).nonzero().tolist()]
        print("NAR ids differing from the oracle (teacher-forced) -> oracle top-2 margin:", bad)
        assert bad and len(bad) <= 1 and all(m < 1e-5 for _i, m in bad), bad
    # Mimi: decode the product's own tokens with the oracle
    ref_wav = M.mimi_decode(mimi_sd, toks.cpu().permute(1, 0).unsqueeze(0))
    err = float((wav.cpu() - ref_wav).abs().max())
    assert tts.codec.engine.precision == "bf16_tc"  # the default: tensor-core contractions, stated tolerance 2e-2 of peak
    assert err <= 2e-2 * float(ref_wav.abs().max()), err
    tts.codec.engine.set_precision("fp32")
    try:
        wav32 = tts.codec.decode_full(toks)
    finally:
        tts.codec.engine.set_precision("bf16_tc")
    err = float((wav32.cpu() - ref_wav).abs().max())
    assert err <= 2e-4 * max(1.0, float(ref_wav.abs().max())), err


def test_global_rng_is_consumed_like_the_reference():
    """No seed kwarg: the global CPU generator is used, and left where `n` multinomial calls would leave it."""
    tts, _ = _tts()
    cfg, sd, inp = e2e_inputs()
    ref = tts.prepare_reference(ref_tokens_tq=inp["ref_tokens_tq"])
    ids = tts.encode_text(TEXT)
    torch.manual_seed(5)
    a = tts.model.generate_tokens(ids, ref, max_frames=24, style_strength=1.0, min_gen_frames=10 ** 9)
    after = torch.get_rng_state()
    torch.manual_seed(5)
    b = tts.model.generate_tokens(ids, ref, max_frames=24, style_strength=1.0, min_gen_frames=10 ** 9)
    assert torch.equal(a, b)
    torch.manual_seed(5)
    torch.empty(a.size(0), cfg.ar_vocab()).exponential_(1.0)
    assert torch.equal(torch.get_rng_state(), after)
    c = tts.model.generate_tokens(ids, ref, max_frames=24, style_strength=1.0, min_gen_frames=10 ** 9, seed=5)
    assert torch.equal(a, c)


def test_stream_chunks():
    tts, _ = _tts()
    cfg, sd, inp = e2e_inputs()
    ref = tts.prepare_reference(ref_tokens_tq=inp["ref_tokens_tq"])
    chunks = list(tts.stream(TEXT, ref=ref, max_frames=20, seed=3, min_gen_frames=10 ** 9))
    # the stream ends at the first EOS whatever min_gen_frames says (reference streaming.py:114-115)
    prep = tts.model.prepare_conditioning(tts.encode_text(TEXT), ref, max_frames=20, style_strength=cfg.style_strength)
    toks = [tok for _t, tok, _e in tts.model.ar_stream(prep, max_frames=20, seed=3, min_gen_frames=10 ** 9)]
    n = toks.index(2048) if 2048 in toks else len(toks)
    want = [6] * (n // 6) + ([n % 6] if n % 6 else [])
    assert [c.shape for c in chunks] == [(1, k * 1920) for k in want]
    assert all(torch.isfinite(c).all() for c in chunks)
    again = list(tts.stream(TEXT, ref=ref, max_frames=20, seed=3, min_gen_frames=10 ** 9))
    assert all(torch.equal(a, b) for a, b in zip(chunks, again))


def test_batch_synthesis_equals_single():
    tts, _ = _tts()
    cfg, sd, inp = e2e_inputs()
    ref = tts.prepare_reference(ref_tokens_tq=inp["ref_tokens_tq"])
    texts = [TEXT, " ".join(str(i) for i in range(3, 40, 3)), "5 9"]
    wavs = tts.synthesize_batch(texts, ref=ref, max_frames=16, seeds=[1, 2, 3], min_gen_frames=10 ** 9)
    for t, s, w in zip(texts, [1, 2, 3], wavs):
        single = tts.synthesize(t, ref=ref, max_frames=16, seed=s, min_gen_frames=10 ** 9)
        assert torch.equal(single, w)


def test_batch_synthesis_equals_single_across_noise_blocks():
    """At 101 steps a seeded batch draws its tapes and launches in blocks of 24, 36 and 41 frames; each utterance still
    equals synthesize(text, seed=s), a batch of one, bit for bit."""
    tts, _ = _tts()
    cfg, sd, inp = e2e_inputs()
    ref = tts.prepare_reference(ref_tokens_tq=inp["ref_tokens_tq"])
    texts = [TEXT, " ".join(str(i) for i in range(3, 40, 3)), "5 9", " ".join(str(11 * i + 2) for i in range(30))]
    seeds = [1, 2, 3, 4]
    wavs = tts.synthesize_batch(texts, ref=ref, max_frames=100, seeds=seeds)
    frames = [w.shape[-1] // 1920 for w in wavs]
    assert max(frames) > 24, f"no utterance ran past the first block: {frames}"
    for t, s, w in zip(texts, seeds, wavs):
        single = tts.synthesize(t, ref=ref, max_frames=100, seed=s)
        assert torch.equal(single, w)


def test_prepared_reference_roundtrips_through_torch_save():
    tts, _ = _tts()
    cfg, sd, inp = e2e_inputs()
    ref = tts.prepare_reference(ref_tokens_tq=inp["ref_tokens_tq"])
    assert ref.ref_tokens_btq.shape == (1, 38, 32) and ref.sv_ref.shape == (1, 192) and ref.ref_seq.shape == (1, 38, 384)
    assert len(ref.ref_kv_caches) == 3 and ref.ref_kv_caches[0]["k"].shape == (1, 2, 38, 192)
    buf = io.BytesIO()
    torch.save(ref, buf)
    buf.seek(0)
    back = torch.load(buf, weights_only=False)
    assert torch.equal(back.ref_seq, ref.ref_seq)
    with pytest.raises(RuntimeError):
        tts.prepare_reference()
    with pytest.raises(RuntimeError):
        tts.prepare_reference(ref_tokens_tq=inp["ref_tokens_tq"], ref_audio_path="x.wav")


def test_stream_concat_equals_synthesize():
    """Through the public API only.  (a) One chunk covering the whole utterance: stream() == synthesize() for the same
    seed, sample for sample (same AR ids, the NAR refiner sees the same window, the stream decoder equals the one-shot
    decode).  (b) Chunked: the AR ids are synthesize()'s; the NAR refiner is not causal, so (as in the reference,
    streaming.py:81-104) a chunk's codes come from a window that ends at the chunk; the concatenated audio equals
    decode_full of exactly those window-refined codes -- the stream decoder adds no error of its own."""
    tts, _ = _tts()
    cfg, sd, inp = e2e_inputs()
    ref = tts.prepare_reference(ref_tokens_tq=inp["ref_tokens_tq"])
    F = 25
    tts.codec.engine.set_precision("fp32")
    try:
        full = tts.synthesize(TEXT, ref=ref, max_frames=F, seed=9, min_gen_frames=10 ** 9)
        T = full.shape[-1] // 1920
        one = list(tts.stream(TEXT, ref=ref, max_frames=F, seed=9, min_gen_frames=10 ** 9, chunk_frames=64))
        assert len(one) == 1 and torch.equal(one[0].reshape(-1), full.reshape(-1))
        chunks = list(tts.stream(TEXT, ref=ref, max_frames=F, seed=9, min_gen_frames=10 ** 9, chunk_frames=6))
        audio = torch.cat(chunks, dim=1)
        assert audio.shape[-1] == T * 1920
        # the same windows through the public model API
        ids = tts.encode_text(TEXT)
        prep = tts.model.prepare_conditioning(ids, ref, max_frames=F, style_strength=cfg.style_strength)
        toks = tts.model.generate_tokens(ids, ref, max_frames=F, style_strength=cfg.style_strength, seed=9, min_gen_frames=10 ** 9)
        ar = toks[:, 0].tolist()
        assert len(ar) == T
        ctx, rows, emitted = tts.model.rf_nar(), [], 0
        while emitted < T:
            end = min(emitted + 6, T)
            lo = max(0, emitted - ctx)
            win = tts.model.nar_refine(prep["cond_ar"][:, lo:end], torch.tensor(ar[lo:end], device=tts.device).unsqueeze(0))[0]
            rows.append(win[emitted - lo:])
            emitted = end
        emitted_codes = torch.cat(rows, dim=0)
        assert emitted_codes[:, 0].tolist() == ar
        assert torch.equal(audio.reshape(-1), tts.codec.decode_full(emitted_codes).reshape(-1))
    finally:
        tts.codec.engine.set_precision("bf16_tc")


def test_interleaved_streams_do_not_share_ar_state():
    """ADVICE r1: two suspended stream() generators (a server interleaving requests) must each equal their solo run."""
    tts, _ = _tts()
    cfg, sd, inp = e2e_inputs()
    ref = tts.prepare_reference(ref_tokens_tq=inp["ref_tokens_tq"])
    t2 = " ".join(str(5 * i + 1) for i in range(20))  # same token count -> same session geometry
    solo_a = list(tts.stream(TEXT, ref=ref, max_frames=18, seed=21, min_gen_frames=10 ** 9))
    solo_b = list(tts.stream(t2, ref=ref, max_frames=18, seed=22, min_gen_frames=10 ** 9))
    ga = tts.stream(TEXT, ref=ref, max_frames=18, seed=21, min_gen_frames=10 ** 9)
    gb = tts.stream(t2, ref=ref, max_frames=18, seed=22, min_gen_frames=10 ** 9)
    mixa, mixb = [], []
    for _ in range(max(len(solo_a), len(solo_b))):
        for g, out in ((ga, mixa), (gb, mixb)):
            c = next(g, None)
            if c is not None:
                out.append(c)
    mid = tts.synthesize(TEXT, ref=ref, max_frames=12, seed=5, min_gen_frames=10 ** 9)  # a synthesize in between
    assert mid.shape[-1] == 13 * 1920
    assert len(mixa) == len(solo_a) and all(torch.equal(x, y) for x, y in zip(mixa, solo_a))
    assert len(mixb) == len(solo_b) and all(torch.equal(x, y) for x, y in zip(mixb, solo_b))


def test_no_top_p_takes_the_unsorted_multinomial_branch():
    """top_p=1.0 / None (reference sampling.py:88-93: multinomial over vocabulary order, noise index = token id)."""
    tts, _ = _tts()
    cfg, sd, inp = e2e_inputs()
    ref = tts.prepare_reference(ref_tokens_tq=inp["ref_tokens_tq"])
    ids = tts.encode_text(TEXT)
    F = 12
    prep = tts.model.prepare_conditioning(ids, ref, max_frames=F, style_strength=cfg.style_strength)
    for tp in (1.0, None):
        got = [tok for _t, tok, _e in tts.model.ar_stream(prep, max_frames=F, top_p=tp, seed=31, min_gen_frames=10 ** 9, anti_loop=False)]
        want = O.ar_generate(sd, cfg, prep["cond_ar"].cpu(), prep["txt_seq"].cpu(), torch.ones(1, prep["txt_seq"].size(1), dtype=torch.bool),
                             max_frames=F, sampling=O.ArSampling(top_p=1.0, anti_loop=False, min_gen_frames=10 ** 9),
                             noise_tv=O.noise_tape(31, F + 1, cfg.ar_vocab()))
        assert got == want
