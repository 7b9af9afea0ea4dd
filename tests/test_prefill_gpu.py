"""GPU parity of the CUDA prefill (sopro_prefill_run through the C-ABI) against (a) rows the unmodified reference
wrote (tests/golden/e2e_prefill.npz) and (b) the torch-CPU restatement sopro_b200/prefill.py, which is bit-equal to the
reference on CPU (tests/test_host_cpu.py).  cond_ar / txt_seq are inputs of the id-exact AR kernel: tolerance 2e-5."""
import dataclasses
import os

import numpy as np
import pytest
import torch

from tests.cases import e2e_inputs

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
torch.set_grad_enabled(False)
_S = {}


def _setup():
    from sopro_b200 import prefill as P
    from sopro_b200.prefill_cuda import PrefillEngine

    if "e" not in _S:
        cfg, sd, inp = e2e_inputs()
        tpos = P.sinusoid_table(int(cfg.max_text_len) + 8, int(cfg.d_model), "cpu")
        fpos = P.sinusoid_table(int(cfg.pos_emb_max) + 8, int(cfg.d_model), "cpu")
        _S["e"] = PrefillEngine(cfg, sd, 0, tpos, fpos)
        _S["pos"] = (tpos, fpos)
        _S["ref"] = P.prepare_reference(sd, cfg, inp["ref_tokens_tq"], torch.device("cpu"))
    return _S["e"], _S["ref"], _S["pos"]


def test_prefill_matches_reference_fixture_rows():
    eng, ref, _ = _setup()
    cfg, sd, inp = e2e_inputs()
    g = np.load(os.path.join(GOLD, "e2e_prefill.npz"))
    txt, lens, pool, cond = eng.run([inp["text_ids"]], ref, n_frames=inp["max_frames"] + 1, style_strength=inp["style_strength"])
    tol = dict(rtol=0, atol=2e-5)
    np.testing.assert_allclose(txt[0, :4].cpu().numpy(), g["txt_seq_rows"], **tol)
    np.testing.assert_allclose(pool.cpu().numpy(), g["txt_pool"], **tol)
    np.testing.assert_allclose(cond[0, g["cond_rows_idx"].tolist()].cpu().numpy(), g["cond_rows"], **tol)
    assert abs(float(cond.abs().mean()) - float(g["cond_absmean"])) < 1e-5
    assert cond.shape == (1, inp["max_frames"] + 1, 384) and lens == [52]


def test_batched_prefill_equals_the_cpu_restatement_per_text():
    """Ragged texts (1 .. 300 ids) in one pass: every utterance equals the batch-1 restatement on its own text."""
    from sopro_b200 import prefill as P

    eng, ref, (tpos, fpos) = _setup()
    cfg, sd, inp = e2e_inputs()
    g = torch.Generator().manual_seed(8)
    texts = [torch.randint(0, 1000, (n,), generator=g) for n in (52, 1, 7, 300, 52, 33)]
    F = 60
    txt, lens, pool, cond = eng.run(texts, ref, n_frames=F + 1, style_strength=1.2)
    assert lens == [52, 1, 7, 300, 52, 33]
    worst = 0.0
    for i, ids in enumerate(texts):
        want = P.prepare_conditioning(sd, cfg, ids, ref, max_frames=F, device="cpu", style_strength=1.2, text_pos=tpos, frame_pos=fpos)
        for got, w in ((txt[i, : lens[i]], want["txt_seq"][0]), (pool[i], want["txt_pool"][0]), (cond[i], want["cond_ar"][0])):
            err = float((got.cpu() - w).abs().max())
            worst = max(worst, err)
            assert err <= 2e-5, (i, err)
    print(f"batched prefill vs CPU restatement: max abs err {worst:.2e}")
    # batch invariance.  Stages with more than 16 rows run the 128x128 tile kernel, whose per-output summation order does
    # not depend on the row count: a 52-token text alone (M = 52) equals its rows in the batch (M = 6 x 300) bit for bit.
    t0, _, p0, c0 = eng.run([texts[0]], ref, n_frames=F + 1, style_strength=1.2)
    assert torch.equal(c0[0], cond[0]) and torch.equal(t0[0, :52], txt[0, :52]) and torch.equal(p0[0], pool[0])
    # A 7-token text alone (M <= 16) takes the skinny kernel (lanes split K: another summation order): equal to rounding
    t1, _, p1, c1 = eng.run([texts[2]], ref, n_frames=F + 1, style_strength=1.2)
    assert float((c1[0] - cond[2]).abs().max()) <= 2e-5 and float((t1[0, :7] - txt[2, :7]).abs().max()) <= 2e-5


def test_public_prepare_conditioning_feeds_the_ar_kernel():
    """Through SoproModel: prep dict shapes/keys of reference model.py:210-216."""
    from oracle import mimi_oracle as M
    from sopro_b200 import SoproTTS
    from sopro_b200.tokenizer import IdsTokenizer

    cfg, sd, inp = e2e_inputs()
    if "tts" not in _S:
        _S["tts"] = SoproTTS.from_state_dict(cfg, sd, IdsTokenizer(1000), M.synth_mimi_state_dict(), device="cuda:0")
    tts = _S["tts"]
    ref = tts.prepare_reference(ref_tokens_tq=inp["ref_tokens_tq"])
    prep = tts.model.prepare_conditioning(inp["text_ids"], ref, max_frames=40, style_strength=1.0)
    assert set(prep) == {"txt_seq", "text_mask", "txt_pool", "sv_ref", "cond_ar"}
    assert prep["txt_seq"].shape == (1, 52, 384) and prep["cond_ar"].shape == (1, 41, 384) and prep["text_mask"].all()
    txt, lens, _pool, cond = tts.model.prefill.run([inp["text_ids"], inp["text_ids"][:9]], ref, n_frames=41, style_strength=1.0)
    assert torch.equal(cond[0:1], prep["cond_ar"]) and torch.equal(txt[0:1], prep["txt_seq"]) and lens == [52, 9]


# ---------------------------------------------------------------------------------------------------------------
# reference preparation (sopro_refprep_*: Token2SV, reference encoder, cached K / V; reference model.py:152-170)
# ---------------------------------------------------------------------------------------------------------------
def _refprep():
    from sopro_b200.prefill_cuda import RefPrepEngine

    if "rp" not in _S:
        cfg, sd, _ = e2e_inputs()
        _S["rp"] = RefPrepEngine(cfg, sd, 0)
    return _S["rp"]


def test_refprep_matches_reference_fixture_rows():
    """sv_ref, ref_seq rows and cached-K rows the unmodified reference wrote (tests/golden/e2e_prefill.npz)."""
    rp = _refprep()
    _, _, inp = e2e_inputs()
    g = np.load(os.path.join(GOLD, "e2e_prefill.npz"))
    sv, seq, caches = rp.run(inp["ref_tokens_tq"])
    assert sv.shape == (1, 192) and seq.shape == (1, 38, 384) and len(caches) == 3 and caches[0]["k"].shape == (1, 2, 38, 192)
    np.testing.assert_allclose(sv.cpu().numpy(), g["sv_ref"], rtol=0, atol=2e-6)
    np.testing.assert_allclose(seq[0, :4].cpu().numpy(), g["ref_seq_rows"], rtol=0, atol=2e-5)
    assert abs(float(seq.abs().mean()) - float(g["ref_seq_absmean"])) < 1e-5
    np.testing.assert_allclose(caches[2]["k"][0, :, :2].cpu().numpy(), g["k2_rows"], rtol=0, atol=2e-5)
    assert abs(float(sv.norm()) - 1.0) < 1e-5 and caches[0]["key_padding_mask"] is None


@pytest.mark.parametrize("Tr,seed", [(1, 3), (5, 4), (38, 5), (150, 6), (769, 7), (1500, 8), (4096, 9)])
def test_refprep_equals_the_cpu_restatement(Tr, seed):
    """Every output tensor against sopro_b200/prefill.py on the CPU, short and long voices (up to the 4096-frame limit)."""
    from sopro_b200 import prefill as P

    rp = _refprep()
    cfg, sd, _ = e2e_inputs()
    tok = torch.randint(0, 2048, (Tr, 32), generator=torch.Generator().manual_seed(seed))
    want = P.prepare_reference(sd, cfg, tok, torch.device("cpu"))
    sv, seq, caches = rp.run(tok)
    assert float((sv.cpu() - want.sv_ref).abs().max()) <= 2e-6
    assert float((seq.cpu() - want.ref_seq).abs().max()) <= 2e-5 * max(1.0, float(want.ref_seq.abs().max()))
    for got, ref in zip(caches, want.ref_kv_caches):
        for n in ("k", "v"):
            assert got[n].shape == ref[n].shape
            assert float((got[n].cpu() - ref[n]).abs().max()) <= 2e-5 * max(1.0, float(ref[n].abs().max()))


@pytest.mark.parametrize("Tr", [769, 1500, 4096])
def test_prefill_with_a_long_reference_equals_the_cpu_restatement(Tr):
    """Above 768 reference frames the cross-attention kernel needs more than 48 KB of shared memory per CTA (its opt-in
    branch); up to the 4096-frame limit it must still equal the CPU restatement.  4097 frames are refused."""
    from sopro_b200 import _lib
    from sopro_b200 import prefill as P

    eng, _, (tpos, fpos) = _setup()
    rp = _refprep()
    cfg, sd, inp = e2e_inputs()
    tok = torch.randint(0, 2048, (Tr, 32), generator=torch.Generator().manual_seed(Tr))
    ref = P.prepare_reference(sd, cfg, tok, torch.device("cpu"))
    texts = [inp["text_ids"], inp["text_ids"][:9]]
    F = 40
    txt, lens, pool, cond = eng.run(texts, ref, n_frames=F + 1, style_strength=1.0)
    for i, ids in enumerate(texts):
        want = P.prepare_conditioning(sd, cfg, ids, ref, max_frames=F, device="cpu", style_strength=1.0, text_pos=tpos, frame_pos=fpos)
        err = float((cond[i].cpu() - want["cond_ar"][0]).abs().max())
        assert err <= 2e-5, (Tr, i, err)
    long_tok = torch.zeros((4097, 32), dtype=torch.long)
    with pytest.raises(_lib.SoproError):
        rp.run(long_tok)
    kv = [{"k": c["k"].new_zeros((1, c["k"].shape[1], 4097, c["k"].shape[3])), "v": c["v"].new_zeros((1, c["v"].shape[1], 4097, c["v"].shape[3])),
           "key_padding_mask": None} for c in ref.ref_kv_caches]
    with pytest.raises(_lib.SoproError):
        eng.run(texts, dataclasses.replace(ref, ref_kv_caches=kv), n_frames=F + 1, style_strength=1.0)


def test_refprep_rejects_codes_outside_the_codebook():
    rp = _refprep()
    tok = torch.randint(0, 2048, (7, 32), generator=torch.Generator().manual_seed(1))
    tok[3, 5] = 2048
    with pytest.raises(IndexError):
        rp.run(tok)
    rp.run(tok.clamp(max=2047))  # the flag was cleared
    with pytest.raises(ValueError):
        rp.run(tok[:, :31])


def test_public_prepare_reference_runs_on_the_engine_and_feeds_the_prefill():
    from sopro_b200 import SoproTTS
    from sopro_b200 import prefill as P
    from sopro_b200.tokenizer import IdsTokenizer
    from sopro_b200.weights import synth_mimi_state_dict

    cfg, sd, inp = e2e_inputs()
    if "tts" not in _S:
        _S["tts"] = SoproTTS.from_state_dict(cfg, sd, IdsTokenizer(1000), synth_mimi_state_dict(), device="cuda:0")
    tts = _S["tts"]
    ref = tts.prepare_reference(ref_tokens_tq=inp["ref_tokens_tq"])
    want = P.prepare_reference(sd, cfg, inp["ref_tokens_tq"], torch.device("cpu"))
    assert ref.ref_tokens_btq.shape == (1, 38, 32) and ref.ref_tokens_btq.dtype == torch.long
    assert float((ref.sv_ref.cpu() - want.sv_ref).abs().max()) <= 2e-6
    sv = tts.encode_speaker(ref_tokens_tq=inp["ref_tokens_tq"])
    assert sv.shape == (192,) and float((sv.cpu() - want.sv_ref[0]).abs().max()) <= 2e-6
    prep = tts.model.prepare_conditioning(inp["text_ids"], ref, max_frames=inp["max_frames"], style_strength=inp["style_strength"])
    g = np.load(os.path.join(GOLD, "e2e_prefill.npz"))
    np.testing.assert_allclose(prep["cond_ar"][0, g["cond_rows_idx"].tolist()].cpu().numpy(), g["cond_rows"], rtol=0, atol=2e-5)
