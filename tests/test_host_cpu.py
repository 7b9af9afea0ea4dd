"""CPU: host logic that needs no GPU - prefill/NAR against the reference fixtures, the API surface, the C-ABI
library's exported symbols, the synthetic checkpoint generator, audio I/O."""
import ctypes
import inspect
import os
import re

import numpy as np
import pytest
import torch

from tests.cases import e2e_inputs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
torch.set_grad_enabled(False)


def test_prefill_and_nar_match_reference_fixtures():
    from sopro_b200 import prefill as P

    cfg, sd, inp = e2e_inputs()
    g = np.load(os.path.join(GOLD, "e2e_prefill.npz"))
    dev = torch.device("cpu")
    pr = P.prepare_reference(sd, cfg, inp["ref_tokens_tq"], dev)
    tpos = P.sinusoid_table(int(cfg.max_text_len) + 8, int(cfg.d_model), dev)
    fpos = P.sinusoid_table(int(cfg.pos_emb_max) + 8, int(cfg.d_model), dev)
    prep = P.prepare_conditioning(sd, cfg, inp["text_ids"], pr, max_frames=inp["max_frames"], device=dev,
                                  style_strength=inp["style_strength"], text_pos=tpos, frame_pos=fpos)
    tol = dict(rtol=0, atol=2e-5)
    np.testing.assert_allclose(pr.sv_ref.numpy(), g["sv_ref"], **tol)
    np.testing.assert_allclose(pr.ref_seq[0, :4].numpy(), g["ref_seq_rows"], **tol)
    np.testing.assert_allclose(pr.ref_kv_caches[2]["k"][0, :, :2].numpy(), g["k2_rows"], **tol)
    np.testing.assert_allclose(prep["txt_seq"][0, :4].numpy(), g["txt_seq_rows"], **tol)
    np.testing.assert_allclose(prep["txt_pool"].numpy(), g["txt_pool"], **tol)
    np.testing.assert_allclose(prep["cond_ar"][0, g["cond_rows_idx"].tolist()].numpy(), g["cond_rows"], **tol)
    assert abs(float(prep["cond_ar"].abs().mean()) - float(g["cond_absmean"])) < 1e-5
    nar = P.nar_refine(sd, cfg, prep["cond_ar"][:, : inp["nar_T"]], inp["rvq1"].unsqueeze(0))[0]
    assert float((nar.numpy() == g["nar_tokens"].astype(np.int64)).mean()) >= 0.999
    assert nar[:, 0].tolist() == inp["rvq1"].tolist()


def test_api_surface_mirrors_the_reference():
    """Signatures of SURVEY.md §8b (reference model.py:419-428, 516-523, 531-546, 577-580; streaming.py:134-143)."""
    from sopro_b200 import SoproTTS
    from sopro_b200.streaming import stream

    def params(f):
        return list(inspect.signature(f).parameters)

    assert params(SoproTTS.__init__) == ["self", "model", "cfg", "tokenizer", "codec", "device"]
    assert params(SoproTTS.from_pretrained)[:5] == ["repo_id", "revision", "cache_dir", "token", "device"]
    assert params(SoproTTS.prepare_reference) == ["self", "ref_audio_path", "ref_tokens_tq", "ref_seconds"]
    ref_syn = ["self", "text", "ref", "ref_audio_path", "ref_tokens_tq", "max_frames", "top_p", "temperature", "anti_loop",
               "style_strength", "ref_seconds", "min_gen_frames"]
    assert params(SoproTTS.synthesize)[: len(ref_syn)] == ref_syn
    d = inspect.signature(SoproTTS.synthesize).parameters
    assert (d["max_frames"].default, d["top_p"].default, d["temperature"].default, d["anti_loop"].default) == (400, 0.9, 1.05, True)
    assert inspect.signature(stream).parameters["chunk_frames"].default == 6
    for name in ("encode_text", "encode_reference", "encode_speaker", "save_wav", "stream"):
        assert callable(getattr(SoproTTS, name))
    assert "nar_context_frames" in params(stream)


def test_shared_library_exports_every_declared_symbol():
    from sopro_b200 import _lib

    hdr = open(os.path.join(ROOT, "include", "sopro_b200.h")).read()
    declared = set(re.findall(r"\b(sopro_[a-z0-9_]+)\s*\(", hdr))
    declared -= {"sopro_status"}
    assert declared == set(_lib.SYMBOLS), declared ^ set(_lib.SYMBOLS)
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in declared:
        assert hasattr(lib, name), name
    assert _lib.load().sopro_version().startswith(b"sopro_b200")


def test_no_cpu_fallback():
    if torch.cuda.is_available():
        pytest.skip("needs a GPU-less host")
    from sopro_b200 import _lib
    from sopro_b200.config import SoproTTSConfig
    from sopro_b200.engine import ArEngine
    from sopro_b200.model import SoproModel

    with pytest.raises(RuntimeError):
        SoproModel(SoproTTSConfig(), {}, "cpu")
    from tests.cases import AR_CASES, ar_case_inputs

    cfg, sd, _ = ar_case_inputs(AR_CASES["small_fp32"])
    with pytest.raises(_lib.SoproError):
        ArEngine(cfg, sd, 0)  # no device: the C-ABI refuses, nothing silently runs on the host


def test_synthetic_checkpoint_is_deterministic_and_complete():
    from sopro_b200.config import SoproTTSConfig
    from sopro_b200.weights import ar_step_param_names, hash_uniform, param_specs, synth_state_dict

    u = hash_uniform(5, 42)
    np.testing.assert_array_equal(u, hash_uniform(5, 42))
    assert u.dtype == np.float32 and np.all(np.abs(u) <= 1)
    cfg = SoproTTSConfig()
    specs = param_specs(cfg, 128257)
    assert sum(int(np.prod(s)) if s else 1 for s, _, _ in specs.values()) == 132260272  # + 32 for the ref_cb_weights buffer
    sd = synth_state_dict(cfg, 64, 0, only_prefix=("ar.",))
    n_step = sum(sd[k].numel() for k in ar_step_param_names(cfg))
    assert n_step == 10575492  # SURVEY.md §8d W_step


def test_wav_roundtrip(tmp_path):
    from sopro_b200.audio import load_audio_file, save_audio, trim_silence_energy

    sr = 24000
    t = torch.arange(sr) / sr
    wav = torch.cat([torch.zeros(sr // 2), 0.5 * torch.sin(2 * np.pi * 440 * t), torch.zeros(sr // 2)])
    p = str(tmp_path / "a.wav")
    save_audio(p, wav.view(1, 1, -1), sr)
    back, sr2 = load_audio_file(p)
    assert sr2 == sr and back.shape == (1, wav.numel())
    assert float((back[0] - wav).abs().max()) < 1e-3
    trimmed = trim_silence_energy(back, sr)
    assert sr * 0.9 < trimmed.shape[-1] < wav.numel()


def test_noise_tape_blocks_equal_one_tape_and_settle_rewinds():
    """ar_stream draws the sampler's Exp(1) rows launch by launch: the blocks must concatenate to the one-shot tape
    (== what `steps` multinomial calls consume) and settle() must leave the global generator after exactly the
    consumed rows."""
    from sopro_b200.sampling import NoiseTape

    V = 2049
    torch.manual_seed(3)
    full = torch.empty(20, V).exponential_(1.0)
    after_full = torch.get_rng_state()
    torch.manual_seed(3)
    n = NoiseTape(20, V, V)
    got = np.zeros((20, V), dtype=np.float32)
    for up in (6, 12, 18, 24):
        n.draw(up, got)
    assert torch.equal(torch.from_numpy(got), full) and torch.equal(torch.get_rng_state(), after_full)
    n.settle(8)
    state = torch.get_rng_state()
    torch.manual_seed(3)
    torch.empty(8, V).exponential_(1.0)
    assert torch.equal(state, torch.get_rng_state())
    # a private seed never touches the global generator
    before = torch.get_rng_state()
    p = NoiseTape(5, V, V, seed=11)
    tape = np.zeros((5, V), dtype=np.float32)
    p.draw(5, tape)
    p.close()
    assert torch.equal(torch.from_numpy(tape), torch.empty(5, V).exponential_(1.0, generator=torch.Generator().manual_seed(11)))
    assert torch.equal(before, torch.get_rng_state())


def test_public_header_is_plain_c():
    """The drop-in boundary is a C ABI: the header must compile as C99 on its own (no C++ or torch types)."""
    import shutil
    import subprocess

    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no gcc")
    hdr = os.path.join(ROOT, "include", "sopro_b200.h")
    r = subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-fsyntax-only", "-x", "c", hdr], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_missing_checkpoint_tensors_get_reference_defaults_or_one_clear_error():
    """The reference loads strict=False: omitted buffers keep their init values (model.py:113-117, 70-72; nn/nar.py:79)."""
    from sopro_b200.config import SoproTTSConfig
    from sopro_b200.model import _complete_state_dict
    from sopro_b200.weights import synth_state_dict

    cfg = SoproTTSConfig()
    sd = synth_state_dict(cfg, text_vocab=64)
    cut = {k: v for k, v in sd.items() if k not in ("ref_cb_weights", "nar_prev_cb_weights") and not k.startswith("nar.head_id_emb.")}
    full = _complete_state_dict(cfg, cut)
    assert torch.equal(full["ref_cb_weights"], torch.linspace(1.0, 0.1, int(cfg.num_codebooks)))
    assert float(full["nar_prev_cb_weights"].abs().sum()) == 0.0
    assert all(float(full[k].abs().sum()) == 0.0 for k in sd if k.startswith("nar.head_id_emb."))
    del cut["ar.head.weight"], cut["cond_norm.weight"]
    with pytest.raises(KeyError) as ei:
        _complete_state_dict(cfg, cut)
    assert "ar.head.weight" in str(ei.value) and "cond_norm.weight" in str(ei.value)


def test_native_noise_tape_draws_are_bit_equal_to_torch_and_skip_the_unread_draws():
    """csrc/noise_host.cu (host-side mt19937 + ATen's uniform -> -log1p(-u) transform) against this torch build's CPU
    exponential_: same bits for private generators, also when only the first `keep` columns of each row are materialised
    and across blocks of rows; the Python NoiseTape wrapper uses it only after this check (sampling._native_noise_ok)."""
    import ctypes as C

    from sopro_b200 import _lib
    from sopro_b200.sampling import NoiseTape, _native_noise_ok

    lib = _lib.load()
    for seed in (0, 1, 1234, 2 ** 31 + 7, 2 ** 40 + 3):
        h = C.c_void_p()
        _lib.check(lib.sopro_noise_create(C.c_uint64(seed), C.byref(h)))
        g = torch.Generator().manual_seed(seed)
        for n, V, keep in ((3, 2049, 50), (1, 33, 33), (5, 2049, 2049), (2, 257, 50), (700, 5, 2)):
            want = torch.empty(n, V).exponential_(1.0, generator=g)[:, :keep].contiguous()
            got = torch.empty(n, keep)
            _lib.check(lib.sopro_noise_rows(h, n, V, keep, got.data_ptr()))
            assert torch.equal(got, want), (seed, n, V, keep)
        lib.sopro_noise_destroy(h)
    assert _native_noise_ok()
    a = NoiseTape(40, 2049, 50, seed=77)
    assert a._native is not None  # a private seed >= 0 draws through the library
    got = np.zeros((40, 50), dtype=np.float32)
    a.draw(13, got)
    a.draw(40, got)
    a.close()
    ref = torch.empty(40, 2049).exponential_(1.0, generator=torch.Generator().manual_seed(77))[:, :50]
    assert torch.equal(torch.from_numpy(got), ref)


def test_ctypes_mirrors_match_the_header_layout(tmp_path):
    """sopro_b200/_lib.py restates every struct of include/sopro_b200.h in ctypes: sizes and the offset of every field
    must equal what the C compiler lays out (a drifted field silently shifts every pointer behind it)."""
    import ctypes as C
    import shutil
    import subprocess

    from sopro_b200 import _lib

    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no gcc")
    pairs = {
        "sopro_ar_config_t": _lib.ArConfig, "sopro_ar_layer_weights_t": _lib.ArLayerWeights, "sopro_ar_weights_t": _lib.ArWeights,
        "sopro_ar_sampling_t": _lib.ArSampling, "sopro_mimi_config_t": _lib.MimiConfigC,
        "sopro_mimi_layer_weights_t": _lib.MimiLayerWeights, "sopro_mimi_stage_weights_t": _lib.MimiStageWeights,
        "sopro_mimi_weights_t": _lib.MimiWeights, "sopro_mimi_enc_stage_weights_t": _lib.MimiEncStageWeights,
        "sopro_mimi_encoder_weights_t": _lib.MimiEncoderWeights, "sopro_ssm_block_weights_t": _lib.SsmBlockWeights,
        "sopro_nar_config_t": _lib.NarConfig, "sopro_nar_weights_t": _lib.NarWeights, "sopro_prefill_config_t": _lib.PrefillConfig,
        "sopro_prefill_ref_layer_t": _lib.PrefillRefLayer, "sopro_prefill_weights_t": _lib.PrefillWeights,
        "sopro_refprep_config_t": _lib.RefPrepConfig, "sopro_refprep_kv_layer_t": _lib.RefPrepKvLayer,
        "sopro_refprep_weights_t": _lib.RefPrepWeights,
    }
    hdr = open(os.path.join(ROOT, "include", "sopro_b200.h")).read()
    import re

    declared = set(re.findall(r"^\} (sopro_[a-z0-9_]+_t);", hdr, flags=re.M))
    assert declared == set(pairs), (declared ^ set(pairs))
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "sopro_b200.h"', "int main(void) {"]
    for cname, cls in pairs.items():
        lines.append(f'  printf("{cname} %zu\\n", sizeof({cname}));')
        for fname, _ in cls._fields_:
            lines.append(f'  printf("{cname}.{fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ["  return 0;", "}"]
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines))
    r = subprocess.run([gcc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr  # also fails when a ctypes field name does not exist in the C struct
    got = dict(l.split() for l in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    for cname, cls in pairs.items():
        assert int(got[cname]) == C.sizeof(cls), (cname, got[cname], C.sizeof(cls))
        for fname, _ in cls._fields_:
            assert int(got[f"{cname}.{fname}"]) == getattr(cls, fname).offset, (cname, fname)


def test_encode_file_host_preparation_matches_the_reference_fixture():
    """tests/golden/audio_prep.json: what the reference's trim_silence_energy + center_crop_audio keep of seeded signals
    (reference audio.py:30-87, 148-155; written by tests/golden/make_audio_golden.py)."""
    import json

    from sopro_b200.audio import center_crop_audio, trim_silence_energy
    from tests.golden.make_audio_golden import CASES, signal

    with open(os.path.join(ROOT, "tests", "golden", "audio_prep.json")) as f:
        g = json.load(f)
    for i, (name, sr, n, lo, hi, floor) in enumerate(CASES):
        w = signal(sr, n, lo, hi, floor, i)
        t = trim_silence_energy(w, sr)
        c = center_crop_audio(t, 12 * 1920)
        want = g[name]
        assert int(t.shape[-1]) == want["trim_len"] and int(c.shape[-1]) == want["crop_len"], name
        assert float(t[0, 0]) == want["trim_first"] and float(t[0, -1]) == want["trim_last"], name
        assert abs(float(t.double().sum()) - want["trim_sum"]) < 1e-9 and abs(float(c.double().sum()) - want["crop_sum"]) < 1e-9, name
        assert float(c[0, 0]) == want["crop_first"], name
    assert g["margins_24k"]["trim_len"] < 72000 and g["short_burst_24k"]["trim_len"] == 48000
