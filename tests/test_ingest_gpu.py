"""GPU: voice ingestion (sopro_b200/csrc/ingest.cu, sopro_mimi_encode_batch, SoproTTS.prepare_references).
  - the trim extents against the float64 oracle, on the reference's fixture signals and on seeded clips at mixed rates;
  - every row of the batched encoder equal to the single-clip encoder bit for bit, codes and latent;
  - prepare_references equal to its parts (oracle extents -> Resampler -> crop -> encode_wav -> prepare_reference);
  - against today's host path (prepare_reference(ref_audio_path=...)) within the stated differences;
  - synthesis from a reference prepared here."""
import math

import numpy as np
import pytest
import torch

from oracle import ingest_oracle as O
from oracle import mimi_oracle as M
from tests.golden.make_audio_golden import CASES, signal
from tests.golden.make_mimi_encode_golden import waveform
from tests.test_ingest_cpu import near_tie, seeded_clip
from tests.test_mimi_encode_gpu import _compare_codes

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
_S = {}
DEV = torch.device("cuda", 0)


def _mimi_sd():
    if "msd" not in _S:
        sd = dict(M.synth_mimi_state_dict())
        sd.update(M.synth_mimi_encoder_state_dict())
        _S["msd"] = sd
    return _S["msd"]


def _tts():
    if "tts" not in _S:
        from sopro_b200 import SoproTTS
        from sopro_b200.tokenizer import IdsTokenizer
        from tests.cases import e2e_inputs

        cfg, sd, _ = e2e_inputs()
        _S["tts"] = SoproTTS.from_state_dict(cfg, sd, IdsTokenizer(1000), _mimi_sd(), device="cuda:0", mimi_precision="fp32")
    return _S["tts"]


def _enc():
    return _tts().codec.encoder


# ---- trim

def _check_extents(xs, rates):
    from sopro_b200 import ingest

    rows = [torch.from_numpy(x).to(DEV) for x in xs]
    got = ingest.trim_extents(rows, rates).cpu().tolist()
    ties = 0
    for x, sr, g in zip(xs, rates, got):
        want = list(O.trim_extent(x, sr))
        if g != want:
            assert near_tie(x, sr), (sr, x.size, g, want)
            ties += 1
    return ties


def test_trim_extents_on_the_fixture_signals():
    xs, rates = [], []
    for i, (name, sr, n, lo, hi, floor) in enumerate(CASES):
        xs.append(signal(sr, n, lo, hi, floor, i)[0].numpy())
        rates.append(sr)
    assert _check_extents(xs, rates) == 0


def test_trim_extents_on_seeded_clips_at_mixed_rates():
    rates = [8000, 11025, 16000, 22050, 24000, 32000, 44100, 48000, 96000, 12345]
    xs, srs = [], []
    for k in range(70):  # more than one launch of 64 rows
        sr = rates[k % len(rates)]
        xs.append(seeded_clip(sr, 77 + k))
        srs.append(sr)
    ties = _check_extents(xs, srs)
    trimmed = sum(O.trim_extent(x, sr) != (0, x.size) for x, sr in zip(xs, srs))
    print(f"{len(xs)} clips: {trimmed} trimmed, {ties} near-tie differences")
    assert trimmed >= 20


# ---- batched encoder

def _batch(lens, seed):
    g = torch.Generator().manual_seed(seed)
    L = max(lens)
    x = torch.randn((len(lens), L), generator=g) * 30.0  # loud padding: a row that read it would show
    for b, n in enumerate(lens):
        x[b, :n] = waveform(n).reshape(-1)
    return x.to(DEV)


def _check_rows(lens, seed, oracle=False):
    eng = _enc()
    x = _batch(lens, seed)
    codes, lats = eng.encode_batch(x, lens, return_latent=True)
    for b, n in enumerate(lens):
        want, lat = eng.encode(x[b, :n].clone(), return_latent=True)
        assert codes[b].shape == want.shape == (32, eng.frames(n))
        assert torch.equal(codes[b], want), (b, n)
        assert torch.equal(lats[b], lat), (b, n)
        if oracle:
            lat_want = M.mimi_encode_latent(_mimi_sd(), x[b, :n].cpu()[None, None])[0]
            _compare_codes(_mimi_sd(), lat_want, codes[b].cpu(), M.rvq_encode(_mimi_sd(), lat_want[None])[0])


def test_batched_encoder_batch_of_one():
    _check_rows([13951], 1)


def test_batched_encoder_ragged_at_every_stride():
    _check_rows([1, 7, 999, 1921, 5760, 13951, 289234], 2, oracle=True)


@pytest.mark.parametrize("B", [16, 64])
def test_batched_encoder_random_lengths(B):
    g = np.random.default_rng(B)
    _check_rows([int(v) for v in g.integers(1, 96000, B)], B)


def test_batched_encoder_splits_an_oversized_batch():
    """Ten 70 s rows: the padded batch exceeds one call's bound, so the rows go in several calls, longest first."""
    lens = [24000 * 70 - 37 * k for k in range(10)]
    eng = _enc()
    x = _batch(lens, 5)
    codes = eng.encode_batch(x, lens)
    for b in (0, 9):
        assert torch.equal(codes[b], eng.encode(x[b, : lens[b]].clone()))


def test_batched_encoder_refusals():
    from sopro_b200 import _lib
    import ctypes as C

    eng = _enc()
    x = torch.zeros((2, 4000), device=DEV)
    c = torch.empty((2, 32, 8), dtype=torch.int32, device=DEV)
    st = _lib.stream_ptr(DEV)
    f = eng.lib.sopro_mimi_encode_batch
    assert f(eng._h, x.data_ptr(), 0, 4000, (C.c_int64 * 1)(10), c.data_ptr(), None, st) == -1
    assert f(eng._h, x.data_ptr(), 2, 4000, (C.c_int64 * 2)(10, 0), c.data_ptr(), None, st) == -1
    assert f(eng._h, x.data_ptr(), 2, 4000, (C.c_int64 * 2)(10, 24000 * 600 + 1), c.data_ptr(), None, st) == -1
    assert f(eng._h, x.data_ptr(), 2, 3999, (C.c_int64 * 2)(10, 4000), c.data_ptr(), None, st) == -1
    assert f(eng._h, None, 2, 4000, (C.c_int64 * 2)(10, 4000), c.data_ptr(), None, st) == -1
    assert f(eng._h, x.data_ptr(), 2, 4000, (C.c_int64 * 2)(10, 4000), None, None, st) == -1
    assert f(eng._h, x.data_ptr(), 2, 24000 * 600, (C.c_int64 * 2)(24000 * 600, 10), c.data_ptr(), None, st) == -1
    with pytest.raises(ValueError):
        eng.encode_batch(x, [10, 4001])


# ---- end to end

def _clips(tmp_path):
    """Mixed tensor clips (16 / 22.05 / 44.1 / 48 kHz, mono and stereo, CPU and GPU) and one PCM16 WAV file."""
    from sopro_b200.audio import save_audio

    out = []
    for k, (sr, ch, secs) in enumerate([(16000, 1, 3.1), (22050, 2, 2.4), (44100, 1, 5.0), (48000, 2, 1.7),
                                        (44100, 2, 14.2), (24000, 1, 2.2)]):
        n = int(sr * secs)
        g =np.random.default_rng(900 + k)
        t = np.arange(n) / sr
        env = ((t > 0.3) & (t < secs - 0.4)).astype(np.float64)
        x = np.stack([(0.3 + 0.1 * c) * np.sin(2 * np.pi * (150 + 40 * c) * t) * env + 1e-3 * g.standard_normal(n)
                      for c in range(ch)]).astype(np.float32)
        w = torch.from_numpy(x if ch > 1 else x[0])
        out.append((w.to(DEV) if k % 2 else w, sr))
    sr = 16000
    n = int(sr * 2.6)
    t = np.arange(n) / sr
    x = (0.5 * np.sin(2 * np.pi * 310 * t) * ((t > 0.5) & (t < 2.2))).astype(np.float32)
    path = str(tmp_path / "voice.wav")
    save_audio(path, torch.from_numpy(x), sr)
    out.append((path, None))
    return out


def _expected_24k(w, sr, win):
    """oracle extents -> Resampler alone -> crop, from the same mono row the pipeline averages"""
    from sopro_b200 import ingest
    from sopro_b200.resample import Resampler

    row = ingest.mono_rows([w], DEV)[0]
    s, e = O.trim_extent(row.cpu().numpy(), sr)
    y = row[s:e]
    if sr != 24000:
        y = Resampler(sr, 24000, DEV)(y.clone())
    o, m = O.crop_plan(int(y.numel()), win)
    return y[o:o + m], (s, e)


def _equal_refs(a, b):
    assert torch.equal(a.ref_tokens_btq, b.ref_tokens_btq)
    assert torch.equal(a.sv_ref, b.sv_ref) and torch.equal(a.ref_seq, b.ref_seq)
    assert len(a.ref_kv_caches) == len(b.ref_kv_caches)
    for ca, cb in zip(a.ref_kv_caches, b.ref_kv_caches):
        assert ca.keys() == cb.keys()
        for k in ca:
            assert (ca[k] is None and cb[k] is None) or torch.equal(ca[k], cb[k]), k


@pytest.mark.parametrize("ref_seconds", [None, 3.0, 0])
def test_prepare_references_equals_its_parts(tmp_path, ref_seconds):
    from sopro_b200 import ingest
    from sopro_b200.audio import load_audio_file

    tts = _tts()
    items = _clips(tmp_path)
    clips = [c for c, _ in items]
    rates = [sr for _, sr in items]
    refs = tts.prepare_references(clips, sample_rates=rates, ref_seconds=ref_seconds)
    assert len(refs) == len(clips)
    win = ingest.crop_samples(ingest.DEFAULT_REF_SECONDS if ref_seconds is None else ref_seconds)
    wavs, srs = ingest.load_clips(clips, rates)
    wav_bl, lens = tts.codec.prepare_wavs(wavs, srs, 12.0 if ref_seconds is None else ref_seconds)
    assert srs[-1] == 16000 and torch.equal(wavs[-1], load_audio_file(clips[-1])[0])
    for b, (w, sr) in enumerate(zip(wavs, srs)):
        want, _ = _expected_24k(w, sr, win)
        assert lens[b] == want.numel() and torch.equal(wav_bl[b, : lens[b]], want), b
        assert not bool(wav_bl[b, lens[b]:].any())
        codes = tts.codec.encode_wav(want)
        assert torch.equal(refs[b].ref_tokens_btq[0], codes), b
        _equal_refs(refs[b], tts.model.prepare_reference(codes, device=tts.device))
    # one clip: the single-voice in-memory case
    one = tts.prepare_references([clips[2]], sample_rates=[rates[2]], ref_seconds=ref_seconds)[0]
    _equal_refs(one, refs[2])


def _oracle64(x, sr):
    """torchaudio's resample sr -> 24 kHz in float64, and §5d's per-element bound (S + 2) 2^-24 sum|k64 x|"""
    F = pytest.importorskip("torchaudio.functional.functional")
    from sopro_b200.resample import filter_taps

    g = math.gcd(24000, sr)
    k64, width = F._get_sinc_resample_kernel(sr, 24000, g, device=x.device, dtype=torch.float64)
    x64 = x.double().reshape(1, -1)
    y64 = F._apply_sinc_resample_kernel(x64, sr, 24000, g, k64, width)[0]
    mag = F._apply_sinc_resample_kernel(x64.abs(), sr, 24000, g, k64.abs(), width)[0]
    _o, n, _w, _f, span, _t = filter_taps(sr, 24000)
    S = torch.as_tensor(span, dtype=torch.float64)[torch.arange(y64.numel()) % n]
    return y64, (S + 2) * 2.0 ** -24 * mag


def test_against_the_host_path_of_encode_file(tmp_path):
    """prepare_reference(ref_audio_path=...) trims, resamples (torchaudio, fp32 on the CPU) and crops on the host: the
    extents are equal, the 24 kHz waveforms within §5d's distance, and a differing id only at an oracle near tie."""
    AF = pytest.importorskip("torchaudio.functional")
    from sopro_b200 import ingest
    from sopro_b200.audio import load_audio_file, save_audio, trim_silence_energy

    tts = _tts()
    sd = _mimi_sd()
    for i, (name, sr, n, lo, hi, floor) in enumerate(CASES):
        path = str(tmp_path / f"{name}.wav")
        save_audio(path, signal(sr, n, lo, hi, floor, i)[0], sr)
        w, fsr = load_audio_file(path)
        assert fsr == sr
        t = trim_silence_energy(w, sr)
        host_ext = [t.storage_offset(), t.storage_offset() + t.shape[-1]]
        assert ingest.trim_extents([w[0].to(DEV)], [sr]).cpu().tolist()[0] == host_ext, name
        host = AF.resample(t, sr, 24000)[0] if sr != 24000 else t[0]
        wav_bl, lens = tts.codec.prepare_wavs([w], [sr], 12.0)
        o, m = ingest.crop_plan(int(host.numel()), ingest.crop_samples(12.0))
        assert lens[0] == m
        ours = wav_bl[0, : m].cpu()
        if sr == 24000:
            assert torch.equal(ours, host[o:o + m])
        else:
            y64, bound = _oracle64(t[0], sr)
            assert bool(((ours.double() - y64[o:o + m]).abs() <= bound[o:o + m]).all()), name
            assert float((ours - host[o:o + m]).abs().max()) <= 5e-4 * max(1.0, float(host.abs().max())), name
        want = tts.prepare_reference(ref_audio_path=path).ref_tokens_btq[0].cpu()
        got = tts.prepare_references([path])[0].ref_tokens_btq[0].cpu()
        assert got.shape == want.shape, name
        if not torch.equal(got, want):
            lat = M.mimi_encode_latent(sd, host[o:o + m][None, None])[0]
            _compare_codes(sd, lat, got.permute(1, 0), want.permute(1, 0))


def test_synthesize_with_a_reference_prepared_here():
    tts = _tts()
    g = np.random.default_rng(3)
    sr = 22050
    t = np.arange(int(sr * 4.0)) / sr
    x = torch.from_numpy((0.4 * np.sin(2 * np.pi * 200 * t) + 0.01 * g.standard_normal(t.size)).astype(np.float32))
    ref = tts.prepare_references([x], sample_rates=[sr])[0]
    text = " ".join(str(7 * i + 3) for i in range(12))
    a = tts.synthesize(text, ref=ref, max_frames=24, seed=5)
    b = tts.synthesize(text, ref_tokens_tq=ref.ref_tokens_btq[0], max_frames=24, seed=5)
    assert a.shape == b.shape and a.shape[-1] > 0 and torch.equal(a, b)
