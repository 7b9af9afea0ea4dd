"""GPU: reference-voice denoising (sopro_b200/csrc/denoise.cu, SoproTTS.prepare_references(denoise=True)).
  - the device against the float64 oracle: the selected noise frames equal, the output within 1e-4 of the row's peak;
  - every row of a ragged batch equal to the row alone, bit for bit, with loud noise in the padding;
  - prepare_references(denoise=True) equal to its parts composed by hand, and each row equal to the single-clip call;
  - denoise=False equal to omitting the argument; the C-ABI's refusals of bad geometry."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import denoise_oracle as O

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
DEV = torch.device("cuda", 0)
_S = {}


def _tts():
    if "tts" not in _S:
        from oracle import mimi_oracle as M
        from sopro_b200 import SoproTTS
        from sopro_b200.tokenizer import IdsTokenizer
        from tests.cases import e2e_inputs

        msd = dict(M.synth_mimi_state_dict())
        msd.update(M.synth_mimi_encoder_state_dict())
        cfg, sd, _ = e2e_inputs()
        _S["tts"] = SoproTTS.from_state_dict(cfg, sd, IdsTokenizer(1000), msd, device="cuda:0", mimi_precision="fp32")
    return _S["tts"]


def _noisy(n: int, seed: int) -> np.ndarray:
    """The voiced test signal (or its start) at 5 dB SNR in white noise, any length."""
    s = np.resize(O.voiced(), n)
    return s + O.at_snr(s, O.white(n, seed), 5.0)


def _selected(ws: torch.Tensor, B: int, most: int) -> np.ndarray:
    kmax = O.n_noise(most) if most >= O.N else 1
    return ws[: B * kmax * 4].view(torch.int32).reshape(B, kmax).cpu().numpy()


@pytest.mark.parametrize("n", [1, 511, 512, 513, 1001, 24000, 24001, 77777, 240000])
def test_against_the_oracle(n):
    from sopro_b200.denoising import _run

    x = _noisy(n, n).astype(np.float32)
    y, ws = _run(torch.from_numpy(x).to(DEV), None)
    d = O.denoise_detail(x)
    got = y.cpu().numpy().astype(np.float64)
    sel = _selected(ws, 1, n)[0]
    if d["sel"] is None:
        assert np.array_equal(got, x.astype(np.float64)) and (sel == -1).all()
        return
    assert sel[: d["sel"].size].tolist() == d["sel"].tolist() and (sel[d["sel"].size:] == -1).all()
    peak = float(np.abs(x).max())
    err = float(np.abs(got - d["y"]).max())
    assert err <= 1e-4 * peak, (n, err, peak)


def test_pass_through_rows_on_the_device():
    from sopro_b200.denoising import denoise

    x = torch.from_numpy(_noisy(30000, 3).astype(np.float32)).to(DEV)
    x[1234] = float("nan")
    assert torch.equal(denoise(x).isnan(), x.isnan()) and torch.equal(denoise(x).nan_to_num(), x.nan_to_num())
    s = torch.from_numpy(O.voiced().astype(np.float32)).to(DEV)  # digital-silence gaps: lambda = 0, G = 1
    assert float((denoise(s) - s).abs().max()) <= 1e-5


def test_noise_is_reduced_on_the_device():
    from sopro_b200.denoising import denoise

    s = O.voiced()
    x = s + O.at_snr(s, O.white(s.size, 1), 0)
    y = denoise(torch.from_numpy(x.astype(np.float32)).to(DEV)).cpu().numpy().astype(np.float64)
    assert O.snr_db(s, y) >= 7.0


@pytest.mark.parametrize("B", [7, 64])
def test_each_row_of_a_batch_equals_the_row_alone(B):
    from sopro_b200.denoising import denoise

    g = np.random.default_rng(B)
    lens = [int(v) for v in g.integers(1, 60000, B)]
    lens[0], lens[1] = 511, 512
    L = max(lens) + 37
    x = torch.randn((B, L), generator=torch.Generator().manual_seed(B)) * 30.0  # loud padding
    for b, n in enumerate(lens):
        x[b, :n] = torch.from_numpy(_noisy(n, 100 + b).astype(np.float32))
    x = x.to(DEV)
    y = denoise(x, lens)
    assert y.shape == (B, L)
    for b, n in enumerate(lens):
        assert torch.equal(y[b, :n], denoise(x[b, :n].clone())), (b, n)
        assert not bool(y[b, n:].any()), b


def test_leading_dims_are_rows():
    from sopro_b200.denoising import denoise

    x = torch.from_numpy(np.stack([_noisy(9000, k) for k in range(6)]).astype(np.float32)).to(DEV).reshape(2, 3, 9000)
    y = denoise(x)
    assert y.shape == x.shape and torch.equal(y[1, 2], denoise(x[1, 2].clone()))


def _clips():
    out = []
    for k, (sr, secs) in enumerate([(16000, 3.3), (24000, 4.1), (44100, 2.7), (24000, 13.5), (16000, 1.2)]):
        n = int(sr * secs)
        t = np.arange(n) / sr
        g = np.random.default_rng(500 + k)
        env = ((t > 0.4) & (t < secs - 0.3)) * np.abs(np.sin(2 * np.pi * 1.5 * t))
        x = 0.4 * np.sin(2 * np.pi * (130 + 25 * k) * t) * env + 0.03 * g.standard_normal(n)
        w = torch.from_numpy(x.astype(np.float32))
        out.append((w.to(DEV) if k % 2 else w, sr))
    return out


@pytest.mark.parametrize("ref_seconds", [None, 3.0])
def test_prepare_references_denoised_equals_its_parts(ref_seconds):
    from sopro_b200 import ingest
    from sopro_b200.denoising import denoise
    from sopro_b200.resample import Resampler

    tts = _tts()
    items = _clips()
    clips, rates = [c for c, _ in items], [sr for _, sr in items]
    refs = tts.prepare_references(clips, sample_rates=rates, ref_seconds=ref_seconds, denoise=True)
    win = ingest.crop_samples(ingest.DEFAULT_REF_SECONDS if ref_seconds is None else ref_seconds)
    wav_bl, lens = tts.codec.prepare_wavs(clips, rates, 12.0 if ref_seconds is None else ref_seconds, denoise=True)
    for b, (w, sr) in enumerate(items):
        row = ingest.mono_rows([w], DEV)[0]
        s, e = ingest.trim_extents([row], [sr]).cpu().tolist()[0]
        z = row[s:e].clone()
        if sr != 24000:
            z = Resampler(sr, 24000, DEV)(z)
        z = denoise(z)
        o, m = ingest.crop_plan(int(z.numel()), win)
        want = z[o:o + m]
        assert lens[b] == m and torch.equal(wav_bl[b, :m], want), b
        codes = tts.codec.encode_wav(want)
        assert torch.equal(refs[b].ref_tokens_btq[0], codes), b
        one = tts.prepare_references([clips[b]], sample_rates=[sr], ref_seconds=ref_seconds, denoise=True)[0]
        assert torch.equal(one.ref_tokens_btq, refs[b].ref_tokens_btq) and torch.equal(one.sv_ref, refs[b].sv_ref), b
    plain = tts.prepare_references(clips, sample_rates=rates, ref_seconds=ref_seconds)
    assert any(not torch.equal(p.ref_tokens_btq, r.ref_tokens_btq) for p, r in zip(plain, refs))


def test_a_file_equals_its_samples(tmp_path):
    from sopro_b200.audio import load_audio_file, save_audio

    tts = _tts()
    w, sr = _clips()[2]
    path = str(tmp_path / "voice.wav")
    save_audio(path, w, sr)
    a = tts.prepare_references([path], ref_seconds=3.0, denoise=True)[0]
    x, fsr = load_audio_file(path)
    b = tts.prepare_references([x], sample_rates=[fsr], ref_seconds=3.0, denoise=True)[0]
    assert torch.equal(a.ref_tokens_btq, b.ref_tokens_btq) and torch.equal(a.sv_ref, b.sv_ref)


def test_default_is_unchanged():
    tts = _tts()
    items = _clips()
    clips, rates = [c for c, _ in items], [sr for _, sr in items]
    a = tts.prepare_references(clips, sample_rates=rates, denoise=False)
    b = tts.prepare_references(clips, sample_rates=rates)
    for p, q in zip(a, b):
        assert torch.equal(p.ref_tokens_btq, q.ref_tokens_btq) and torch.equal(p.sv_ref, q.sv_ref)


def test_c_abi_refusals():
    from sopro_b200 import _lib
    from sopro_b200.denoising import workspace_bytes

    lib = _lib.load()
    x = torch.zeros((2, 4000), device=DEV)
    y = torch.empty_like(x)
    ws = torch.empty(workspace_bytes(2, 4000), dtype=torch.uint8, device=DEV)
    st = _lib.stream_ptr(DEV)
    f = lib.sopro_denoise
    ok = (C.c_int64 * 2)(4000, 3000)
    assert f(x.data_ptr(), 2, 4000, ok, ws.data_ptr(), y.data_ptr(), 4000, st) == 0
    assert f(x.data_ptr(), 0, 4000, ok, ws.data_ptr(), y.data_ptr(), 4000, st) == -1
    assert f(x.data_ptr(), 2, 3999, ok, ws.data_ptr(), y.data_ptr(), 4000, st) == -1
    assert f(x.data_ptr(), 2, 4000, (C.c_int64 * 2)(4001, 10), ws.data_ptr(), y.data_ptr(), 4000, st) == -1
    assert f(x.data_ptr(), 2, 4000, ok, None, y.data_ptr(), 4000, st) == -1
    assert f(x.data_ptr(), 2, 4000, ok, ws.data_ptr(), None, 4000, st) == -1
    assert f(x.data_ptr(), 2, 4000, ok, ws.data_ptr(), y.data_ptr(), 3999, st) == -1
    torch.cuda.synchronize()
    from sopro_b200.denoising import denoise

    with pytest.raises(ValueError):
        denoise(x, [10, 4001])
