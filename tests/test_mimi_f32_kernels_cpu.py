"""Without a GPU: the float64 references that tests/test_mimi_f32_kernels_gpu.py holds Mimi's fp32 kernels to
(tests/mimi_f32_refs.py) against oracle/mimi_oracle.py, the restatement of the reference's model, and the refusals of
non-finite audio, which come before any device work."""
import pytest
import torch
import torch.nn.functional as F

from oracle import mimi_oracle as M
from sopro_b200 import ingest
from tests import mimi_f32_refs as R

torch.set_grad_enabled(False)


@pytest.mark.parametrize("r,L", [(4, 37), (4, 40), (5, 1), (6, 17), (8, 64), (8, 65)])
def test_superrow_two_tap_view_is_the_strided_conv(r, L):
    """A conv of kernel 2r and stride r (MimiConv1d, with its causal left pad of r rows and the extra right padding) is
    the 2-tap stride-1 conv over the superrow view [ceil(L/r)][r*C] with the repacked weight and pad 1 (the tap at
    superrow -1 is the left padding)."""
    g = torch.Generator().manual_seed(r * 100 + L)
    C, N = 12, 8
    x = torch.randn(2, L, C, generator=g, dtype=torch.float64)
    w = torch.randn(N, C, 2 * r, generator=g, dtype=torch.float64)
    b = torch.randn(N, generator=g, dtype=torch.float64)
    want = M.conv1d_mimi(x, w, b, stride=r)
    s = R.superrows(x, r)
    Ms = s.shape[1]
    got, _ = R.gemm_ref(s, R.conv_repack(w), Ms, Ms, 2, 1, 1, bias=b, bias_mod=N)
    assert got.shape == want.shape
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("r", [8, 6, 5, 4])
def test_convtranspose_as_two_tap_gemm(r):
    """The decoder's ConvTranspose1d (stride r, kernel 2r, causal trim) is the 2-tap conv over its input rows with the
    weight repacked to [(phase, co)][(tap, ci)] and bias_mod = Cout: its [T][r*Cout] output is the [T*r][Cout] upsampled
    activation."""
    g = torch.Generator().manual_seed(r)
    T, cin, cout = 9, 10, 6
    x = torch.randn(2, T, cin, generator=g, dtype=torch.float64)
    w = torch.randn(cin, cout, 2 * r, generator=g, dtype=torch.float64)
    b = torch.randn(cout, generator=g, dtype=torch.float64)
    want = M.conv_transpose_causal(x, w, b, r)
    got, _ = R.gemm_ref(x, R.convT_as_2tap(w, r), T, T, 2, 1, 1, bias=b, bias_mod=cout)
    torch.testing.assert_close(got.reshape(2, T * r, cout), want, rtol=1e-12, atol=1e-12)


def test_chunked_ring_attention_is_the_windowed_attention():
    """window_attention over chunks (each chunk's queries against the earlier positions plus its own) equals the
    oracle's one-shot sliding-window attention (mimi_oracle.transformer's mask and softmax, RoPE left out)."""
    g = torch.Generator().manual_seed(3)
    B, T, H, Dh, window = 2, 70, 2, 8, 9
    q, k, v = (torch.randn(B, T, H, Dh, generator=g, dtype=torch.float64) for _ in range(3))
    i = torch.arange(T)
    allowed = (i[None, :] <= i[:, None]) & (i[:, None] - i[None, :] < window)
    bias = torch.zeros(T, T, dtype=torch.float64).masked_fill(~allowed, float("-inf"))
    qt, kt, vt = (t.transpose(1, 2) for t in (q, k, v))
    w = F.softmax(torch.matmul(qt, kt.transpose(2, 3)) / Dh ** 0.5 + bias, dim=-1)
    want = torch.matmul(w, vt).transpose(1, 2)
    pos = 0
    for n in (1, 7, 2, 13, 20, 27):
        got, _ = R.window_attention(q[:, pos:pos + n], k[:, pos:pos + n], v[:, pos:pos + n], window, pos,
                                    k[:, :pos] if pos else None, v[:, :pos] if pos else None)
        torch.testing.assert_close(got, want[:, pos:pos + n], rtol=1e-12, atol=1e-12)
        pos += n
    assert pos == T


def test_rope64_is_the_oracle_rotation():
    """rope64 with make_rope's table is the oracle's rotation (mimi_oracle.rope) to fp32 table precision."""
    g = torch.Generator().manual_seed(4)
    B, H, T, Dh = 1, 2, 40, 16
    x = torch.randn(B, H, T, Dh, generator=g)
    want, _ = M.rope(x, x)
    tab = R.rope_table(64, Dh)
    got, _ = R.rope64(x.transpose(1, 2), torch.arange(T), tab, 64)
    torch.testing.assert_close(got.transpose(1, 2).float(), want, rtol=0, atol=1e-4)


def test_oracle_codes_of_non_finite_rows_are_zero():
    """The reference's codeword search (torch.cdist(...).argmin()) over a NaN, an infinite or an overflowing frame picks
    code 0 at every codebook: the codes the fixed CUDA search must give."""
    sd = M.synth_mimi_state_dict()
    g = torch.Generator().manual_seed(5)
    emb = torch.randn(1, 6, 512, generator=g) * 0.3
    emb[0, 1] = float("nan")
    emb[0, 3] = float("inf")
    emb[0, 4] = 1e30
    codes = M.rvq_encode(sd, emb, n_q=4)
    assert bool((codes[0, :, [1, 3, 4]] == 0).all()), codes[0]
    assert bool((codes[0, :, [0, 2, 5]] != 0).any())


def _tts_stub():
    from sopro_b200.model import SoproTTS

    return SoproTTS.__new__(SoproTTS)  # no codec, no model, no device: a refusal must come first


def _float_file(monkeypatch, bad):
    """audio.load_audio_file reading a float file that holds `bad` at sample 7 (soundfile reads float WAVs as they are)"""
    from sopro_b200 import audio

    def load(path):
        y = torch.zeros(1, 4000)
        y[0, 7] = bad
        return y, 16000

    monkeypatch.setattr(audio, "load_audio_file", load)


@pytest.mark.parametrize("bad", [float("nan"), float("inf"), -float("inf")])
def test_prepare_references_refuses_non_finite_clips(bad, monkeypatch):
    """Every clip, tensor or file, is checked for finite samples before the first launch; the error names the clip."""
    good = torch.zeros(4000)
    x = torch.zeros(2, 4000)
    x[1, 1234] = bad
    with pytest.raises(ValueError, match="clip 1 "):
        _tts_stub().prepare_references([good, x], sample_rates=[16000, 16000])
    silent = torch.zeros(4000)
    with pytest.raises(ValueError, match="clip 0 "):  # peak-normalising a silent clip: 0 / 0
        _tts_stub().prepare_references([silent / silent.abs().max()], sample_rates=16000)
    _float_file(monkeypatch, bad)
    path = "voice.wav"
    with pytest.raises(ValueError, match="clip 2 "):
        _tts_stub().prepare_references([good, good, path], sample_rates=[16000, 16000, None])
    with pytest.raises(ValueError, match="clip 0 "):
        ingest.load_clips([path])


def test_codec_encode_refuses_non_finite_audio(monkeypatch):
    """MimiCodec.encode_wav and encode_file refuse non-finite audio before the encoder is built or launched (the stub
    has no encoder: reaching it would raise something else)."""
    from sopro_b200.codec import MimiCodec

    codec = MimiCodec.__new__(MimiCodec)
    wav = torch.zeros(1, 4800)
    wav[0, 100] = float("nan")
    with pytest.raises(ValueError, match="non-finite"):
        codec.encode_wav(wav)
    _float_file(monkeypatch, float("inf"))
    with pytest.raises(ValueError, match="non-finite"):
        codec.encode_file("voice.wav")
