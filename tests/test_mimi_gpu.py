"""GPU parity of the CUDA Mimi decoder against the CPU oracle (which is pinned to transformers' MimiModel)."""
import numpy as np
import pytest
import torch

from oracle import mimi_oracle as M

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
_ENG = {}

# Tensor-core mode against oracle.mimi_decode_bf16_operands, the model of the mode's own bf16 rounding: max distance as
# a fraction of the model waveform's peak, RMS distance as a fraction of its RMS.  attention="tc" models the one-shot
# decode, attention="fp32" the stream.  Measured on an H100 80GB HBM3 at a 700 W power limit: one-shot max 4.2e-3 ..
# 5.5e-3, rms 5.0e-3 .. 5.2e-3 (six shapes below, and frames [0, 300) of the 10k-frame decode); stream max 5.1e-3, rms
# 5.0e-3.  That is as far as the fp32 oracle, not the "accumulation order only" distance one might expect: every SEANet
# stage re-rounds its activations to bf16, so any difference in fp32 summation order (GPU vs CPU) decorrelates the
# roundings by the waveform.  The model itself moves as far when only its accumulation goes from fp32 to fp64
# (DESIGN.md section 7).  So these bounds are ~2-3x the worst measurement and no waveform-level bound can see a window
# one key off (8e-4 of the peak); tests/test_mimi_tc_kernels_gpu.py checks the kernels where that bug lives.
TC_MODEL_MAX, TC_MODEL_RMS = 1.5e-2, 1e-2
STREAM_MODEL_MAX, STREAM_MODEL_RMS = 1.5e-2, 1e-2


def _model_distance(got, model):
    """(max |got - model| / peak(model), rms(got - model) / rms(model))"""
    d = got.cpu().reshape(model.shape) - model
    return float(d.abs().max()) / float(model.abs().max()), float(d.pow(2).mean().sqrt()) / float(model.pow(2).mean().sqrt())


def _engine(precision="fp32"):
    from sopro_b200.codec import MimiEngine

    if "e" not in _ENG:
        _ENG["sd"] = M.synth_mimi_state_dict()
        _ENG["e"] = MimiEngine(_ENG["sd"], 0, 32)
    _ENG["e"].set_precision(precision)
    return _ENG["e"], _ENG["sd"]


@pytest.mark.parametrize("B,T", [(1, 1), (2, 9), (1, 37), (3, 16)])
def test_decode_matches_oracle(B, T):
    """fp32 mode; the contraction order differs from the CPU's: tolerance 2e-4 of the waveform's peak."""
    eng, sd = _engine("fp32")
    codes = torch.randint(0, 2048, (B, 32, T), generator=torch.Generator().manual_seed(100 + T))
    want = M.mimi_decode(sd, codes)
    got = eng.decode(codes).cpu()
    assert got.shape == want.shape
    peak = float(want.abs().max())
    assert peak > 1e-3
    assert float((got - want).abs().max()) <= 2e-4 * max(1.0, peak)


@pytest.mark.parametrize("B,T", [(1, 1), (2, 9), (1, 37), (3, 16), (1, 150), (2, 203)])
def test_decode_tensor_core_mode(B, T):
    """Default mode: bf16 operands on the tensor cores, fp32 accumulation.  Stated tolerance: max error
    2e-2 of the waveform's peak and relative RMS error 1e-2 against the fp32 oracle.  Against the model of this mode's
    rounding (oracle.mimi_decode_bf16_operands): max 1.5e-2 of the peak and relative RMS 1e-2 (TC_MODEL_MAX /
    TC_MODEL_RMS; measured on an H100 at 700 W: max <= 5.5e-3, rms <= 5.2e-3 over these six shapes).  The model is no
    closer than the fp32 oracle at the waveform: the SEANet's bf16 re-rounding turns the GPU's other fp32 summation
    order into a distance as large as the rounding itself (see TC_MODEL_MAX)."""
    eng, sd = _engine("bf16_tc")
    codes = torch.randint(0, 2048, (B, 32, T), generator=torch.Generator().manual_seed(100 + T))
    want = M.mimi_decode(sd, codes)
    got = eng.decode(codes).cpu()
    assert got.shape == want.shape and bool(torch.isfinite(got).all())
    peak = float(want.abs().max())
    err = got - want
    emu = M.mimi_decode_bf16_operands(sd, codes)
    dmax, drms = _model_distance(got, emu)
    print(f"tensor-core mode B={B} T={T}: max err vs fp32 oracle {float(err.abs().max()) / peak:.2e} of peak; "
          f"vs bf16-operand model max {dmax:.2e} of peak, rms {drms:.2e} of rms")
    assert float(err.abs().max()) <= 2e-2 * peak, (float(err.abs().max()), peak)
    assert float(err.pow(2).mean().sqrt()) <= 1e-2 * float(want.pow(2).mean().sqrt())
    assert dmax <= TC_MODEL_MAX and drms <= TC_MODEL_RMS, (dmax, drms)


def test_full_size_decode_properties():
    """BASELINE.json's standalone configuration (10k frames) through size-independent properties: the decoder is
    causal, so the first 300 frames of the 10k-frame waveform equal a 300-frame decode bit for bit (same kernels, other
    grid sizes); the tensor-core result stays within the stated tolerance of the fp32 mode at full size; a batch of 25
    x 400 frames equals the same utterances decoded one by one.  Frames [0, 300) are also held to the bounds against the
    model of the mode's rounding (TC_MODEL_MAX / TC_MODEL_RMS)."""
    eng, _ = _engine("bf16_tc")
    codes = torch.randint(0, 2048, (1, 32, 10000), generator=torch.Generator().manual_seed(5))
    big = eng.decode(codes)
    assert big.shape == (1, 1, 10000 * 1920) and bool(torch.isfinite(big).all())
    small = eng.decode(codes[:, :, :300])
    assert torch.equal(big[..., : 300 * 1920], small)
    eng.set_precision("fp32")
    ref32 = eng.decode(codes[:, :, :2000])
    eng.set_precision("bf16_tc")
    err = (big[..., : 2000 * 1920] - ref32).abs().max()
    assert float(err) <= 2e-2 * float(ref32.abs().max())
    # against the CPU oracle directly: the decoder is causal, so the oracle's decode of the first 700 frames is the
    # reference for frames [0, 700) of the 10k-frame waveform: the start [0, 300) and a mid-stream slice [400, 700)
    # (past the 125-frame attention window) in both modes
    want = M.mimi_decode(_ENG["sd"], codes[:, :, :700])
    peak = float(want.abs().max())
    for lo, hi in ((0, 300), (400, 700)):
        sl = slice(lo * 1920, hi * 1920)
        e_tc = float((big[..., sl].cpu() - want[..., sl]).abs().max())
        e_32 = float((ref32[..., sl].cpu() - want[..., sl]).abs().max())
        print(f"10k-frame decode vs oracle, frames [{lo},{hi}): tensor-core {e_tc / peak:.2e} of peak, fp32 {e_32 / peak:.2e} of peak")
        assert e_tc <= 2e-2 * peak, (lo, hi, e_tc, peak)
        assert e_32 <= 2e-4 * max(1.0, peak), (lo, hi, e_32, peak)
    dmax, drms = _model_distance(big[..., : 300 * 1920], M.mimi_decode_bf16_operands(_ENG["sd"], codes[:, :, :300]))
    print(f"10k-frame decode vs bf16-operand model, frames [0,300): max {dmax:.2e} of peak, rms {drms:.2e} of rms")
    assert dmax <= TC_MODEL_MAX and drms <= TC_MODEL_RMS, (dmax, drms)
    batch = codes.view(1, 32, 25, 400).permute(2, 1, 0, 3).reshape(25, 32, 400).contiguous()
    wb = eng.decode(batch)
    for i in (0, 11, 24):
        assert torch.equal(wb[i: i + 1], eng.decode(batch[i: i + 1]))


@pytest.mark.parametrize("precision", ["fp32", "bf16_tc"])
def test_host_buffer_path_and_stream_decoder(precision):
    from sopro_b200.codec import MimiCodec, MimiStreamDecoder

    eng, sd = _engine(precision)
    codes = torch.randint(0, 2048, (1, 32, 20), generator=torch.Generator().manual_seed(3))
    full = eng.decode(codes).cpu().numpy()
    np.testing.assert_array_equal(eng.decode_host(codes.numpy()), full)
    codec = MimiCodec(32, device="cuda:0", state_dict=sd, precision=precision)
    dec = MimiStreamDecoder(codec)
    state, parts = None, []
    for a, b in [(0, 6), (6, 12), (12, 13), (13, 20)]:
        wav, state = dec.decode_step(codes[0, :, a:b].permute(1, 0), state)
        parts.append(wav.cpu().numpy())
    got = np.concatenate(parts, axis=1)
    assert got.shape == (1, 20 * 1920) and state.frames_seen == 20
    if precision == "fp32":  # the persistent-state stream decoder computes every sample in the one-shot decode's order
        np.testing.assert_array_equal(got[0], full[0, 0])
    else:  # tensor-core mode: same tensor-core tiles, the attention core runs in fp32 over the K/V ring (tolerance 1e-2 of peak)
        np.testing.assert_allclose(got[0], full[0, 0], rtol=0, atol=1e-2 * float(np.abs(full).max()))


def test_small_decodes_replay_from_graphs_identically():
    """<= 64 frames go through the library's CUDA-graph cache: first call captures, later calls replay; both equal the
    plain launches bit for bit, also after a large decode reallocated the workspace (graphs are dropped then)."""
    eng, _ = _engine("bf16_tc")
    codes = torch.randint(0, 2048, (2, 32, 7), generator=torch.Generator().manual_seed(9))
    other = torch.randint(0, 2048, (2, 32, 7), generator=torch.Generator().manual_seed(10))
    eng.set_graphs(False)
    want, want_other = eng.decode(codes).cpu(), eng.decode(other).cpu()
    eng.set_graphs(True)
    assert torch.equal(eng.decode(codes).cpu(), want)        # capture + first replay
    assert torch.equal(eng.decode(other).cpu(), want_other)  # replay with new inputs
    eng.decode(torch.randint(0, 2048, (4, 32, 120)))         # grows the workspace
    assert torch.equal(eng.decode(codes).cpu(), want)


def test_decode_full_signature():
    from sopro_b200.codec import MimiCodec

    _, sd = _engine()
    codec = MimiCodec(32, device="cuda:0", state_dict=sd)
    codes_tq = torch.randint(0, 2048, (5, 32), generator=torch.Generator().manual_seed(4))
    wav = codec.decode_full(codes_tq)
    assert wav.shape == (1, 1, 5 * 1920) and wav.dtype == torch.float32


@pytest.mark.parametrize("mode", ["fp32", "bf16_tc"])
def test_stream_decode_step_equals_the_full_decode(mode):
    """sopro_mimi_decode_step carries the K/V rings and every conv's left context: chunks of ragged sizes (1 frame,
    the default 6, 16, a 40-frame chunk that is split internally, ...) over 310 frames -- 620 transformer positions,
    far past the 250-position window and past the ring's wrap-around -- concatenate to the one-shot decode.  fp32
    mode: bit for bit (every output element is computed in the same order).  Tensor-core mode: the dense blocks are the
    same tensor-core tiles, only the attention core runs in fp32 on the ring.  Every kernel of the tensor-core stream is
    row-local with a fixed summation order, so one-frame chunks give the ragged schedule's output bit for bit; against
    the model of the stream's rounding (oracle.mimi_decode_bf16_operands(attention="fp32")) the first 150 frames are
    held to max 1.5e-2 of the peak and relative RMS 1e-2 (STREAM_MODEL_MAX / STREAM_MODEL_RMS; measured on an H100 at
    700 W: max 5.1e-3, rms 5.0e-3), and to the mode's 2e-2 vs the fp32 oracle.  The distance to the one-shot
    tensor-core decode (the two attention roundings differ; measured 5.3e-3) is reported and held to 1e-2 of the peak."""
    eng, sd = _engine(mode)
    T = 310
    codes = torch.randint(0, 2048, (1, 32, T), generator=torch.Generator().manual_seed(77))
    full = eng.decode(codes).reshape(1, -1)
    st = eng.stream(16)
    sizes, pos, parts = [1, 6, 6, 16, 3, 40, 6, 2, 64, 6], 0, []
    i = 0
    while pos < T:
        n = min(sizes[i % len(sizes)], T - pos)
        parts.append(st.step(codes[0, :, pos:pos + n]))
        pos += n
        i += 1
    assert st.frames == T
    got = torch.cat(parts, dim=1)
    assert got.shape == full.shape
    peak = float(full.abs().max())
    err = float((got - full).abs().max())
    print(f"stream vs one-shot [{mode}]: max err {err / peak:.2e} of peak")
    if mode == "fp32":
        assert torch.equal(got, full)
    else:
        ones = eng.stream(16)
        one_by_one = torch.cat([ones.step(codes[0, :, t:t + 1]) for t in range(T)], dim=1)
        assert torch.equal(one_by_one, got), f"chunk schedules differ at {int((one_by_one != got).sum())} samples"
        dmax, drms = _model_distance(got[:, : 150 * 1920], M.mimi_decode_bf16_operands(sd, codes[:, :, :150], attention="fp32"))
        print(f"stream [{mode}] vs its bf16-operand model (fp32 attention), frames [0,150): max {dmax:.2e} of peak, rms {drms:.2e} of rms")
        assert dmax <= STREAM_MODEL_MAX and drms <= STREAM_MODEL_RMS, (dmax, drms)
        want = M.mimi_decode(sd, codes[:, :, :150]).reshape(1, -1)
        assert float((got[:, : 150 * 1920].cpu() - want).abs().max()) <= 2e-2 * float(want.abs().max())
        assert err <= 1e-2 * peak, (err, peak)
    # reset -> the same stream object decodes a new utterance from frame 0; host-buffer entry point
    st.reset()
    assert st.frames == 0
    again = st.step_host(codes[0, :, :9].numpy())
    one = eng.decode(codes[:, :, :9]).reshape(1, -1).cpu().numpy()
    if mode == "fp32":
        assert np.array_equal(again, one)
    else:
        assert float(np.abs(again - one).max()) <= 1e-2 * peak


def test_two_streams_are_independent_and_state_is_per_stream():
    eng, _ = _engine("fp32")
    a = torch.randint(0, 2048, (32, 30), generator=torch.Generator().manual_seed(1))
    b = torch.randint(0, 2048, (32, 30), generator=torch.Generator().manual_seed(2))
    sa, sb = eng.stream(8), eng.stream(8)
    outa, outb = [], []
    for lo in range(0, 30, 6):  # interleaved
        outa.append(sa.step(a[:, lo:lo + 6]))
        outb.append(sb.step(b[:, lo:lo + 6]))
    assert torch.equal(torch.cat(outa, 1), eng.decode(a.unsqueeze(0)).reshape(1, -1))
    assert torch.equal(torch.cat(outb, 1), eng.decode(b.unsqueeze(0)).reshape(1, -1))


def test_out_of_range_codes_are_reported_not_read():
    """An uncut EOS id (2048) must not index past the codebook: the Python layer raises IndexError like the reference's
    embedding lookup, the host C-ABI path returns an error, and the device path clamps + flags (sopro_mimi_check)."""
    import ctypes as C

    from sopro_b200 import _lib

    eng, _ = _engine("fp32")
    bad = torch.randint(0, 2048, (1, 32, 4))
    bad[0, 3, 2] = 2048
    with pytest.raises(IndexError):
        eng.decode(bad)
    with pytest.raises(_lib.SoproError):
        eng.decode_host(bad.numpy())
    dev = bad.to("cuda:0", torch.int32).contiguous()
    wav = torch.empty(1, 1, 4 * 1920, device="cuda:0")
    _lib.check(eng.lib.sopro_mimi_decode(eng._h, dev.data_ptr(), 1, 4, wav.data_ptr(), int(torch.cuda.current_stream().cuda_stream)))
    with pytest.raises(_lib.SoproError):
        eng.check()
    eng.check()  # the flag is cleared by the failed check
    assert bool(torch.isfinite(wav).all())
