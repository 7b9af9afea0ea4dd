"""Without a GPU: the float64 model and the checks that tests/test_mimi_tc_kernels_gpu.py holds the tensor-core implicit
GEMM to (tests/mimi_tc_refs.py).  The model, in the decoder's pitched, ctx-aware operand geometry, is pinned to
oracle/mimi_oracle.py's convolutions; the dyadic operands are shown to make every fp32 sum exact in any order; and
emulated wrong kernels (a row shifted, a tap dropped, a K chunk skipped or doubled, an item pitch off by one, the bf16
output one row late, a write one row past M) are shown to fail the very checks the GPU tests apply."""
import dataclasses

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import mimi_oracle as M
from tests import mimi_f32_refs as R
from tests import mimi_tc_refs as T

torch.set_grad_enabled(False)
CPU = torch.device("cpu")
F64 = torch.float64


def _ops64(L, x, w_gemm, bias=None, r=None, scale=None):
    """float64 operands in the launch's buffers (NaN operand rows past ctx + M, NaN residual rows past M)"""
    X = T.pitched_rows(x, L.a_pitch, float("nan"))
    Rb = T.pitched_rows(r, L.r_pitch, float("nan")) if r is not None else None
    return T.Operands(X, w_gemm, bias, Rb, scale)


@pytest.mark.parametrize("pitched", [False, True])
@pytest.mark.parametrize("taps", [1, 3, 7])
def test_reference_is_the_oracle_conv(taps, pitched):
    """T.reference over the items' ctx context rows (then the causal zero pad) is MimiConv1d's causal conv
    (mimi_oracle.conv1d_causal) at the chunk's rows: a chunk starting at row ctx with every ctx in [0, taps-1], and
    a mid-sequence chunk with taps-1 context rows; each epilogue (GELU, R + acc, R + scale acc) on top."""
    g = torch.Generator().manual_seed(10 * taps + pitched)
    B, Lx, cin, N = 2, 40, 6, 8
    x = torch.randn(B, Lx, cin, generator=g, dtype=F64)
    w = torch.randn(N, cin, taps, generator=g, dtype=F64)
    b = torch.randn(N, generator=g, dtype=F64)
    r = torch.randn(B, Lx, N, generator=g, dtype=F64)
    scale = torch.randn(N, generator=g, dtype=F64)
    conv = M.conv1d_causal(x, w, b)
    want = {T.EPI_NONE: conv, T.EPI_GELU: F.gelu(conv), T.EPI_RES: r + conv, T.EPI_RES_SCALE: r + scale * conv}
    chunks = [(ctx, ctx, 11) for ctx in range(taps)] + [(17, taps - 1, 23)]
    for epi, wv in want.items():
        layer = T.Layer("conv", cin, taps, N, N, epi, True, False, False)
        for s, ctx, m in chunks:
            L = T.launch(layer, B, m, ctx, pitched)
            res = epi in (T.EPI_RES, T.EPI_RES_SCALE)
            ops = _ops64(L, x[:, s - ctx: s + m], R.conv_repack(w), b, r[:, s: s + m] if res else None,
                         scale if epi == T.EPI_RES_SCALE else None)
            y, _, _ = T.reference(L, ops)
            torch.testing.assert_close(y, wv[:, s: s + m], rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("r", [8, 6, 5, 4])
def test_reference_is_the_oracle_conv_transpose(r):
    """With convT_as_2tap's weight and bias_mod = Cout, T.reference is the ConvTranspose1d (mimi_oracle.
    conv_transpose_causal): one-shot (ctx 0, packed) and as a stream chunk with the previous input row as context
    (pitched); each output row's r * Cout columns are r upsampled rows."""
    g = torch.Generator().manual_seed(r)
    B, Tn, cin, cout = 2, 12, 5, 3
    x = torch.randn(B, Tn, cin, generator=g, dtype=F64)
    w = torch.randn(cin, cout, 2 * r, generator=g, dtype=F64)
    b = torch.randn(cout, generator=g, dtype=F64)
    want = M.conv_transpose_causal(x, w, b, r)
    layer = T.Layer("convT", cin, 2, r * cout, cout, T.EPI_NONE, True, True, True)
    for s, ctx, m, pitched in ((0, 0, Tn, False), (4, 1, 7, True)):
        L = T.launch(layer, B, m, ctx, pitched)
        y, _, _ = T.reference(L, _ops64(L, x[:, s - ctx: s + m], R.convT_as_2tap(w, r), b))
        torch.testing.assert_close(y.reshape(B, m * r, cout), want[:, s * r: (s + m) * r], rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("layer", [l for l in T.PRODUCTION + T.TILES if l.K >= 2048], ids=lambda l: l.name)
def test_dyadic_operands_are_exact_in_fp32(layer):
    """The dyadic grids (T.dyadic_values) at the longest K: every product is exact in fp32, fp32 sums in four random
    orders equal the float64 sum, and every epilogue result (bias, R + acc, fmaf(scale, acc, R)) is exact in fp32."""
    L = T.launch(layer, 2, 5, layer.taps - 1, pitched=True)
    ops = T.operands(L, "dyadic", 5, CPU)
    A = R.im2col(ops.X[:, : L.ctx + L.M].double(), L.M, L.ctx + L.M, L.taps, 1, L.taps - 1 - L.ctx).reshape(-1, L.K)
    Wd = ops.W.double()
    rng = np.random.default_rng(6)
    for n in rng.choice(L.N, size=8, replace=False):
        p = A * Wd[n]  # [rows][K]
        assert torch.equal(p.float().double(), p)
        assert T.seq_sums_match(p.numpy(), rng)
    y, a, _ = T.reference(L, ops)
    assert torch.equal(a.float().double(), a) and torch.equal(y.float().double(), y)
    assert float(y.abs().max()) < 2 ** 9 and bool(((y * 2 ** 14).frac() == 0).all())
    # the extremes of the grids: every product +1/16 (K <= 4096: the sum <= 2^8), bias 1, scale 1, R 64
    top = L.K / 16 + 1
    assert top * 1 + 64 < 2 ** 9 and float(np.float32(top) + np.float32(64)) == top + 64


# ---------------------------------------------------------------------------------------------------------------
# controls: emulated wrong kernels must fail the GPU tests' checks
# ---------------------------------------------------------------------------------------------------------------
FAULTS = [None, "row_shifted", "tap_dropped", "chunk_skipped", "chunk_doubled", "item_pitch_off_by_one", "bf16_one_row_late",
          "write_past_M"]
CONTROL_LAYERS = [
    # the ConvTranspose's outputs (fp32 + bf16 ELU behind context elements) with a residual; conv0's (bf16 ELU only)
    T.Layer("f32_and_elu_bf16", 64, 3, 64, 32, T.EPI_RES, True, True, True, h_ctx=64),
    T.Layer("elu_bf16_only", 64, 3, 128, 128, T.EPI_NONE, False, True, True, h_ctx=128),
]


def _emulate(L, ops, fault):
    """what a kernel with `fault` writes into sentinel-filled buffers (CPU): the float64 result rounded to fp32, and
    to bf16 through fp32 ELU"""
    W = ops.W.clone()
    if fault == "tap_dropped":  # the tap of the row itself
        W[:, (L.taps - 1) * L.cin: L.taps * L.cin] = 0
    elif fault == "chunk_skipped":
        W[:, 64:128] = 0
    elif fault == "chunk_doubled":
        W[:, 64:128] *= 2
    y, _, _ = T.reference(L, dataclasses.replace(ops, W=W))
    if fault == "row_shifted":
        k = L.M // 2
        y[:, k] = y[:, k - 1]
    n = L.B * L.c_pitch * L.N
    of = T.f32_sentinel(n, CPU) if L.f32 else None
    oh = T.bf16_sentinel(L.h_off + n, CPU) if L.bf16 else None
    pitch = L.c_pitch + (1 if fault == "item_pitch_off_by_one" else 0)
    rows = L.M + (1 if fault == "write_past_M" else 0)
    h_off = L.h_off + (L.N if fault == "bf16_one_row_late" else 0)
    vf = y.float()
    vh = (F.elu(vf) if L.elu else vf).to(T.BF16)
    for b in range(L.B):
        for m in range(rows):
            src = min(m, L.M - 1)
            o = (b * pitch + m) * L.N
            if of is not None and o + L.N <= n:
                of[o: o + L.N] = vf[b, src]
            if oh is not None and h_off + o + L.N <= oh.numel():
                oh[h_off + o: h_off + o + L.N] = vh[b, src]
    return of, oh, y if fault is None else T.reference(L, ops)[0]


@pytest.mark.parametrize("fault", FAULTS, ids=lambda f: f or "correct")
@pytest.mark.parametrize("layer", CONTROL_LAYERS, ids=lambda l: l.name)
def test_checks_catch_emulated_wrong_kernels(layer, fault):
    """A correct emulation passes T.check_launch (the GPU tests' check, dyadic mode); each fault fails it."""
    L = T.launch(layer, 3, 9, 1, pitched=True)
    ops = T.operands(L, "dyadic", 11, CPU)
    of, oh, y = _emulate(L, ops, fault)
    if fault is None:
        T.check_launch(L, of, oh, y, None, "correct emulation")
    else:
        with pytest.raises(AssertionError):
            T.check_launch(L, of, oh, y, None, fault)


def test_launch_sweeps_cover_the_geometry():
    """Every layer's sweep reaches M in {1, 127, 128, 129, 383} and a multi-tile M, every ctx, B in {1, 3, 64},
    packed and pitched items with three distinct pitches, and the bf16 output behind the stream's context
    elements; the tile table reaches every (BN, BK) instantiation of tc::launch and the stage-ring edges."""
    for layer in T.PRODUCTION + T.TILES:
        ls = T.launches(layer)
        assert {1, 127, 128, 129, 383} <= {L.M for L in ls} and max(L.M for L in ls) > 3 * 128
        assert {L.ctx for L in ls} == set(range(layer.taps)) and {L.B for L in ls} == {1, 3, 64}
        packed = [L for L in ls if L.a_pitch == L.ctx + L.M and L.c_pitch == L.M]
        pitched = [L for L in ls if L not in packed]
        assert packed and pitched
        for L in pitched:
            assert L.a_pitch > L.ctx + L.M and L.c_pitch > L.M and L.h_off == layer.h_ctx
            if L.r_pitch and not layer.inplace:
                assert len({L.a_pitch, L.c_pitch, L.r_pitch}) == 3

    def bn(N):
        return 128 if N % 128 == 0 else 64 if N % 64 == 0 else 32

    def bk(cin):
        return 64 if cin % 64 == 0 else 32

    tiles = {(bn(l.N), bk(l.cin)) for l in T.PRODUCTION + T.TILES}
    assert tiles == {(n, k) for n in (128, 64, 32) for k in (64, 32)}
    nks = {l.K // bk(l.cin) for l in T.TILES}
    assert {1, 2, 3, 4, 5} <= nks and max(nks) >= 64
