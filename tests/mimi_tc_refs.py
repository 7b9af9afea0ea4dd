"""Float64 model of one launch of Mimi's tensor-core implicit GEMM (igemm_tc_kernel, launched by gemm_tc in
mimi_engine.cu) in the decoder's operand geometry, and the checks a launch is held to.  tests/test_mimi_tc_kernels_gpu.py
holds the kernel to them; tests/test_mimi_tc_gemm_cpu.py pins the model to oracle/mimi_oracle.py and shows that emulated
wrong kernels fail the same checks.

A launch (Launch) runs one layer (Layer) over B items.  Item b of the bf16 operand X starts a_pitch rows after item
b - 1 and holds ctx context rows, then M rows of cin channels.  Output row m of item b is

    y[b][m][n] = epi( sum_{j < taps} sum_ci X_b[m + ctx + j - (taps - 1)][ci] W[n][j cin + ci] + bias[n % bias_mod] )

(rows before X_b's first row read as zero: the causal pad), written to the fp32 output at (b c_pitch + m) N + n and to
the bf16 output at h_off + that offset (h_off: the context rows a stream keeps in front of a bf16 activation).  epi
RES adds R[(b r_pitch + m) N + n], RES_SCALE adds it to scale[n] times the sum; an in-place launch reads R from the
fp32 output itself.  Nothing else of either output buffer may change.
"""
import dataclasses

import numpy as np
import torch

from tests import mimi_f32_refs as R_

U = R_.U
EPI_NONE, EPI_GELU, EPI_RES_SCALE, EPI_RES = 0, 1, 2, 3
BF16 = torch.bfloat16
F32_SENTINEL = 0x7FC0DEAD  # a NaN payload no kernel computes: rows a launch must not write are filled with it
BF16_SENTINEL = 0x7FAD
# elu_fast(v) = __expf(v) - 1 for v <= 0 (mimi_tc.cuh).  __expf(v) is within 2 + floor(1.173 |v|) ulp of e^v (CUDA C
# Programming Guide, intrinsic functions); an ulp of e^v is at most 2^-23 e^v, and (2 + 1.173 t) e^-t <= 2 for t >= 0,
# so the exponential is within 2^-22 of e^v.  The subtraction of 1 is exact for e^v >= 1/2 (Sterbenz) and rounds
# by at most half an ulp of a result in (-1, -1/2], 2^-25, otherwise.  So elu_fast is within this ABSOLUTE floor of
# ELU(v) for every fp32 v (v > 0 passes through).
ELU_FLOOR = 2.0 ** -22 + 2.0 ** -25


@dataclasses.dataclass(frozen=True)
class Layer:
    """one contraction gemm_tc issues: its shape, epilogue and outputs"""
    name: str
    cin: int
    taps: int
    N: int
    bias_mod: int  # 0: no bias
    epi: int
    f32: bool  # writes the fp32 output
    bf16: bool  # writes the bf16 output
    elu: bool  # the bf16 output goes through ELU
    inplace: bool = False  # R is the fp32 output (the transformer's residual stream)
    h_ctx: int = 0  # elements a stream keeps in front of the bf16 output (its consumer's context rows)

    @property
    def K(self):
        return self.taps * self.cin


# Every gemm_tc call of the decoder, at Mimi's geometry (hidden 512, FFN 2048, 64 filters, ratios 8 6 5 4, conv0 k7,
# ResnetBlock k3 with compress 2; stage 0's block (hidden 256) is too wide for the fused kernel and runs as two GEMMs):
#   run_layers' `lin`            qkv, out_proj (in place on x), fc1 (bf16 hidden), fc2 (in place on x)
#   seanet_tc conv0              conv0: bf16 ELU'd a0, behind a0's context row in a stream
#   seanet_tc ConvTranspose      convT_r*: fp32 zf and bf16 ELU(z) behind z's two context rows, one launch
#   seanet_tc unfused block      res0_k3 (bf16 ELU'd h), res0_k1 (EPI_RES on zf at z's pitch, bf16 ELU'd o at o's pitch)
PRODUCTION = [
    Layer("qkv", 512, 1, 1536, 0, EPI_NONE, True, False, False),
    Layer("out_proj", 512, 1, 512, 0, EPI_RES_SCALE, True, False, False, inplace=True),
    Layer("fc1", 512, 1, 2048, 0, EPI_GELU, False, True, False),
    Layer("fc2", 2048, 1, 512, 0, EPI_RES_SCALE, True, False, False, inplace=True),
    Layer("conv0", 512, 7, 1024, 1024, EPI_NONE, False, True, True, h_ctx=1024),
    Layer("convT_r8", 1024, 2, 8 * 512, 512, EPI_NONE, True, True, True, h_ctx=2 * 512),
    Layer("convT_r6", 512, 2, 6 * 256, 256, EPI_NONE, True, True, True, h_ctx=2 * 256),
    Layer("convT_r5", 256, 2, 5 * 128, 128, EPI_NONE, True, True, True, h_ctx=2 * 128),
    Layer("convT_r4", 128, 2, 4 * 64, 64, EPI_NONE, True, True, True, h_ctx=2 * 64),
    Layer("res0_k3", 512, 3, 256, 256, EPI_NONE, False, True, True),
    Layer("res0_k1", 256, 1, 512, 512, EPI_RES, False, True, True, h_ctx=512),
]

# The tile instantiations production does not reach and the edges of the stage ring (tc::launch_bn: BN = 128 takes up
# to 3 stages, narrower tiles 4; nk = K / BK <= 4 chunks take 2).  name: BK x BN, nk.
TILES = [
    Layer("bk64_bn32_nk3", 64, 3, 32, 32, EPI_NONE, True, True, False),
    Layer("bk64_bn64_nk1", 64, 1, 192, 64, EPI_RES, True, True, True),
    Layer("bk64_bn128_nk2", 128, 1, 256, 256, EPI_RES_SCALE, True, True, False),
    Layer("bk64_bn128_nk4", 64, 4, 128, 128, EPI_NONE, True, True, True),
    Layer("bk64_bn64_nk4", 256, 1, 64, 0, EPI_GELU, True, True, False),
    Layer("bk64_bn128_nk5", 64, 5, 128, 128, EPI_RES, True, True, True),
    Layer("bk64_bn32_nk5", 320, 1, 96, 96, EPI_NONE, True, True, True),
    Layer("bk64_bn128_nk9_3ch", 192, 3, 384, 128, EPI_NONE, True, True, True),
    Layer("bk64_bn128_longk", 1024, 4, 256, 256, EPI_RES_SCALE, True, True, False, inplace=True),
    Layer("bk32_bn128_nk3", 32, 3, 128, 0, EPI_NONE, True, True, False),
    Layer("bk32_bn64_nk1", 32, 1, 64, 64, EPI_RES, True, True, True),
    Layer("bk32_bn32_nk2", 32, 2, 32, 32, EPI_RES_SCALE, True, True, False),
    Layer("bk32_bn64_nk21", 96, 7, 64, 64, EPI_NONE, True, True, True),
]


@dataclasses.dataclass(frozen=True)
class Launch:
    layer: Layer
    B: int
    M: int
    ctx: int
    a_pitch: int
    c_pitch: int
    r_pitch: int  # 0 without a residual
    h_off: int

    def __getattr__(self, k):  # the layer's fields
        return getattr(self.__dict__["layer"], k)


def launch(layer, B, M, ctx, pitched, h_off=None):
    """the packed geometry (items back to back, as the one-shot decode lays them out) or a pitched one (as a stream
    does): the operand, output and residual each at its own pitch, the bf16 output behind the layer's context rows"""
    res = layer.epi in (EPI_RES, EPI_RES_SCALE)
    if pitched:
        a_pitch, c_pitch, r_pitch = ctx + M + 3, M + 5, M + 2
        h = layer.h_ctx if h_off is None else h_off
    else:
        a_pitch, c_pitch, r_pitch, h = ctx + M, M, M, 0 if h_off is None else h_off
    if layer.inplace:
        r_pitch = c_pitch
    return Launch(layer, B, M, ctx, a_pitch, c_pitch, r_pitch if res else 0, h)


def launches(layer):
    """the sweep of one layer: M in {1, 127, 128, 129, 383} plus a multi-tile M, every ctx in [0, taps-1], B in
    {1, 3, 64}, packed and pitched"""
    geo = [(1, 1), (3, 127), (1, 128), (3, 129), (1, 383), (3, 2053), (64, 12), (64, 1)]
    out = []
    for i, (B, M) in enumerate(geo):
        ctx = i % layer.taps if B < 64 else layer.taps - 1
        out.append(launch(layer, B, M, ctx, pitched=i % 2 == 1))
    assert {L.ctx for L in out} == set(range(layer.taps))
    return out


# ---------------------------------------------------------------------------------------------------------------
# operands
# ---------------------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class Operands:
    X: torch.Tensor  # bf16 [B][a_pitch][cin], rows [ctx + M, a_pitch) NaN
    W: torch.Tensor  # bf16 [N][K]
    bias: torch.Tensor  # fp32 [bias_mod] or None
    R: torch.Tensor  # fp32 [B][r_pitch][N] (rows [M, r_pitch) the sentinel) or None
    scale: torch.Tensor  # fp32 [N] or None


def signed_ints(gen, shape, hi, device, dtype=torch.int32):
    """integers +-k, k uniform in 1..hi"""
    k = torch.randint(1, hi + 1, shape, generator=gen, device=device, dtype=dtype)
    k *= torch.randint(0, 2, shape, generator=gen, device=device, dtype=dtype) * 2 - 1
    return k


def _signed(gen, shape, hi, device):
    return signed_ints(gen, shape, hi, device).double()


def dyadic_values(gen, L, device):
    """X, W, bias, R, scale values on grids that make every sum and epilogue of the launch exact in fp32 (nonzero, so
    every dropped or doubled product changes an output):
      x = +-k/16 and w = +-k/256, k in 1..16: each product is a multiple of 2^-12 of magnitude <= 2^-4, so with
        K <= 4096 every partial sum, in any order, is a multiple of 2^-12 of magnitude <= 2^8: at most 21 bits;
      bias = +-k/64, k in 1..64 (|bias| <= 1): the biased sum stays a multiple of 2^-12 below 2^9 (21 bits);
      R = +-k/4096, k in 1..2^18 (|R| <= 64): RES's sum stays a multiple of 2^-12 below 2^9 (21 bits);
      scale = +-k/4, k in 1..4: scale * v is a multiple of 2^-14 of magnitude <= 2^8 + 1, and fmaf(scale, v, R) a
        multiple of 2^-14 below 2^9: at most 23 bits.
    So every fp32 value the kernel forms equals the float64 value, and its bf16 output is RNE of it."""
    assert L.K <= 4096
    B, N = L.B, L.N
    x = _signed(gen, (B, L.ctx + L.M, L.cin), 16, device) / 16
    w = _signed(gen, (N, L.K), 16, device) / 256
    bias = _signed(gen, (L.bias_mod,), 64, device) / 64 if L.bias_mod else None
    r = _signed(gen, (B, L.M, N), 2 ** 18, device) / 4096 if L.r_pitch else None
    scale = _signed(gen, (N,), 4, device) / 4 if L.epi == EPI_RES_SCALE else None
    return x, w, bias, r, scale


def random_values(gen, L, device):
    """unit-sized activations, weights scaled by 1/sqrt(K) as trained layers are, a bias and a residual of the
    activations' size and a LayerScale of mixed sign"""
    B, N = L.B, L.N
    x = torch.randn(B, L.ctx + L.M, L.cin, generator=gen, device=device, dtype=torch.float64)
    w = torch.randn(N, L.K, generator=gen, device=device, dtype=torch.float64) / L.K ** 0.5
    bias = torch.randn(L.bias_mod, generator=gen, device=device, dtype=torch.float64) * 0.3 if L.bias_mod else None
    r = torch.randn(B, L.M, N, generator=gen, device=device, dtype=torch.float64) if L.r_pitch else None
    scale = torch.randn(N, generator=gen, device=device, dtype=torch.float64) * 0.5 if L.epi == EPI_RES_SCALE else None
    return x, w, bias, r, scale


def f32_sentinel(n, device):
    return torch.full((n,), F32_SENTINEL, dtype=torch.int32, device=device).view(torch.float32)


def bf16_sentinel(n, device):
    return torch.full((n,), BF16_SENTINEL, dtype=torch.int16, device=device).view(BF16)


def pitched_rows(v, pitch, fill):
    """[B][rows][C] -> [B][pitch][C] with rows [rows, pitch) = fill (a float, or a sentinel buffer's element)"""
    B, rows, Cc = v.shape
    if isinstance(fill, torch.Tensor):
        out = fill.reshape(1, 1, 1).expand(B, pitch, Cc).clone()
    else:
        out = torch.full((B, pitch, Cc), fill, dtype=v.dtype, device=v.device)
    out[:, :rows] = v
    return out


def operands(L, kind, seed, device):
    """the launch's operands in their buffers: X rows past ctx + M of each item NaN (a launch must not read them),
    R rows past M the fp32 sentinel"""
    gen = torch.Generator(device=device).manual_seed(seed)
    x, w, bias, r, scale = (dyadic_values if kind == "dyadic" else random_values)(gen, L, device)
    X = pitched_rows(x.to(BF16), L.a_pitch, float("nan"))
    Rb = pitched_rows(r.float(), L.r_pitch, f32_sentinel(1, device)) if r is not None else None
    return Operands(X, w.to(BF16).contiguous(), None if bias is None else bias.float(), Rb, None if scale is None else scale.float())


# ---------------------------------------------------------------------------------------------------------------
# float64 reference
# ---------------------------------------------------------------------------------------------------------------
def reference(L, ops):
    """float64 (y, a, mag) [B][M][N] of the launch on the operand values: y the epilogue's result, a the biased sum it
    starts from, mag = sum |x w| + |bias| (the size of the sum's roundings).  Built on mimi_f32_refs.gemm_ref over the
    rows of each item the launch may read."""
    Xi = ops.X[:, : L.ctx + L.M]
    a, mag = R_.gemm_ref(Xi, ops.W, L.M, L.ctx + L.M, L.taps, 1, L.taps - 1 - L.ctx, bias=ops.bias, bias_mod=L.bias_mod or None)
    if ops.bias is not None:
        mag = mag + ops.bias.double().abs()[torch.arange(L.N, device=a.device) % L.bias_mod]
    if L.epi == EPI_GELU:
        y = 0.5 * a * (1 + torch.erf(a / 2 ** 0.5))
    elif L.epi == EPI_RES:
        y = ops.R[:, : L.M].double() + a
    elif L.epi == EPI_RES_SCALE:
        y = ops.R[:, : L.M].double() + ops.scale.double() * a
    else:
        y = a
    return y, a, mag


def bound(L, y, a, mag, ops, exact_sum=False):
    """per-element bound on |fp32 result - y| for random operands.  Products of bf16 values are exact in fp32; wgmma's
    accumulation order is undocumented, so each of the K - 1 additions (and the bias's) may round by up to 2u of the
    sum of magnitudes: 2u K mag.  GELU (|gelu'| <= 1.13) carries that and adds its own roundings (erff within 2 ulp,
    the products and 1 + erf: 8u |a|); RES adds one rounding of the result, RES_SCALE scales the sum's error by
    |scale| and rounds once (fmaf).  exact_sum: the sum is exact (dyadic operands), only GELU's roundings remain."""
    e = torch.zeros_like(mag) if exact_sum else 2 * U * L.K * mag
    if L.epi == EPI_GELU:
        return 1.13 * e + 8 * U * a.abs()
    if L.epi == EPI_RES:
        return e + U * y.abs()
    if L.epi == EPI_RES_SCALE:
        return ops.scale.double().abs() * e + U * y.abs()
    return e


def bf16_ulp(x):
    """spacing of bf16 values at |x| (float64; the subnormal spacing near 0)"""
    x = x.double().abs()
    _, e = torch.frexp(x)
    return torch.where(x == 0, torch.full_like(x, 2.0 ** -133), torch.ldexp(torch.ones_like(x), (e - 8).clamp(min=-133)))


# ---------------------------------------------------------------------------------------------------------------
# checks
# ---------------------------------------------------------------------------------------------------------------
def _first(mask, n=4):
    return mask.nonzero()[:n].tolist()


def check_values(L, f32, bf, y, err=None, what=""):
    """The written values of a launch: f32 / bf ([..., N] fp32 / bf16, or None when the layer writes no such output)
    against the float64 y.  err None: the operands are dyadic, so the fp32 result equals y exactly and the plain bf16
    result is RNE(y); the ELU'd bf16 result is within half a bf16 ulp of ELU(y) plus ELU_FLOOR.  Otherwise per element:
    fp32 within err, bf16 within err plus half an ulp, ELU'd bf16 within err + ELU_FLOOR plus half an ulp.  Returns the
    worst |got - want| / tolerance of each output checked against a tolerance: {"fp32": .., "bf16": ..}."""
    worst = {}
    y = y.double()
    if err is None:
        assert torch.equal(y.float().double(), y), f"{what}: the reference is not exact in fp32 (operands off their grids)"
    e = torch.zeros_like(y) if err is None else err.double()
    if L.f32:
        assert f32 is not None
        g = f32.double()
        if err is None:
            bad = g != y
        else:
            d = (g - y).abs()
            bad = ~(d <= e)
            worst["fp32"] = float((d / e.clamp(min=1e-300)).max())
        assert not bool(bad.any()), f"{what} fp32: {int(bad.sum())} of {bad.numel()} differ, first {_first(bad)}"
    if L.bf16:
        assert bf is not None
        g = bf.double()
        if L.elu:
            want = torch.nn.functional.elu(y)
            tol = e + ELU_FLOOR + bf16_ulp(want.abs() + e + ELU_FLOOR) / 2
        elif err is None:
            want, tol = y.float().to(BF16).double(), None
        else:
            want = y
            tol = e + bf16_ulp(y.abs() + e) / 2
        if tol is None:
            bad = g != want
        else:
            d = (g - want).abs()
            bad = ~(d <= tol)
            worst["bf16"] = float((d / tol).max())
        kind = "bf16(ELU)" if L.elu else "bf16"
        assert not bool(bad.any()), f"{what} {kind}: {int(bad.sum())} of {bad.numel()} differ, first {_first(bad)}"
    return worst


def f32_rows(L, buf):
    """the fp32 output buffer (B items of c_pitch rows, then anything) -> [B][c_pitch][N]"""
    return buf[: L.B * L.c_pitch * L.N].view(L.B, L.c_pitch, L.N)


def bf16_rows(L, buf):
    """the bf16 output buffer (h_off elements, then B items of c_pitch rows) -> ([B][c_pitch][N], the h_off front)"""
    return buf[L.h_off: L.h_off + L.B * L.c_pitch * L.N].view(L.B, L.c_pitch, L.N), buf[: L.h_off]


def check_guards(L, f32_buf, bf_buf, what=""):
    """every element of the output buffers outside rows [0, M) of an item still holds its sentinel: rows [M, c_pitch)
    of each item, the h_off elements in front of the bf16 output and anything past the last item"""
    if f32_buf is not None:
        bits = f32_buf.view(torch.int32)
        rows = bits[: L.B * L.c_pitch * L.N].view(L.B, L.c_pitch, L.N)
        bad = rows[:, L.M:] != F32_SENTINEL
        assert not bool(bad.any()), f"{what} fp32: {int(bad.sum())} guard elements written past row M, first {_first(bad)}"
        tail = bits[L.B * L.c_pitch * L.N:] != F32_SENTINEL
        assert not bool(tail.any()), f"{what} fp32: written past the last item"
    if bf_buf is not None:
        bits = bf_buf.view(torch.int16)
        rows, front = bf16_rows(L, bits)
        assert bool((front == BF16_SENTINEL).all()), f"{what} bf16: the {L.h_off} context elements in front were written"
        bad = rows[:, L.M:] != BF16_SENTINEL
        assert not bool(bad.any()), f"{what} bf16: {int(bad.sum())} guard elements written past row M, first {_first(bad)}"
        tail = bits[L.h_off + L.B * L.c_pitch * L.N:] != BF16_SENTINEL
        assert not bool(tail.any()), f"{what} bf16: written past the last item"


def check_launch(L, f32_buf, bf_buf, y, err=None, what=""):
    """check_guards, then check_values on rows [0, M) of every item; returns check_values' worst ratios"""
    check_guards(L, f32_buf if L.f32 else None, bf_buf if L.bf16 else None, what)
    f = f32_rows(L, f32_buf)[:, : L.M] if L.f32 else None
    b = bf16_rows(L, bf_buf)[0][:, : L.M] if L.bf16 else None
    return check_values(L, f, b, y, err, what)


def seq_sums_match(products, rng, orders=4):
    """True when fp32 sums of `products` [n][K] (fp32-exact values) in `orders` random orders all equal the float64
    sums"""
    p = np.asarray(products, dtype=np.float64)
    want = p.sum(axis=1)
    for _ in range(orders):
        perm = rng.permutation(p.shape[1])
        got = R_.seq_sum_f32(p[:, perm].astype(np.float32), axis=1).astype(np.float64)
        if not np.array_equal(got, want):
            return False
    return True
