"""Mimi's fp32 kernels one at a time against float64 references on the same fp32 operands.

Every decode and stream runs the RVQ gather, the fp32 implicit GEMM (the RVQ projection), the upsampler and the
LayerNorm; the tensor-core stream runs RoPE and the fp32 attention over its K/V rings; the encoder (voice ingestion) is
fp32 throughout and ends in the codeword search.  End to end these are held to waveform or latent bounds that a kernel
bug of the size of one key or one row can hide under.  Here each kernel goes through its test hook (include/sopro_b200.h),
launched as the codec launches it, and is held to a bound derived from its arithmetic (u = 2^-24, gamma_n = n u /
(1 - n u); CUDA Programming Guide maximum errors without fast-math: expm1f 1 ulp, expf 2 ulp, erff 2 ulp, sqrtf and
division correctly rounded), or bit-exact where the operands make every rounding exact.  Each test prints its worst
error-to-bound ratio.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from tests.mimi_f32_refs import U, gamma, gemm_ref, rope64, rope_table, seq_sum_f32, window_attention

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
DEV = torch.device("cuda:0")
ULP1 = 2.0 ** -23  # one ulp relative to the value, an upper bound for a 1-ulp function error


def _lib():
    from sopro_b200 import _lib

    return _lib, _lib.load()


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ratio(err, bound):
    err, bound = err.double(), bound.double()
    r = torch.where(bound > 0, err / bound.clamp(min=1e-300), torch.where(err > 0, float("inf"), 0.0))
    return float(r.max())


# ---------------------------------------------------------------------------------------------------------------
# implicit GEMM
# ---------------------------------------------------------------------------------------------------------------
EPI_NONE, EPI_GELU, EPI_RES_SCALE, EPI_RES = 0, 1, 2, 3

# (name, cin, taps, N, bias_mod or None, epi, elu): every geometry the fp32 codec issues
GEMM_GEOMS = [
    ("rvq projection", 512, 1, 512, None, EPI_NONE, 0),
    ("qkv", 512, 1, 1536, None, EPI_NONE, 0),
    ("out-proj", 512, 1, 512, None, EPI_RES_SCALE, 0),
    ("fc1", 512, 1, 2048, None, EPI_GELU, 0),
    ("fc2", 2048, 1, 512, None, EPI_RES_SCALE, 0),
    ("conv0", 512, 7, 1024, 1024, EPI_NONE, 0),
    ("convT r=8", 1024, 2, 8 * 512, 512, EPI_NONE, 1),
    ("convT r=6", 512, 2, 6 * 256, 256, EPI_NONE, 1),
    ("convT r=5", 256, 2, 5 * 128, 128, EPI_NONE, 1),
    ("convT r=4", 128, 2, 4 * 64, 64, EPI_NONE, 1),
    ("dec res k3 512", 512, 3, 256, 256, EPI_NONE, 1),
    ("dec res k3 256", 256, 3, 128, 128, EPI_NONE, 1),
    ("dec res k3 128", 128, 3, 64, 64, EPI_NONE, 1),
    ("dec res k3 64 (32-col tile)", 64, 3, 32, 32, EPI_NONE, 1),
    ("dec res k1 256", 256, 1, 512, 512, EPI_RES, 1),
    ("dec res k1 32", 32, 1, 64, 64, EPI_RES, 1),
    ("enc strided r=4", 4 * 64, 2, 128, 128, EPI_NONE, 1),
    ("enc strided r=5", 5 * 128, 2, 256, 256, EPI_NONE, 1),
    ("enc strided r=6", 6 * 256, 2, 512, 512, EPI_NONE, 1),
    ("enc strided r=8", 8 * 512, 2, 1024, 1024, EPI_NONE, 1),
    ("enc last conv", 1024, 3, 512, 512, EPI_NONE, 1),
    ("enc downsample", 1024, 2, 512, None, EPI_NONE, 0),
    ("enc input projections", 512, 1, 512, None, EPI_NONE, 0),
    ("enc res k3 64 (32-col tile)", 64, 3, 32, 32, EPI_NONE, 1),
]
M_EDGES = [1, 63, 64, 65, 1100]


def _gemm_case(i):
    """geometry i with an M of the edge list, a context of 0..taps-1 rows, B = 3 on every other case"""
    name, cin, taps, N, bias_mod, epi, elu = GEMM_GEOMS[i]
    M = M_EDGES[i % len(M_EDGES)]
    ctx = i % taps
    B = 3 if i % 2 == 0 else 1
    return name, cin, taps, N, bias_mod, epi, elu, M, ctx, B


def _run_gemm(X, W, bias, bias_mod, R, scale, M, ctx, taps, N, epi, elu, B, a_pitch, c_pitch, r_pitch, ldc):
    """X [B][a_pitch][cin] (rows [0, M + ctx) read), out [B][c_pitch][ldc] NaN-filled, R [B][r_pitch][N]"""
    lib_mod, lib = _lib()
    cin = X.shape[-1]
    out = torch.full((B, c_pitch, ldc), float("nan"), device=DEV)
    lib_mod.check(lib.sopro_debug_mimi_gemm(_p(X), _p(W), _p(bias), _p(R), _p(scale), _p(out), B, M, N, taps * cin, M + ctx, cin, taps, 1,
                                            taps - 1 - ctx, ldc, bias_mod or N, epi, elu, a_pitch * cin, c_pitch * ldc, r_pitch * N, _st()))
    torch.cuda.synchronize()
    return out


def _gemm_operands(cin, taps, N, M, ctx, B, g, dyadic, elu):
    a_pitch, c_pitch, r_pitch = M + ctx + 3, M + 2, M + 5
    if dyadic:  # a, w on a 2^-6 grid with |.| <= 1/4 (a >= 0 under ELU, where ELU is the identity), bias on 2^-12:
        # every partial sum is a multiple of 2^-12 below 2^9 (K <= 8192), 21 significant bits, exact in fp32
        lo = 0 if elu else -16
        X = torch.randint(lo, 17, (B, a_pitch, cin), generator=g).float() / 64
        W = torch.randint(-16, 17, (N, taps * cin), generator=g).float() / 64
        bias = torch.randint(-64, 65, (N,), generator=g).float() / 4096
        R = torch.randint(-64, 65, (B, r_pitch, N), generator=g).float() / 64
    else:
        X = torch.randn(B, a_pitch, cin, generator=g)
        W = torch.randn(N, taps * cin, generator=g) / math.sqrt(taps * cin)
        bias = torch.randn(N, generator=g) * 0.1
        R = torch.randn(B, r_pitch, N, generator=g)
    scale = 0.3 + 0.1 * torch.randn(N, generator=g)
    return X, W, bias, R, scale, a_pitch, c_pitch, r_pitch


def _gemm_bound(v64, mag, K, epi, R64, scale64):
    """per output: the fma chain over K (gamma_K sum|a'w|), the ELU on load (expm1f <= 1 ulp: 2^-23 |elu(a)| per
    operand, so 2^-23 sum|elu(a) w|), then the epilogue's roundings propagated through it:
      bias add: u (|v| + E);  GELU 0.5 x (1 + erff(x c)): its slope |GELU'| <= 1.13 times the input error, plus x c off
      by 2u |x c| (c = fp32(1/sqrt 2) and the product's rounding; erff' <= 2/sqrt(pi)), erff's 2 ulp, the sum 1 + erf
      and the product (u each), 0.5 exact;  R + scale v (fused or not): |scale| E + u |scale v| + u |out|;  R + v: E + u |out|.
    Returns (reference value, bound)."""
    E = (gamma(K) * (1 + ULP1) + ULP1) * mag
    E = E + U * (v64.abs() + E)
    if epi == EPI_GELU:
        x = v64
        erf = torch.erf(x / math.sqrt(2))
        out = 0.5 * x * (1 + erf)
        ev = 0.5 * x.abs() * (2 * ULP1 * erf.abs() + 2 / math.sqrt(math.pi) * 2 * U * (x / math.sqrt(2)).abs() + 2 * U * (1 + erf.abs()))
        return out, 1.13 * E + ev + U * out.abs()
    if epi == EPI_RES_SCALE:
        out = R64 + scale64 * v64
        return out, scale64.abs() * E + U * (scale64 * v64).abs() + U * out.abs()
    if epi == EPI_RES:
        out = R64 + v64
        return out, E + U * out.abs()
    return v64, E


def _check_gemm(i, dyadic):
    name, cin, taps, N, bias_mod, epi, elu, M, ctx, B = _gemm_case(i)
    if dyadic and epi in (EPI_GELU, EPI_RES_SCALE):
        epi = EPI_NONE  # GELU and the LayerScale multiply are not exact: their arithmetic is held to the random bound
    g = torch.Generator().manual_seed(1000 * i + dyadic)
    X, W, bias, R, scale, a_pitch, c_pitch, r_pitch = _gemm_operands(cin, taps, N, M, ctx, B, g, dyadic, elu)
    ldc = N + (8 if i % 3 == 0 else 0)
    d = {k: t.to(DEV) for k, t in dict(X=X, W=W, bias=bias, R=R, scale=scale).items()}
    use_bias = bias_mod is not None
    out = _run_gemm(d["X"], d["W"], d["bias"] if use_bias else None, bias_mod, d["R"], d["scale"], M, ctx, taps, N, epi, elu, B, a_pitch,
                    c_pitch, r_pitch, ldc)
    got = out[:, :M, :N]
    assert bool(torch.isnan(out[:, M:]).all()) and bool(torch.isnan(out[:, :, N:]).all()), f"{name}: wrote outside [M, N]"
    v64, mag = gemm_ref(d["X"], d["W"], M, M + ctx, taps, 1, taps - 1 - ctx, d["bias"] if use_bias else None, bias_mod, bool(elu))
    want, bound = _gemm_bound(v64, mag, taps * cin, epi, d["R"][:, :M].double(), d["scale"].double())
    if dyadic:
        bad = int((got.double() != want).sum())
        print(f"igemm {name} dyadic M={M} ctx={ctx} B={B} ldc={ldc}: {bad} outputs differ from the exact sum")
        assert bad == 0, name
        return
    err = (got.double() - want).abs()
    r = _ratio(err, bound)
    print(f"igemm {name} M={M} ctx={ctx} B={B} ldc={ldc} epi={epi}: max |err| {float(err.max()):.2e}, worst err / bound {r:.3f}")
    assert r <= 1.0, name


@pytest.mark.parametrize("i", range(len(GEMM_GEOMS)))
def test_igemm_production_geometries(i):
    """Every fp32 GEMM geometry of the decoder and the encoder, bit-exact on dyadic operands and within the derived
    bound on random ones; context rows, operand / output / residual pitches larger than their rows, ldc > N, B = 3.
    Rows past M and columns past N of the output stay untouched."""
    _check_gemm(i, dyadic=True)
    _check_gemm(i, dyadic=False)


@pytest.mark.parametrize("M", M_EDGES)
def test_igemm_row_edges(M):
    """M around the 64-row tile with both column tiles (N = 32 and N = 512) and every context of a k = 3 conv."""
    for ctx in range(3):
        for N in (32, 512):
            g = torch.Generator().manual_seed(M * 10 + ctx + N)
            B, cin, taps = 3, 64, 3
            X, W, bias, R, _, a_pitch, c_pitch, r_pitch = _gemm_operands(cin, taps, N, M, ctx, B, g, True, True)
            d = [t.to(DEV) for t in (X, W, bias, R)]
            out = _run_gemm(d[0], d[1], d[2], N, d[3], None, M, ctx, taps, N, EPI_RES, 1, B, a_pitch, c_pitch, r_pitch, N)
            v64, _ = gemm_ref(d[0], d[1], M, M + ctx, taps, 1, taps - 1 - ctx, d[2], N, True)
            want = v64 + d[3][:, :M].double()
            assert torch.equal(out[:, :M].double(), want), (M, ctx, N)
            assert bool(torch.isnan(out[:, M:]).all())


def test_igemm_refuses_unsupported_shapes():
    lib_mod, lib = _lib()
    X = torch.zeros(1, 64, 64, device=DEV)
    W = torch.zeros(64, 192, device=DEV)
    out = torch.full((1, 64, 64), 7.0, device=DEV)
    base = dict(B=1, M=8, N=64, K=192, Min=8, Cin=64, taps=3, pad=2, ldc=64, epi=0, a_bs=0)
    for k, v in (("K", 190), ("Cin", 62), ("Min", 7), ("ldc", 63), ("epi", 2), ("epi", 3), ("B", 0), ("M", 0), ("a_bs", 6)):
        a = dict(base, **{k: v})
        if k == "Cin":
            a["K"] = 3 * v
        rc = lib.sopro_debug_mimi_gemm(_p(X), _p(W), None, None, None, _p(out), a["B"], a["M"], a["N"], a["K"], a["Min"], a["Cin"], a["taps"],
                                       1, a["pad"], a["ldc"], 64, a["epi"], 0, a["a_bs"], 0, 0, _st())
        assert rc != 0, (k, v)
    torch.cuda.synchronize()
    assert bool((out == 7.0).all())


# ---------------------------------------------------------------------------------------------------------------
# codeword search
# ---------------------------------------------------------------------------------------------------------------
DC = 256


def _rvq_encode(proj, embed, n_sem, frames=None, fill=-7):
    """proj [B][T][512] fp32, embed [n_q][V][256] -> codes [B][n_q][T] (pre-filled with `fill`)"""
    lib_mod, lib = _lib()
    B, T, _ = proj.shape
    n_q, V, _ = embed.shape
    p, e = proj.to(DEV).contiguous(), embed.to(DEV).contiguous()
    codes = torch.full((B, n_q, T), fill, dtype=torch.int32, device=DEV)
    fr = torch.tensor(frames, dtype=torch.int32, device=DEV) if frames is not None else None
    lib_mod.check(lib.sopro_debug_mimi_rvq_encode(_p(p), _p(e), _p(codes), T, n_q, n_sem, V, _p(fr), B, _st()))
    torch.cuda.synchronize()
    return codes.cpu()


def _synth_codebooks():
    from sopro_b200.codec import _codebooks
    from sopro_b200.weights import synth_mimi_state_dict

    return _codebooks(synth_mimi_state_dict(), 32)  # [32][2048][256] fp32, as the encoder uploads them


def test_codeword_search_random_latents():
    """Random projections through the synthetic codebooks (n_q 32, n_sem 1).  The residual chain is replayed in fp32
    from the GPU's own codes (exact: each step is one subtraction, as in the kernel).  Each distance the kernel forms
    (a rounded difference per channel, an fma chain of 8 per lane, a 5-level shuffle tree) is within gamma_15 d of the
    float64 distance d of the same fp32 residual, all terms being non-negative.  So at every codebook the GPU's pick
    is within gamma_15 (d_pick + d_min) of the float64 minimum, and equals the float64 argmin wherever the float64
    margin to the runner-up exceeds gamma_15 (d_1 + d_2)."""
    E = _synth_codebooks()
    E64 = E.double().to(DEV)
    g = torch.Generator().manual_seed(11)
    B, T = 2, 150
    proj = torch.randn(B, T, 2 * DC, generator=g) * 0.8
    codes = _rvq_encode(proj, E, 1)
    assert bool(((codes >= 0) & (codes < 2048)).all())
    tol = gamma(15)
    worst, ties, checked = 0.0, 0, 0
    for half, qs in ((0, range(0, 1)), (1, range(1, 32))):
        r = proj[:, :, half * DC:(half + 1) * DC].clone().to(DEV)  # fp32 residual [B][T][256]
        for q in qs:
            d = torch.cdist(r.double().reshape(-1, DC), E64[q], compute_mode="donot_use_mm_for_euclid_dist") ** 2  # [B*T][V]
            top, arg = d.topk(2, dim=1, largest=False)
            c = codes[:, q].reshape(-1).to(DEV).long()
            dg = d.gather(1, c[:, None])[:, 0]
            slack = tol * (dg + top[:, 0])
            worst = max(worst, _ratio(dg - top[:, 0], slack))
            clear = (top[:, 1] - top[:, 0]) > tol * (top[:, 0] + top[:, 1])
            assert bool((c[clear] == arg[clear, 0]).all()), f"codebook {q}: a pick differs from a clear float64 argmin"
            ties += int((~clear).sum())
            checked += int(c.numel())
            r = (r.reshape(-1, DC) - E[q].to(DEV)[c]).reshape(B, T, DC)  # the kernel's fp32 subtraction
    print(f"codeword search: {checked} picks, {ties} near ties, worst (d_pick - d_min) / bound {worst:.3f}")
    assert worst <= 1.0


@pytest.mark.parametrize("V", [2048, 13, 5, 1])
def test_codeword_search_exact_ties(V):
    """Small-integer residuals and codebooks make every distance exact in fp32, so the float64 argmin with the lowest
    index first is the only right answer.  V = 2048: frame t's semantic residual is a codeword held at indices a, a + 3
    and a + 8 (a + 8 in the same warp, a + 3 in another, with a = 5 mod 8 making a + 3 the higher index in the lower
    warp); the acoustic residual is 0 and each acoustic codebook holds the zero vector at indices in one warp and in
    others.  V = 13, 5, 1: codewords repeat every 3 indices (V = 5 leaves three warps without a codeword)."""
    g = torch.Generator().manual_seed(V)
    B, T, n_q = 1, 24, 4
    E = torch.randint(-3, 4, (n_q, V, DC), generator=g).float()
    proj = torch.zeros(B, T, 2 * DC)
    if V >= 64:
        for t in range(T):
            a = 32 * t + (t % 8)
            E[0, [a + 3, a + 8]] = E[0, a].clone()
            proj[0, t, :DC] = E[0, a]
        for q in range(1, n_q):
            E[q, [40 + q, 48 + q, 41 + q, 1000]] = 0
    else:
        for q in range(n_q):
            E[q] = E[q, torch.arange(V) % 3]
        proj[0, :, :DC] = E[0, torch.arange(T) % V]
        proj[0, :, DC:] = E[1, (torch.arange(T) + 1) % V]
    ref = torch.zeros(B, n_q, T, dtype=torch.int32)
    ties = 0
    for h, qs in ((0, [0]), (1, list(range(1, n_q)))):
        r = proj[0, :, h * DC:(h + 1) * DC].double()
        for q in qs:
            d = ((r[:, None, :] - E[q].double()[None]) ** 2).sum(-1)  # [T][V], exact integers
            at_min = d == d.min(dim=1, keepdim=True).values
            ties += int((at_min.sum(1) > 1).sum())
            idx = torch.where(at_min, torch.arange(V)[None].expand_as(d), V).min(dim=1).values
            ref[0, q] = idx.int()
            r = r - E[q].double()[idx]
    got = _rvq_encode(proj, E, 1)
    print(f"codeword search ties V={V}: {ties} of {n_q * T} picks among tied minima")
    assert V == 1 or ties >= T
    assert torch.equal(got, ref), (V, (got != ref).nonzero()[:5].tolist())


def test_codeword_search_ragged_batch():
    """Frames at or past a clip's own length are left untouched (pre-filled with a sentinel); the others equal the
    single-clip search of the same projections."""
    E = _synth_codebooks()[:6]
    g = torch.Generator().manual_seed(12)
    B, T = 4, 40
    proj = torch.randn(B, T, 2 * DC, generator=g) * 0.8
    frames = [40, 1, 17, 39]
    got = _rvq_encode(proj, E, 1, frames=frames, fill=-7)
    for b, n in enumerate(frames):
        assert bool((got[b, :, n:] == -7).all()), b
        alone = _rvq_encode(proj[b:b + 1, :n], E, 1)
        assert torch.equal(got[b, :, :n], alone[0]), b


def test_codeword_search_non_finite_rows():
    """A NaN, +Inf, -Inf or overflowing (1e30: every squared distance is +Inf) frame gives oracle.rvq_encode's codes,
    0 at every codebook; every code is in [0, V) and the neighbouring frames equal a run without the bad frames."""
    from oracle import mimi_oracle as Mo

    sd = Mo.synth_mimi_state_dict()
    E = _synth_codebooks()[:8]
    g = torch.Generator().manual_seed(13)
    T = 9
    emb = torch.randn(1, T, 512, generator=g) * 0.3
    bad = {1: float("nan"), 3: float("inf"), 5: -float("inf"), 7: 1e30}
    for t, v in bad.items():
        emb[0, t] = v
    proj = torch.cat([torch.nn.functional.linear(emb, sd[f"quantizer.{grp}_residual_vector_quantizer.input_proj.weight"].squeeze(-1))
                      for grp in ("semantic", "acoustic")], dim=-1)
    want = Mo.rvq_encode(sd, emb, n_q=8).int()
    got = _rvq_encode(proj, E, 1)
    assert bool(((got >= 0) & (got < 2048)).all())
    rows = sorted(bad)
    assert bool((got[0, :, rows] == 0).all()) and torch.equal(got[0, :, rows], want[0, :, rows])
    good = [t for t in range(T) if t not in bad]
    clean = _rvq_encode(proj[:, good], E, 1)
    assert torch.equal(got[0, :, good], clean[0])


def test_codeword_search_refuses_unsupported_shapes():
    _, lib = _lib()
    proj = torch.zeros(1, 4, 512, device=DEV)
    E = torch.zeros(2, 8, 256, device=DEV)
    codes = torch.full((1, 2, 4), -7, dtype=torch.int32, device=DEV)
    for T, n_q, n_sem, V, B in ((0, 2, 1, 8, 1), (4, 0, 1, 8, 1), (4, 2, 0, 8, 1), (4, 2, 3, 8, 1), (4, 2, 1, 0, 1), (4, 2, 1, 8, 0)):
        assert lib.sopro_debug_mimi_rvq_encode(_p(proj), _p(E), _p(codes), T, n_q, n_sem, V, None, B, _st()) != 0
    torch.cuda.synchronize()
    assert bool((codes == -7).all())


# ---------------------------------------------------------------------------------------------------------------
# RVQ gather, upsample, LayerNorm
# ---------------------------------------------------------------------------------------------------------------
def test_rvq_gather_exact_and_clamped():
    """Bit-exact against the float32 sum in q order, semantic and acoustic sums apart; codes read from columns [0, T) of
    a wider [Q][code_T] buffer; out-of-range codes (-1, 2048, INT32_MAX) are clamped and set the sticky flag."""
    lib_mod, lib = _lib()
    g = torch.Generator().manual_seed(21)
    B, Q, T, code_T, Dc, V, n_sem = 3, 32, 37, 45, 256, 2048, 1
    embed = torch.randn(Q, V, Dc, generator=g)
    for with_bad in (False, True):
        codes = torch.randint(0, V, (B, Q, code_T), generator=g, dtype=torch.int32)
        if with_bad:
            codes[0, 3, 5], codes[1, 0, 0], codes[2, 31, T - 1] = -1, V, 2 ** 31 - 1
            codes[2, 7, T] = -5  # past column T: never read
        S = torch.full((B, T, 2 * Dc), float("nan"), device=DEV)
        flag = torch.zeros(1, dtype=torch.int32, device=DEV)
        cd, ed = codes.to(DEV), embed.to(DEV)
        lib_mod.check(lib.sopro_debug_mimi_rvq_gather(_p(cd), _p(ed), _p(S), B, Q, T, code_T, Dc, V, n_sem, _p(flag), _st()))
        torch.cuda.synchronize()
        cl = codes[:, :, :T].long().clamp(0, V - 1)
        e = embed[torch.arange(Q)[None, :, None], cl]  # [B][Q][T][Dc]
        want = np.concatenate([seq_sum_f32(e[:, :n_sem].numpy(), 1), seq_sum_f32(e[:, n_sem:].numpy(), 1)], axis=-1)
        assert np.array_equal(S.cpu().numpy(), want), with_bad
        assert int(flag.item()) == int(with_bad)
    assert lib.sopro_debug_mimi_rvq_gather(_p(cd), _p(ed), _p(S), B, Q, T, T - 1, Dc, V, n_sem, _p(flag), _st()) != 0


@pytest.mark.parametrize("with_prev", [False, True])
def test_upsample(with_prev):
    """y[2t+r] = x[t] w[r] + x[t-1] w[r+2]: at most two roundings (u |x w| each; fused or not), row pair 0 reads
    `prev` (the carried frame) or, without it, is the single fp32 product, bit-exact."""
    lib_mod, lib = _lib()
    g = torch.Generator().manual_seed(22 + with_prev)
    B, T, Cc = 3, 29, 512
    x = torch.randn(B, T, Cc, generator=g)
    w = torch.randn(Cc, 4, generator=g)
    prev = torch.randn(B, Cc, generator=g) if with_prev else None
    y = torch.full((B, 2 * T, Cc), float("nan"), device=DEV)
    xd, wd, pd = x.to(DEV), w.to(DEV), prev.to(DEV) if with_prev else None
    lib_mod.check(lib.sopro_debug_mimi_upsample(_p(xd), _p(wd), _p(y), _p(pd), B, T, Cc, _st()))
    torch.cuda.synchronize()
    y = y.cpu().double()
    xm1 = torch.cat([prev[:, None] if with_prev else torch.zeros(B, 1, Cc), x[:, :-1]], dim=1).double()
    x64, w64 = x.double(), w.double()
    worst = 0.0
    for r in (0, 1):
        a, b = x64 * w64[:, r], xm1 * w64[:, r + 2]
        want, bound = a + b, 2 * U * (1 + 2.0 ** -20) * (a.abs() + b.abs())  # (the u^2 term of three roundings)
        got = y[:, r::2]
        worst = max(worst, _ratio((got - want).abs(), bound))
        assert bool(((got - want).abs() <= bound).all()), r
        if not with_prev:
            assert torch.equal(got[:, 0].float(), x[:, 0] * w[:, r]), r
    print(f"upsample prev={with_prev}: worst err / bound {worst:.3f}")


def _layernorm_bound(x, w, b, eps):
    """float64 LayerNorm and its bound for the kernel's arithmetic (n = ceil(C/32) + 5 additions per sum: one lane's
    chain and the shuffle tree): mean error Em = gamma_n sum|x| / C + u |mean|; d error Ed = Em + u (|d| + Em); variance
    error Ev = (gamma_n sum d^2 + sum (2 |d| Ed + Ed^2)) / C + u var; z = var + eps: Ez = Ev + u (z + Ev); inv =
    1/sqrtf(z) (two correct roundings): Einv = inv (Ez / (2 (z - Ez)) + 2u) (1 + 4u); y = d inv w + b (three
    roundings): Ey = |w| (Ed inv + |d| Einv + Ed Einv) (1 + u) + 2u |d inv w| + u |y| (1 + u)."""
    x, w, b = x.double(), w.double(), b.double()
    Cc = x.shape[-1]
    n = -(-Cc // 32) + 5
    mean = x.mean(-1, keepdim=True)
    d = x - mean
    var = (d * d).mean(-1, keepdim=True)
    Em = gamma(n) * x.abs().sum(-1, keepdim=True) / Cc + U * mean.abs()
    Ed = Em + U * (d.abs() + Em)
    Ev = (gamma(n) * (d * d).sum(-1, keepdim=True) + (2 * d.abs() * Ed + Ed * Ed).sum(-1, keepdim=True)) / Cc + U * var
    z = var + eps
    Ez = Ev + U * (z + Ev)
    inv = 1 / torch.sqrt(z)
    Einv = inv * (Ez / (2 * (z - Ez)) + 2 * U) * (1 + 4 * U)
    y = d * inv * w + b
    Ey = w.abs() * (Ed * inv + d.abs() * Einv + Ed * Einv) * (1 + U) + 2 * U * (d * inv * w).abs() + U * y.abs() * (1 + U)
    return y, Ey


@pytest.mark.parametrize("rows", [1, 7, 13, 1001])
def test_layernorm(rows):
    """fp32 output within the derived bound; bf16 output within half a bf16 ulp (at most 2^-8 |y|: 8 significant bits)
    plus the fp32 bound.
    Row counts that are not a multiple of the 8 rows per block; a constant row (variance 0: only eps keeps it finite)
    and a row with a large common offset."""
    lib_mod, lib = _lib()
    g = torch.Generator().manual_seed(rows)
    Cc, eps = 512, 1e-5
    x = torch.randn(rows, Cc, generator=g) * 2
    x[0] = 0.75  # constant row
    if rows > 2:
        x[2] += 300.0
    w = 1 + 0.2 * torch.randn(Cc, generator=g)
    b = 0.1 * torch.randn(Cc, generator=g)
    xd, wd, bd = x.to(DEV), w.to(DEV), b.to(DEV)
    want, bound = _layernorm_bound(x, w, b, eps)
    for bf in (0, 1):
        y = torch.full((rows + 1, Cc), float("nan"), dtype=torch.bfloat16 if bf else torch.float32, device=DEV)
        lib_mod.check(lib.sopro_debug_mimi_layernorm(_p(xd), _p(wd), _p(bd), _p(y), rows, Cc, eps, bf, _st()))
        torch.cuda.synchronize()
        y = y.cpu().double()
        assert bool(torch.isnan(y[rows]).all())
        tol = bound + (2.0 ** -8 * (want.abs() + bound) if bf else 0)
        err = (y[:rows] - want).abs()
        r = _ratio(err, tol)
        print(f"layernorm rows={rows} {'bf16' if bf else 'fp32'}: max |err| {float(err.max()):.2e}, worst err / bound {r:.3f}")
        assert r <= 1.0, bf


# ---------------------------------------------------------------------------------------------------------------
# RoPE + fp32 attention, one-shot and over the ring
# ---------------------------------------------------------------------------------------------------------------
H, CH, DH, WINDOW = 8, 512, 64, 250


def _attn_call(qkv, tab, tab_n, T2, window, pos0=0, ring=None, bf=0):
    """qkv [B][T2][3C] fp32 on the device (rotated in place) -> out [B][T2][C] (fp32 or bf16)"""
    lib_mod, lib = _lib()
    B = qkv.shape[0]
    out = torch.full((B, T2, CH), float("nan"), dtype=torch.bfloat16 if bf else torch.float32, device=DEV)
    kr, vr, R = ring if ring is not None else (None, None, 0)
    lib_mod.check(lib.sopro_debug_mimi_attn(_p(qkv), _p(tab), tab_n, _p(out), B, T2, CH, H, window, pos0, _p(kr), _p(vr), R, bf, _st()))
    torch.cuda.synchronize()
    return out


_SEQ = {}


def _seq_copies(n, count):
    """the float32 sequential sum of `count` copies of fp32(1/n), as the kernel forms an output of the probe"""
    if n not in _SEQ:
        inv = np.float32(1.0) / np.float32(n)
        s, acc = [np.float32(0)], np.float32(0)
        for _ in range(n):
            acc = np.float32(acc + inv)
            s.append(acc)
        _SEQ[n] = s
    return _SEQ[n][count]


def _probe(B, T_total, window, pos0, T2):
    """q = 0 (every probability exactly 1) and v one-hot by absolute position p in channel (7p + 3h + 5b) % 64: the
    output channel c of the query at position i counts the window's keys in channel c, each adding fp32(1/n)"""
    p = torch.arange(T_total)
    ch = (7 * p[None, :, None] + 3 * torch.arange(H)[None, None, :] + 5 * torch.arange(B)[:, None, None]) % DH  # [B][P][H]
    v = torch.nn.functional.one_hot(ch, DH).float()  # [B][P][H][DH]
    want = np.zeros((B, T2, H, DH), dtype=np.float32)
    for i in range(T2):
        a = pos0 + i
        j0 = max(0, a - window + 1)
        n = a - j0 + 1
        cnt = v[:, j0:a + 1].sum(1).long().numpy()  # [B][H][DH]
        _seq_copies(n, 0)
        want[:, i] = np.asarray(_SEQ[n], dtype=np.float32)[cnt]
    return v, torch.from_numpy(want)


def _qkv(q, k, v):
    B, T2 = q.shape[:2]
    return torch.cat([q.reshape(B, T2, CH), k.reshape(B, T2, CH), v.reshape(B, T2, CH)], dim=-1).contiguous()


@pytest.mark.parametrize("T2", [1, 9, 250, 251, 600])
def test_attention_probes_one_shot(T2):
    """Exact probes over the whole window range (partial and full windows, the first position past the window), fp32
    and bf16 output, B = 3."""
    B = 3
    g = torch.Generator().manual_seed(T2)
    tab = rope_table(T2 + 5, DH).to(DEV)
    v, want = _probe(B, T2, WINDOW, 0, T2)
    k = torch.randn(B, T2, H, DH, generator=g)
    for bf in (0, 1):
        qkv = _qkv(torch.zeros(B, T2, H, DH), k, v).to(DEV)
        got = _attn_call(qkv, tab, T2 + 5, T2, WINDOW, bf=bf).cpu().float().reshape(B, T2, H, DH)
        w = want.to(torch.bfloat16).float() if bf else want
        bad = (got != w).nonzero()
        assert bad.numel() == 0, f"T2={T2} bf16={bf}: {bad.shape[0]} differ, first {bad[:4].tolist()}"


def _attn_bound(q, k, v, window, pos0, kp, vp):
    """float64 attention of the kernel's own rotated fp32 q / k and the fp32 v over the window, and the bound: score
    s_j = scale q.k_j (Dh products and sums in any order: gamma_Dh sum|q k_j|; scale = 1/8 exact); the exponent argument
    s_j - max is off by delta_j <= scale gamma_Dh (sum|q k_j| + sum|q k_max|) + u |s_j - max|, expf adds 2 ulp, so e_j
    is off by rho_j = expm1(delta_j) + 2^-22 relative; the sum adds gamma_nk, 1/sum and e_j * inv one rounding each, so
    p_j is off by rho_j + max rho + gamma_nk + 3u relative; the output sum over nk adds gamma_nk sum |p v|.  The final
    factor 1.0001 covers the products of these first-order terms."""
    out, p = window_attention(q, k, v, window, pos0, kp, vp)
    kk = torch.cat([kp, k], 1) if pos0 else k
    vv = torch.cat([vp, v], 1) if pos0 else v
    mag = torch.einsum("bqhd,bkhd->bhqk", q.double().abs(), kk.double().abs()) / math.sqrt(DH)  # [B][H][T][P]
    s = torch.einsum("bqhd,bkhd->bhqk", q.double(), kk.double()) / math.sqrt(DH)
    ok = p > 0
    mx_idx = s.masked_fill(~ok, float("-inf")).argmax(-1, keepdim=True)
    mag_mx = mag.gather(-1, mx_idx)
    s_mx = s.gather(-1, mx_idx)
    nk = ok.sum(-1, keepdim=True).double()
    gn = nk * U / (1 - nk * U)
    delta = gamma(DH) * (mag + mag_mx) + U * (s - s_mx).abs()
    rho = torch.where(ok, torch.expm1(delta) + 2.0 ** -22, torch.zeros_like(delta))
    rel = rho + rho.amax(-1, keepdim=True) + gn + 3 * U
    bound = torch.einsum("bhqk,bkhd->bqhd", p * (rel + gn), vv.double().abs()) * 1.0001
    return out, bound


def _check_random_chunk(got, qr, kr, v, window, pos0, kp, vp, bf, tag):
    ref, bound = _attn_bound(qr, kr, v, window, pos0, kp, vp)
    if bf:
        bound = bound + 2.0 ** -8 * (ref.abs() + bound)  # the bf16 rounding: half an ulp, <= 2^-8 |out|
    err = (got.double() - ref).abs()
    r = _ratio(err, bound)
    assert r <= 1.0, tag
    return r


def _check_rope(qkv_rot, qkv_in, pos0, tab, tab_n):
    """the kernel's rotated q and k against the float64 rotation of the same fp32 inputs with the fp32 table:
    x1 c - x2 s and x2 c + x1 s, two products and a difference (fused or not): <= 2u (|x1 c| + |x2 s|) up to a u^2 term"""
    B, T2, _ = qkv_in.shape
    pos = torch.arange(pos0, pos0 + T2)
    worst = 0.0
    for which in (0, 1):
        x = qkv_in[:, :, which * CH:(which + 1) * CH].reshape(B, T2, H, DH)
        ref, mag = rope64(x, pos, tab, tab_n)
        got = qkv_rot[:, :, which * CH:(which + 1) * CH].reshape(B, T2, H, DH).double()
        r = _ratio((got - ref).abs(), 2.0 ** -23 * (1 + 2.0 ** -20) * mag)
        assert r <= 1.0, which
        worst = max(worst, r)
    assert torch.equal(qkv_rot[:, :, 2 * CH:], qkv_in[:, :, 2 * CH:])  # v untouched
    return worst


@pytest.mark.parametrize("T2", [1, 250, 600])
def test_attention_random_one_shot(T2):
    """Random q / k / v (scores of unit size and scores scaled until the softmax is peaked), fp32 and bf16 output:
    RoPE against float64, the attention within the derived bound against float64 attention over the window."""
    B = 2
    tab = rope_table(T2, DH)
    tab_d = tab.to(DEV)
    worst_a = worst_r = 0.0
    for sc in (1.0, 4.0):
        g = torch.Generator().manual_seed(T2 + int(sc))
        qkv_in = torch.cat([torch.randn(B, T2, 2 * CH, generator=g) * sc, torch.randn(B, T2, CH, generator=g)], -1)
        for bf in (0, 1):
            qkv = qkv_in.to(DEV)
            got = _attn_call(qkv, tab_d, T2, T2, WINDOW, bf=bf).cpu().reshape(B, T2, H, DH)
            rot = qkv.cpu()
            worst_r = max(worst_r, _check_rope(rot, qkv_in, 0, tab, T2))
            q, k, v = (rot[:, :, i * CH:(i + 1) * CH].reshape(B, T2, H, DH) for i in range(3))
            worst_a = max(worst_a, _check_random_chunk(got, q, k, v, WINDOW, 0, None, None, bf, (T2, sc, bf)))
    print(f"fp32 attention one-shot T2={T2}: worst err / bound {worst_a:.3f}, rope {worst_r:.3f}")


@pytest.mark.parametrize("max_chunk", [1, 4, 16])
def test_attention_over_the_ring(max_chunk):
    """The stream's geometry: chunks of 2n rows, n <= max_chunk, at pos0 advancing, the keys and values appended to a
    ring of R = (window + 2 max_chunk + 7) / 8 * 8 rows (as sopro_mimi_stream_create_rows sizes it) and read back from
    it, past two wrap-arounds, B = 2.  Each chunk: exact probes (fp32 and bf16 output), then random operands within the
    derived bound; the ring rows of the chunk's positions hold the kernel's rotated keys and the values exactly."""
    B = 2
    R = (WINDOW + 2 * max_chunk + 7) // 8 * 8
    total = 2 * R + 3 * WINDOW // 2
    tab_n = total + 64
    tab = rope_table(tab_n, DH)
    tab_d = tab.to(DEV)
    g = torch.Generator().manual_seed(max_chunk)
    sched = []
    pos = 0
    while pos < total:
        n = 1 + int(torch.randint(0, max_chunk, (1,), generator=g))
        sched.append((pos, 2 * n))
        pos += 2 * n
    vprobe, _ = _probe(B, pos, WINDOW, 0, 1)
    kin = torch.randn(B, pos, H, DH, generator=g)
    qkv_rand = torch.cat([torch.randn(B, pos, 2 * CH, generator=g), torch.randn(B, pos, CH, generator=g)], -1)
    worst = 0.0
    for kind in ("probe", "random"):
        for bf in ((0, 1) if kind == "probe" else (0,)):
            kring = torch.full((B, R, CH), float("nan"), device=DEV)
            vring = torch.full((B, R, CH), float("nan"), device=DEV)
            rot_all = []
            for pos0, T2 in sched:
                if kind == "probe":
                    qkv_in = _qkv(torch.zeros(B, T2, H, DH), kin[:, pos0:pos0 + T2], vprobe[:, pos0:pos0 + T2])
                else:
                    qkv_in = qkv_rand[:, pos0:pos0 + T2].contiguous()
                qkv = qkv_in.to(DEV)
                got = _attn_call(qkv, tab_d, tab_n, T2, WINDOW, pos0, (kring, vring, R), bf).cpu().reshape(B, T2, H, DH)
                rot = qkv.cpu()
                rot_all.append(rot)
                slots = torch.arange(pos0, pos0 + T2) % R
                kr, vr = kring.cpu(), vring.cpu()
                assert torch.equal(kr[:, slots], rot[:, :, CH:2 * CH]) and torch.equal(vr[:, slots], rot[:, :, 2 * CH:]), (kind, pos0)
                if kind == "probe":
                    _, want = _probe(B, pos0 + T2, WINDOW, pos0, T2)
                    w = want.to(torch.bfloat16).float() if bf else want
                    bad = (got.float() != w).nonzero()
                    assert bad.numel() == 0, f"ring probe chunk at {pos0} (R={R}, bf16={bf}): {bad.shape[0]} differ, first {bad[:4].tolist()}"
                else:
                    worst = max(worst, _check_rope(rot, qkv_in, pos0, tab, tab_n))
                    allr = torch.cat(rot_all, 1)
                    q, k, v = (allr[:, pos0:, i * CH:(i + 1) * CH].reshape(B, T2, H, DH) for i in range(3))
                    kp = allr[:, :pos0, CH:2 * CH].reshape(B, pos0, H, DH) if pos0 else None
                    vp = allr[:, :pos0, 2 * CH:].reshape(B, pos0, H, DH) if pos0 else None
                    worst = max(worst, _check_random_chunk(got, q, k, v, WINDOW, pos0, kp, vp, 0, pos0))
    print(f"fp32 attention over a ring of R={R} rows, {len(sched)} chunks to position {pos}: probes exact, worst err / bound {worst:.3f}")


def test_attention_refuses_unsupported_shapes():
    _, lib = _lib()
    qkv = torch.zeros(1, 8, 3 * CH, device=DEV)
    tab = rope_table(16, DH).to(DEV)
    out = torch.full((1, 8, CH), 7.0, device=DEV)
    ring = torch.zeros(1, 256, CH, device=DEV)
    for T2, H_, window, pos0, kr, vr, R, tab_n in ((8, 7, 250, 0, None, None, 0, 16), (8, H, 0, 0, None, None, 0, 16),
                                                  (8, H, 250, 4, None, None, 0, 16), (8, H, 250, 0, ring, None, 256, 16),
                                                  (8, H, 250, 0, ring, ring, 256, 16), (8, H, 200, 9, ring, ring, 256, 16),
                                                  (8, H, 6000, 0, None, None, 0, 16)):
        assert lib.sopro_debug_mimi_attn(_p(qkv), _p(tab), tab_n, _p(out), 1, T2, CH, H_, window, pos0, _p(kr), _p(vr), R, 0, _st()) != 0
    torch.cuda.synchronize()
    assert bool((out == 7.0).all()) and bool((qkv == 0).all())


# ---------------------------------------------------------------------------------------------------------------
# final conv
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Tn", [1, 253, 254, 255, 256, 257, 508, 509, 512, 1000])
def test_final_conv(Tn):
    """Both kernels, lo = 0 (the causal zero pad) and lo = -(taps-1) (context rows in front), B = 3 at a batch stride
    larger than the item, against float64:
      fp32 input, ELU on load (final_conv_kernel): gamma_{taps Cin + 1} (|bias| + sum |elu(x) w|) for the sum in any
      order, plus 2^-23 sum |elu(x) w| (1 + gamma) for expm1f's 1 ulp;
      bf16 input already ELU'd (final_conv_h_kernel, 254 outputs per block): a Cin-long fma chain per tap, then the
      bias and the taps: gamma_{Cin + taps + 1} (|bias| + sum |x w|)."""
    lib_mod, lib = _lib()
    B, Cin, taps = 3, 64, 3
    g = torch.Generator().manual_seed(Tn)
    w = torch.randn(taps * Cin, generator=g) / math.sqrt(taps * Cin)
    bias = torch.randn(1, generator=g) * 0.1
    wd, bd = w.to(DEV), bias.to(DEV)
    worst = 0.0
    for bf in (0, 1):
        for lo in (0, -(taps - 1)):
            ctx = -lo
            pitch = ctx + Tn + 5
            xall = torch.randn(B, pitch, Cin, generator=g)
            if bf:
                xall = torch.nn.functional.elu(xall).to(torch.bfloat16)
            xd = xall.to(DEV)
            y = torch.full((B, Tn + 3), float("nan"), device=DEV)
            lib_mod.check(lib.sopro_debug_mimi_final_conv(C.c_void_p(xd.data_ptr() + ctx * Cin * xd.element_size()), bf, _p(wd), _p(bd),
                                                          _p(y), B, Tn, Cin, taps, lo, pitch * Cin, Tn + 3, _st()))
            torch.cuda.synchronize()
            y = y.cpu().double()
            assert bool(torch.isnan(y[:, Tn:]).all())
            xin = xall.double() if bf else torch.nn.functional.elu(xall.double())
            rows = torch.zeros(B, taps - 1 + Tn, Cin, dtype=torch.float64)  # rows -(taps-1) .. Tn-1
            rows[:, taps - 1 - ctx:] = xin[:, :ctx + Tn]
            cols = torch.cat([rows[:, j:j + Tn] for j in range(taps)], dim=-1)  # tap j reads row t + j - (taps-1)
            want = cols @ w.double() + float(bias)
            mag = cols.abs() @ w.double().abs() + abs(float(bias))
            bound = gamma(Cin + taps + 1) * mag if bf else (gamma(taps * Cin + 1) + ULP1 * (1 + gamma(taps * Cin + 1))) * mag
            err = (y[:, :Tn] - want).abs()
            r = _ratio(err, bound)
            worst = max(worst, r)
            assert r <= 1.0, (bf, lo)
    print(f"final conv Tn={Tn}: worst err / bound {worst:.3f}")


def test_final_conv_refuses_unsupported_shapes():
    _, lib = _lib()
    x = torch.zeros(2, 20, 64, device=DEV)
    w = torch.zeros(3 * 64, device=DEV)
    b = torch.zeros(1, device=DEV)
    y = torch.full((2, 16), 7.0, device=DEV)
    for bf, B, Tn, Cin, taps, lo, xbs in ((0, 1, 16, 62, 3, 0, 0), (1, 1, 16, 60, 3, 0, 0), (0, 1, 16, 64, 9, 0, 0), (0, 1, 16, 64, 3, 1, 0),
                                          (0, 1, 16, 64, 3, -3, 0), (0, 2, 16, 64, 3, -2, 16 * 64), (0, 1, 0, 64, 3, 0, 0)):
        assert lib.sopro_debug_mimi_final_conv(_p(x), bf, _p(w), _p(b), _p(y), B, Tn, Cin, taps, lo, xbs, 16, _st()) != 0
    torch.cuda.synchronize()
    assert bool((y == 7.0).all())
