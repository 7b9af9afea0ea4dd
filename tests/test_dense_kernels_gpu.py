"""The NAR refiner's and the prefill's contractions one kernel at a time, against float64 (oracle/dense_probes.py).

End to end the refiner is checked through argmax ids, which a split that is wrong at the 2^-17 level can pass.  Here each
kernel runs through its test hook (include/sopro_b200.h: sopro_debug_dense / _tc6 / _dwconv_res / _argmax_heads, which call
the engine's own launchers) and is held to what its arithmetic allows:
  * dense_tile_kernel (32 / 64 / 128) and dense_skinny_kernel: bit-equal to float64 on dyadic operands (every epilogue,
    production and edge shapes), bit-equal to each other across tile edges and row counts, within gamma_K sum|a w| of
    float64 on random operands; first-maximum argmax ties inside and across tiles, skinny CTA parts and groups;
  * split3_rows_kernel + the six-product wgmma GEMM: an exact three-term split, pair probes returned exactly, an elementwise
    bound and an RMS error within 2x of the fp32 FMA kernel's;
  * dwconv_res_kernel: ragged lengths, padding rows never read (NaN there) nor written;
  * argmax_heads_kernel: first maximum across lanes and lane strides.
Float64 references run on the GPU (torch float64 matmul), operands are generated on the host from seeded generators.
"""
import ctypes as C
import math

import pytest
import torch

from oracle import dense_probes as P

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
DEV = "cuda:0"
EPI_BIAS, EPI_GELU, EPI_RES, EPI_GLU, EPI_ARGMAX, EPI_RES_GATE = range(6)
TC_NONE, TC_GELU, TC_RES = 0, 1, 3
U = P.U


def _lib():
    from sopro_b200 import _lib

    return _lib, _lib.load()


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _d(t):
    return None if t is None else t.to(DEV, torch.float32).contiguous()


def _dense(A, W, bias=None, norm_w=None, a_add=None, R=None, gate=0.0, epi=EPI_BIAS, groups=1, kernel=0, ldc=None, C_out=None):
    """one DenseOp through sopro_debug_dense -> C [M][ldc] (fp32, device) or, for EPI_ARGMAX, ids [M][groups]"""
    lib_mod, lib = _lib()
    M, K = A.shape
    N = W.shape[-2]
    A, W, bias, norm_w, a_add, R = (_d(t) for t in (A, W, bias, norm_w, a_add, R))
    ncol = N // 2 if epi == EPI_GLU else N
    ldc = ldc or ncol
    ids = ws = None
    if epi == EPI_ARGMAX:
        ids = torch.full((M, groups), -1, dtype=torch.int32, device=DEV)
        ws = torch.empty(8 * groups * M * ((N + 7) // 8), dtype=torch.uint8, device=DEV)
    elif C_out is None:
        C_out = torch.full((M, ldc), float("nan"), device=DEV)
    zW, zB, zA = N * K, N, K
    rc = lib.sopro_debug_dense(_p(A), _p(W), _p(bias), _p(norm_w), _p(a_add), _p(R), _p(C_out), float(gate), M, N, K, ldc, epi, groups,
                               zW, zB, zA, kernel, _p(ids), _p(ws), ws.numel() if ws is not None else 0, _st())
    lib_mod.check(rc)
    return ids if epi == EPI_ARGMAX else C_out


def _ref(A, W, bias=None, norm_w=None, a_add=None, R=None, gate=0.0, epi=EPI_BIAS):
    """float64 of the same op -> (out, pre-activation acc, sum |a w|) on the device"""
    A64, W64 = A.to(DEV, torch.float64), W.to(DEV, torch.float64)
    if norm_w is not None:
        A64 = A64 * torch.rsqrt(A64.pow(2).mean(-1, keepdim=True) + 1e-6) * norm_w.to(DEV, torch.float64)
    if a_add is not None:
        A64 = A64 + a_add.to(DEV, torch.float64)
    acc = A64 @ W64.T
    mag = A64.abs() @ W64.abs().T
    if bias is not None:
        acc = acc + bias.to(DEV, torch.float64)
    if epi == EPI_GELU:
        out = 0.5 * acc * (1 + torch.erf(acc / math.sqrt(2)))
    elif epi == EPI_RES:
        out = R.to(DEV, torch.float64) + acc
    elif epi == EPI_RES_GATE:
        out = R.to(DEV, torch.float64) + gate * acc
    elif epi == EPI_GLU:
        D = W.shape[0] // 2
        out = acc[:, :D] * torch.sigmoid(acc[:, D:])
    else:
        out = acc
    return out, acc, mag


# (name, N, K, epi): the refiner's / prefill's production contractions
PROD = [("glu", 768, 384, EPI_GLU), ("ffn1", 1536, 384, EPI_GELU), ("ffn2", 384, 1536, EPI_RES), ("pre", 256, 384, EPI_BIAS),
        ("film0", 384, 192, EPI_GELU), ("film2", 768, 384, EPI_BIAS), ("xattn_o", 384, 384, EPI_RES_GATE)]
EDGE_M = [1, 15, 16, 17, 31, 33, 63, 65, 127, 129, 401, 1203]


def _kernels(M, epi):
    ks = [0, 64, 128] + ([] if epi == EPI_GLU else [32])
    return ks + ([16] if M <= 16 else [])


def _exact_operands(M, N, K, epi, seed, norm=False):
    """dyadic A (2^-6 grid, |a| <= 1/4), W (2^-6, |w| <= 1/4), bias / R on 2^-12: every sum is exact in fp32 for K <= 2048"""
    g = torch.Generator().manual_seed(seed)
    A = P.dyadic((M, K), -16, 16, -6, g)
    W = P.dyadic((N, K), -16, 16, -6, g)
    bias = P.dyadic((N,), -64, 64, -12, g)
    add = P.dyadic((K,), -8, 8, -6, g)
    R = P.dyadic((M, N // 2 if epi == EPI_GLU else N), -64, 64, -12, g) if epi in (EPI_RES, EPI_RES_GATE) else None
    return A, W, bias, add, R


def _check_exact(got, out64, acc64, epi):
    """bit-exact for the linear epilogues; GELU / GLU: the exact pre-activation through erff / expf (few ulps)"""
    got = got.double()
    if epi in (EPI_BIAS, EPI_RES, EPI_RES_GATE):
        bad = (got != out64).nonzero()
        assert bad.numel() == 0, f"{bad.shape[0]} outputs differ from float64, first {bad[:4].tolist()}"
        return
    if epi == EPI_GELU:
        tol = 8 * U * (out64.abs() + 0.5 * acc64.abs()) + 1e-30
    else:
        D = acc64.shape[1] // 2
        tol = 8 * U * (out64.abs() + 0.25 * acc64[:, :D].abs() * acc64[:, D:].abs()) + 1e-30
    err = (got - out64).abs()
    assert bool((err <= tol).all()), f"max error / tol {float((err / tol).max()):.2f}"


@pytest.mark.parametrize("name,N,K,epi", PROD, ids=[p[0] for p in PROD])
@pytest.mark.parametrize("M", [1, 17, 401, 1203])
def test_production_ops_bit_exact_on_dyadic_operands(name, N, K, epi, M):
    A, W, bias, add, R = _exact_operands(M, N, K, epi, seed=M * 131 + N + K)
    gate = 0.5 if epi == EPI_RES_GATE else 0.0
    for use_add in (False, True):
        out64, acc64, _ = _ref(A, W, bias, None, add if use_add else None, R, gate, epi)
        for kern in _kernels(M, epi):
            got = _dense(A, W, bias, None, add if use_add else None, R, gate, epi, kernel=kern)
            try:
                _check_exact(got, out64, acc64, epi)
            except AssertionError as e:
                raise AssertionError(f"{name} M={M} kernel={kern} a_add={use_add}: {e}") from None


@pytest.mark.parametrize("M", EDGE_M)
@pytest.mark.parametrize("N,K", [(40, 16), (200, 48), (96, 2048)])
@pytest.mark.parametrize("epi", [EPI_BIAS, EPI_GELU, EPI_RES, EPI_GLU, EPI_RES_GATE])
def test_edge_shapes_bit_exact_on_dyadic_operands(M, N, K, epi):
    """N not a multiple of any tile, K = 16 (one k-tile), 48 (three), 2048 (the skinny kernel's shared-memory limit); a
    result row pitch ldc > N (the tile kernels must write only columns < N)"""
    A, W, bias, add, R = _exact_operands(M, N, K, epi, seed=M + 7 * N + K + epi)
    gate = 0.25 if epi == EPI_RES_GATE else 0.0
    ncol = N // 2 if epi == EPI_GLU else N
    ldc = ncol + 5
    Rp = None
    if R is not None:
        Rp = torch.zeros((M, ldc))
        Rp[:, :ncol] = R
    out64, acc64, _ = _ref(A, W, bias, None, add, R, gate, epi)
    for kern in _kernels(M, epi):
        got = _dense(A, W, bias, None, add, Rp, gate, epi, kernel=kern, ldc=ldc)
        assert bool(got[:, ncol:].isnan().all()), f"kernel {kern} wrote past column {ncol}"
        try:
            _check_exact(got[:, :ncol], out64, acc64, epi)
        except AssertionError as e:
            raise AssertionError(f"kernel={kern}: {e}") from None


def test_ffn2_residual_in_place():
    """R aliased to C (the refiner's FFN2): every output reads its own residual before it is overwritten"""
    M, N, K = 129, 384, 1536
    A, W, bias, _, R = _exact_operands(M, N, K, EPI_RES, seed=5)
    out64, _, _ = _ref(A, W, bias, None, None, R, 0.0, EPI_RES)
    for kern in (0, 32, 64, 128):
        Cb = R.to(DEV).clone()
        _dense(A, W, bias, None, None, Cb, 0.0, EPI_RES, kernel=kern, C_out=Cb)
        assert torch.equal(Cb.double(), out64), kern
    Cb = R[:9].to(DEV).clone()
    _dense(A[:9], W, bias, None, None, Cb, 0.0, EPI_RES, kernel=16, C_out=Cb)
    assert torch.equal(Cb.double(), out64[:9])


def _rand_operands(M, N, K, epi, seed):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn((M, K), generator=g)
    W = torch.randn((N, K), generator=g) / math.sqrt(K)
    bias = torch.randn((N,), generator=g) * 0.1
    nw = 1 + 0.1 * torch.randn((K,), generator=g)
    add = 0.1 * torch.randn((K,), generator=g)
    R = torch.randn((M, N // 2 if epi == EPI_GLU else N), generator=g) if epi in (EPI_RES, EPI_RES_GATE) else None
    return A, W, bias, nw, add, R


@pytest.mark.parametrize("name,N,K,epi", PROD, ids=[p[0] for p in PROD])
def test_tile_edges_and_row_count_never_change_a_bit(name, N, K, epi):
    """dense_f32.cuh: every output is one fma chain over k whatever the tile, so 32 / 64 / 128 agree bit for bit, and a row's
    output does not depend on how many rows the op has once it runs on a tile kernel"""
    M = 1203
    A, W, bias, nw, add, R = _rand_operands(M, N, K, epi, seed=N + K)
    gate = 0.75 if epi == EPI_RES_GATE else 0.0
    for norm in (None, nw):
        outs = {k: _dense(A, W, bias, norm, add, R, gate, epi, kernel=k) for k in _kernels(M, epi) if k}
        first = next(iter(outs.values()))
        for k, o in outs.items():
            assert torch.equal(o, first), (name, k, norm is not None)
        auto = _dense(A, W, bias, norm, add, R, gate, epi)
        assert torch.equal(auto, first)
        for r0, rows in ((700, 17), (0, 33), (1202, 1)):
            sub = _dense(A[r0:r0 + rows], W, bias, norm, add, None if R is None else R[r0:r0 + rows], gate, epi,
                         kernel=0 if rows > 16 else 64)
            assert torch.equal(sub, first[r0:r0 + rows]), (name, r0, rows)


def _bound(epi, K, acc64, mag, bias, R, gate, norm):
    """|c - c64| bound: gamma_K sum|a w| for the chain (any order), the bias / residual roundings, the RMSNorm prologue's
    relative error (sum of squares over K in ~K/32 + 5 sequential steps, sqrtf, one division, two products), propagated
    through GELU (|gelu'| <= 1.13, erff <= 2 ulp) and GLU (|sigmoid'| <= 1/4, expf <= 2 ulp)"""
    extra = (K // 32 + 12) * U if norm else 0.0
    b = (P.gamma(K + 2) + extra) * mag + 2 * U * (acc64.abs() + (bias.abs() if bias is not None else 0))
    if epi == EPI_GELU:
        return 1.2 * b + 8 * U * (acc64.abs() + 1e-30)
    if epi == EPI_GLU:
        D = acc64.shape[1] // 2
        v, g = acc64[:, :D], acc64[:, D:]
        return torch.sigmoid(g) * b[:, :D] + 0.25 * v.abs() * b[:, D:] + 8 * U * v.abs()
    if epi == EPI_RES:
        return b + 2 * U * (R.abs() + acc64.abs())
    if epi == EPI_RES_GATE:
        return abs(gate) * b + 2 * U * (R.abs() + abs(gate) * acc64.abs())
    return b


@pytest.mark.parametrize("name,N,K,epi", PROD, ids=[p[0] for p in PROD])
@pytest.mark.parametrize("M", [7, 16, 129, 1203])
def test_random_operands_within_the_summation_bound(name, N, K, epi, M):
    A, W, bias, nw, add, R = _rand_operands(M, N, K, epi, seed=3 * M + N + K)
    gate = 0.75 if epi == EPI_RES_GATE else 0.0
    Rd = None if R is None else R.to(DEV, torch.float64)
    for norm in (None, nw):
        out64, acc64, mag = _ref(A, W, bias, norm, add, R, gate, epi)
        bound = _bound(epi, K, acc64, mag, bias.to(DEV, torch.float64), Rd, gate, norm is not None)
        for kern in _kernels(M, epi):
            got = _dense(A, W, bias, norm, add, R, gate, epi, kernel=kern).double()
            ratio = float(((got - out64).abs() / bound).max())
            assert ratio <= 1.0, (name, M, kern, norm is not None, ratio)


# ---------------------------------------------------------------------------------------------------------------
# argmax ties
# ---------------------------------------------------------------------------------------------------------------
def _skinny_cols(ncol, groups):
    """columns per CTA of the skinny kernel (nar_engine.cu launch_dense)"""
    cols = max(8, (ncol * groups + 295) // 296)
    return (cols + 7) // 8 * 8


@pytest.mark.parametrize("M", [5, 16, 17, 129, 401])
@pytest.mark.parametrize("groups", [1, 3, 16])
def test_argmax_ties_take_the_first_index(M, groups):
    """Heads (V = 2048, K = 256) with a_add: in every group, every row's maximum is shared bit for bit by two columns -- inside
    one tile, across the 32 / 64 / 128 tile boundaries, across the skinny kernel's CTA parts and warps -- and the id must
    be the first one, as torch.argmax gives"""
    N, K = 2048, 256
    cols = _skinny_cols(N, groups)
    bounds = [32, 64, 96, 128, 256, 1024, 2047, cols, 2 * cols, 5 * cols, 9]
    g = torch.Generator().manual_seed(M * 17 + groups)
    A, Ws, Bs, adds, wants = None, [], [], [], []
    for z in range(groups):  # row m aims at pair m % 24 of every group; the groups' pairs sit at different columns
        pairs = P.tie_pairs(N, 24, bounds[z % 3:] + bounds[: z % 3], g)
        assert len(pairs) == 24
        a, w, b, add, want = P.tie_probe(M, N, K, pairs, g, a_add=True)
        A = a if A is None else A  # tie_probe's A has the same structure for every group
        Ws.append(w), Bs.append(b), adds.append(add), wants.append(want)
    W, bias, add, want = torch.stack(Ws), torch.stack(Bs), torch.stack(adds), torch.stack(wants, 1)
    for z in range(groups):  # the float64 logits really tie, and torch.argmax takes the first
        lg = (A.double() + add[z].double()) @ W[z].double().T + bias[z].double()
        top = lg.max(-1, keepdim=True).values
        assert bool(((lg == top).sum(-1) == 2).all()) and torch.equal(lg.argmax(-1), want[:, z])
    for kern in _kernels(M, EPI_ARGMAX):
        ids = _dense(A, W, bias, None, add, epi=EPI_ARGMAX, groups=groups, kernel=kern).cpu().long()
        assert torch.equal(ids, want), (kern, (ids != want).nonzero()[:4].tolist())


def test_argmax_heads_kernel_takes_the_first_maximum():
    """argmax_heads_kernel (the tensor-core path's head argmax, one warp per row and head, lanes stride 4 columns by 128):
    ties inside one lane's float4, across neighbouring lanes, across a lane's strides and across the whole row"""
    _lib_mod, lib = _lib()
    rows, heads, V, Q = 37, 5, 2048, 9
    g = torch.Generator().manual_seed(11)
    lg = torch.randn((rows, heads, V), generator=g)
    ties = [(1, 2), (3, 4), (0, 4), (5, 133), (127, 128), (7, 2047), (0, 2047), (130, 258), (1000, 1001), (2046, 2047)]
    want = torch.empty((rows, heads), dtype=torch.long)
    for r in range(rows):
        for h in range(heads):
            c1, c2 = ties[(r * heads + h) % len(ties)]
            lg[r, h, c1] = lg[r, h, c2] = 10.0 + (r % 3)
            want[r, h] = c1
    assert torch.equal(lg.argmax(-1), want)
    codes = torch.full((rows, Q), -1, dtype=torch.int32, device=DEV)
    d = lg.to(DEV).contiguous()
    _lib_mod.check(lib.sopro_debug_argmax_heads(_p(d), rows, heads, V, _p(codes), Q, _st()))
    got = codes.cpu().long()
    assert torch.equal(got[:, :heads], want) and bool((got[:, heads:] == -1).all())
    assert lib.sopro_debug_argmax_heads(_p(d), rows, heads, V - 2, _p(codes), Q, _st()) != 0  # V % 4 != 0
    assert lib.sopro_debug_argmax_heads(_p(d), rows, heads, V, _p(codes), heads - 1, _st()) != 0


def test_dense_hook_refuses_what_the_kernels_do_not_take():
    _lib_mod, lib = _lib()
    A = torch.zeros((32, 64), device=DEV)
    W = torch.zeros((64, 64), device=DEV)
    b = torch.zeros(64, device=DEV)
    Cb = torch.full((32, 64), 7.0, device=DEV)

    def rc(M=32, N=64, K=64, epi=EPI_BIAS, kernel=0, groups=1, ldc=64):
        return lib.sopro_debug_dense(_p(A), _p(W), _p(b), None, None, None, _p(Cb), 0.0, M, N, K, ldc, epi, groups, 0, 0, 0, kernel,
                                     None, None, 0, _st())

    assert rc() == 0
    Cb.fill_(7.0)
    bad = [dict(kernel=16), dict(kernel=48), dict(epi=EPI_GLU, kernel=32, ldc=32), dict(K=40), dict(ldc=63), dict(epi=9),
           dict(epi=EPI_ARGMAX), dict(groups=2), dict(epi=EPI_RES), dict(M=16, K=4096, kernel=16)]
    for kw in bad:
        assert rc(**kw) != 0, kw
    torch.cuda.synchronize()
    assert bool((Cb == 7.0).all())  # nothing was launched


# ---------------------------------------------------------------------------------------------------------------
# the six-product tensor-core GEMM
# ---------------------------------------------------------------------------------------------------------------
def _pack_w6(W):
    lib_mod, lib = _lib()
    N, K = W.shape
    Wc = W.float().contiguous().cpu()
    out = torch.empty((N, 6 * K), dtype=torch.int16)
    lib_mod.check(lib.sopro_debug_pack_w6(_p(Wc), N, K, _p(out)))
    return out.to(DEV)


def _tc6(X, W6, bias=None, R=None, epi=TC_NONE, norm_w=None, C_out=None):
    """-> (C [M][N] fp32, A3 [M][3K] bf16 as the kernel split X)"""
    lib_mod, lib = _lib()
    M, K = X.shape
    N = W6.shape[0]
    Xd, bias, R, norm_w = _d(X), _d(bias), _d(R), _d(norm_w)
    A3 = torch.full((M, 3 * K), float("nan"), dtype=torch.bfloat16, device=DEV)
    C_out = torch.full((M, N), float("nan"), device=DEV) if C_out is None else C_out
    lib_mod.check(lib.sopro_debug_tc6(_p(Xd), _p(norm_w), _p(W6), _p(bias), _p(R), _p(C_out), _p(A3), M, N, K, epi, _st()))
    return C_out, A3


def test_device_split_is_exact_and_round_to_nearest():
    """split3_rows_kernel without norm_w: h + m + l == x bit for bit, each term the RNE bf16 of the previous residual,
    |m| <= 2^-8 |h|, |l| <= 2^-16 |h|.  Checked for 2^-100 <= |x| <= 2^100: below about 2^-110 the bf16 l underflows
    (its exponent leaves the normal range while x itself is still an fp32 normal) and h + m + l == x no longer holds."""
    M, K, N = 129, 384, 64
    g = torch.Generator().manual_seed(2)
    e = torch.randint(-100, 100, (M, K), generator=g).double()
    X = ((1 + torch.rand((M, K), generator=g, dtype=torch.float64)) * torch.exp2(e) *
         torch.where(torch.rand((M, K), generator=g) < 0.5, -1.0, 1.0).double()).float()
    X[0, :8] = torch.tensor([1.0, -1.0, 2.0 ** -100, 2.0 ** 100, 1 + 2.0 ** -23, 3.0, -0.1, 1e-20])
    W6 = _pack_w6(torch.zeros((N, K)))
    _C, A3 = _tc6(X, W6)
    a = A3.cpu().float().view(M, 3, K)
    h, m, l = a[:, 0], a[:, 1], a[:, 2]
    assert torch.equal(h, X.to(torch.bfloat16).float())
    r1 = X - h  # exact in fp32
    assert torch.equal(m, r1.to(torch.bfloat16).float())
    assert torch.equal(l, (r1 - m).to(torch.bfloat16).float())
    assert torch.equal(h.double() + m.double() + l.double(), X.double())
    assert bool((m.abs() <= 2.0 ** -8 * h.abs()).all()) and bool((l.abs() <= 2.0 ** -16 * h.abs()).all())


@pytest.mark.parametrize("M", [17, 129, 2049])
@pytest.mark.parametrize("N,K", [(64, 64), (768, 384), (256, 1536)])
def test_pair_probes_are_returned_exactly(M, N, K):
    """Each output is one probe product x w with x = s (1 + 2^-10 + 2^-19), w = t (1 + 2^-12 + 2^-21): the six kept term
    products are one distinct bit each and their exact sum fits fp32, so the kernel must return it exactly.  A pair with
    the wrong x or w term, a wrong tap column or [h|m|l] block, or a missing term changes the value
    (tests/test_nar_reference_cpu.py proves that for every such change)."""
    g = torch.Generator().manual_seed(M + N + K)
    X, W, want = P.pair_probe(M, N, K, g)
    got, _ = _tc6(X, _pack_w6(W))
    bad = (got.cpu().double() != want).nonzero()
    assert bad.numel() == 0, f"{bad.shape[0]} of {M * N} probe outputs differ, first {bad[:4].tolist()}"


# the refiner's tensor-core contractions: (name, N, K, epi); heads: 3 heads of V = 2048 over Hn = 256
TC_PROD = [("glu", 768, 384, TC_NONE), ("ffn1", 1536, 384, TC_GELU), ("ffn2", 384, 1536, TC_RES), ("pre", 256, 384, TC_NONE),
           ("heads", 3 * 2048, 256, TC_NONE)]


@pytest.mark.parametrize("name,N,K,epi", TC_PROD, ids=[p[0] for p in TC_PROD])
@pytest.mark.parametrize("M", [17, 127, 128, 129, 2047, 2048, 2049, 4097])
def test_tc6_random_operands_against_float64(name, N, K, epi, M):
    """Elementwise: |c - c64| <= (2^-22 + 6K 2^-23) sum|x w| (+ the epilogue's roundings): the three dropped pairs are below
    2^-23 of each product together, and wgmma's fp32 accumulation is not documented as round-to-nearest, so each of the 6K
    additions is allowed a full ulp.  The sharp check: the RMS error over all outputs is at most 2x that of the fp32 FMA
    tile kernel on the same operands -- 'the fp32 result up to summation order'.  FFN2 runs in place (R aliased to C).
    Measured on an H100 80GB HBM3 (400 W): RMS ratio 0.8 - 1.04 at K = 256 / 384, but 2.19 - 2.21 at FFN2's K = 1536 (6K =
    9216 accumulations in wgmma), so FFN2 is held to 2.5x."""
    g = torch.Generator().manual_seed(M * 7 + N)
    X = torch.randn((M, K), generator=g)
    W = torch.randn((N, K), generator=g) / math.sqrt(K)
    bias = 0.1 * torch.randn((N,), generator=g)
    nw = 1 + 0.1 * torch.randn((K,), generator=g)
    norm = nw if name in ("glu", "ffn1", "pre") else None
    R = torch.randn((M, N), generator=g) if epi == TC_RES else None
    depi = {TC_NONE: EPI_BIAS, TC_GELU: EPI_GELU, TC_RES: EPI_RES}[epi]
    Cin = R.to(DEV).clone() if R is not None else None
    got, _ = _tc6(X, _pack_w6(W), bias, Cin, epi, norm, C_out=Cin)
    fma = _dense(X, W, bias, norm, None, R, 0.0, depi, kernel=128)
    A64 = X.to(DEV, torch.float64)
    if norm is not None:
        A64 = A64 * torch.rsqrt(A64.pow(2).mean(-1, keepdim=True) + 1e-6) * norm.to(DEV, torch.float64)
    W64 = W.to(DEV, torch.float64)
    acc = A64 @ W64.T + bias.to(DEV, torch.float64)
    mag = A64.abs() @ W64.abs().T
    out64 = acc if epi == TC_NONE else (0.5 * acc * (1 + torch.erf(acc / math.sqrt(2))) if epi == TC_GELU else R.to(DEV, torch.float64) + acc)
    extra = (K // 32 + 12) * U if norm is not None else 0.0
    b = (2.0 ** -22 + 6 * K * 2.0 ** -23 + extra) * mag + 2 * U * acc.abs()
    if epi == TC_GELU:
        b = 1.2 * b + 8 * U * acc.abs()
    elif epi == TC_RES:
        b = b + 2 * U * out64.abs()
    err = (got.double() - out64).abs()
    assert float((err / (b + 1e-30)).max()) <= 1.0
    rms_tc = float(err.pow(2).mean().sqrt())
    rms_fma = float((fma.double() - out64).pow(2).mean().sqrt())
    print(f"tc6 {name} M={M}: rms error {rms_tc:.3e} (fp32 FMA tile kernel {rms_fma:.3e}, ratio {rms_tc / rms_fma:.2f})")
    assert rms_tc <= (2.5 if K > 1024 else 2.0) * rms_fma, (rms_tc, rms_fma)


def test_tc6_full_stage_e_heads():
    """all 16 heads of the largest stage in one launch (N = 16 x 2048), as the refiner's head chunks run them"""
    M, N, K = 1025, 16 * 2048, 256
    g = torch.Generator().manual_seed(99)
    X, W, want = P.pair_probe(M, N, K, g)
    got, _ = _tc6(X, _pack_w6(W))
    assert torch.equal(got.double(), want.to(DEV))


def test_tc6_refuses_unsupported_shapes():
    lib_mod, lib = _lib()
    X = torch.zeros((64, 128), device=DEV)
    W6 = torch.zeros((64, 6 * 128), dtype=torch.int16, device=DEV)
    A3 = torch.zeros((64, 3 * 128), dtype=torch.bfloat16, device=DEV)
    Cb = torch.full((64, 64), 7.0, device=DEV)
    for M, N, K, epi in ((64, 40, 128, 0), (64, 64, 48, 0), (64, 64, 100, 0), (0, 64, 128, 0), (64, 64, 128, 2), (64, 64, 128, TC_RES)):
        assert lib.sopro_debug_tc6(_p(X), None, _p(W6), None, None, _p(Cb), _p(A3), M, N, K, epi, _st()) != 0, (M, N, K, epi)
    torch.cuda.synchronize()
    assert bool((Cb == 7.0).all()) and bool((A3 == 0).all())


# ---------------------------------------------------------------------------------------------------------------
# depthwise conv + residual
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [1, 7, 11])
@pytest.mark.parametrize("dil", [1, 2, 4, 8])
@pytest.mark.parametrize("causal", [False, True])
def test_dwconv_res_ragged_rows(k, dil, causal):
    """out[b][t] = x + bias + sum_j h[t + j dil - left] w_j over t < lens[b], zero outside [0, lens[b]).  Rows of h at or past
    lens[b] hold NaN (a read would poison the output); output rows at or past lens[b] start as NaN and must stay NaN."""
    lib_mod, lib = _lib()
    lens = torch.tensor([1, 37, 64, 2, 60, 19])
    B, T, D = len(lens), 64, 384
    total = (k - 1) * dil
    left = total if causal else total // 2
    g = torch.Generator().manual_seed(k * 100 + dil + causal)
    h = torch.randn((B, T, D), generator=g)
    x = torch.randn((B, T, D), generator=g)
    w = torch.randn((D, k), generator=g) / math.sqrt(k)
    bias = 0.1 * torch.randn((D,), generator=g)
    valid = torch.arange(T)[None, :] < lens[:, None]
    h[~valid] = float("nan")
    out = torch.full((B, T, D), float("nan"), device=DEV)
    hd, xd, wd, bd = (t.to(DEV).contiguous() for t in (h, x, w, bias))
    ln = lens.to(DEV, torch.int32)
    lib_mod.check(lib.sopro_debug_dwconv_res(_p(hd), _p(xd), _p(wd), _p(bd), _p(out), _p(ln), B, T, D, k, dil, left, _st()))
    got = out.cpu().double()
    h0 = torch.where(valid[..., None], h, torch.zeros(())).double()
    acc = torch.zeros((B, T, D), dtype=torch.float64)
    mag = torch.zeros((B, T, D), dtype=torch.float64)
    for j in range(k):
        s = j * dil - left  # out[t] reads h[t + s]
        sh = torch.zeros_like(h0)
        lo, hi = max(0, -s), min(T, T - s)
        if lo < hi:
            sh[:, lo:hi] = h0[:, lo + s:hi + s]
        acc += sh * w[:, j].double()
        mag += (sh * w[:, j].double()).abs()
    want = x.double() + (acc + bias.double())
    bound = P.gamma(k + 2) * (mag + bias.double().abs() + x.double().abs())
    assert bool(got[~valid].isnan().all()), "an output row past lens[b] was written"
    assert bool(torch.isfinite(got[valid]).all()), "a padding row of h was read"
    assert float(((got - want).abs()[valid] / bound[valid].clamp_min(1e-30)).max()) <= 1.0
