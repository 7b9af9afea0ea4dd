"""The tensor-core mode's Mimi kernels one at a time, against float64 references on the same bf16 operands.

End to end, the tensor-core decode is compared with models whose own bf16 rounding is larger than many kernel bugs
(a window off by one key moves the waveform by ~8e-4 of its peak).  Here each kernel is driven through its test hook
(include/sopro_b200.h) and held to what its arithmetic allows:
  * attn_tc_kernel (sliding-window attention): bit-exact on probes whose softmax is exact (every key count is an integer),
    and a per-element bound on random operands;
  * resblock_tc_kernel (fused ResnetBlock): bit-equal to the unfused pair of tensor-core GEMMs and to itself with
    context rows (the stream's geometry), near a float64 reference;
  * rope_pack_kernel (RoPE + bf16 packing of the attention operands): one bf16 ulp of the float64 rotation, v exact;
  * igemm_tc_kernel (every other contraction of the mode, through the decoder's launcher gemm_tc) at every geometry
    the decoder and its streams launch: bit-exact on dyadic operands, a derived per-element bound on random ones,
    sentinels around every item, and output rows that do not depend on the launch around them (tests/mimi_tc_refs.py).
"""
import ctypes as C
import dataclasses

import pytest
import torch

from tests import mimi_tc_refs as T

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
BF16 = torch.bfloat16
DH = 64  # head dim of the tensor-core attention


def _lib():
    from sopro_b200 import _lib

    return _lib, _lib.load()


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _bf(x):
    """round to bf16 (round to nearest even), back in the input's dtype"""
    return x.to(BF16).to(x.dtype)


def _bf16_ulp(x):
    """spacing of bf16 values at |x| (0 where x == 0)"""
    _, e = torch.frexp(x.double())
    return torch.where(x == 0, torch.zeros_like(x, dtype=torch.float64), torch.ldexp(torch.ones_like(x, dtype=torch.float64), e - 8))


# ---------------------------------------------------------------------------------------------------------------
# attention
# ---------------------------------------------------------------------------------------------------------------
ATTN_T2 = [1, 5, 127, 128, 129, 250, 251, 256, 257, 300, 383, 384, 385, 1000, 2503]
WINDOWS = [1, 2, 127, 128, 129, 250, 256, 257]  # 257: the largest window the 384-key tile takes


def _attn(q, k, v, H, window):
    """q, k, v: bf16 [B][T2][C] on the device -> the kernel's bf16 output.  v goes in transposed with a NaN pad up to
    the 8-aligned pitch: the kernel must never read past key T2 - 1."""
    lib_mod, lib = _lib()
    B, T2, Cc = q.shape
    T2p = (T2 + 7) // 8 * 8
    vt = torch.full((B, Cc, T2p), float("nan"), dtype=BF16, device=q.device)
    vt[:, :, :T2] = v.transpose(1, 2)
    out = torch.full((B, T2, Cc), float("nan"), dtype=BF16, device=q.device)
    lib_mod.check(lib.sopro_debug_tc_attn(_p(q), _p(k), _p(vt), _p(out), B, T2, T2p, Cc, H, window, _st()))
    torch.cuda.synchronize()
    return out.cpu()


def _probe_v(B, T2, H):
    """v of key j, head h, item b: one-hot in channel (j + 7h + 13b) % 64 -- every key of a window is a different
    channel pattern, shifted per head and per item"""
    j = torch.arange(T2)[None, :, None]
    h = torch.arange(H)[None, None, :]
    b = torch.arange(B)[:, None, None]
    ch = (j + 7 * h + 13 * b) % DH  # [B][T2][H]
    return torch.nn.functional.one_hot(ch, DH)  # [B][T2][H][64] int


def _probe_want(B, T2, H, window):
    """the exact output when every probability is 1: per query, (keys of the window in channel c) / (window length),
    as the kernel rounds it: bf16(fp32(count) * fp32(1 / n))"""
    cs = torch.cumsum(_probe_v(B, T2, H), dim=1)  # [B][T2][H][64]
    i = torch.arange(T2)
    lo = (i - window).clamp(min=-1)  # count = cs[i] - cs[i - window] (cs[-1] = 0)
    prev = torch.where((lo >= 0)[None, :, None, None], cs[:, lo.clamp(min=0)], torch.zeros_like(cs))
    count = (cs - prev).float()
    n = (i - lo).float()
    inv = torch.ones(()) / n  # fp32 division, correctly rounded like the kernel's 1.0f / sum
    return (count * inv[None, :, None, None]).to(BF16).reshape(B, T2, H * DH)


def _probes(B, T2, H, window, dev):
    """window probe (q = 0: every score 0) and masked-max probe (every in-window score -900, every zero-filled key of
    the tile 0); both must give the exact output"""
    Cc = H * DH
    g = torch.Generator().manual_seed(T2 * 1000 + window)
    v = _probe_v(B, T2, H).reshape(B, T2, Cc).to(BF16).to(dev)
    want = _probe_want(B, T2, H, window)
    q = torch.zeros(B, T2, Cc, dtype=BF16, device=dev)
    k = torch.randn(B, T2, Cc, generator=g).to(BF16).to(dev)
    got = _attn(q, k, v, H, window)
    bad = (got != want).nonzero()
    assert bad.numel() == 0, f"window probe B={B} T2={T2} H={H} window={window}: {bad.shape[0]} elements differ, first {bad[:4].tolist()}"
    q = torch.zeros(B, T2, Cc)
    k = torch.zeros(B, T2, Cc)
    q[:, :, ::DH] = 30.0
    k[:, :, ::DH] = -30.0
    got2 = _attn(q.to(BF16).to(dev), k.to(BF16).to(dev), v, H, window)
    assert bool(torch.isfinite(got2.float()).all()), f"masked-max probe B={B} T2={T2} window={window}: non-finite output"
    assert torch.equal(got2, got), f"masked-max probe B={B} T2={T2} H={H} window={window}"


def _attn_ref(q, k, v, window):
    """float64 model of attn_tc_kernel on the bf16 operands q, k, v [B][T2][H][64] (CPU): S = q.k^T, the max over the
    valid keys (i - window < j <= i), P = bf16(exp((S - max) / 8)), out = (P.V) / sum(P), computed per block of 128
    queries over its key band only.  Returns the output (before its bf16 rounding) and a per-element allowance for
    probabilities whose float64 value lies so close to a bf16 rounding boundary that the kernel's fp32 exponent
    argument may round it the other way (each such flip moves the output by one ulp of P times |v| / sum(P))."""
    B, T2, H, D = q.shape
    q, k, v = q.double(), k.double(), v.double()
    out = torch.empty(B, T2, H, D, dtype=torch.float64)
    flip = torch.empty(B, T2, H, D, dtype=torch.float64)
    for q0 in range(0, T2, 128):
        q1 = min(q0 + 128, T2)
        k0 = max(0, q0 - window + 1)
        i = torch.arange(q0, q1)[:, None]
        j = torch.arange(k0, q1)[None, :]
        ok = (j <= i) & (j > i - window)  # [nq][nk]
        qb, kb, vb = q[:, q0:q1], k[:, k0:q1], v[:, k0:q1]
        s = torch.einsum("bqhd,bkhd->bhqk", qb, kb)
        mag = torch.einsum("bqhd,bkhd->bhqk", qb.abs(), kb.abs())  # sum |q_d k_d|: the size of the fp32 rounding in S
        s = s.masked_fill(~ok, float("-inf"))
        mx, arg = s.max(dim=-1, keepdim=True)
        x = torch.exp((s - mx) / 8)  # 0 outside the window
        pr = _bf(x)
        den = pr.sum(dim=-1, keepdim=True)
        o = torch.einsum("bhqk,bkhd->bqhd", pr, vb) / den.permute(0, 2, 1, 3)
        # rounding-boundary allowance: the kernel's exponent argument carries ~2^-23 of (|S| terms + |max| terms) / 8
        # plus exp2f's own error; flag probabilities within 2^-19 of that (relative) of a bf16 midpoint
        mag_mx = torch.gather(mag, -1, arg)
        delta = 2.0 ** -19 * (1.0 + (mag + mag_mx) / 8 + (s - mx).abs().nan_to_num(0.0, 0.0, 0.0) / 8)
        ulp = _bf16_ulp(x)
        near = ok & (x > 0) & ((ulp / 2 - (x - pr).abs()).abs() <= delta * x)
        w = torch.where(near, ulp, torch.zeros_like(ulp)) / den  # [B][H][nq][nk]
        flip[:, q0:q1] = torch.einsum("bhqk,bkhd->bqhd", w, vb.abs()) + w.sum(-1).permute(0, 2, 1)[..., None] * o.abs()
        out[:, q0:q1] = o
    return out, flip


def _attn_random(B, T2, H, window, score_scale, seed, dev):
    Cc = H * DH
    g = torch.Generator().manual_seed(seed)
    q = (torch.randn(B, T2, H, DH, generator=g) * score_scale).to(BF16)
    k = (torch.randn(B, T2, H, DH, generator=g) * score_scale).to(BF16)
    v = torch.randn(B, T2, H, DH, generator=g).to(BF16)
    got = _attn(q.reshape(B, T2, Cc).to(dev), k.reshape(B, T2, Cc).to(dev), v.reshape(B, T2, Cc).to(dev), H, window)
    got = got.reshape(B, T2, H, DH).double()
    ref, flip = _attn_ref(q, k, v, window)
    vmax = float(v.float().abs().max())
    tol = 2.0 ** -7 * ref.abs() + 2.0 ** -10 * vmax + flip
    d = (got - ref).abs()
    worst = float((d / (2.0 ** -7 * ref.abs() + 2.0 ** -10 * vmax)).max())
    print(f"tc attention B={B} T2={T2} H={H} window={window} scale={score_scale}: max |got-ref| {float(d.max()):.2e}, "
          f"worst / (2^-7|ref| + 2^-10 max|v|) = {worst:.3f}, {int((flip > 0).sum())} outputs see a probability at a rounding boundary")
    assert bool(torch.isfinite(got).all())
    bad = (d > tol).nonzero()
    assert bad.numel() == 0, (B, T2, H, window, score_scale, bad[:4].tolist(), float(d.max()))


@pytest.mark.parametrize("T2", ATTN_T2)
def test_attention_probes_are_exact(T2):
    """Exact-softmax probes over B = 1..3 and every window of the sweep at Mimi's geometry (H = 8, C = 512): partial
    query tiles, a second warpgroup without rows, key tiles starting before position 0 and reaching past T2.  One key
    too many or too few, a key of another item, or a key block skipped wrongly changes a channel by 1 / n."""
    dev = torch.device("cuda:0")
    for wi, window in enumerate(WINDOWS):
        _probes(1 + (wi % 3), T2, 8, window, dev)
    for B in (1, 2, 3):
        _probes(B, T2, 8, 250, dev)


@pytest.mark.parametrize("H", [1, 2, 8])
def test_attention_window_sweep(H):
    """T2 = 700 (past two query tiles of 128 + the window): every window of the sweep, probes and random operands."""
    dev = torch.device("cuda:0")
    for window in WINDOWS:
        _probes(2, 700, H, window, dev)
        _attn_random(2, 700, H, window, 1.0, 7 * window + H, dev)


@pytest.mark.parametrize("B", [1, 2, 3])
@pytest.mark.parametrize("T2", ATTN_T2)
def test_attention_random_operands(B, T2):
    """Random bf16 q / k / v at Mimi's geometry (H = 8, C = 512, window 250), unit-sized scores and scores scaled until
    the softmax is peaked (|S / 8| up to ~60).  Per element: |got - ref| <= 2^-7 |ref| + 2^-10 max|v| (one bf16
    rounding of the output, accumulation order), plus the allowance for probabilities at a bf16 rounding boundary."""
    dev = torch.device("cuda:0")
    for score_scale in (1.0, 3.8):
        _attn_random(B, T2, 8, 250, score_scale, 1000 * B + T2 + int(10 * score_scale), dev)


# ---------------------------------------------------------------------------------------------------------------
# fused ResnetBlock
# ---------------------------------------------------------------------------------------------------------------
def _resblock(X, W1, W2, b1, b2, Z, ctx, hid, taps, out_elu, want_f32=True, want_bf16=True):
    lib_mod, lib = _lib()
    B, M, cout = Z.shape
    of = torch.full((B, M, cout), float("nan"), device=Z.device) if want_f32 else None
    oh = torch.full((B, M, cout), float("nan"), dtype=BF16, device=Z.device) if want_bf16 else None
    lib_mod.check(lib.sopro_debug_tc_resblock(_p(X), _p(W1), _p(W2), _p(b1), _p(b2), _p(Z), _p(of), _p(oh), B, M, ctx, hid, taps,
                                              out_elu, _st()))
    torch.cuda.synchronize()
    return of, oh


def _resblock_pitched(X, W1, W2, b1, b2, Z, ctx, hid, taps):
    """The stream's layout of the same launch (seanet_tc: X and Z at z's pitch, the bf16 output at o's pitch behind o's
    context row): X, Z and both outputs each at its own item pitch, X's rows past ctx + M and Z's past M NaN (never
    read), every output element outside rows [0, M) of an item a sentinel (never written).  Returns the packed
    [B][M][2 hid] outputs after checking the sentinels."""
    lib_mod, lib = _lib()
    B, M, cout = Z.shape
    a_pitch, z_pitch, o_pitch = ctx + M + 3, M + 2, M + 5
    Xp = T.pitched_rows(X, a_pitch, float("nan"))
    Zp = T.pitched_rows(Z, z_pitch, float("nan"))
    L = T.Launch(T.Layer("resblock", cout, taps, cout, 0, T.EPI_RES, True, True, True), B, M, ctx, a_pitch, o_pitch, 0, cout)
    of = T.f32_sentinel(B * o_pitch * cout + cout, Z.device)
    oh = T.bf16_sentinel(cout + B * o_pitch * cout + cout, Z.device)
    lib_mod.check(lib.sopro_debug_tc_resblock_pitched(_p(Xp), _p(W1), _p(W2), _p(b1), _p(b2), _p(Zp), _p(of), _p(oh[cout:]), B, M, ctx,
                                                      a_pitch, z_pitch, o_pitch, hid, taps, 1, _st()))
    torch.cuda.synchronize()
    T.check_guards(L, of, oh, f"fused ResnetBlock hid={hid} taps={taps} B={B} M={M} pitched")
    return T.f32_rows(L, of)[:, :M], T.bf16_rows(L, oh)[0][:, :M]


def _gemm(X, rows, cin, taps, pad, W, N, bias, epi, R, of, oh, out_elu):
    lib_mod, lib = _lib()
    lib_mod.check(lib.sopro_debug_tc_gemm(_p(X), X.shape[0], rows, cin, taps, 1, pad, _p(W), N, _p(bias), N, epi, _p(R), None,
                                          _p(of), _p(oh), out_elu, _st()))


def _resblock_ref(X, W1, W2, b1, b2, Z, taps):
    """float64: Z + W2 . bf16(ELU(causal conv_taps(X; W1) + b1)) + b2 on the bf16 operands (CPU).  Also returns, per
    output element, an allowance for hidden values whose float64 value lies so close to a bf16 rounding boundary that
    the kernel's fp32 accumulation (error ~2^-23 of sum |x w|) may round them the other way: each such flip moves the
    output by one ulp of the hidden value times |W2|."""
    X, W1, W2 = X.double(), W1.double(), W2.double()
    B, M, cin = X.shape
    cols = []
    for j in range(taps):
        sh = j - (taps - 1)
        y = torch.zeros_like(X)
        y[:, -sh if sh < 0 else 0:] = X[:, : M + sh if sh < 0 else M]
        cols.append(y)
    a = torch.cat(cols, dim=-1)
    e = torch.nn.functional.elu(a @ W1.t() + b1.double())
    h = _bf(e.float()).double()
    ulp = _bf16_ulp(e)
    near = (ulp / 2 - (e - h).abs()).abs() <= 2.0 ** -20 * (a.abs() @ W1.abs().t() + b1.double().abs()) + 4e-7
    allow = torch.where(near, ulp, torch.zeros_like(ulp)) @ W2.abs().t()
    return Z.double() + h @ W2.t() + b2.double(), allow


RES_CASES = [(hid, taps, B, M) for hid in (32, 64, 128) for taps in (1, 3) for B in (1, 3) for M in (1, 5, 127, 128, 129, 1000, 20000)
             if not (M == 20000 and B != 1)]


@pytest.mark.parametrize("hid,taps,B,M", RES_CASES)
def test_fused_resblock(hid, taps, B, M):
    """One fused ResnetBlock launch (hid 32 / 64 / 128: the stages that take it; taps 1 gives a one- or two-stage ring):
      * bit-equal to the unfused path on the same inputs (conv k=taps with out_elu, then the 1x1 conv with EPI_RES):
        same wgmma shapes, the same K-chunk order and the same bias / skip / ELU arithmetic;
      * with ctx = taps - 1 context rows in front (the stream's geometry), bit-equal to the ctx = 0 launch over the
        concatenated rows, restricted to the last M rows;
      * near the float64 reference: per element, the effect of hidden values at a bf16 rounding boundary (one such
        flip at M = 20000 moved an output by 1.03e-3 of the scale on an H100) plus 1e-5 of the output scale for fp32,
        1e-3 of the scale plus one bf16 ulp of the scale for bf16 (an absolute floor: elu_fast's error is absolute,
        see mimi_tc.cuh)."""
    dev = torch.device("cuda:0")
    cout = 2 * hid
    g = torch.Generator().manual_seed(hid * 100000 + taps * 10000 + B * 1000 + M)
    ctx = taps - 1
    Xall = torch.randn(B, ctx + M, cout, generator=g).to(BF16)
    W1 = (torch.randn(hid, taps * cout, generator=g) / (taps * cout) ** 0.5).to(BF16)
    W2 = (torch.randn(cout, hid, generator=g) / hid ** 0.5).to(BF16)
    b1 = torch.randn(hid, generator=g) * 0.3
    b2 = torch.randn(cout, generator=g) * 0.3
    Zall = torch.randn(B, ctx + M, cout, generator=g)
    X, Z = Xall[:, ctx:].contiguous(), Zall[:, ctx:].contiguous()
    d = {n: t.to(dev) for n, t in dict(X=X, W1=W1, W2=W2, b1=b1, b2=b2, Z=Z, Xall=Xall.contiguous(), Zall=Zall).items()}
    of, oh = _resblock(d["X"], d["W1"], d["W2"], d["b1"], d["b2"], d["Z"], 0, hid, taps, 1)
    _, oh0 = _resblock(d["X"], d["W1"], d["W2"], d["b1"], d["b2"], d["Z"], 0, hid, taps, 0, want_f32=False)
    # unfused: conv k=taps -> bf16 ELU(h), then the 1x1 conv + bias + fp32 skip
    h = torch.full((B, M, hid), float("nan"), dtype=BF16, device=dev)
    uf = torch.full((B, M, cout), float("nan"), device=dev)
    uh = torch.full((B, M, cout), float("nan"), dtype=BF16, device=dev)
    _gemm(d["X"], M, cout, taps, taps - 1, d["W1"], hid, d["b1"], 0, None, None, h, 1)
    _gemm(h, M, hid, 1, 0, d["W2"], cout, d["b2"], 3, d["Z"], uf, uh, 1)
    torch.cuda.synchronize()
    assert torch.equal(of, uf), f"fp32 out: fused vs unfused differ at {int((of != uf).sum())} elements, max {float((of - uf).abs().max()):.2e}"
    assert torch.equal(oh, uh), f"bf16 out: fused vs unfused differ at {int((oh != uh).sum())} elements"
    # the stream's geometry: ctx context rows in front, no zero pad; equals the one-shot launch over all rows
    cf, ch = of, oh
    if ctx:
        cf, ch = _resblock(d["Xall"], d["W1"], d["W2"], d["b1"], d["b2"], d["Z"], ctx, hid, taps, 1)
        af, ah = _resblock(d["Xall"], d["W1"], d["W2"], d["b1"], d["b2"], d["Zall"], 0, hid, taps, 1)
        assert torch.equal(cf, af[:, ctx:]) and torch.equal(ch, ah[:, ctx:])
    # the same launch over pitched items (the stream's buffers): bit-equal, nothing outside the items' rows touched
    pf, ph = _resblock_pitched(d["Xall"] if ctx else d["X"], d["W1"], d["W2"], d["b1"], d["b2"], d["Z"], ctx, hid, taps)
    assert torch.equal(pf, cf) and torch.equal(ph, ch), "pitched items differ from packed ones"
    ref, allow = _resblock_ref(X, W1, W2, b1, b2, Z, taps)
    s = float(ref.abs().max())
    e32 = (of.cpu().double() - ref).abs() - allow
    eh = (oh.cpu().double() - torch.nn.functional.elu(ref)).abs() - allow
    eh0 = (oh0.cpu().double() - ref).abs() - allow
    e32, eh, eh0 = float(e32.max()), float(eh.max()), float(eh0.max())
    print(f"fused ResnetBlock hid={hid} taps={taps} B={B} M={M}: beyond the flip allowance: fp32 {e32 / s:.2e}, "
          f"bf16(ELU) {eh / s:.2e}, bf16 {eh0 / s:.2e} of scale; {int((allow > 0).sum())} outputs see a flip allowance")
    assert e32 <= 1e-5 * s  # beyond the flips only accumulation order remains (measured <= 1.7e-7 on an H100)
    assert eh <= 2 ** -8 * s + 1e-3 * s
    assert eh0 <= 2 ** -8 * s + 1e-3 * s


# ---------------------------------------------------------------------------------------------------------------
# RoPE pack
# ---------------------------------------------------------------------------------------------------------------
def _rope_table(n, Dh=DH, theta=10000.0):
    """make_rope's table in its layout [cos rows 0..n) | sin rows 0..n)], fp32 arithmetic as there"""
    d = torch.arange(Dh // 2, dtype=torch.float32)
    inv = torch.ones(()) / torch.pow(torch.tensor(theta, dtype=torch.float32), (2 * d) / Dh)
    f = torch.arange(n, dtype=torch.float32)[:, None] * inv[None, :]
    return torch.cat([torch.cos(f), torch.sin(f)], dim=0).contiguous()


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("T2", [1, 31, 32, 33, 300])
def test_rope_pack(B, T2):
    """rope_pack_kernel with a table built for 4096 positions (as streams size it), more than T2: rotated q and k within
    one bf16 ulp of bf16(float64 rotation of the same fp32 inputs and table) plus 2^-20 (|x1| + |x2|) (the kernel's
    fp32 x1*c - x2*s can cancel); v^T exactly bf16(v) transposed, its pad columns T2..T2p zero."""
    lib_mod, lib = _lib()
    dev = torch.device("cuda:0")
    H, Cc, tab_T2 = 8, 512, 4096
    T2p = (T2 + 7) // 8 * 8
    g = torch.Generator().manual_seed(10 * T2 + B)
    qkv = torch.randn(B, T2, 3 * Cc, generator=g) * 2
    tab = _rope_table(tab_T2)
    qh = torch.full((B, T2, Cc), float("nan"), dtype=BF16, device=dev)
    kh = torch.full((B, T2, Cc), float("nan"), dtype=BF16, device=dev)
    vt = torch.full((B, Cc, T2p), float("nan"), dtype=BF16, device=dev)
    qkv_d, tab_d = qkv.to(dev), tab.to(dev)  # held until the kernel has run
    lib_mod.check(lib.sopro_debug_rope_pack(_p(qkv_d), _p(tab_d), tab_T2, _p(qh), _p(kh), _p(vt), B, T2, Cc, H, _st()))
    torch.cuda.synchronize()
    cos, sin = tab[:T2].double()[None, :, None, :], tab[tab_T2: tab_T2 + T2].double()[None, :, None, :]
    for which, got in ((0, qh), (1, kh)):
        x = qkv[:, :, which * Cc: (which + 1) * Cc].double().view(B, T2, H, DH)
        x1, x2 = x[..., : DH // 2], x[..., DH // 2:]
        ref = torch.cat([x1 * cos - x2 * sin, x2 * cos + x1 * sin], dim=-1)
        want = _bf(ref.float()).double()
        floor = 2.0 ** -20 * torch.cat([x1.abs() + x2.abs()] * 2, dim=-1)
        d = (got.cpu().double().view(B, T2, H, DH) - want).abs()
        tol = _bf16_ulp(want) + floor
        print(f"rope pack B={B} T2={T2} {'qk'[which]}: max distance / tolerance {float((d / tol).max()):.3f}")
        assert bool((d <= tol).all()), ("qk"[which], (d > tol).nonzero()[:4].tolist())
    vt = vt.cpu()
    assert torch.equal(vt[:, :, :T2], qkv[:, :, 2 * Cc:].to(BF16).transpose(1, 2))
    assert bool((vt[:, :, T2:] == 0).all())


# ---------------------------------------------------------------------------------------------------------------
# tensor-core implicit GEMM (igemm_tc_kernel through gemm_tc)
# ---------------------------------------------------------------------------------------------------------------
def _tc_gemm(L, ops):
    """one launch through sopro_debug_tc_gemm_pitched into fresh output buffers filled with the sentinels -> (fp32 buffer,
    bf16 buffer), flat; an in-place launch's fp32 buffer starts as a copy of the residual buffer and is its R"""
    lib_mod, lib = _lib()
    dev = ops.X.device
    n = L.B * L.c_pitch * L.N
    of = ops.R.clone().view(-1) if L.inplace else (T.f32_sentinel(n, dev) if L.f32 else None)
    oh = T.bf16_sentinel(L.h_off + n, dev) if L.bf16 else None
    R = of if L.inplace else ops.R
    lib_mod.check(lib.sopro_debug_tc_gemm_pitched(_p(ops.X), L.B, L.M, L.ctx, L.a_pitch, L.cin, L.taps, _p(ops.W), L.N, _p(ops.bias),
                                                  L.bias_mod, L.epi, _p(R), L.r_pitch, _p(ops.scale), _p(of),
                                                  _p(oh[L.h_off:] if L.bf16 else None), L.c_pitch, int(L.elu), _st()))
    torch.cuda.synchronize()
    return of, oh


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


def _rows(L, of, oh, lo=0, hi=None):
    """rows [lo, hi) of every item of both outputs (None where the layer writes no such output)"""
    hi = L.M if hi is None else hi
    return (T.f32_rows(L, of)[:, lo:hi] if L.f32 else None, T.bf16_rows(L, oh)[0][:, lo:hi] if L.bf16 else None)


def _same_rows(got, want, what):
    for g, w, kind in zip(got, want, ("fp32", "bf16")):
        if g is not None:
            bad = _bits(g) != _bits(w)
            assert not bool(bad.any()), f"{what} {kind}: {int(bad.sum())} elements differ, first {bad.nonzero()[:4].tolist()}"


def _check(L, kind, seed):
    """launch L on `kind` operands and hold it to the float64 reference (T.check_launch); an in-place launch must also
    equal, bit for bit, the same launch with R in a buffer of its own.  Returns the worst ratios to the bound per output."""
    dev = torch.device("cuda:0")
    ops = T.operands(L, kind, seed, dev)
    of, oh = _tc_gemm(L, ops)
    y, a, mag = T.reference(L, ops)
    if kind == "dyadic":  # the sums are exact; only GELU rounds
        err = T.bound(L, y, a, mag, ops, exact_sum=True) if L.epi == T.EPI_GELU else None
    else:
        err = T.bound(L, y, a, mag, ops)
    what = f"{L.name} B={L.B} M={L.M} ctx={L.ctx} pitches a/c/r {L.a_pitch}/{L.c_pitch}/{L.r_pitch} h_off={L.h_off} {kind}"
    worst = T.check_launch(L, of, oh, y, err, what)
    if L.inplace:
        Ls = dataclasses.replace(L, layer=dataclasses.replace(L.layer, inplace=False), r_pitch=L.M + 2)
        sops = dataclasses.replace(ops, R=T.pitched_rows(ops.R[:, : L.M], Ls.r_pitch, T.f32_sentinel(1, dev)))
        sf, sh = _tc_gemm(Ls, sops)
        _same_rows(_rows(Ls, sf, sh), _rows(L, of, oh), what + ": in place vs R apart")
    return worst


LAYERS = T.PRODUCTION + T.TILES


@pytest.mark.parametrize("layer", LAYERS, ids=lambda l: l.name)
def test_tc_gemm_exact_on_dyadic_operands(layer):
    """Every contraction gemm_tc issues (T.PRODUCTION: the transformer's four linears, conv0, the four ConvTransposes,
    stage 0's unfused ResnetBlock) and every tile instantiation and stage-ring edge (T.TILES), over M in {1, 127,
    128, 129, 383, 2053}, every ctx in [0, taps-1], B in {1, 3, 64}, packed and pitched items (T.launches).  Operands
    on the grids of T.dyadic_values, so every fp32 sum is exact: the fp32 output equals float64 bit for bit for NONE,
    RES and RES_SCALE (the fp32 copy next to an ELU'd bf16 copy is not ELU'd), the plain bf16 output is RNE of it,
    the ELU'd bf16 output is within half a bf16 ulp of ELU plus elu_fast's absolute floor (T.ELU_FLOOR), and GELU is
    within its own roundings.  A dropped, doubled or misplaced product, tap or K chunk changes an output.  Operand rows
    past ctx + M are NaN; every output element outside rows [0, M) of an item must keep its sentinel; in-place
    residual launches equal the same launch with R apart."""
    for i, L in enumerate(T.launches(layer)):
        _check(L, "dyadic", 7919 * i + 1)


@pytest.mark.parametrize("layer", LAYERS, ids=lambda l: l.name)
def test_tc_gemm_random_operands(layer):
    """The same sweep on random operands (unit activations, weights scaled by 1/sqrt(K), a bias, a residual, a
    LayerScale of mixed sign), per element within T.bound: the accumulation at 2u per addition of the sum of
    magnitudes, then each epilogue's own roundings and half a bf16 ulp for the bf16 output.  This covers GELU, the
    LayerScale and the rounding of the bf16 output away from exact values."""
    worst = {}
    for i, L in enumerate(T.launches(layer)):
        for k, v in _check(L, "random", 104729 * i + 3).items():
            worst[k] = max(worst.get(k, 0.0), v)
    print(f"tc gemm {layer.name}: random operands, worst |got - ref| / bound: " + ", ".join(f"{k} {v:.3e}" for k, v in worst.items()))


@pytest.mark.parametrize("layer", T.PRODUCTION, ids=lambda l: l.name)
def test_tc_gemm_rows_do_not_depend_on_the_launch(layer):
    """An output row's bits do not depend on M, its row within a tile, ctx, the pitches or B:
      * a stream's chunks (each a pitched launch with the previous chunk's last taps-1 operand rows as context; zero
        rows before the first) equal the one-shot launch (ctx 0, packed) over all 700 rows, row for row;
      * item b of a 64-item launch equals item b launched alone, for every b."""
    dev = torch.device("cuda:0")
    pad = layer.taps - 1
    one = T.launch(layer, 2, 700, 0, pitched=False)
    ops = T.operands(one, "random", 31, dev)
    of, oh = _tc_gemm(one, ops)
    xz = torch.cat([torch.zeros(2, pad, layer.cin, dtype=BF16, device=dev), ops.X], dim=1)
    s = 0
    for cs in (1, 127, 129, 5, 256, 182):
        L = T.launch(layer, 2, cs, pad, pitched=True)
        R = T.pitched_rows(ops.R[:, s: s + cs], L.r_pitch, T.f32_sentinel(1, dev)) if ops.R is not None else None
        cops = T.Operands(T.pitched_rows(xz[:, s: s + pad + cs], L.a_pitch, float("nan")), ops.W, ops.bias, R, ops.scale)
        cf, ch = _tc_gemm(L, cops)
        T.check_guards(L, cf if L.f32 else None, ch, f"{layer.name} chunk at {s}")
        _same_rows(_rows(L, cf, ch), _rows(one, of, oh, s, s + cs), f"{layer.name}: chunk rows [{s}, {s + cs}) vs one-shot")
        s += cs
    assert s == one.M
    L64 = T.launch(layer, 64, 129, pad, pitched=True)
    ops = T.operands(L64, "random", 37, dev)
    of, oh = _tc_gemm(L64, ops)
    L1 = dataclasses.replace(L64, B=1)
    for b in range(64):
        R = ops.R[b: b + 1].clone() if ops.R is not None else None
        f1, h1 = _tc_gemm(L1, T.Operands(ops.X[b: b + 1].clone(), ops.W, ops.bias, R, ops.scale))
        got = _rows(L64, of, oh)
        _same_rows(_rows(L1, f1, h1), tuple(t[b: b + 1] if t is not None else None for t in got), f"{layer.name}: item {b} of 64 vs alone")


@pytest.mark.parametrize("name,M", [("convT_r4", 4_800_000), ("conv0", 20_000)])
def test_tc_gemm_full_size_decode_launches(name, M):
    """The unfused launches of a 10k-frame one-shot decode at full size: the last ConvTranspose over 4.8M input rows
    (a 4.9 GB fp32 output: byte offsets past 2^32) and conv0 over 20000 rows, dyadic operands generated on the device.
    Sampled rows equal float64 exactly (fp32; bf16 ELU within its bound): the first and the last tile, the rows around
    every 2^k * 128 and the last row; one guard row past M keeps its sentinel."""
    dev = torch.device("cuda:0")
    layer = next(l for l in T.PRODUCTION if l.name == name)
    L = dataclasses.replace(T.launch(layer, 1, M, 0, pitched=False), c_pitch=M + 1)
    gen = torch.Generator(device=dev).manual_seed(M)
    X = T.signed_ints(gen, (1, M, layer.cin), 16, dev, torch.int8).to(BF16).div_(16)
    W = (T.signed_ints(gen, (layer.N, layer.K), 16, dev).double() / 256).to(BF16)
    bias = T.signed_ints(gen, (layer.bias_mod,), 64, dev).float() / 64
    ops = T.Operands(X, W, bias, None, None)
    of, oh = _tc_gemm(L, ops)
    T.check_guards(L, of if L.f32 else None, oh, f"{name} M={M}")
    last = (M - 1) // 128 * 128
    windows = [(0, 128), (last, M)] + [(max(0, (128 << k) - 3), (128 << k) + 3) for k in range(20) if (128 << k) + 3 <= M]
    for lo, hi in windows:
        c = min(lo, layer.taps - 1)  # the operand rows the window reads, as context rows in front of it
        Lw = T.launch(layer, 1, hi - lo, c, pitched=False)
        y, _, _ = T.reference(Lw, T.Operands(X[:, lo - c: hi], W, bias, None, None))
        f, b = _rows(L, of, oh, lo, hi)
        T.check_values(Lw, f, b, y, None, f"{name} M={M} rows [{lo}, {hi})")
    print(f"tc gemm {name} M={M}: {len(windows)} sampled row windows exact")
    del X, of, oh, ops
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------
# refusals: a shape the kernels do not take is an error and launches nothing
# ---------------------------------------------------------------------------------------------------------------
def test_tc_gemm_hook_refuses_and_launches_nothing():
    """sopro_debug_tc_gemm_pitched refuses null pointers, B outside [1, 65535], M < 1, ctx outside [0, taps-1], pitches
    shorter than an item, an unknown epilogue, a bias period that is no multiple of 4 or wider than N, misaligned
    pointers and shapes tc::supported rejects, and writes nothing; the same call with valid arguments runs.  Its packed
    form sopro_debug_tc_gemm refuses a dilation or a pad the decoder never issues."""
    _, lib = _lib()
    dev = torch.device("cuda:0")
    cin, N, M = 64, 64, 8
    X = torch.zeros(1, M + 2, cin, dtype=BF16, device=dev)
    W = torch.zeros(N, 3 * cin, dtype=BF16, device=dev)
    bias = torch.zeros(N, device=dev)
    R = torch.zeros(1, M, N, device=dev)
    scale = torch.zeros(N, device=dev)
    of = torch.full((1, M, N), 7.0, device=dev)
    oh = torch.full((1, M, N), 7.0, dtype=BF16, device=dev)
    good = dict(X=_p(X), B=1, M=M, ctx=2, a_pitch=M + 2, cin=cin, taps=3, W=_p(W), N=N, bias=_p(bias), bias_mod=N, epi=T.EPI_RES,
                R=_p(R), r_pitch=M, scale=None, of=_p(of), oh=_p(oh), c_pitch=M, elu=1)

    def call(**kw):
        a = {**good, **kw}
        return lib.sopro_debug_tc_gemm_pitched(a["X"], a["B"], a["M"], a["ctx"], a["a_pitch"], a["cin"], a["taps"], a["W"], a["N"],
                                               a["bias"], a["bias_mod"], a["epi"], a["R"], a["r_pitch"], a["scale"], a["of"], a["oh"],
                                               a["c_pitch"], a["elu"], _st())

    refused = [dict(X=None), dict(W=None), dict(of=None, oh=None), dict(R=None), dict(epi=T.EPI_RES_SCALE), dict(B=0),
               dict(B=65536), dict(M=0), dict(ctx=-1), dict(ctx=3), dict(a_pitch=M + 1), dict(c_pitch=M - 1), dict(r_pitch=M - 1),
               dict(epi=4), dict(epi=-1), dict(bias_mod=2), dict(bias_mod=2 * N), dict(taps=0, ctx=0), dict(cin=48),
               dict(N=48, bias_mod=48), dict(of=C.c_void_p(of.data_ptr() + 4)), dict(X=C.c_void_p(X.data_ptr() + 2))]
    for kw in refused:
        assert call(**kw) != 0, kw
    for dil, pad in ((2, 4), (1, 1), (1, 0)):  # packed form: rows M + 2 of X, 3 taps
        assert lib.sopro_debug_tc_gemm(_p(X), 1, M + 2, cin, 3, dil, pad, _p(W), N, _p(bias), N, T.EPI_NONE, None, None, _p(of), _p(oh), 1,
                                       _st()) != 0, (dil, pad)
    torch.cuda.synchronize()
    assert bool((of == 7.0).all()) and bool((oh.float() == 7.0).all())
    of2, oh2 = torch.full_like(of, 7.0), torch.full_like(oh, 7.0)
    assert call(of=_p(of2), oh=_p(oh2)) == 0
    torch.cuda.synchronize()
    assert bool((of2 == 0).all()) and bool((oh2.float() == 0).all())  # zero operands: R + 0, ELU(0)


def test_hooks_refuse_unsupported_shapes():
    _, lib = _lib()
    dev = torch.device("cuda:0")
    B, T2, H, Cc = 1, 16, 8, 512
    q = torch.zeros(B, T2, Cc, dtype=BF16, device=dev)
    vt = torch.zeros(B, Cc, 24, dtype=BF16, device=dev)
    out = torch.full((B, T2, Cc), 7.0, dtype=BF16, device=dev)
    for T2p, C_, H_, window in ((16, Cc, H, 258), (16, Cc, H, 0), (17, Cc, H, 250), (8, Cc, H, 250), (16, 384, H, 250)):
        assert lib.sopro_debug_tc_attn(_p(q), _p(q), _p(vt), _p(out), B, T2, T2p, C_, H_, window, _st()) != 0
    hid, M = 256, 8
    X = torch.zeros(1, M + 2, 2 * hid, dtype=BF16, device=dev)
    W = torch.zeros(3 * 2 * hid * hid, dtype=BF16, device=dev)
    b = torch.zeros(2 * hid, device=dev)
    Z = torch.zeros(1, M, 2 * hid, device=dev)
    of = torch.full((1, M, 2 * hid), 7.0, device=dev)
    for hid_, taps, ctx in ((256, 3, 0), (48, 3, 0), (64, 3, 3), (64, 3, -1), (64, 1, 1), (64, 0, 0)):
        assert lib.sopro_debug_tc_resblock(_p(X), _p(W), _p(W), _p(b), _p(b), _p(Z), _p(of), None, 1, M, ctx, hid_, taps, 1, _st()) != 0
    for ctx, a_pitch, z_pitch, o_pitch in ((2, M + 1, M, M), (0, M, M - 1, M), (0, M, M, M - 1)):  # an item shorter than its rows
        assert lib.sopro_debug_tc_resblock_pitched(_p(X), _p(W), _p(W), _p(b), _p(b), _p(Z), _p(of), None, 1, M, ctx, a_pitch, z_pitch,
                                                   o_pitch, 64, 3, 1, _st()) != 0
    qkv = torch.zeros(B, T2, 3 * Cc, device=dev)
    tab = _rope_table(T2).to(dev)
    for tab_T2, C_, H_ in ((T2 - 1, Cc, H), (T2, 500, H), (T2, 32 * H, H)):
        assert lib.sopro_debug_rope_pack(_p(qkv), _p(tab), tab_T2, _p(out), _p(out), _p(vt), B, T2, C_, H_, _st()) != 0
    torch.cuda.synchronize()
    assert bool((out.float() == 7.0).all()) and bool((of == 7.0).all())
