"""Float64 references of Mimi's fp32 kernels, in the operand layouts the kernels take (channel-last, convs as implicit
GEMMs over [rows][Cin]).  tests/test_mimi_f32_kernels_gpu.py holds each kernel to them; tests/test_mimi_f32_kernels_cpu.py
pins them to oracle/mimi_oracle.py, the restatement of the reference's model."""
import math

import numpy as np
import torch

U = 2.0 ** -24  # unit roundoff of fp32 (round to nearest)


def gamma(n):
    """gamma_n = n u / (1 - n u): the relative error bound of a length-n chain of fp32 roundings"""
    return n * U / (1 - n * U)


def im2col(X, M, Min, taps, dil, pad):
    """X [B][>= Min][Cin] -> A' [B][M][taps*Cin] with A'[m][(j, ci)] = X[m + j*dil - pad][ci], zero outside [0, Min)"""
    B, _, Cin = X.shape
    cols = []
    m = torch.arange(M, device=X.device)
    for j in range(taps):
        r = m + j * dil - pad
        ok = (r >= 0) & (r < Min)
        g = X[:, r.clamp(0, Min - 1)]
        cols.append(torch.where(ok[None, :, None], g, torch.zeros((), dtype=X.dtype, device=X.device)))
    return torch.cat(cols, dim=-1)


def gemm_ref(X, W, M, Min, taps, dil, pad, bias=None, bias_mod=None, elu=False):
    """float64 sum_k act(A'[m][k]) W[n][k] + bias[n % bias_mod] -> (value [B][M][N], sum_k |act(A') W| [B][M][N])"""
    X, W = X.double(), W.double()
    if elu:
        X = torch.nn.functional.elu(X)
    A = im2col(X, M, Min, taps, dil, pad)
    v = A @ W.t()
    mag = A.abs() @ W.abs().t()
    if bias is not None:
        N = W.shape[0]
        v = v + bias.double()[torch.arange(N, device=W.device) % bias_mod]
    return v, mag


def convT_as_2tap(w, r):
    """A ConvTranspose1d weight [Cin][Cout][2r] (stride r) -> the GEMM weight [(phase, co)][(tap, ci)] of the 2-tap conv
    over the input rows: output row t*r + phase = x[t-1] . w[.., phase + r] + x[t] . w[.., phase] (sopro_mimi_create's
    repack); bias index n % Cout."""
    cin, cout, k = w.shape
    assert k == 2 * r
    tw = torch.empty(r * cout, 2 * cin, dtype=w.dtype)
    for ph in range(r):
        tw[ph * cout: (ph + 1) * cout, :cin] = w[:, :, ph + r].t()
        tw[ph * cout: (ph + 1) * cout, cin:] = w[:, :, ph].t()
    return tw


def conv_repack(w):
    """A conv weight [Cout][Cin][k] -> [Cout][(tap, ci)]; a stride-r conv of kernel 2r is then the 2-tap conv over the
    superrow view [L/r][r*Cin] with this same weight (taps j = j2*r + rr ordered (j2, rr, ci))"""
    co, ci, k = w.shape
    return w.permute(0, 2, 1).reshape(co, k * ci)


def superrows(x, r):
    """[B][L][C] -> [B][ceil(L/r)][r*C]: the rows zero padded to a multiple of r (MimiConv1d's extra padding), then
    read r rows at a time"""
    B, L, C = x.shape
    Lp = -(-L // r) * r
    y = torch.zeros(B, Lp, C, dtype=x.dtype)
    y[:, :L] = x
    return y.reshape(B, Lp // r, r * C)


def rope_table(n, Dh, theta=10000.0):
    """make_rope's table [cos rows 0..n) | sin rows 0..n)] of Dh/2 floats, in its fp32 arithmetic"""
    d = torch.arange(Dh // 2, dtype=torch.float32)
    inv = torch.ones(()) / torch.pow(torch.tensor(theta, dtype=torch.float32), (2 * d) / Dh)
    f = torch.arange(n, dtype=torch.float32)[:, None] * inv[None, :]
    return torch.cat([torch.cos(f), torch.sin(f)], dim=0).contiguous()


def rope64(x, pos, table, tab_n):
    """float64 rotation of fp32 x [..., T][H][Dh] at positions pos [T] with the fp32 table's values -> (rotation, the
    sum of its two products' magnitudes)"""
    half = x.shape[-1] // 2
    c = table[pos].double()[:, None, :]
    s = table[tab_n + pos].double()[:, None, :]
    x = x.double()
    x1, x2 = x[..., :half], x[..., half:]
    return (torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], dim=-1),
            torch.cat([(x1 * c).abs() + (x2 * s).abs(), (x2 * c).abs() + (x1 * s).abs()], dim=-1))


def window_attention(q, k, v, window, pos0=0, k_past=None, v_past=None):
    """float64 causal sliding-window attention of the queries at positions pos0 + i over the keys at positions
    (p - window, p]; q, k, v [B][T][H][Dh] are this chunk's rows, k_past / v_past the earlier positions [B][pos0][H][Dh]
    (None when pos0 = 0).  Returns out [B][T][H][Dh] and the probabilities [B][H][T][pos0 + T]."""
    if pos0:
        k = torch.cat([k_past, k], dim=1)
        v = torch.cat([v_past, v], dim=1)
    q, k, v = q.double(), k.double(), v.double()
    T, P = q.shape[1], k.shape[1]
    i = torch.arange(T)[:, None] + pos0
    j = torch.arange(P)[None, :]
    ok = (j <= i) & (j > i - window)
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) / math.sqrt(q.shape[-1])
    p = torch.softmax(s.masked_fill(~ok, float("-inf")), dim=-1)
    return torch.einsum("bhqk,bkhd->bqhd", p, v), p


def seq_sum_f32(x, axis):
    """float32 sum along `axis` in index order, one rounding per addition (numpy, no pairwise summation)"""
    x = np.moveaxis(np.asarray(x, dtype=np.float32), axis, 0)
    s = np.zeros(x.shape[1:], dtype=np.float32)
    for t in x:
        s = (s + t).astype(np.float32)
    return s
