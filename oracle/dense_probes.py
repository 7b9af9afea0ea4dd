"""TEST INFRASTRUCTURE (never imported by the product): operand constructions and error bounds for the NAR refiner's and
the prefill's contractions (sopro_b200/csrc/dense_f32.cuh, the six-product tensor-core GEMM of nar_engine.cu).

  * dyadic operands: every product and partial sum is exact in fp32, so a kernel's output equals float64 bit for bit
    whatever its summation order -- a wrong row, column, k-tile or stride cannot hide inside rounding;
  * pair probes: x = s (1 + 2^-10 + 2^-19), w = t (1 + 2^-12 + 2^-21) split into three bf16 terms each; the six kept term
    products (mm, lh, hl, mh, hm, hh) are one distinct bit each, the three dropped ones are <= 2^-31 of the product;
  * tie probes: duplicated weight rows, so two columns give bit-identical logits and the first index must win;
  * the rounding-error bound gamma_n = n u / (1 - n u) of any order of n fp32 additions.
"""
from __future__ import annotations

from fractions import Fraction
from typing import List, Sequence, Tuple

import torch

U = 2.0 ** -24  # fp32 unit roundoff
# the refiner's pre-head activation z on the GPU must stay within KAPPA x the fp32 CPU oracle's error (both against the
# float64 oracle, tests/test_nar_gpu.py); the RMS error of the two-term control must exceed it
# (tests/test_nar_reference_cpu.py: 6.7x).  Measured on an H100 80GB HBM3 (400 W): at most 2.13x (max) and 2.08x (RMS).
# The AR step is held to the same KAPPA per utterance, layer residual, logits and text K / V (tests/test_ar_float64_gpu.py;
# controls in tests/test_ar_float64_cpu.py: 17x and up).  Measured on an H100 80GB HBM3 (700 W): at most 1.34x.
KAPPA = 3.0

# the tensor-core path's kept term pairs (x term, w term), 0 = h, 1 = m, 2 = l: mm, lh, hl, mh, hm, hh
PAIRS: Tuple[Tuple[int, int], ...] = ((1, 1), (2, 0), (0, 2), (1, 0), (0, 1), (0, 0))
PROBE_X = (Fraction(1), Fraction(1, 2 ** 10), Fraction(1, 2 ** 19))  # h, m, l of x = 1 + 2^-10 + 2^-19
PROBE_W = (Fraction(1), Fraction(1, 2 ** 12), Fraction(1, 2 ** 21))  # h, m, l of w = 1 + 2^-12 + 2^-21


def gamma(n) -> torch.Tensor | float:
    return n * U / (1 - n * U)


def dyadic(shape, lo: int, hi: int, scale_log2: int, gen: torch.Generator) -> torch.Tensor:
    """integers in [lo, hi] times 2^scale_log2, float32"""
    return torch.randint(lo, hi + 1, shape, generator=gen).float() * 2.0 ** scale_log2


def pair_value(pairs: Sequence[Tuple[int, int]] = PAIRS, x=PROBE_X, w=PROBE_W) -> Fraction:
    """the exact sum of the kept term products of one pair probe"""
    return sum((x[i] * w[j] for i, j in pairs), Fraction(0))


def fits_fp32(v: Fraction) -> bool:
    """v exactly representable in fp32 (normal range)"""
    return float(v) == v and float(torch.tensor(float(v), dtype=torch.float32)) == v


def pair_probe(M: int, N: int, K: int, gen: torch.Generator):
    """X [M][K], W [N][K] fp32 and the exact C [M][N] (float64) of the six kept pairs.  Row m of X holds pair-probe values
    s(m,k) (1 + 2^-10 + 2^-19) at every k with s a signed power of two in [2^-12, 2^12]; row n of W is zero except at one k_n
    (k_n covers every K chunk) where it holds t(n) (1 + 2^-12 + 2^-21).  Each output is then ONE probe product: exact,
    and different for every (m, k, n) mapping."""
    xv, wv = float(sum(PROBE_X)), float(sum(PROBE_W))
    e_x = torch.randint(-12, 13, (M, K), generator=gen).double()
    sx = torch.where(torch.rand((M, K), generator=gen) < 0.5, -1.0, 1.0).double()
    X = (sx * torch.exp2(e_x) * xv).float()
    kn = torch.randperm(K, generator=gen)[torch.arange(N) % K]
    e_w = torch.randint(-12, 13, (N,), generator=gen).double()
    W = torch.zeros((N, K), dtype=torch.float64)
    W[torch.arange(N), kn] = torch.exp2(e_w) * wv
    W = W.float()
    keep = float(pair_value())
    C = (sx * torch.exp2(e_x))[:, kn] * torch.exp2(e_w)[None, :] * keep
    return X, W, C


def tie_pairs(N: int, n_pairs: int, boundaries: Sequence[int], gen: torch.Generator) -> List[Tuple[int, int]]:
    """disjoint column pairs (c1 < c2): one straddling each of `boundaries` (b - 1, b), the rest random"""
    used, out = set(), []
    for b in boundaries:
        if 1 <= b < N and b - 1 not in used and b not in used:
            out.append((b - 1, b))
            used |= {b - 1, b}
    perm = torch.randperm(N, generator=gen).tolist()
    free = [c for c in perm if c not in used]
    while len(out) < n_pairs and len(free) >= 2:
        a, b = free.pop(), free.pop()
        out.append((min(a, b), max(a, b)))
    return out


def tie_probe(M: int, N: int, K: int, pairs: Sequence[Tuple[int, int]], gen: torch.Generator, a_add: bool = False):
    """Dyadic A [M][K], W [N][K], bias [N] (and a_add [K]) where row m's largest logit is shared bit for bit by the two
    columns of pair m % len(pairs): W[c2] = W[c1], bias[c2] = bias[c1], and pair j has 64 at k = j while |other W| <= 1,
    |A| <= 1/8 except A[m][j_m] = 1.  -> (A, W, bias, add, want ids [M] = c1 of each row's pair)."""
    P = len(pairs)
    assert P <= K
    W = dyadic((N, K), -16, 16, -4, gen)
    for j, (c1, c2) in enumerate(pairs):
        W[c1, j] = 64.0
        W[c2] = W[c1]
    bias = dyadic((N,), -16, 16, -10, gen)
    for c1, c2 in pairs:
        bias[c2] = bias[c1]
    A = dyadic((M, K), -4, 4, -6, gen)
    j_m = torch.arange(M) % P
    A[torch.arange(M), j_m] = 1.0
    add = dyadic((K,), -2, 2, -6, gen) if a_add else None
    want = torch.tensor([pairs[j][0] for j in j_m.tolist()])
    return A, W, bias, add, want


def two_term(w: torch.Tensor) -> torch.Tensor:
    """h + m of the three-term bf16 split of an fp32 tensor (what a kernel without the l terms multiplies by)"""
    w = w.float()
    h = w.to(torch.bfloat16).float()
    m = (w - h).to(torch.bfloat16).float()
    return (h.double() + m.double())


def rel_errors(z: torch.Tensor, z64: torch.Tensor) -> Tuple[float, float]:
    """(max |z - z64| / max |z64|, rms(z - z64) / rms(z64))"""
    d = z.double() - z64.double()
    return float(d.abs().max() / z64.abs().max()), float(d.pow(2).mean().sqrt() / z64.double().pow(2).mean().sqrt())
