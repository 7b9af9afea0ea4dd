"""CPU checks (no GPU) of the references the NAR kernel tests rely on: the float64 mode of oracle/nar_oracle.py, the probe
constructions of oracle/dense_probes.py (exact, and each one discriminates the change it is meant to catch) and the
two-term control that shows the float64 trace comparison in tests/test_nar_gpu.py can see a dropped l term."""
import itertools

import numpy as np
import pytest
import torch

from oracle import dense_probes as P
from oracle import nar_oracle as N
from sopro_b200 import _lib
from tests.cases import _unit, e2e_inputs

torch.set_grad_enabled(False)


def _inputs(T, key):
    cfg, sd, _ = e2e_inputs()
    cond = _unit(T * int(cfg.d_model), key).view(1, T, int(cfg.d_model))
    rvq1 = torch.randint(0, 2048, (1, T), generator=torch.Generator().manual_seed(key))
    return cfg, sd, cond, rvq1


def test_float64_mode_keeps_float64_and_fp32_mode_is_unchanged():
    cfg, sd, cond, rvq1 = _inputs(23, 501)
    x = torch.randn(3, 384, dtype=torch.float64)
    assert N.rms_norm(x, sd["nar.norm.weight"]).dtype == torch.float64
    z32, z64 = [], []
    ids32, m32 = N.nar_refine(sd, cfg, cond, rvq1, z_out=z32)
    ids_plain, m_plain = N.nar_refine(sd, cfg, cond, rvq1)
    assert torch.equal(ids32, ids_plain) and torch.equal(m32, m_plain)
    ids64, _ = N.nar_refine(sd, cfg, cond, rvq1, forced=ids32, dtype=torch.float64, z_out=z64)
    n_stages = len([1 for idx in cfg.stage_indices().values() if len(idx)])
    assert len(z32) == len(z64) == n_stages
    for a, b in zip(z32, z64):
        assert a.dtype == torch.float32 and b.dtype == torch.float64 and a.shape == b.shape == (1, 23, int(cfg.nar_head_dim))
        e_max, _ = P.rel_errors(a, b)
        assert 1e-9 < e_max < 1e-4, e_max  # fp32 rounding, neither zero nor a different computation
    # teacher-forced on the fp32 ids, the float64 refiner agrees except where the fp32 argmax was a near-tie
    diff = (ids64 != ids32).nonzero().tolist()
    assert all(float(m32[tuple(i)]) < 1e-5 for i in diff), diff


def test_pair_probe_is_exact_and_every_pair_is_discriminated():
    """The six kept pairs of x = 1 + 2^-10 + 2^-19, w = 1 + 2^-12 + 2^-21 are one distinct bit each, their sum fits fp32,
    and the fp32 result changes if any pair is dropped, if the x terms of two pairs with different x terms are swapped
    (kPairX), if the w terms likewise (kPairW), or if l is lost on either side."""
    keep = P.pair_value()
    prods = [P.PROBE_X[i] * P.PROBE_W[j] for i, j in P.PAIRS]
    assert len(set(prods)) == 6 and all(p.numerator == 1 and (p.denominator & (p.denominator - 1)) == 0 for p in prods)
    assert P.fits_fp32(keep) and float(keep) == 1 + 2 ** -10 + 2 ** -12 + 2 ** -19 + 2 ** -21 + 2 ** -22
    dropped = [P.PROBE_X[i] * P.PROBE_W[j] for i in range(3) for j in range(3) if (i, j) not in P.PAIRS]
    assert max(dropped) <= P.Fraction(1, 2 ** 31)

    def f32(v):
        return float(np.float32(float(v)))

    want = f32(keep)
    for j in range(6):
        assert f32(P.pair_value(P.PAIRS[:j] + P.PAIRS[j + 1:])) != want, f"dropping pair {j} is invisible"
    for a, b in itertools.combinations(range(6), 2):
        for side in (0, 1):  # swap the x (0) or the w (1) terms of pairs a and b; a swap that keeps the pair set is no change
            pairs = [list(p) for p in P.PAIRS]
            pairs[a][side], pairs[b][side] = pairs[b][side], pairs[a][side]
            pairs = [tuple(p) for p in pairs]
            if sorted(pairs) != sorted(P.PAIRS):
                assert f32(P.pair_value(pairs)) != want, f"swapping the {'xw'[side]} terms of pairs {a}, {b} is invisible"
    no_xl = (P.PROBE_X[0], P.PROBE_X[1], P.Fraction(0))
    no_wl = (P.PROBE_W[0], P.PROBE_W[1], P.Fraction(0))
    assert f32(P.pair_value(x=no_xl)) != want and f32(P.pair_value(w=no_wl)) != want


def test_pair_order_matches_the_packed_weight_image():
    """P.PAIRS's w terms are the order in which pack_w6 lays out W6's K blocks (host hook, no device)"""
    lib = _lib.load()
    K = 64
    W = np.full((1, K), float(sum(P.PROBE_W)), dtype=np.float32)
    out = np.zeros((1, 6, K), dtype=np.uint16)
    _lib.check(lib.sopro_debug_pack_w6(W.ctypes.data, 1, K, out.ctypes.data))
    blocks = (out.astype(np.uint32) << 16).view(np.float32)[0, :, 0]
    assert [float(b) for b in blocks] == [float(P.PROBE_W[j]) for _i, j in P.PAIRS]


def test_pair_probe_operands():
    g = torch.Generator().manual_seed(1)
    X, W, C = P.pair_probe(33, 70, 128, g)
    assert bool(((W != 0).sum(1) == 1).all())
    exact = X.double() @ W.double().T  # one nonzero product per output: float64 holds it exactly
    # the probe's kept-pair value differs from the full product only by the dropped pairs (<= 2^-30 relative)
    assert float(((exact - C).abs() / C.abs()).max()) < 2.0 ** -29
    assert bool((C != 0).all()) and all(P.fits_fp32(P.Fraction(float(v))) for v in C.flatten()[:200].tolist())


@pytest.mark.parametrize("groups", [1, 3])
def test_tie_probe_ties_exactly_and_first_index_wins(groups):
    g = torch.Generator().manual_seed(groups)
    N_, K = 2048, 256
    pairs = P.tie_pairs(N_, 24, [32, 64, 128, 112, 2047], g)
    assert len(pairs) == 24 and len({c for p in pairs for c in p}) == 48
    assert all((b - 1, b) in pairs for b in (32, 64, 128, 112, 2047))
    A, W, bias, add, want = P.tie_probe(40, N_, K, pairs, g, a_add=True)
    lg32 = ((A + add) @ W.T + bias)  # fp32, any order: the dyadic grid makes it exact
    lg64 = (A.double() + add.double()) @ W.double().T + bias.double()
    assert torch.equal(lg32.double(), lg64)
    top = lg64.max(-1, keepdim=True).values
    assert bool(((lg64 == top).sum(-1) == 2).all())
    assert torch.equal(lg64.argmax(-1), want)
    # the last maximum is a different column in every row: a kernel keeping the last maximum fails
    last = lg64.shape[1] - 1 - lg64.flip(-1).argmax(-1)
    assert bool((last != want).all())


def test_two_term_control_exceeds_kappa():
    """A refiner whose weights lose their l terms (every weight reduced to h + m, what a kernel without the l products
    computes) must be visible to the z comparison: its error against float64 exceeds KAPPA x the fp32 oracle's, per stage."""
    cfg, sd, cond, rvq1 = _inputs(129, 777)
    forced, _ = N.nar_refine(sd, cfg, cond, rvq1)
    z64, z32, z2 = [], [], []
    N.nar_refine(sd, cfg, cond, rvq1, forced=forced, dtype=torch.float64, z_out=z64)
    N.nar_refine(sd, cfg, cond, rvq1, forced=forced, z_out=z32)
    sd2 = {k: (P.two_term(v) if k.startswith("nar.") and v.is_floating_point() and v.dim() == 2 else v) for k, v in sd.items()}
    N.nar_refine(sd2, cfg, cond, rvq1, forced=forced, dtype=torch.float64, z_out=z2)
    ratios = []
    for s, (a, b, c) in enumerate(zip(z32, z2, z64)):
        e32, r32 = P.rel_errors(a, c)
        e2, r2 = P.rel_errors(b, c)
        print(f"stage {s}: fp32 oracle max {e32:.2e} rms {r32:.2e} | two-term weights max {e2:.2e} rms {r2:.2e} "
              f"(x{e2 / e32:.1f}, x{r2 / r32:.1f})")
        ratios.append((e2 / e32, r2 / r32))
    assert all(r > P.KAPPA for _m, r in ratios), ratios
