"""CPU: the float64 sampler reference (tests/sampler_refs.py) is right, reaches every top-k path, and has teeth.

- Wherever every margin is clear, `sample64` equals `oracle.ar_oracle.sample_token` (the reference semantics in torch
  fp32) on the known-answer rows and on the whole sweep; on exact ties it draws the same rank and probability.
- Each mutated copy of the reference (ties by descending index, a 49- or 51-token penalty window, `>=` at the top-p
  cut, the recovery pair swapped, the noise read one rank late, x / T at T = 0) gives another token on at least one
  row the GPU test checks exactly, so a kernel with that bug fails there.  Two more mutants are harmless, and the test
  pins why: x / T at T = 1 leaves x bit-equal, and the penalty before the temperature moves x by at most two ulp.
- The sweep's predicted kernel paths reach the minimum counts asserted below.
"""
import collections
import json
import os

import numpy as np
import pytest
import torch

from oracle import ar_oracle as O
from tests import sampler_refs as S

GOLD = os.path.join(os.path.dirname(__file__), "golden")
_CACHE = {}

# the fraction of sweep rows allowed to be unclear (the float64 decision sits within SAFETY x the bound of a flip)
MAX_UNCLEAR = 0.08
MIN_PATHS = {"fits": 150, "cold": 60, "cold_tie": 20, "fallback": 2, "n_cand=128 fits": 3, "n_cand=129 cold": 3,
             "fewer nonzero than k": 10, "tie": 40}


def _sweep():
    if "rows" not in _CACHE:
        rows = S.sweep()
        _CACHE["rows"] = [(r, S.sample64(r.logits, r.hist, r.params, r.noise, r.recovery),
                           S.torch_rank(r.logits, r.hist, r.params, r.noise, r.recovery)) for r in rows]
    return _CACHE["rows"]


def coverage(decisions):
    c = collections.Counter()
    for d in decisions:
        c[d.path] += 1
        c["n_cand=128 fits"] += d.n_cand == 128 and d.path == "fits"
        c["n_cand=129 cold"] += d.n_cand == 129 and d.path != "fits"
        c["fewer nonzero than k"] += d.n_nonzero < d.kk
        c["tie"] += d.tie
    return c


def test_known_answer_rows_match_the_reference():
    from tests.cases import SAMPLER_CASES, sampler_case_inputs

    with open(os.path.join(GOLD, "sampler_kat.json")) as f:
        kat = json.load(f)
    clear = 0
    for name, spec in SAMPLER_CASES.items():
        logits, hist, kw, seed = sampler_case_inputs(spec)
        if int(kw["top_k"]) < 1:
            continue
        V = logits.numel()
        prm = S.Params(top_p=kw["top_p"], top_k=min(int(kw["top_k"]), 64), temperature=kw["temperature"],
                       rec_top_p=kw["top_p"], rec_temp=kw["temperature"], rep=kw["repetition_penalty"])
        tape = O.noise_tape(seed, 1, V)[0]
        d = S.sample64(logits, hist, prm, tape)
        if d.clear and not d.tie:
            assert d.token == kat[name], (name, d.token, kat[name])
            clear += 1
        else:  # near a flip: the reference's token is one the float64 decision reaches inside the bound
            assert kat[name] in S.reachable(logits, hist, prm, tape), (name, kat[name], d.token, d.slack)
    print(f"[sampler-f64 cpu] known-answer rows: {clear} of 27 clear")
    assert clear >= 20, clear


def test_sweep_matches_sample_token_where_clear():
    rows = _sweep()
    n_clear = n_tie = 0
    for r, d, (tok, rank) in rows:
        if d.zero_draw:
            continue
        if d.tie:
            # the same tie class: the same probability; with top_p < 1 also the same drawn rank
            n_tie += 1
            assert d.p[tok] == d.p[d.token], (r.name, tok, d.token)
            if d.top_p < 1.0:
                assert rank == d.rank, (r.name, rank, d.rank)
        elif d.clear:
            n_clear += 1
            assert tok == d.token, (r.name, tok, d.token, d.slack)
    unclear = sum(not d.clear and not d.tie for _r, d, _t in rows)
    print(f"[sampler-f64 cpu] rows {len(rows)} clear {n_clear} ties {n_tie} unclear {unclear}")
    assert unclear <= MAX_UNCLEAR * len(rows), unclear


def test_sweep_reaches_every_path():
    c = coverage([d for _r, d, _t in _sweep()])
    print("[sampler-f64 cpu] paths " + " ".join(f"{k}={c[k]}" for k in MIN_PATHS))
    short = {k: (c[k], m) for k, m in MIN_PATHS.items() if c[k] < m}
    assert not short, short


@pytest.mark.parametrize("mutate", S.MUTATIONS)
def test_mutations_are_caught(mutate):
    """A mutant gives another token on a row the GPU test checks exactly (clear, or an exact tie)."""
    caught = []
    for r, d, _t in _sweep():
        if not (d.clear or d.tie):
            continue
        m = S.sample64(r.logits, r.hist, r.params, r.noise, r.recovery, mutate=mutate)
        if m.token != d.token:
            caught.append(r.name)
    print(f"[sampler-f64 cpu] mutation {mutate}: caught on {len(caught)} rows, e.g. {caught[:3]}")
    assert caught, mutate


@pytest.mark.parametrize("mutate", S.NULL_MUTATIONS)
def test_null_mutations_leave_the_shared_operand(mutate):
    for r, d, _t in _sweep():
        T = r.params.rec_temp if r.recovery else r.params.temperature
        m = S.shared_x(r.logits, r.hist, T, r.params.rep, mutate)
        if mutate == "div_at_t1":
            assert np.array_equal(m, d.x), r.name
        else:
            with np.errstate(invalid="ignore"):  # inf - inf on the overflow rows, where both are inf
                near = (m == d.x) | (np.abs(m.astype(np.float64) - d.x) <= 2 * np.spacing(np.abs(d.x)))
            assert near.all(), r.name


def test_zero_draw_semantics_are_pinned():
    """A draw of exactly 0: sample_token's 0 / 0 at a zero-probability rank is NaN, which torch.argmax takes as the
    maximum, so it returns a token outside the top-p set; the device (and sample64) never draws a zero probability.
    A positive probability with a zero draw is +inf on both and wins."""
    lg = torch.tensor([3.0, 2.0, 1.0, 0.0, -5.0, -6.0])
    prm = S.Params(top_p=0.5, top_k=3, temperature=1.0, rep=1.0)
    q = torch.ones(6)
    q[5] = 0.0
    d = S.sample64(lg, [], prm, q)
    tok, _ = S.torch_rank(lg, [], prm, q)
    assert d.zero_draw and tok == 5 and d.token == 0
    q = torch.ones(6) * 2.0
    q[1] = 0.0
    d = S.sample64(lg, [], S.Params(top_p=0.999, top_k=3, temperature=1.0, rep=1.0), q)
    tok, _ = S.torch_rank(lg, [], S.Params(top_p=0.999, top_k=3, temperature=1.0, rep=1.0), q)
    assert d.token == tok == 1


def test_fp32_pipeline_stays_inside_the_bound():
    """An fp32 restatement of the device's softmax and renormalisation (numpy's float32 exp) stays within the
    per-probability bound of the module docstring on every sweep row."""
    worst = 0.0
    for r, d, _t in _sweep():
        if d.path == "fallback" or d.exact:
            continue
        x = d.x
        mx = x.max()
        e = np.exp((x - mx).astype(np.float32)).astype(np.float32)
        se = np.float32(e.sum(dtype=np.float32))
        q = (e / se).astype(np.float32)
        sel = np.lexsort((np.arange(x.size), -d.p))[: d.kk]
        s1 = np.float32(q[sel].astype(np.float64).sum())
        a = (q[sel] / s1).astype(np.float64)
        p = d.p[sel] / d.p[sel].sum()
        ok = p >= S.TINY
        eps = S._eps(d.p, (mx - x).astype(np.float64))[sel]
        ratio = np.abs(a[ok] - p[ok]) / (p[ok] * eps[ok])
        worst = max(worst, float(ratio.max()) if ratio.size else 0.0)
    print(f"[sampler-f64 cpu] fp32 restatement: worst error / bound {worst:.3f}")
    assert worst <= 1.0, worst


def test_recovery_flags_follow_the_reference_rule():
    eos = 2048
    base = list(range(100, 140))
    for n in range(3, 17):
        pat = list(range(500, 500 + n))
        f = S.recovery_flags(base + pat + pat, 8)
        assert f[-1] and not f[-2], n
    pat2 = [7, 9]
    assert not S.recovery_flags(base + pat2 + pat2, 8)[-1]  # n = 2 is below the detector
    pat17 = list(range(600, 617))
    assert not any(S.recovery_flags(base + pat17 + pat17, 8))  # n = 17 is above it
    run = base + [eos] * 3
    assert not S.recovery_flags(run, 3)[-1] and S.recovery_flags(run + [eos], 3)[-1]  # streak 2 / 3 of 3
    assert not any(S.recovery_flags(base + pat2 + pat2, 8, anti_loop=False))
    assert O.repeated_tail(base + list(range(3)) * 2) and not O.repeated_tail(base + pat2 * 2)
