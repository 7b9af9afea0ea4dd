"""GPU: the device sampler against the float64 reference of tests/sampler_refs.py.

1. The sampler alone, through `sopro_debug_sample`, over the sweep of `sampler_refs.sweep()`: vocabularies 2 ... 4096,
   top_k 1 ... 64 and above V, flat / mid / peaked rows, k-th values 17-40 octaves down, subnormal and zero tails,
   128 / 129 / 200 equal values, NaN / +-inf, temperatures 0 ... 5, penalties 0.8 / 1 / 1.1 over windows 0 ... 80, top_p
   1e-6 ... 1, exact top_p hits, exact p / q ties, tiny and zero draws, recovery pairs.
2. The sampler inside teacher-forced batched launches (batch 1, 19 in ragged teams of 8 with the LL fetch, 64) of the
   head_gain = 12 weights: every sampled token against `sample64` on the traced device logits, with the recovery flag
   the forced history gives; n_tokens and done against the stop rule.

Clear rows must equal sample64 (and sample_token, section 1); rows with an exact tie must equal sample64 under the
index-ascending rule, sample_token drawing the same rank and probability; an unclear row's token must be one the float64
decision reaches within the bound, and unclear rows must stay under MAX_UNCLEAR of the rows.
"""
import collections
import ctypes as C

import numpy as np
import pytest
import torch

from tests import sampler_refs as S

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

MAX_UNCLEAR = 0.08


def _device_token(lib, row):
    from sopro_b200 import _lib

    p = row.params
    q = _lib.ArSampling(p.top_p, p.temperature, p.rec_top_p, p.rec_temp, p.rep, p.top_k, 0, 8, 2 ** 31 - 1, 0)
    lg = row.logits.to(torch.float32).contiguous()
    nz = row.noise.to(torch.float32).contiguous()
    h = np.asarray(row.hist, dtype=np.int32)
    out = C.c_int32(-1)
    _lib.check(lib.sopro_debug_sample(lg.data_ptr(), lg.numel(), h.ctypes.data if len(h) else None, len(h), nz.data_ptr(),
                                      nz.numel(), C.byref(q), int(row.recovery), 0, C.byref(out)))
    return out.value


def _report(label, counts, paths):
    print(f"[sampler-f64] {label}: rows {counts['rows']} clear {counts['clear']} unclear {counts['unclear']} "
          f"ties {counts['tie']} | paths " + " ".join(f"{k}={v}" for k, v in sorted(paths.items())))


def test_sampler_alone_against_float64():
    from sopro_b200 import _lib

    lib = _lib.load()
    counts, paths, bad = collections.Counter(), collections.Counter(), []
    for row in S.sweep():
        d = S.sample64(row.logits, row.hist, row.params, row.noise, row.recovery)
        got = _device_token(lib, row)
        counts["rows"] += 1
        paths[d.path] += 1
        paths["n_cand=128 fits"] += d.n_cand == 128 and d.path == "fits"
        paths["n_cand=129 cold"] += d.n_cand == 129 and d.path != "fits"
        paths["fewer nonzero than k"] += d.n_nonzero < d.kk
        tok, rank = S.torch_rank(row.logits, row.hist, row.params, row.noise, row.recovery)
        if d.tie:
            counts["tie"] += 1
            if got != d.token:
                bad.append(f"{row.name}: tie row, device {got}, index-ascending rule {d.token}")
            elif not d.zero_draw and (d.p[tok] != d.p[got] or (d.top_p < 1.0 and rank != d.rank)):
                bad.append(f"{row.name}: sample_token {tok} (rank {rank}) is not in the device's tie class / rank {d.rank}")
        elif d.clear:
            counts["clear"] += 1
            if got != d.token or (not d.zero_draw and tok != d.token):
                bad.append(f"{row.name}: device {got}, float64 {d.token}, sample_token {tok}, slack {d.slack}")
        else:
            counts["unclear"] += 1
            if got not in S.reachable(row.logits, row.hist, row.params, row.noise, row.recovery):
                bad.append(f"{row.name}: unclear row, device {got} unreachable from float64 {d.token} (slack {d.slack})")
    _report("sampler alone", counts, paths)
    assert not bad, f"{len(bad)} rows: " + "; ".join(bad[:10])
    assert counts["unclear"] <= MAX_UNCLEAR * counts["rows"], counts
    assert paths["fits"] and paths["cold"] and paths["cold_tie"] and paths["n_cand=128 fits"] and paths["n_cand=129 cold"]


def test_top_k_above_64_is_refused():
    from sopro_b200 import _lib

    lib = _lib.load()
    row = S.sweep()[0]
    bad = S.Row(row.name, row.logits, row.hist, S.Params(top_k=65), row.noise)
    with pytest.raises(_lib.SoproError, match="top_k"):
        _device_token(lib, bad)


# ---------------------------------------------------------------------------
# 2. batched launches
# ---------------------------------------------------------------------------
STEPS = 80
KINDS = 6


def _forced_histories(B, eos, rng):
    """[B, STEPS] forced ids (distinct apart from the planted repeats) and per-utterance Sampling overrides.
    kind 0: a repeated tail of n = 3 ... 13 at step 8 and a 2-long repeat at 40; kind 1: a 17-long repeat (misses the
    detector) then n = 16 ... 6; kind 2: loop_streak 3 with runs of 3 (streak 2) and 4 (streak 3); kind 3: EOS at
    min_gen - 1 frames (goes on) and at min_gen (stops); kind 4: stop_on_first_eos; kind 5: anti_loop off."""
    forced = np.zeros((B, STEPS), dtype=np.int64)
    over = []
    for b in range(B):
        f = rng.permutation(eos)[:STEPS]
        kind, j = b % KINDS, b // KINDS
        o = dict(temperature=(1.05, 0.05, 0.7, 1.0, 5.0, 0.3)[b % 6 if B > 1 else 1], top_p=(0.9, 0.95, 0.8)[b % 3],
                 repetition_penalty=(1.1, 0.8, 1.0, 1.1)[b % 4], top_k=(50, 64, 33, 50, 2)[b % 5], min_gen_frames=10 ** 9)
        if kind == 0:
            n = 3 + j % 14
            f[8 + n: 8 + 2 * n] = f[8: 8 + n]
            f[40:42] = f[38:40]
        elif kind == 1:
            f[22:39] = f[5:22]
            n = 16 - j % 11
            f[42 + n: 42 + 2 * n] = f[42: 42 + n]
        elif kind == 2:
            o["loop_streak"] = 3
            f[10:13] = f[10]
            f[20:24] = f[20]
        elif kind == 3:
            o["min_gen_frames"] = 40
            f[38] = f[39] = eos
        elif kind == 4:
            o["stop_on_first_eos"] = True
            f[25] = eos
        else:
            o["anti_loop"] = False
            f[10 + 5: 20] = f[10:15]
            f[40:50] = f[40]
        forced[b] = f
        over.append(o)
    return forced, over


def _stop(f, o, eos):
    for t in range(STEPS):
        if f[t] == eos and (o.get("stop_on_first_eos") or t + 1 >= o["min_gen_frames"]):
            return t + 1
    return STEPS


def _min_rep_n(hist):
    L = len(hist)
    for n in range(3, min(16, L // 2) + 1):
        if hist[L - n:] == hist[L - 2 * n: L - n]:
            return n
    return 0


_ENG = {}


@pytest.mark.parametrize("B", [1, 19, 64])
def test_sampler_in_batched_launches(B):
    from sopro_b200.engine import ArEngine, Sampling
    from tests.cases import AR_CASES, ar_case_inputs, ar_forced_batch

    spec = AR_CASES["peaked_nostop"]  # head_gain = 12
    cfg, sd, _ = ar_case_inputs(spec)
    if "e" not in _ENG:
        _ENG["e"] = ArEngine(cfg, sd, device=0, weight_dtype="fp32")
    eng = _ENG["e"]
    eos, V = int(cfg.codebook_size), cfg.ar_vocab()
    lens = ([52, 7, 23, 33, 1, 12, 5, 40, 17, 9, 52, 3, 28, 44, 2, 36, 11, 6, 50] * 4)[:B]
    cond, txt, _ = ar_forced_batch(cfg, lens, STEPS, 70 + B)
    forced, over = _forced_histories(B, eos, np.random.default_rng(B))
    samp = [Sampling(**o) for o in over]
    noise = torch.empty(B, STEPS, 64).exponential_(1.0, generator=torch.Generator().manual_seed(B))
    dev = eng.device
    ses = eng.session(B, STEPS, max(lens))
    ses.set_forced(torch.from_numpy(forced).to(torch.int32))
    tr_b = torch.zeros(STEPS, int(cfg.n_layers_ar), B, int(cfg.d_model), device=dev)
    tr_l = torch.zeros(STEPS, B, V, device=dev)
    ses.set_trace(tr_b, tr_l)
    ses.begin(cond, txt, lens, noise, samp)
    ses.run()
    toks, n, done = ses.read()
    sampled = ses.sampled().cpu().numpy()
    logits = tr_l.cpu()
    ses.set_forced(None)
    ses.close()

    counts, paths, rep_ns, bad = collections.Counter(), collections.Counter(), collections.Counter(), []
    for b in range(B):
        o, f = over[b], forced[b].tolist()
        n_ref = _stop(f, o, eos)
        if n[b] != n_ref or done[b] != 1 or toks[b, :n_ref].tolist() != f[:n_ref]:
            bad.append(f"utterance {b}: n_tokens {n[b]} done {done[b]}, the stop rule gives {n_ref}")
        prm = S.Params(top_p=samp[b].top_p, top_k=samp[b].top_k, temperature=samp[b].temperature,
                       rec_top_p=samp[b].recovery_top_p, rec_temp=samp[b].recovery_temp, rep=samp[b].repetition_penalty)
        rec = S.recovery_flags(f, samp[b].loop_streak, samp[b].anti_loop)
        for t in range(n_ref):
            counts["recovery"] += rec[t]
            if rec[t] and _min_rep_n(f[:t]):
                rep_ns[_min_rep_n(f[:t])] += 1
            d = S.sample64(logits[t, b], f[:t], prm, noise[b, t], rec[t])
            counts["rows"] += 1
            paths[d.path] += 1
            got = int(sampled[b, t])
            if d.clear or d.tie:
                counts["tie" if d.tie else "clear"] += 1
                if got != d.token:
                    bad.append(f"utterance {b} step {t} (recovery {rec[t]}, path {d.path}): device {got}, float64 "
                               f"{d.token}, slack {d.slack}")
            else:
                counts["unclear"] += 1
                if got not in S.reachable(logits[t, b], f[:t], prm, noise[b, t], rec[t]):
                    bad.append(f"utterance {b} step {t}: unclear, device {got} unreachable from float64 {d.token}")
    _report(f"batch {B}", counts, paths)
    print(f"[sampler-f64] batch {B}: recovery steps {counts['recovery']}, repeated tails by n {dict(sorted(rep_ns.items()))}")
    assert not bad, f"{len(bad)} mismatches: " + "; ".join(bad[:10])
    assert counts["unclear"] <= MAX_UNCLEAR * counts["rows"], counts
    assert paths["fits"] > 0 and paths["cold"] + paths["cold_tie"] > 0, paths
    if B == 64:
        assert set(rep_ns) >= set(range(3, 17)), rep_ns
