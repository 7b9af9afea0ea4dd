"""A float64 reference of the AR sampler (`sample_utterance` in sopro_b200/csrc/ar_kernel.cuh), with the margins that
decide each draw and a bound on how far the device's fp32 arithmetic can move them.

**Shared operand.**  The penalised, temperature-scaled logits x are built in fp32, the same IEEE operations the kernel
and `oracle.ar_oracle.sample_token` perform: nan_to_num to +-1e9, x / T unless T is 0 or 1, then the repetition
penalty on set(hist[-50:]) (x * r below zero, x / r otherwise).  So x is bit-identical on all three.

**Float64 from there.**  Softmax, top-k, renormalisation, the cumulative sum, the top-p cut (a rank j >= 1 is removed
when cum[j-1] > top_p) and the draw argmax(p / q) are float64.  The noise q is indexed by rank when top_p < 1 and by
token id when top_p = 1.  A zero-probability candidate is never drawn (its 0 / q is 0, and 0 / 0 loses every
comparison); a positive one with q = 0 gets +inf.

**The device's tie contract.**  Everywhere (top-k membership, rank order, the argmax fallback) equal values are ordered
by index ascending; equal p / q ratios go to the smaller key (the rank, or the token id when top_p = 1).  torch's CPU
topk and sort do not define an order among equal values, so on an exact tie `sample_token` can give the tied ranks to
other tokens of the same value: it then draws the same rank and the same probability, not always the same id.

**Error bound.**  For a probability p_i whose logit sits d_i = mx - x_i below the maximum, the device's fp32 value
differs from float64 by at most eps_i relative, where

    eps_i = 2^-24 (d_i + 32) + 2^-147 / p_i

- fl(x_i - mx) is off by at most 2^-24 d_i absolute, which expf turns into 2^-24 d_i relative;
- expf is within 2 ulp (4 units of 2^-24; the build does not use -use_fast_math);
- the sum of the exponentials is a tree of at most 8 serial + 5 warp + 4 block additions of positive terms (17 units);
- q = e / se, the renormalisation sums (double sums rounded to float, one unit each, twice), the two divisions by
  them and the division by the noise add 1 unit each (6 units);
- the remaining 5 units are slack for the double sums' own rounding;
- a result in the subnormal range carries an absolute error of at most 2 subnormal ulp (2^-148) from expf plus half
  an ulp (2^-150) from the division, below 2^-147 absolute.

Two compared values a > b (probabilities, or ratios p / q) can swap only if a - b <= a eps_a + b eps_b; the
cumulative sum's error is bounded by sum_i eps_i a_i plus one float rounding of the sum.  A decision counts as
**clear** when its margin exceeds SAFETY = 4 times the bound of the quantities it compares.  Rows whose nonzero
probabilities are all equal and a power of two in number are **exact**: every device operation on them is exact
(expf(0) = 1, n * 1, 1 / n), so their bound is 0 and exact hits of top_p are decided by the strict `>` alone.
Membership and order among probabilities below 2^-126 (subnormal or zero on the device) are not margins: such a
candidate's p / q stays below 2^-126 / q, far under the winning ratio for every draw the sweep uses.
"""
from __future__ import annotations

import dataclasses
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

U = 2.0 ** -24
C_UNITS = 32.0
SUBNORMAL_ABS = 2.0 ** -147
SAFETY = 4.0
K_MAX, K_CAND, K_BINS = 64, 128, 1024
EPS = 1e-12  # the renormalisation floor below which both fall back to argmax(x)
TINY = 2.0 ** -126  # below: subnormal or zero on the device; such a candidate's p / q cannot win against the sweep's draws

MUTATIONS = ("tie_desc", "window49", "window51", "cut_ge", "recovery_swap", "noise_rank1", "div_at_t0")
# x / T at T = 1 is the identity in IEEE arithmetic, and the penalty before the temperature moves x by at most one
# ulp or two (x r / T against (x / T) r): no token can tell these two from the reference outside a near-tie
NULL_MUTATIONS = ("div_at_t1", "penalty_first")


@dataclasses.dataclass(frozen=True)
class Params:
    top_p: float = 0.9
    top_k: int = 50
    temperature: float = 1.05
    rec_top_p: float = 0.85
    rec_temp: float = 1.2
    rep: float = 1.1


@dataclasses.dataclass
class Decision:
    token: int
    path: str  # "fits" | "cold" | "cold_tie" (the predicted top-k path) ; "fallback" when argmax(x) decides
    kk: int
    n_cand: int  # candidates down to the threshold bin (the fits test compares it with 128)
    b_sel: int  # the threshold bin (1023 = everything below 16 octaves, zeros included)
    n_nonzero: int
    top_p: float
    rank: int  # the drawn rank (top_p < 1) or -1
    kept: int  # ranks kept by the top-p cut
    margins: Dict[str, float]  # relative: topk (k-th vs (k+1)-th), topp (|cum[j-1] - top_p| at the cut), draw
    slack: Dict[str, float]  # margin / (SAFETY x bound); > 1 is clear
    tie: bool  # an exact tie decides the token: a tie class straddling the cut, holding the drawn rank, or a p / q tie
    exact: bool
    zero_draw: bool  # a draw of exactly 0 lies among the noise sample_token reads
    p: np.ndarray = dataclasses.field(repr=False)
    x: np.ndarray = dataclasses.field(repr=False)

    @property
    def clear(self) -> bool:
        return all(s > 1.0 for s in self.slack.values())


def shared_x(logits: torch.Tensor, hist: Sequence[int], temp: float, rep: float, mutate: Optional[str] = None) -> np.ndarray:
    """The fp32 penalised, temperature-scaled logits (the kernel's and sample_token's shared operand)."""
    x = torch.nan_to_num(logits.reshape(-1).to(torch.float32), nan=-1e9, posinf=1e9, neginf=-1e9)
    win = {"window49": 49, "window51": 51}.get(mutate, 50)
    ids = sorted(set(int(h) for h in list(hist)[-win:])) if (rep != 1.0 and len(hist)) else []
    T = np.float32(temp)

    def scale(x):
        if (T != 0 and T != 1) or (mutate == "div_at_t1" and T == 1) or (mutate == "div_at_t0" and T == 0):
            return x / torch.tensor(T)
        return x

    def penal(x):
        if ids:
            x = x.clone()
            v = x[ids]
            r = torch.tensor(np.float32(rep))
            x[ids] = torch.where(v < 0, v * r, v / r)
        return x

    x = scale(penal(x)) if mutate == "penalty_first" else penal(scale(x))
    return x.numpy().astype(np.float32)


def _eps(p: np.ndarray, d: np.ndarray) -> np.ndarray:
    """the per-probability relative bound of the module docstring; an exact float64 zero is a device zero too"""
    pos = p > 0
    return np.where(pos, U * (np.where(pos, d, 0.0) + C_UNITS) + SUBNORMAL_ABS / np.where(pos, p, 1.0), 0.0)


def _bits_key(q32: np.ndarray) -> np.ndarray:
    return (q32.view(np.uint32) >> 17).astype(np.int64)


def _predict_path(p: np.ndarray, kk: int, order: np.ndarray):
    """The kernel's fits test on float32(p): the 1024-bin histogram (64 bins per octave) below the maximum."""
    q32 = p.astype(np.float32)
    top = _bits_key(np.array([q32.max()], dtype=np.float32))[0]
    rel = np.minimum(top - _bits_key(q32), K_BINS - 1)
    b_sel = int(np.sort(rel)[kk - 1])
    n_cand = int((rel <= b_sel).sum())
    fits = b_sel < K_BINS - 1 and n_cand <= K_CAND
    if fits:
        path = "fits"
    else:
        tie = kk < p.size and p[order[kk - 1]] == p[order[kk]]
        path = "cold_tie" if tie else "cold"
    return path, n_cand, b_sel


def _draw(vals: np.ndarray, keys: np.ndarray):
    """argmax with the smaller key on ties; NaN (0 / 0) never wins -> (position, best, second best other value)"""
    r = np.where(np.isnan(vals), -np.inf, vals)
    best = r.max()
    pos = int(np.flatnonzero(r == best)[np.argmin(keys[r == best])])
    rest = np.delete(r, pos)
    return pos, best, (rest.max() if rest.size else -np.inf)


def _decide(x, p, eps, V, kk, top_p, noise, mutate):
    """top-k, renormalise, top-p, draw on float64 p -> dict of the decision and its margins"""
    idx = np.arange(V)
    order = np.lexsort((-idx if mutate == "tie_desc" else idx, -p))
    sel = order[:kk]
    out = dict(order=order, sel=sel, rank=-1, kept=kk, fallback=False, tie=False)
    m, bnd = {}, {}
    if kk < V:
        a, b = p[order[kk - 1]], p[order[kk]]
        if a == b:
            out["tie"] = a > 0  # a tie class straddles the cut: decided by index, exactly
        elif a >= TINY:
            m["topk"] = (a - b) / a
            bnd["topk"] = (a * eps[order[kk - 1]] + b * eps[order[kk]]) / a
    s1 = p[sel].sum()
    if s1 <= EPS:
        out.update(fallback=True, token=int(np.lexsort((idx, -x.astype(np.float64)))[0]))
        return out, m, bnd
    a = p[sel] / s1
    if top_p < 1.0:
        if kk > 1:  # the order inside the top-k assigns the noise
            sv = p[sel]
            d = sv[:-1] - sv[1:]
            nz = (d > 0) & (sv[:-1] >= TINY)
            if nz.any():
                rel = d[nz] / sv[:-1][nz]
                b2 = ((sv * eps[sel])[:-1] + (sv * eps[sel])[1:])[nz] / sv[:-1][nz]
                j = int(np.argmin(rel / np.maximum(b2, 1e-300)))
                if "topk" not in m or rel[j] / b2[j] < m["topk"] / bnd["topk"]:
                    m["topk"], bnd["topk"] = float(rel[j]), float(b2[j])
        cum = np.cumsum(a)
        prev = np.concatenate([[0.0], cum[:-1]])
        removed = (prev >= top_p) if mutate == "cut_ge" else (prev > top_p)
        removed[0] = False
        kept = int((~removed).sum())
        out["kept"] = kept
        if kk > 1:
            # the last kept and the first removed rank, where the cut moves a drawable probability
            js = [j for j in (kept - 1, kept) if 1 <= j < kk and a[j] >= TINY]
            cb = np.cumsum(a * eps[sel]) + (U * cum + U if eps.any() else 0.0)
            if js:
                dist = [abs(prev[j] - top_p) for j in js]
                j = int(np.argmin(dist))
                m["topp"], bnd["topp"] = float(dist[j]), float(cb[js[j] - 1])
        a = np.where(removed, 0.0, a)
        s2 = a.sum()
        a = a / s2
        q = noise[np.minimum(np.arange(kk) + (1 if mutate == "noise_rank1" else 0), noise.size - 1)].astype(np.float64)
        keys = np.arange(kk)
    else:
        q = noise[sel].astype(np.float64)
        keys = sel.copy()
    with np.errstate(divide="ignore", invalid="ignore"):
        r = a / q
    pos, best, second = _draw(r, keys)
    out["rank"] = pos if top_p < 1.0 else -1
    out["token"] = int(sel[pos])
    if top_p < 1.0 and p[sel[pos]] > 0 and (p[sel] == p[sel[pos]]).sum() > 1:
        out["tie"] = True  # the drawn rank belongs to a tie class: which tied token holds it is the index rule
    if np.isfinite(best) and best > 0 and second > 0:
        w = int(np.flatnonzero(np.where(np.isnan(r), -np.inf, r) == second)[0])
        if second == best and p[sel[pos]] == p[sel[w]] and q[pos] == q[w]:
            out["tie"] = True  # the same value and the same draw: decided by the key, exactly
        else:
            m["draw"] = (best - second) / best
            bnd["draw"] = (best * eps[sel[pos]] + second * eps[sel[w]]) / best
    return out, m, bnd


def sample64(logits: torch.Tensor, hist: Sequence[int], params: Params, noise: torch.Tensor, recovery: bool = False,
             mutate: Optional[str] = None) -> Decision:
    """The device sampler's decision in float64 on the shared fp32 operand; `mutate` names one of MUTATIONS."""
    rec = bool(recovery) != (mutate == "recovery_swap")
    top_p = float(np.float32(params.rec_top_p if rec else params.top_p))
    temp = params.rec_temp if rec else params.temperature
    x = shared_x(logits, hist, temp, params.rep, mutate)
    V = x.size
    kk = min(int(params.top_k), V, K_MAX)
    xd = x.astype(np.float64)
    if np.isinf(xd).any():  # inf - inf: the softmax is NaN, nan_to_num makes it 0 everywhere
        p = np.zeros(V)
        d = np.zeros(V)
    else:
        mx = xd.max()
        d = mx - xd
        e = np.exp(-d)
        p = e / e.sum()
    nzn = np.asarray(noise, dtype=np.float32).reshape(-1)
    nzp = p[p > 0]
    n = nzp.size
    exact = n > 0 and bool((nzp == nzp[0]).all()) and (n & (n - 1)) == 0
    with np.errstate(divide="ignore"):
        eps = np.zeros(V) if exact else _eps(p, d)
    out, m, bnd = _decide(xd, p, eps, V, kk, top_p, nzn, mutate)
    order = out["order"]
    path, n_cand, b_sel = _predict_path(p, kk, order) if not out["fallback"] else ("fallback", V, 0)
    slack = {k: (np.inf if bnd[k] == 0 else m[k] / (SAFETY * bnd[k])) for k in m}
    zero_draw = bool((nzn[:V] == 0).any())  # sample_token reads the first V draws in either branch
    return Decision(token=out["token"], path=path, kk=kk, n_cand=n_cand, b_sel=b_sel, n_nonzero=int((p > 0).sum()),
                    top_p=top_p, rank=out["rank"], kept=out["kept"], margins=m, slack=slack, tie=out["tie"],
                    exact=exact, zero_draw=zero_draw, p=p, x=x)


def reachable(logits: torch.Tensor, hist: Sequence[int], params: Params, noise: torch.Tensor, recovery: bool = False,
              trials: int = 96, seed: int = 0) -> set:
    """Tokens the float64 decision reaches when each probability moves by up to SAFETY x its bound (random moves and
    the two uniform extremes, renormalised): the tokens an unclear row may legitimately give."""
    dec = sample64(logits, hist, params, noise, recovery)
    rec = bool(recovery)
    top_p = float(np.float32(params.rec_top_p if rec else params.top_p))
    V = dec.x.size
    xd = dec.x.astype(np.float64)
    d = xd.max() - xd
    p = dec.p
    eps = _eps(p, d)
    nzn = np.asarray(noise, dtype=np.float32).reshape(-1)
    rng = np.random.default_rng(seed)
    toks = {dec.token}
    for t in range(trials):
        s = rng.uniform(-1.0, 1.0, V) if t >= 2 else np.full(V, (-1.0, 1.0)[t])
        if t % 3 == 2:
            s = np.sign(s)
        pp = p * (1.0 + SAFETY * eps * s)
        out, _m, _b = _decide(xd, pp / pp.sum(), eps, V, dec.kk, top_p, nzn, None)
        toks.add(out["token"])
    return toks


def torch_rank(logits: torch.Tensor, hist: Sequence[int], params: Params, noise: torch.Tensor, recovery: bool = False):
    """sample_token's token and, when top_p < 1, the rank it drew (from its sorted order)."""
    from oracle.ar_oracle import sample_token

    rec = bool(recovery)
    top_p = params.rec_top_p if rec else params.top_p
    trace: dict = {}
    tok = sample_token(logits.reshape(1, 1, -1).to(torch.float32), list(hist), top_p=top_p, top_k=params.top_k,
                       temperature=params.rec_temp if rec else params.temperature, repetition_penalty=params.rep,
                       noise_v=noise.reshape(-1).to(torch.float32), trace=trace)
    rank = -1
    if "sorted_idx" in trace:
        hits = (trace["sorted_idx"] == tok).nonzero()
        rank = int(hits[0, 0]) if hits.numel() else -1
    return tok, rank


def recovery_flags(hist: Sequence[int], loop_streak: int, anti_loop: bool = True) -> List[bool]:
    """The recovery flag at every step t of a forced history (model.py:274-279): repeated_tail(hist[:t], 16), or a
    streak of loop_streak repeats of the last token."""
    from oracle.ar_oracle import repeated_tail

    out, streak, last = [], 0, None
    for t in range(len(hist) + 1):
        out.append(bool(anti_loop and (repeated_tail(hist[:t], 16) or (last is not None and streak >= loop_streak))))
        if t < len(hist):
            streak = streak + 1 if (last is not None and hist[t] == last) else 0
            last = hist[t]
    return out


# ---------------------------------------------------------------------------
# the sweep: every row is (name, logits [V] fp32, history, Params, noise [V] fp32, recovery)
# ---------------------------------------------------------------------------
@dataclasses.dataclass
class Row:
    name: str
    logits: torch.Tensor
    hist: List[int]
    params: Params
    noise: torch.Tensor
    recovery: bool = False


VOCABS = (2, 3, 5, 33, 63, 64, 65, 511, 512, 513, 2049, 4095, 4096)
TOP_KS = (1, 2, 31, 32, 33, 50, 63, 64)
TEMPS = (0.0, 1.0, 0.05, 1.05, 5.0)
TOP_PS = (1.0, 0.9, 0.85, 1e-6, 0.999999)
REPS = (1.0, 1.1, 0.8)
HLENS = (0, 1, 49, 50, 51, 80)
LN2 = float(np.log(2.0))


def _tape(seed: int, V: int) -> torch.Tensor:
    from oracle.ar_oracle import noise_tape

    return noise_tape(seed, 1, V)[0].contiguous()


def _f32(a) -> torch.Tensor:
    return torch.from_numpy(np.asarray(a, dtype=np.float32).copy())


def _shape(kind: str, V: int, rng) -> np.ndarray:
    s = {"flat": 0.5, "mid": 3.0, "peaked": 9.0}[kind] * np.sqrt(3.0)
    return rng.uniform(-1.0, 1.0, V) * s


def _deep(V: int, octaves: float, n_top: int, rng) -> np.ndarray:
    """one logit at 0, n_top - 1 about `octaves` octaves below it and the rest lower still: the k-th value far below
    the histogram's 16 octaves"""
    x = -octaves * LN2 - 3.0 - rng.uniform(0.0, 4.0, V)
    top = rng.permutation(V)[:n_top]
    x[top[0]] = 0.0
    x[top[1:]] = -octaves * LN2 + rng.uniform(-0.5, 0.5, top.size - 1)
    return x


def _hist_window(V: int, x: np.ndarray, n: int, rng) -> List[int]:
    """a history of length n whose hist[-51] is the best token and hist[-50] the second (each only there), so a
    49- or 51-token window flips a penalty; duplicates and the EOS id (V - 1) among the rest"""
    order = np.argsort(-x, kind="stable")
    best, second = int(order[0]), int(order[1])
    pool = [int(t) for t in rng.permutation(V) if t not in (best, second)] or [V - 1]
    h = [pool[i % len(pool)] for i in range(n)]
    if n >= 51:
        h[n - 51] = best
    if n >= 50:
        h[n - 50] = second
    if n >= 4:
        h[n - 2] = h[n - 3]  # a duplicate
        h[n - 4] = V - 1  # the EOS id
    return h


def sweep() -> List[Row]:
    rows: List[Row] = []
    seed = [1000]

    def add(name, x, hist=(), noise=None, recovery=False, **kw):
        x = np.asarray(x, dtype=np.float64)
        V = x.size
        seed[0] += 1
        rows.append(Row(name, _f32(x), list(hist), Params(**kw), _tape(seed[0], V) if noise is None else _f32(noise),
                        recovery))

    # 1. base sweep: every vocabulary x shape, top_k / temperature / top_p / penalty / history cycling
    i = 0
    for V in VOCABS:
        for kind in ("flat", "mid", "peaked"):
            for j in range(4):
                rng = np.random.default_rng(10 * i + j)
                x = _shape(kind, V, rng)
                n = HLENS[(i + j) % len(HLENS)]
                add(f"base/V{V}/{kind}/{j}", x, rng.integers(0, V, n).tolist(), top_k=TOP_KS[(i + 3 * j) % len(TOP_KS)],
                    temperature=TEMPS[(i + j) % len(TEMPS)], top_p=TOP_PS[(2 * i + j) % len(TOP_PS)],
                    rep=REPS[(i + 2 * j) % len(REPS)])
                i += 1
        rng = np.random.default_rng(5000 + V)
        add(f"base/V{V}/topk_gt_v", _shape("mid", V, rng), top_k=64 if V < 64 else 50)
    # 2. deep rows: the k-th value 17 ... 40 octaves down (cold path without ties)
    for V in (2049, 4096, 513, 65):
        for o in (17.5, 20, 25, 30, 40):
            for k in (33, 50, 64):
                if k >= V:
                    continue
                rng = np.random.default_rng(int(V * 100 + o * 3 + k))
                add(f"deep/V{V}/o{o}/k{k}", _deep(V, o, k + 8, rng), top_k=k, top_p=(0.9, 1.0, 0.95)[k % 3],
                    temperature=1.0, rep=1.0)
    # 3. tails in subnormals and exact zeros; a single +-1e9 spike
    for V in (2049, 4096, 64):
        rng = np.random.default_rng(V + 7)
        x = np.full(V, -300.0)
        top = rng.permutation(V)
        x[top[:5]] = rng.uniform(-1.0, 0.0, 5)
        x[top[5:40]] = -rng.uniform(88.0, 102.0, 35)  # subnormal probabilities
        add(f"tail/V{V}/subnormal", x, temperature=1.0, rep=1.0, top_p=0.999999)
        add(f"tail/V{V}/subnormal_nop", x, temperature=1.0, rep=1.0, top_p=1.0)
        y = _shape("mid", V, rng)
        y[top[0]] = 1e9
        add(f"tail/V{V}/spike+1e9", y, top_p=0.9)
        y = _shape("mid", V, rng)
        y[top[1]] = -1e9
        add(f"tail/V{V}/spike-1e9", y, top_p=1.0)
        add(f"tail/V{V}/fewer_than_k", np.where(np.arange(V) % 5 == 0, rng.uniform(-1, 0, V), -1e9)[:V] if V < 64 else
            np.where(rng.permutation(V) < 10, rng.uniform(-1, 0, V), -1e9), top_k=50, top_p=0.93)
    # 4. ties and the fits boundary
    for V in (2049, 4096, 513):
        for n_eq in (128, 129, 200):
            rng = np.random.default_rng(V + n_eq)
            x = np.full(V, -40.0) - rng.uniform(0, 1, V)
            x[rng.permutation(V)[:n_eq]] = 0.0  # n_eq equal maxima: the threshold bin holds exactly n_eq
            for tp in (0.93, 1.0):
                add(f"tie/V{V}/eq{n_eq}/p{tp}", x, top_p=tp, temperature=1.0, rep=1.0)
        for n_eq in (60, 200):  # 20 distinct values above a tie class straddling rank 50
            rng = np.random.default_rng(V + 3 * n_eq)
            x = np.full(V, -40.0) - rng.uniform(0, 1, V)
            perm = rng.permutation(V)
            x[perm[:20]] = rng.uniform(0.5, 2.0, 20)
            x[perm[20:20 + n_eq]] = 0.0
            add(f"tie/V{V}/straddle{n_eq}", x, top_p=0.999999, temperature=1.0, rep=1.0)
        for n_in in (128, 129):  # distinct values, all in the maximum's bin
            for s in range(40):
                rng = np.random.default_rng(V * 1000 + n_in * 10 + s)
                x = np.full(V, -40.0) - rng.uniform(0, 1, V)
                x[rng.permutation(V)[:n_in]] = -rng.uniform(0.0, 0.004, n_in)
                p = np.exp(x - x.max())
                p /= p.sum()
                ok = all(_predict_path(p * f, 50, np.lexsort((np.arange(V), -p)))[1] == n_in for f in (1 - 1e-4, 1 + 1e-4))
                if ok:
                    add(f"bin/V{V}/n{n_in}", x, top_p=0.9, temperature=1.0, rep=1.0)
                    break
    # 5. special values
    for V in (2049, 33, 4096):
        rng = np.random.default_rng(V + 11)
        x = _shape("mid", V, rng)
        x[1], x[V // 2], x[V - 2] = np.nan, np.inf, -np.inf
        add(f"special/V{V}/nan_inf", x, rng.integers(0, V, 20).tolist())
        y = _shape("mid", V, rng)
        y[[0, 5, V - 1]] = np.inf  # three-way tie at 1e9
        add(f"special/V{V}/inf3", y, top_p=0.9)
        y[7 % V] = np.inf  # four-way: exact probabilities 1/4
        add(f"special/V{V}/inf4", y, top_p=1.0)
        add(f"special/V{V}/all_nan", np.full(V, np.nan), top_p=0.93)
        z = _shape("mid", V, rng)
        z[3] = np.inf
        add(f"special/V{V}/overflow_fallback", z, temperature=1e-35)
    # 6. repetition penalty over negative, zero and positive logits; windows of 49 / 50 / 51 / 80
    for V in (2049, 513):
        for n in HLENS:
            for rep in (1.1, 0.8):
                for sign in (1.0, -1.0):
                    rng = np.random.default_rng(V + n * 7 + int(rep * 10) + int(sign))
                    x = rng.uniform(-1, 1, V) * 0.3 + sign * 1.5
                    x[rng.integers(0, V, 3)] = 0.0
                    order = np.argsort(-x)
                    x[order[0]] = x[order[1]] + 0.05 * sign  # best and second close: a penalty decides
                    add(f"pen/V{V}/h{n}/r{rep}/s{sign:+.0f}", x, _hist_window(V, x, n, rng), rep=rep, temperature=1.0,
                        top_p=0.999999, top_k=2, noise=np.ones(V))
    # 7. top-p: an exact hit of top_p (strict >), cuts inside ranks 33-63, the extremes
    for V in (2049, 64, 5):
        for n_top, tp in ((4, 0.5), (8, 0.375), (2, 0.5), (4, 0.75)):
            if n_top > V:
                continue
            x = np.full(V, -1e9)
            x[np.arange(n_top) * (V // n_top)] = 0.0
            noise = np.ones(V)
            noise[int(round(tp * n_top))] = 0.25  # the rank just past the last kept one with a strict cut
            add(f"topp/V{V}/exact{n_top}_{tp}", x, top_p=tp, temperature=1.0, rep=1.0, noise=noise, top_k=64)
    for V in (2049, 4096):
        for tp in (0.55, 0.7, 0.8):
            rng = np.random.default_rng(V + int(tp * 100))
            add(f"topp/V{V}/upper_half_{tp}", _shape("flat", V, rng), top_p=tp, top_k=64, temperature=1.0)
        for tp in (1e-6, 0.999999):
            rng = np.random.default_rng(V + 17)
            add(f"topp/V{V}/extreme_{tp}", _shape("mid", V, rng), top_p=tp, top_k=64)
    # 8. noise: exact p / q ties (within a lane, between lanes, between the two halves), tiny draws, zero draws
    for V in (2049, 64):
        x = np.full(V, -1e9)
        x[np.arange(64) * (V // 64)] = 0.0  # 64 equal probabilities, exact
        for a, b in ((3, 35), (3, 5), (10, 40), (33, 60)):
            noise = np.ones(V) * 2.0
            noise[a] = noise[b] = 0.5
            add(f"noise/V{V}/ratio_tie_{a}_{b}", x, top_p=0.999999, top_k=64, temperature=1.0, rep=1.0, noise=noise)
            noise = np.ones(V) * 2.0
            toks = np.arange(64) * (V // 64)
            noise[toks[b]] = noise[toks[a]] = 0.5
            add(f"noise/V{V}/ratio_tie_ids_{a}_{b}", x, top_p=1.0, top_k=64, temperature=1.0, rep=1.0, noise=noise)
    for V in (2049, 512):
        rng = np.random.default_rng(V + 23)
        x = _shape("mid", V, rng)
        for small in (1e-30, 1e-37):
            noise = _tape(V + 29, V).numpy().astype(np.float64)
            noise[7] = small  # rank 7 is drawn
            add(f"noise/V{V}/small_{small}", x, top_p=0.9, noise=noise)
            noise2 = _tape(V + 31, V).numpy().astype(np.float64)
            noise2[int(np.argsort(-x)[3])] = small  # the 4th most likely token is drawn
            add(f"noise/V{V}/small_ids_{small}", x, top_p=1.0, noise=noise2)
        noise = _tape(V + 37, V).numpy().astype(np.float64)
        noise[2] = 0.0  # a positive probability with a zero draw: +inf wins
        add(f"noise/V{V}/zero_kept", x, top_p=0.9, noise=noise)
        noise = _tape(V + 41, V).numpy().astype(np.float64)
        noise[V - 3] = 0.0  # a zero draw at a zero-probability rank: never drawn by the device
        add(f"noise/V{V}/zero_removed", x, top_p=0.9, noise=noise)
    # 9. recovery: a recovery pair that differs from the normal pair
    for V in (2049, 4096, 65):
        for j in range(4):
            rng = np.random.default_rng(V * 3 + j)
            add(f"recovery/V{V}/{j}", _shape(("mid", "peaked", "flat", "mid")[j], V, rng), rng.integers(0, V, 30).tolist(),
                recovery=True, top_p=(0.9, 1.0, 0.5, 0.95)[j], temperature=(1.05, 0.7, 1.0, 0.05)[j],
                rec_top_p=(0.5, 0.85, 1.0, 0.6)[j], rec_temp=(1.0, 2.5, 0.3, 1.2)[j])
    return rows
