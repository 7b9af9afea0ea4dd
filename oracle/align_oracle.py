"""CPU oracle for word timestamps (no reference counterpart).  TEST INFRASTRUCTURE ONLY.

`ar_step_attn_probs` is one AR step of oracle/ar_oracle.py that also returns the text cross-attention weights the
kernel exports, in float64.  `first_frames` restates the alignment of include/sopro_b200.h (sopro_b200/csrc/align.cu)
in float64 numpy, in the same order of IEEE double additions and comparisons, so its path equals the device's bit for
bit.  `words_for` and `long_words` restate the host mapping of sopro_b200/timestamps.py independently: tokens -> words
-> seconds."""
from __future__ import annotations

import re
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from oracle.ar_oracle import ArState, _heads, rms_norm, ssm_block_step, xattn_step


def ar_step_attn_probs(sd, cfg, x: torch.Tensor, st: ArState) -> Tuple[torch.Tensor, torch.Tensor]:
    """ar_oracle.ar_step (the same fp32 residual stream; mutates ``st``) that also returns every text cross-attention's
    weights in float64: softmax(q . k / sqrt(Dh)) over the kept keys from the step's fp32 q and cached K, as
    [n_attn, B, H, L] (the attention layers in ascending order) -> (logits [B,1,V], probs)."""
    probs = []
    h = x
    for i, dil in enumerate(cfg.ar_dilations()):
        h, st.rings[i] = ssm_block_step(sd, f"ar.blocks.{i}.", h, st.rings[i], dil)
        if i in st.kv:
            p = f"ar.x_attns.{i}."
            k, v = st.kv[i]
            q = _heads(F.linear(rms_norm(h, sd[p + "nq.weight"]), sd[p + "q_proj.weight"]), cfg.AR_HEADS)  # [B,H,1,Dh]
            s = torch.einsum("bhqd,bhld->bhql", q.double(), k.double())[:, :, 0] / float(q.shape[-1]) ** 0.5
            if st.keep is not None:
                s = s.masked_fill(~st.keep.to(torch.bool)[:, None, :], float("-inf"))
            probs.append(torch.softmax(s, dim=-1))
            h = xattn_step(sd, p, h, k, v, st.keep, cfg.AR_HEADS)
    h = rms_norm(h, sd["ar.norm.weight"])
    return F.linear(h, sd["ar.head.weight"], sd["ar.head.bias"]), torch.stack(probs)


def accumulate(probs: np.ndarray, b: int, T: int, L: int) -> np.ndarray:
    """A[t][l] for t < T, l < L: (double) probs[t][s][b][h][l] summed over s ascending, then h ascending, from 0.0."""
    steps, n_attn, _B, H, _ld = probs.shape
    A = np.zeros((T, L), dtype=np.float64)
    for s in range(n_attn):
        for h in range(H):
            A += probs[:T, s, b, h, :L].astype(np.float64)
    return A


def path_from_scores(A: np.ndarray) -> Optional[np.ndarray]:
    """The DP over A [T, L] -> first frame of each token (int64 [L]), or None when there is no path."""
    T, L = A.shape
    if T == 0 or T < L:
        return None
    S = np.full(L, -np.inf)
    S[0] = A[0, 0]
    moves = np.zeros((T, L), dtype=bool)
    for t in range(1, T):
        stay = S
        move = np.concatenate([[-np.inf], S[:-1]])
        mv = move > stay  # ties: stay
        moves[t] = mv
        S = A[t] + np.where(mv, move, stay)
    first = np.full(L, -1, dtype=np.int64)
    l = L - 1
    for t in range(T - 1, 0, -1):
        if l > 0 and moves[t, l]:
            first[l] = t
            l -= 1
    if l != 0:
        return None
    first[0] = 0
    return first


def first_frames(probs: np.ndarray, text_len: Sequence[int], frames: Sequence[int]) -> np.ndarray:
    """probs [steps, n_attn, B, H, ld] f32 -> first [B, ld] int32, as sopro_align writes it."""
    _steps, _n, B, _H, ld = probs.shape
    out = np.full((B, ld), -1, dtype=np.int32)
    for b in range(B):
        L, T = int(text_len[b]), int(frames[b])
        if T == 0 or T < L:
            continue
        f = path_from_scores(accumulate(probs, b, T, L))
        if f is not None:
            out[b, :L] = f
    return out


# ---- host mapping, restated

def _word_list(text: str) -> List[Tuple[str, int, int]]:
    out, i, n = [], 0, len(text)
    while i < n:
        if text[i].isspace():
            i += 1
            continue
        j = i
        while j < n and not text[j].isspace():
            j += 1
        out.append((text[i:j], i, j))
        i = j
    return out


def _owner(text: str, span, words) -> Optional[int]:
    if span is None:
        return None
    for c in range(span[0], span[1]):
        if not text[c].isspace():
            for k, (_w, a, b) in enumerate(words):
                if a <= c < b:
                    return k
            return None
    return None


def _word_frames(text: str, spans, first, T: int) -> List[Tuple[int, int]]:
    words = _word_list(text)
    L = len(spans)
    ends = [int(first[l + 1]) if l + 1 < L else int(T) for l in range(L)]
    res = []
    last_end = 0
    for k in range(len(words)):
        toks = [l for l in range(L) if _owner(text, spans[l], words) == k]
        if toks:
            res.append((int(first[toks[0]]), ends[toks[-1]]))
            last_end = ends[toks[-1]]
        else:
            res.append((last_end, last_end))
    return res


def _seconds(sample: int, S: Optional[int]) -> float:
    x = float(sample)
    if S is not None:
        x = x * 65536.0 / float(S)
    return x / 24000.0


def words_for(text: str, spans, first, T: int, hop: int, S: Optional[int] = None) -> List[tuple]:
    """(word, start s, end s, char_start, char_end) per word; [] without an alignment."""
    if first is None or len(spans) == 0 or int(first[0]) < 0:
        return []
    words = _word_list(text)
    fr = _word_frames(text, spans, first, T)
    return [(w, _seconds(f0 * hop, S), _seconds(f1 * hop, S), a, b) for (w, a, b), (f0, f1) in zip(words, fr)]


def long_words(text: str, segments: Sequence[str], seg_spans, firsts, Ts, hop: int, extents, pause: int,
               S: Optional[int] = None) -> List[tuple]:
    """synthesize_long's words: segment i's sample x lands at O_i + clamp(x, e0, e1) - e0."""
    all_words = _word_list(text)
    out, k, offset = [], 0, 0
    for i, seg in enumerate(segments):
        e0, e1 = int(extents[i][0]), int(extents[i][1])
        seg_words = _word_list(seg)
        f = firsts[i]
        live = e1 > e0 and f is not None and int(f[0]) >= 0
        fr = _word_frames(seg, seg_spans[i], f, int(Ts[i])) if live else None
        for j, (w, _a, _b) in enumerate(seg_words):
            tw, ta, tb = all_words[k]
            assert tw == w, (tw, w)
            if live:
                x0 = offset + min(max(fr[j][0] * hop, e0), e1) - e0
                x1 = offset + min(max(fr[j][1] * hop, e0), e1) - e0
            else:
                x0 = x1 = offset
            out.append((tw, _seconds(x0, S), _seconds(x1, S), ta, tb))
            k += 1
        if e1 > e0:
            offset += e1 - e0 + pause
    assert k == len(all_words)
    return out


def word_spans_regex(text: str) -> List[Tuple[int, int]]:
    """The words as \\S+ runs (for cross-checking the scanner above)."""
    return [(m.start(), m.end()) for m in re.finditer(r"\S+", text)]
