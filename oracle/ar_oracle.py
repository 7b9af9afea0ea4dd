"""CPU oracle for the autoregressive codec-token path.  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
reference legs may import this module.  The product (sopro_b200/) never does.

This is a functional restatement (flat state_dict in, tensors out) of the
reference's PyTorch-eager algorithm, written with the same torch CPU operators
in the same order so that, on one host, it is bit-identical to the reference
modules.  Each function cites the reference lines it follows
(paths relative to /root/reference/src/sopro/).

Parity pin: the reference ships no tests or golden vectors (SURVEY.md §4), so
this oracle is pinned against the reference itself, imported in the build
container: tests/golden/make_golden.py runs both on the same seeded inputs,
asserts bit-equality, and writes the fixtures tests/test_oracle_golden.py
re-checks anywhere (see DESIGN.md "Oracle").
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, Iterator, List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

from oracle.dense_probes import rel_errors

Tensor = torch.Tensor
SD = Dict[str, Tensor]


# ---------------------------------------------------------------------------
# building blocks
# ---------------------------------------------------------------------------
def _acc(t: Tensor) -> Tensor:
    """The compute type: float64 stays float64 (the float64 oracle), everything else is computed in fp32 as the
    reference does."""
    return t if t.dtype == torch.float64 else t.float()


def rms_norm(x: Tensor, w: Tensor, eps: float = 1e-6) -> Tensor:
    """nn/blocks.py:32-37 — fp32 mean of squares, rsqrt, scale by weight (float64 for float64 input)."""
    x32 = _acc(x)
    var = x32.pow(2).mean(dim=-1, keepdim=True)
    y32 = x32 * torch.rsqrt(var + eps)
    y32 = y32 * w.to(x32.dtype)
    return y32.to(dtype=x.dtype)


def glu(x: Tensor, w: Tensor, b: Tensor) -> Tensor:
    """nn/blocks.py:21-23 — rows [0,d) are the value, rows [d,2d) the gate."""
    a, g = F.linear(x, w, b).chunk(2, dim=-1)
    return a * torch.sigmoid(g)


def dwconv_step(h: Tensor, ring: Tensor, w_dk: Tensor, bias: Tensor, dil: int) -> Tuple[Tensor, Tensor]:
    """nn/blocks.py:92-110 — push one frame into the ring, 13-tap dilated MAC.

    ``ring`` is [B, (k-1)*dil+1, D] with the newest frame LAST; tap j reads row
    j*dil, so w[:, k-1] multiplies the current frame."""
    if ring.size(1) > 1:
        ring = torch.cat([ring[:, 1:, :], h], dim=1)
    else:
        ring = h
    k = int(w_dk.size(-1))
    idx = torch.arange(0, k * dil, dil)
    taps = ring.index_select(1, idx)  # [B,k,D]
    y = (taps.transpose(1, 2) * w_dk.unsqueeze(0)).sum(dim=-1)
    y = y + bias.unsqueeze(0)
    return y.unsqueeze(1), ring


def ssm_block_step(sd: SD, p: str, x: Tensor, ring: Tensor, dil: int) -> Tuple[Tensor, Tensor]:
    """nn/blocks.py:150-162 — norm→GLU→dwconv(+res)→norm→FFN(GELU-erf)(+res)."""
    h = glu(rms_norm(x, sd[p + "norm.weight"]), sd[p + "glu.pro.weight"], sd[p + "glu.pro.bias"])
    y, ring = dwconv_step(h, ring, sd[p + "dw.dw.weight"].squeeze(1), sd[p + "dw.dw.bias"], dil)
    x = x + y
    f = rms_norm(x, sd[p + "ff.0.weight"])
    f = F.linear(f, sd[p + "ff.1.weight"], sd[p + "ff.1.bias"])
    f = F.gelu(f)  # exact erf form, nn.GELU() default (nn/blocks.py:131)
    f = F.linear(f, sd[p + "ff.3.weight"], sd[p + "ff.3.bias"])
    return x + f, ring


def _heads(t: Tensor, n_heads: int) -> Tensor:
    B, T, D = t.shape
    return t.view(B, T, n_heads, D // n_heads).transpose(1, 2)


def text_kv_cache(sd: SD, p: str, txt_seq: Tensor, n_heads: int) -> Tuple[Tensor, Tensor]:
    """nn/text.py:75-83 — K,V = W·RMSNorm_kv(text), split into heads [B,H,L,Dh]."""
    kv = rms_norm(txt_seq, sd[p + "nkv.weight"])
    k = _heads(F.linear(kv, sd[p + "k_proj.weight"]), n_heads)
    v = _heads(F.linear(kv, sd[p + "v_proj.weight"]), n_heads)
    return k, v


def xattn_step(sd: SD, p: str, x: Tensor, k: Tensor, v: Tensor, keep: Optional[Tensor], n_heads: int) -> Tensor:
    """nn/text.py:93-131 — pre-norm q, fp32 SDPA (float64 for float64 input) over the
    cached text K/V with a boolean keep-mask, nan_to_num, out-proj, x + tanh(gate)*a."""
    q = _heads(F.linear(rms_norm(x, sd[p + "nq.weight"]), sd[p + "q_proj.weight"]), n_heads)
    mask = None
    if keep is not None:
        keep = keep.to(torch.bool)
        bad = ~keep.any(dim=1)
        if bad.any():
            keep = keep.clone()
            keep[bad, 0] = True
        mask = keep[:, None, None, :]
    a = F.scaled_dot_product_attention(_acc(q), _acc(k), _acc(v), attn_mask=mask, dropout_p=0.0, is_causal=False)
    a = torch.nan_to_num(a, nan=0.0, posinf=0.0, neginf=0.0).to(x.dtype)
    B, H, T, Dh = a.shape
    a = a.transpose(1, 2).contiguous().view(B, T, H * Dh)
    a = F.linear(a, sd[p + "out_proj.weight"])
    return x + torch.tanh(sd[p + "gate"]) * a


# ---------------------------------------------------------------------------
# the step
# ---------------------------------------------------------------------------
@dataclass
class ArState:
    rings: List[Tensor]
    kv: Dict[int, Tuple[Tensor, Tensor]]
    keep: Optional[Tensor]


def ar_init_state(sd: SD, cfg, txt_seq: Tensor, text_mask: Optional[Tensor], batch: int = 1) -> ArState:
    """nn/generator.py:44-68 — zero rings of (k-1)*dil+1 rows, text K/V per attn layer."""
    D = int(cfg.d_model)
    k = int(cfg.ar_kernel)
    rings = [torch.zeros((batch, (k - 1) * d + 1, D), dtype=txt_seq.dtype) for d in cfg.ar_dilations()]
    kv = {i: text_kv_cache(sd, f"ar.x_attns.{i}.", txt_seq, cfg.AR_HEADS) for i in cfg.ar_attn_layers()}
    return ArState(rings=rings, kv=kv, keep=text_mask)


def ar_step(sd: SD, cfg, x: Tensor, st: ArState, trace: Optional[dict] = None) -> Tensor:
    """nn/generator.py:98-130 — x [B,1,D] → logits [B,1,V]; mutates ``st``."""
    h = x
    for i, dil in enumerate(cfg.ar_dilations()):
        h, st.rings[i] = ssm_block_step(sd, f"ar.blocks.{i}.", h, st.rings[i], dil)
        if i in st.kv:
            k, v = st.kv[i]
            h = xattn_step(sd, f"ar.x_attns.{i}.", h, k, v, st.keep, cfg.AR_HEADS)
        if trace is not None:
            trace[f"h{i}"] = h.clone()
    h = rms_norm(h, sd["ar.norm.weight"])
    return F.linear(h, sd["ar.head.weight"], sd["ar.head.bias"])


@dataclass
class ArTrace:
    """What a teacher-forced run of ar_step computed, in the kernel's trace layouts."""
    blocks: Tensor                    # [steps, n_layers, B, D] residual after every layer
    logits: Tensor                    # [steps, B, V]
    kv: Dict[int, Tuple[Tensor, Tensor]]  # attention layer -> text (K, V), each [B, H, Lmax, Dh]


def ar_teacher_forced(sd: SD, cfg, cond_ar: Tensor, txt_seq: Tensor, text_len: Sequence[int], forced: Tensor,
                      dtype: torch.dtype = torch.float32) -> ArTrace:
    """A ragged batch through ar_step with the tokens forced, every tensor cast to ``dtype`` (float64: the float64
    oracle; float32: the reference's arithmetic).

    cond_ar [B, steps, D], txt_seq [B, Lmax, D] (rows past text_len[b] are padding, masked out through the keep-mask),
    forced [B, steps] token ids: step 0 takes the BOS row, step t the embedding row of forced[:, t - 1] (EOS =
    codebook_size is fed back as table row codebook_size, model.py:266-272)."""
    sd = {k: v.to(dtype) for k, v in sd.items()}
    cond_ar, txt_seq = cond_ar.to(dtype), txt_seq.to(dtype)
    B, steps, _D = cond_ar.shape
    keep = torch.arange(txt_seq.size(1))[None, :] < torch.as_tensor(list(text_len))[:, None]
    st = ar_init_state(sd, cfg, txt_seq, keep, batch=B)
    emb = sd["cb_embed.emb.weight"]
    bos_row = int(cfg.num_codebooks) * int(cfg.codebook_size)
    n_layers = int(cfg.n_layers_ar)
    blocks = torch.empty((steps, n_layers, B, int(cfg.d_model)), dtype=dtype)
    logits = torch.empty((steps, B, int(cfg.ar_vocab())), dtype=dtype)
    for t in range(steps):
        rows = torch.full((B,), bos_row, dtype=torch.long) if t == 0 else forced[:, t - 1].long()
        tr: dict = {}
        logits[t] = ar_step(sd, cfg, cond_ar[:, t: t + 1] + emb[rows].unsqueeze(1), st, tr)[:, 0]
        for i in range(n_layers):
            blocks[t, i] = tr[f"h{i}"][:, 0]
    return ArTrace(blocks=blocks, logits=logits, kv=dict(st.kv))


def ar_trace_labels(cfg) -> List[str]:
    """Names of the quantities ar_trace_errors compares, in its order."""
    attn = list(cfg.ar_attn_layers())
    return ([f"h{i}" for i in range(int(cfg.n_layers_ar))] + ["logits"] + [f"k{i}" for i in attn]
            + [f"v{i}" for i in attn])


def ar_trace_errors(got: ArTrace, ref: ArTrace, text_len: Sequence[int]) -> Tensor:
    """[B, len(ar_trace_labels), 2] float64: for every utterance, the max and RMS error of each layer's residual, of
    the logits, and of every attention layer's text K and V rows [:text_len[b]], against ``ref``, relative to that
    utterance's own peak and RMS (dense_probes.rel_errors) over all its steps."""
    B = got.logits.size(1)
    n_layers = got.blocks.size(1)
    out = torch.empty((B, n_layers + 1 + 2 * len(ref.kv), 2), dtype=torch.float64)
    for b in range(B):
        L = int(text_len[b])
        pairs = [(got.blocks[:, i, b], ref.blocks[:, i, b]) for i in range(n_layers)]
        pairs.append((got.logits[:, b], ref.logits[:, b]))
        pairs += [(got.kv[i][0][b, :, :L], ref.kv[i][0][b, :, :L]) for i in ref.kv]
        pairs += [(got.kv[i][1][b, :, :L], ref.kv[i][1][b, :, :L]) for i in ref.kv]
        for j, (z, z64) in enumerate(pairs):
            out[b, j] = torch.tensor(rel_errors(z, z64), dtype=torch.float64)
    return out


# ---------------------------------------------------------------------------
# sampler
# ---------------------------------------------------------------------------
def repeated_tail(hist: Sequence[int], max_n: int = 16) -> bool:
    """sampling.py:16-21 — last n ids equal the n before them, for some n>=3."""
    L = len(hist)
    for n in range(3, min(max_n, L // 2) + 1):
        if list(hist[L - n:]) == list(hist[L - 2 * n: L - n]):
            return True
    return False


def sample_token(
    logits_1x1v: Tensor,
    history: Sequence[int],
    *,
    top_p: float,
    top_k: int,
    temperature: float,
    repetition_penalty: float,
    noise_v: Optional[Tensor] = None,
    eps: float = 1e-12,
    trace: Optional[dict] = None,
) -> int:
    """sampling.py:24-93.

    ``noise_v`` ([V] Exp(1) draws) replaces the RNG: torch.multinomial(p, 1) on
    CPU is argmax(p / q) with q = empty_like(p).exponential_(1) (ATen
    native/Distributions.cpp multinomial fast path; verified against
    torch.multinomial in tests/test_oracle_golden.py).  When ``noise_v`` is None
    the global generator is consumed exactly as the reference does."""
    x = torch.nan_to_num(logits_1x1v, nan=-1e9, posinf=1e9, neginf=-1e9)
    if temperature and temperature != 1.0:
        x = x / float(temperature)
    if repetition_penalty != 1.0 and len(history) > 0:
        ids = torch.tensor(list(set(history[-50:])), dtype=torch.long)
        if ids.numel() > 0:
            vals = x[0, 0, ids]
            vals = torch.where(vals < 0, vals * repetition_penalty, vals / repetition_penalty)
            x = x.clone()
            x[0, 0, ids] = vals
    probs = torch.softmax(x, dim=-1).view(1, -1)
    probs = torch.nan_to_num(probs, nan=0.0, posinf=0.0, neginf=0.0)
    V = int(probs.size(-1))

    def _draw(p: Tensor) -> int:
        if noise_v is None:
            return int(torch.multinomial(p, 1).item())
        return int(torch.argmax(p / noise_v.view(1, -1), dim=-1).item())

    if top_k and top_k > 0:
        kk = min(int(top_k), V)
        val, idx = torch.topk(probs, kk, dim=-1)
        newp = torch.zeros_like(probs)
        newp.scatter_(1, idx, val)
        probs = newp
        s = probs.sum(dim=-1, keepdim=True)
        if float(s.item()) <= eps:
            return int(torch.argmax(x[0, 0]).item())
        probs = probs / s
    if top_p is not None and top_p < 1.0:
        sp, si = torch.sort(probs, descending=True, dim=-1)
        cum = torch.cumsum(sp, dim=-1)
        if trace is not None:
            trace["cum"] = cum[0, :64].clone()
        remove = cum > float(top_p)
        remove[..., 1:] = remove[..., :-1].clone()
        remove[..., 0] = False
        sp = sp.masked_fill(remove, 0.0)
        s = sp.sum(dim=-1, keepdim=True)
        if float(s.item()) <= eps:
            return int(torch.argmax(x[0, 0]).item())
        sp = sp / s
        if trace is not None:
            trace["sorted_probs"] = sp[0, :64].clone()
            trace["sorted_idx"] = si[0, :64].clone()
        return int(si[0, _draw(sp)].item())
    s = probs.sum(dim=-1, keepdim=True)
    if float(s.item()) <= eps:
        return int(torch.argmax(x[0, 0]).item())
    return _draw(probs / s)


# ---------------------------------------------------------------------------
# the serial driver
# ---------------------------------------------------------------------------
@dataclass
class ArSampling:
    """Per-call knobs of ar_stream (model.py:218-231) + the literals it hard-wires
    (model.py:289-290)."""
    top_p: float = 0.9
    temperature: float = 1.05
    anti_loop: bool = True
    loop_streak: int = 8
    recovery_top_p: float = 0.85
    recovery_temp: float = 1.2
    min_gen_frames: Optional[int] = None
    top_k: int = 50
    repetition_penalty: float = 1.1


def ar_stream(
    sd: SD,
    cfg,
    cond_ar: Tensor,
    txt_seq: Tensor,
    text_mask: Optional[Tensor],
    *,
    max_frames: int,
    sampling: ArSampling = ArSampling(),
    noise_tv: Optional[Tensor] = None,
    logits_out: Optional[List[Tensor]] = None,
    recovery_out: Optional[List[int]] = None,
) -> Iterator[Tuple[int, int, bool]]:
    """model.py:218-305 — yields (t, token, is_eos), batch 1.

    ``noise_tv`` [max_frames+1, V] is the Exp(1) tape, one row per step; None =
    consume the global torch generator like the reference."""
    eos_id = int(cfg.codebook_size)
    min_gen = int(sampling.min_gen_frames if sampling.min_gen_frames is not None else cfg.min_gen_frames)
    steps = int(max_frames) + 1
    emb = sd["cb_embed.emb.weight"]
    bos_row = int(cfg.num_codebooks) * int(cfg.codebook_size)
    st = ar_init_state(sd, cfg, txt_seq, text_mask, batch=1)
    hist: List[int] = []
    streak, last = 0, None
    prev = None
    for t in range(steps):
        row = bos_row if t == 0 else prev  # cb_index 0 → row == token id (embeddings.py:51-55)
        x_t = cond_ar[:, t: t + 1, :] + emb[row].view(1, 1, -1)
        cur_p, cur_t = sampling.top_p, sampling.temperature
        if sampling.anti_loop:
            if repeated_tail(hist, 16) or (last is not None and streak >= sampling.loop_streak):
                cur_p, cur_t = sampling.recovery_top_p, sampling.recovery_temp
                if recovery_out is not None:
                    recovery_out.append(t)
        logits = ar_step(sd, cfg, x_t, st)
        if logits_out is not None:
            logits_out.append(logits[0, 0].clone())
        tok = sample_token(
            logits, hist, top_p=cur_p, top_k=sampling.top_k, temperature=cur_t,
            repetition_penalty=sampling.repetition_penalty,
            noise_v=None if noise_tv is None else noise_tv[t],
        )
        hist.append(tok)
        streak = streak + 1 if (last is not None and tok == last) else 0
        last = tok
        prev = tok
        is_eos = tok == eos_id
        yield t, tok, is_eos
        if is_eos and (t + 1) >= min_gen:
            break


def ar_generate(sd: SD, cfg, cond_ar: Tensor, txt_seq: Tensor, text_mask: Optional[Tensor], **kw) -> List[int]:
    return [tok for _t, tok, _e in ar_stream(sd, cfg, cond_ar, txt_seq, text_mask, **kw)]


def noise_tape(seed: int, steps: int, vocab: int) -> Tensor:
    """The Exp(1) draws `steps` successive torch.multinomial calls would consume
    after torch.manual_seed(seed) (SURVEY.md §0.6): one [steps, V] exponential_
    equals `steps` successive [1, V] calls."""
    g = torch.Generator().manual_seed(int(seed))
    return torch.empty(steps, vocab).exponential_(1.0, generator=g)
