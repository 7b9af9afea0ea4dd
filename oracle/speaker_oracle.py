"""Token2SV (reference nn/speaker.py: Token2SV.forward; nn/blocks.py: DepthwiseConv1d, AttentiveStatsPool) restated in
float64, for a ragged batch whose every row is computed as a sequence of its own length.

Per row b, over its first lens[b] frames only:
  x[t]     = sum_q softmax(cb_weights)[q] * emb[q*V + codes[t, q]]
  h        = GELU(dwconv(GELU(dwconv(x))))      depthwise, kernel k, non-causal: left = (k-1)//2, zero padding both ends
  u[t]     = W0 h[t] + b0;   logit[t] = w2 . tanh(u[t]) + b2;   a = softmax over the row's frames
  mu       = sum_t a[t] h[t];   std = sqrt(max(sum_t a[t] (h[t] - mu)^2, 1e-6))
  e        = P [mu | std] + p;   sv = e / max(||e||, 1e-6)

The reference's own padded batch is not row-wise: its second convolution reads GELU(bias) at the padding frames of a
shorter row.  Its only caller prepares one reference at a time, so every sv it produces is the B = 1 case, which this
restatement reproduces for any batch."""
from __future__ import annotations

import math
from typing import Dict, Optional, Sequence, Tuple

import torch

SD = Dict[str, torch.Tensor]


def _gelu(x: torch.Tensor) -> torch.Tensor:
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def _dwconv_same(x_td: torch.Tensor, w_dk: torch.Tensor, b_d: torch.Tensor) -> torch.Tensor:
    T, D = x_td.shape
    k = int(w_dk.shape[-1])
    left = (k - 1) // 2
    xp = torch.zeros(T + k - 1, D, dtype=x_td.dtype)
    xp[left: left + T] = x_td
    y = b_d.unsqueeze(0).expand(T, D).clone()
    for j in range(k):
        y = y + xp[j: j + T] * w_dk[:, j].unsqueeze(0)
    return y


def speaker_vectors(sd: SD, codebook_size: int, codes_btq: torch.Tensor, lens: Sequence[int],
                    ref_sv: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """codes [B, Tmax, Q] (row b's first lens[b] frames) -> (sv [B, sv_dim] float64, cos [B] float64 with ref_sv)."""
    f = lambda name: sd[name].detach().to("cpu", torch.float64)  # noqa: E731
    emb, cbw = f("token2sv.emb.weight"), torch.softmax(f("token2sv.cb_weights"), dim=0)
    w0, b0 = f("token2sv.enc.0.dw.weight").reshape(emb.shape[1], -1), f("token2sv.enc.0.dw.bias")
    w1, b1 = f("token2sv.enc.3.dw.weight").reshape(emb.shape[1], -1), f("token2sv.enc.3.dw.bias")
    pw0, pb0 = f("token2sv.pool.attn.0.weight"), f("token2sv.pool.attn.0.bias")
    pw2, pb2 = f("token2sv.pool.attn.2.weight").reshape(-1), f("token2sv.pool.attn.2.bias").reshape(-1)[0]
    P, p = f("token2sv.proj.weight"), f("token2sv.proj.bias")
    codes = codes_btq.detach().to("cpu", torch.long)
    Q, V = int(codes.shape[2]), int(codebook_size)
    out = []
    for b, n in enumerate(int(x) for x in lens):
        c = codes[b, :n]
        rows = emb[torch.arange(Q).view(1, Q) * V + c]  # [n, Q, d]
        x = (rows * cbw.view(1, Q, 1)).sum(dim=1)
        h = _gelu(_dwconv_same(_gelu(_dwconv_same(x, w0, b0)), w1, b1))
        logit = torch.tanh(h @ pw0.T + pb0) @ pw2 + pb2
        a = torch.softmax(logit, dim=0).unsqueeze(1)
        mu = (a * h).sum(dim=0)
        std = torch.sqrt((a * (h - mu).pow(2)).sum(dim=0).clamp_min(1e-6))
        e = P @ torch.cat([mu, std]) + p
        out.append(e / e.norm().clamp_min(1e-6))
    sv = torch.stack(out)
    cos = None if ref_sv is None else sv @ ref_sv.detach().to("cpu", torch.float64).reshape(-1)
    return sv, cos
