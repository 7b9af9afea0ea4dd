"""TEST INFRASTRUCTURE (never imported by the product): CPU restatement of the NAR refiner.

Follows the reference op by op: SoproTTSModel.nar_refine (reference src/sopro/model.py:307-347),
NARSinglePass.forward_stage (nn/nar.py:89-116), NARStageAdapter.forward (nn/nar.py:24-32),
CodebookEmbedding.sum_embed_subset (nn/embeddings.py:77-112), SSMLiteBlock.forward (nn/blocks.py:143-148),
DepthwiseConv1d.forward (nn/blocks.py:63-74).  Pinned against tokens the UNMODIFIED reference produced
(tests/golden/e2e_prefill.npz `nar_tokens`, written by tests/golden/make_golden_e2e.py) in
tests/test_oracle_golden.py.  Besides the ids it returns, per id, the relative margin between the two largest
logits (how far the argmax is from a tie) and accepts teacher-forced previous codebooks, so a GPU-vs-oracle
mismatch can be classified as a near-tie or a bug.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

Tensor = torch.Tensor
SD = Dict[str, Tensor]


def rms_norm(x: Tensor, w: Tensor, eps: float = 1e-6) -> Tensor:
    x32 = x if x.dtype == torch.float64 else x.float()  # float64 mode keeps float64
    y = x32 * torch.rsqrt(x32.pow(2).mean(dim=-1, keepdim=True) + eps)
    return (y * w.to(x32.dtype)).to(x.dtype)


def dwconv_same(x_btd: Tensor, w: Tensor, b: Tensor, dilation: int) -> Tensor:
    k = int(w.shape[-1])
    total = (k - 1) * dilation
    left = total // 2
    xt = F.pad(x_btd.transpose(1, 2), (left, total - left))
    return F.conv1d(xt, w, b, groups=w.shape[0], dilation=dilation).transpose(1, 2)


def ssm_block(sd: SD, p: str, x: Tensor, dilation: int) -> Tensor:
    a, g = F.linear(rms_norm(x, sd[p + "norm.weight"]), sd[p + "glu.pro.weight"], sd[p + "glu.pro.bias"]).chunk(2, dim=-1)
    x = x + dwconv_same(a * torch.sigmoid(g), sd[p + "dw.dw.weight"], sd[p + "dw.dw.bias"], dilation)
    f = F.linear(rms_norm(x, sd[p + "ff.0.weight"]), sd[p + "ff.1.weight"], sd[p + "ff.1.bias"])
    return x + F.linear(F.gelu(f), sd[p + "ff.3.weight"], sd[p + "ff.3.bias"])


def nar_refine(sd: SD, cfg, cond_seq: Tensor, rvq1_bt: Tensor, forced: Optional[Tensor] = None,
               dtype: torch.dtype = torch.float32, z_out: Optional[List[Tensor]] = None) -> Tuple[Tensor, Tensor]:
    """-> (codes [B, T, Q] int64, margin [B, T, Q] f32).  margin[..., q] = (top1 - top2) / max|logit| of the head
    that decided codebook q (inf for q = 0).  `forced` [B, T, Q]: the previous codebooks every stage conditions on are
    taken from it instead of from this run's own argmax.  dtype=torch.float64 runs the whole refiner on the state dict
    and the conditioning cast to float64 (the reference the kernels' rounding is measured against).  z_out: a list that
    receives each stage's pre-head activation z [B, T, Hn]."""
    if dtype != torch.float32:
        sd = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in sd.items() if k.startswith(("nar", "cb_embed."))}
        cond_seq = cond_seq.to(dtype)
    B, T, D = cond_seq.shape
    Q, V = int(cfg.num_codebooks), int(cfg.codebook_size)
    out = torch.zeros((B, T, Q), dtype=torch.long)
    margin = torch.full((B, T, Q), float("inf"))
    out[:, :, 0] = rvq1_bt
    emb = sd["cb_embed.emb.weight"]
    stages = [(n, idx) for n, idx in cfg.stage_indices().items() if len(idx) > 0]
    dils = cfg.nar_dilations()
    src = out if forced is None else forced.long()
    for sid, (name, idxs) in enumerate(stages):
        cbs = list(range(0, idxs[0]))
        cbt = torch.tensor(cbs, dtype=torch.long)
        toks = src[:, :, : idxs[0]] if forced is not None else out[:, :, : idxs[0]]
        e = emb[cbt.view(1, 1, -1) * V + toks]
        w = F.softmax(sd["nar_prev_cb_weights"].to(dtype).index_select(0, cbt), dim=0)
        prev_sum = (e * w.view(1, 1, -1, 1)).sum(dim=2)
        mix = torch.softmax(sd[f"nar.mix.{name}"], dim=0)
        x = mix[0] * cond_seq + mix[1] * prev_sum
        sv = sd["nar.stage_emb.weight"][sid].unsqueeze(0).expand(B, -1)
        g, b = F.linear(F.gelu(F.linear(sv, sd["nar.adapter.mlp.0.weight"], sd["nar.adapter.mlp.0.bias"])),
                        sd["nar.adapter.mlp.2.weight"], sd["nar.adapter.mlp.2.bias"]).chunk(2, dim=-1)
        x = rms_norm(x, sd["nar.adapter.norm.weight"]) * (1 + torch.tanh(g.unsqueeze(1))) + torch.tanh(b.unsqueeze(1))
        for i, d in enumerate(dils):
            x = ssm_block(sd, f"nar.blocks.{i}.", x, int(d))
        z = F.linear(rms_norm(x, sd["nar.norm.weight"]), sd["nar.pre.weight"], sd["nar.pre.bias"])
        if z_out is not None:
            z_out.append(z)
        for j, cb in enumerate(idxs):
            hb = sd[f"nar.head_id_emb.{name}.weight"][j].view(1, 1, -1)
            lg = F.linear(z + hb, sd[f"nar.heads.{name}.{j}.weight"], sd[f"nar.heads.{name}.{j}.bias"])
            out[:, :, cb] = lg.argmax(dim=-1)
            top2 = lg.topk(2, dim=-1).values
            margin[:, :, cb] = (top2[..., 0] - top2[..., 1]) / lg.abs().amax(dim=-1).clamp_min(1e-30)
    return out, margin
