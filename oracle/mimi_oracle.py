"""CPU oracle for the Mimi codec: the DECODE path and (further down) the ENCODE path.  TEST INFRASTRUCTURE ONLY (see oracle/ar_oracle.py).

The arithmetic of this path does not live in /root/reference: the reference calls
``transformers.MimiModel.decode`` (reference codec/mimi.py:65-72, 152-156; dependency
``transformers>=4.46``, uv.lock pins 4.57.6 / 5.0.0; installed here: 5.5.0).  This file restates
that published algorithm functionally over the model's state_dict, citing
``transformers/models/mimi/modeling_mimi.py`` (5.5.0) line numbers, and is pinned by
tests/test_mimi_oracle.py against the installed ``MimiModel`` itself on seeded random weights
(no checkpoint exists offline: "parity unpinned by the reference", SURVEY.md §8c).

Layout note: everything here is channel-last [B, T, C] (the CUDA engine's layout); the HF modules
are channel-first, the restatement transposes nothing numerically relevant.
"""
from __future__ import annotations

import math
from typing import Dict

import torch
import torch.nn.functional as F

Tensor = torch.Tensor
SD = Dict[str, Tensor]

UPSAMPLING_RATIOS = (8, 6, 5, 4)  # MimiConfig.upsampling_ratios


def codebook(sd: SD, p: str) -> Tensor:
    """MimiEuclideanCodebook.embed (:1192-1196): embed_sum / clamp(cluster_usage, eps)."""
    return sd[p + "embed_sum"] / sd[p + "cluster_usage"].clamp(min=1e-5)[:, None]


def rvq_decode(sd: SD, codes_bqt: Tensor, n_sem: int = 1) -> Tensor:
    """MimiSplitResidualVectorQuantizer.decode (:1340-1350) + MimiResidualVectorQuantizer.decode
    (:1282-1293): sum of per-codebook embeddings, then a bias-free 1x1 conv 256->512, separately for
    the semantic (first) and acoustic (other) groups.  Returns [B, T, 512]."""
    out = 0.0
    for grp, lo, hi in (("semantic", 0, n_sem), ("acoustic", n_sem, codes_bqt.size(1))):
        if hi <= lo:
            continue
        pre = f"quantizer.{grp}_residual_vector_quantizer."
        q = 0.0
        for i in range(hi - lo):
            q = q + F.embedding(codes_bqt[:, lo + i], codebook(sd, pre + f"layers.{i}.codebook."))  # [B,T,256]
        out = out + F.linear(q, sd[pre + "output_proj.weight"].squeeze(-1))
    return out


def upsample(sd: SD, x_btc: Tensor) -> Tensor:
    """MimiConvTranspose1d (:354-409) with groups=C, kernel 4, stride 2, no bias, causal trim of
    kernel-stride samples on the right (:388-392, :405-408)."""
    y = F.conv_transpose1d(x_btc.transpose(1, 2), sd["upsample.conv.weight"], None, stride=2, groups=x_btc.size(-1))
    return y[..., : y.size(-1) - 2].transpose(1, 2)


def rope(q: Tensor, k: Tensor, theta: float = 10000.0):
    """MimiRotaryEmbedding.forward (:565-577) + apply_rotary_pos_emb (:589-612); q,k [B,H,T,Dh]."""
    Dh, T = q.size(-1), q.size(-2)
    inv = 1.0 / (theta ** (torch.arange(0, Dh, 2, dtype=torch.int64).float() / Dh))
    freqs = torch.arange(T).float()[:, None] * inv[None, :]
    emb = torch.cat((freqs, freqs), dim=-1)
    cos, sin = emb.cos()[None, None], emb.sin()[None, None]
    rot = lambda x: torch.cat((-x[..., Dh // 2:], x[..., : Dh // 2]), dim=-1)  # noqa: E731
    return q * cos + rot(q) * sin, k * cos + rot(k) * sin


def transformer(sd: SD, x: Tensor, n_layers: int = 8, n_heads: int = 8, window: int = 250, eps: float = 1e-5,
                prefix: str = "decoder_transformer") -> Tensor:
    """MimiTransformerModel (:1001-1140) / MimiTransformerLayer.forward (:966-993) /
    MimiAttention.forward (:681-738): pre-LayerNorm, RoPE, causal sliding-window softmax in fp32,
    LayerScale on both residual branches, GELU(erf) MLP."""
    B, T, C = x.shape
    Dh = C // n_heads
    i = torch.arange(T)
    allowed = (i[None, :] <= i[:, None]) & (i[:, None] - i[None, :] < window)
    bias = torch.zeros(T, T).masked_fill(~allowed, float("-inf"))
    for l in range(n_layers):
        p = f"{prefix}.layers.{l}."
        h = F.layer_norm(x, (C,), sd[p + "input_layernorm.weight"], sd[p + "input_layernorm.bias"], eps)
        sp = lambda t: t.view(B, T, n_heads, Dh).transpose(1, 2)  # noqa: E731
        q, k, v = (sp(F.linear(h, sd[p + f"self_attn.{n}_proj.weight"])) for n in ("q", "k", "v"))
        q, k = rope(q, k)
        w = torch.matmul(q, k.transpose(2, 3)) * (1.0 / math.sqrt(Dh)) + bias
        w = F.softmax(w, dim=-1, dtype=torch.float32)
        a = torch.matmul(w, v).transpose(1, 2).contiguous().view(B, T, C)
        x = x + sd[p + "self_attn_layer_scale.scale"] * F.linear(a, sd[p + "self_attn.o_proj.weight"])
        h = F.layer_norm(x, (C,), sd[p + "post_attention_layernorm.weight"], sd[p + "post_attention_layernorm.bias"], eps)
        h = F.linear(F.gelu(F.linear(h, sd[p + "mlp.fc1.weight"])), sd[p + "mlp.fc2.weight"])
        x = x + sd[p + "mlp_layer_scale.scale"] * h
    return x


def conv1d_causal(x_btc: Tensor, w: Tensor, b: Tensor, dilation: int = 1) -> Tensor:
    """MimiConv1d.forward (:331-351), stride 1, causal: left zero-pad (k-1)*dilation (:337-339)."""
    k = w.size(-1)
    xt = F.pad(x_btc.transpose(1, 2), ((k - 1) * dilation, 0))
    return F.conv1d(xt, w, b, dilation=dilation).transpose(1, 2)


def conv_transpose_causal(x_btc: Tensor, w: Tensor, b: Tensor, stride: int) -> Tensor:
    """MimiConvTranspose1d.forward (:402-409): full transposed conv, drop kernel-stride samples on the right."""
    y = F.conv_transpose1d(x_btc.transpose(1, 2), w, b, stride=stride)
    return y[..., : y.size(-1) - (w.size(-1) - stride)].transpose(1, 2)


def seanet_decoder(sd: SD, x: Tensor) -> Tensor:
    """MimiDecoder (:1143-1173): conv k7 -> 4 x [ELU, ConvT(stride r, kernel 2r), ResnetBlock] -> ELU -> conv k3.
    ResnetBlock (:412-451): x + conv1(ELU(conv3(ELU(x)))), true skip."""
    x = conv1d_causal(x, sd["decoder.layers.0.conv.weight"], sd["decoder.layers.0.conv.bias"])
    li = 1
    for r in UPSAMPLING_RATIOS:
        x = conv_transpose_causal(F.elu(x), sd[f"decoder.layers.{li + 1}.conv.weight"], sd[f"decoder.layers.{li + 1}.conv.bias"], r)
        p = f"decoder.layers.{li + 2}.block."
        h = conv1d_causal(F.elu(x), sd[p + "1.conv.weight"], sd[p + "1.conv.bias"])
        h = conv1d_causal(F.elu(h), sd[p + "3.conv.weight"], sd[p + "3.conv.bias"])
        x = x + h
        li += 3
    return conv1d_causal(F.elu(x), sd[f"decoder.layers.{li + 1}.conv.weight"], sd[f"decoder.layers.{li + 1}.conv.bias"])


def mimi_decode(sd: SD, codes_bqt: Tensor) -> Tensor:
    """MimiModel._decode_frame (:1613-1631) + decode (:1633-1680): codes [B,Q,T] int64 -> wav [B,1,T*1920]."""
    x = rvq_decode(sd, codes_bqt)
    x = upsample(sd, x)
    x = transformer(sd, x)
    return seanet_decoder(sd, x).transpose(1, 2)


from sopro_b200.weights import synth_mimi_encoder_state_dict, synth_mimi_state_dict  # noqa: E402,F401  (seeded random weights)


# ---------------------------------------------------------------------------------------------------------------
# ENCODE path (waveform -> codes): what the reference runs once per reference voice, ``MimiCodec.encode_file`` ->
# ``MimiModel.encode`` (reference codec/mimi.py:41-63; modeling_mimi.py:1455-1488, 1522-1611).  Pinned against the
# installed MimiModel.encode by tests/test_mimi_oracle.py.
# ---------------------------------------------------------------------------------------------------------------
def conv1d_mimi(x_btc: Tensor, w: Tensor, b, stride: int = 1, dilation: int = 1, pad_mode: str = "constant") -> Tensor:
    """MimiConv1d.forward (:331-351), causal: left pad (k_eff - stride), right pad the "extra padding" that makes the
    last window full (:273-285), mode "constant" (zeros) or "replicate"."""
    k_eff = (w.size(-1) - 1) * dilation + 1
    pad_total = k_eff - stride
    L = x_btc.size(1)
    n_frames = math.ceil((L - k_eff + pad_total) / stride + 1) - 1
    extra = n_frames * stride + k_eff - pad_total - L
    xt = F.pad(x_btc.transpose(1, 2), (pad_total, extra), mode=pad_mode)
    return F.conv1d(xt, w, b, stride=stride, dilation=dilation).transpose(1, 2)


def encoded_frames(n_samples: int) -> int:
    """MimiModel.get_encoded_length (:1490-1503): every strided conv rounds up."""
    n = int(n_samples)
    for r in reversed(UPSAMPLING_RATIOS):
        n = -(-n // r)
    return -(-n // 2)


def seanet_encoder(sd: SD, x_bt1: Tensor) -> Tensor:
    """MimiEncoder (:454-497): conv k7 -> 4 x [ResnetBlock, ELU, conv(kernel 2r, stride r, C -> 2C)] (r = 4,5,6,8)
    -> ELU -> conv k3 -> [B, T', 512]."""
    x = conv1d_mimi(x_bt1, sd["encoder.layers.0.conv.weight"], sd["encoder.layers.0.conv.bias"])
    li = 1
    for r in reversed(UPSAMPLING_RATIOS):
        p = f"encoder.layers.{li}.block."
        h = conv1d_mimi(F.elu(x), sd[p + "1.conv.weight"], sd[p + "1.conv.bias"])
        h = conv1d_mimi(F.elu(h), sd[p + "3.conv.weight"], sd[p + "3.conv.bias"])
        x = x + h
        x = conv1d_mimi(F.elu(x), sd[f"encoder.layers.{li + 2}.conv.weight"], sd[f"encoder.layers.{li + 2}.conv.bias"], stride=r)
        li += 3
    return conv1d_mimi(F.elu(x), sd[f"encoder.layers.{li + 1}.conv.weight"], sd[f"encoder.layers.{li + 1}.conv.bias"])


def mimi_encode_latent(sd: SD, wav_b1n: Tensor) -> Tensor:
    """MimiModel._encode_frame up to the quantizer (:1469-1484): SEANet encoder, encoder transformer, the 25 -> 12.5 Hz
    conv (kernel 4, stride 2, no bias, replicate padding, :1419-1429).  wav [B,1,N] -> [B, T, 512]."""
    x = seanet_encoder(sd, wav_b1n.transpose(1, 2))
    x = transformer(sd, x, prefix="encoder_transformer")
    return conv1d_mimi(x, sd["downsample.conv.weight"], None, stride=2, pad_mode="replicate")


def rvq_encode(sd: SD, emb_btc: Tensor, n_q: int = 32, n_sem: int = 1) -> Tensor:
    """MimiSplitResidualVectorQuantizer.encode (:1311-1338): the semantic and the acoustic RVQ both start from the same
    embeddings, each through its own bias-free 1x1 input_proj 512 -> 256 (:1267-1268); then residual nearest-neighbour
    search (:1272-1279) with MimiEuclideanCodebook.quantize = argmin of torch.cdist (:1197-1203).  -> codes [B, Q, T]."""
    out = []
    for grp, n in (("semantic", n_sem), ("acoustic", n_q - n_sem)):
        pre = f"quantizer.{grp}_residual_vector_quantizer."
        res = F.linear(emb_btc, sd[pre + "input_proj.weight"].squeeze(-1))  # [B,T,256]
        for i in range(n):
            e = codebook(sd, pre + f"layers.{i}.codebook.")
            idx = torch.cdist(res.reshape(1, -1, res.size(-1)).float(), e[None].float(), p=2)[0].argmin(dim=-1).view(res.shape[:-1])
            res = res - F.embedding(idx, e)
            out.append(idx)
    return torch.stack(out, dim=1)


def mimi_encode(sd: SD, wav_b1n: Tensor, n_q: int = 32) -> Tensor:
    """MimiModel.encode (:1522-1611) without streaming caches: wav [B,1,N] f32 @24 kHz -> codes [B, Q, ceil(N/1920)]."""
    return rvq_encode(sd, mimi_encode_latent(sd, wav_b1n), n_q=n_q)


# ---------------------------------------------------------------------------------------------------------------
# A model of the PRODUCT's tensor-core mode (not of the reference): the same decode with operands rounded to bf16
# exactly where sopro_b200/csrc/mimi_tc.cuh rounds them (weights of every contraction, the activation feeding every
# contraction — after ELU where the layer wants ELU —, q / k / v, the softmax probabilities and the attention output),
# fp32 accumulation and fp32 residual streams everywhere else.  It exists so that the tensor-core kernels can be held to
# a tolerance far tighter than "2e-2 of the fp32 result": what remains between this restatement and the GPU is
# accumulation order and rare one-ulp bf16 rounding flips.  Test infrastructure only.
# ---------------------------------------------------------------------------------------------------------------
def _bf(x: Tensor) -> Tensor:
    return x.to(torch.bfloat16).to(torch.float32)


def transformer_bf16_operands(sd: SD, x: Tensor, n_layers: int = 8, n_heads: int = 8, window: int = 250, eps: float = 1e-5,
                              attention: str = "tc") -> Tensor:
    """attention="tc": the one-shot decode's tensor-core attention (rope_pack_kernel + attn_tc_kernel): q / k / v rounded
    to bf16, probabilities rounded to bf16 before they are summed.  attention="fp32": the tensor-core stream's attention
    (rope_kernel + attn_kernel over the K/V ring): RoPE and softmax in fp32 on the fp32 q / k / v, unrounded
    probabilities.  Both round the attention output to bf16 (the operand of o_proj)."""
    if attention not in ("tc", "fp32"):
        raise ValueError(f"attention must be 'tc' or 'fp32', got {attention!r}")
    B, T, C = x.shape
    Dh = C // n_heads
    i = torch.arange(T)
    allowed = (i[None, :] <= i[:, None]) & (i[:, None] - i[None, :] < window)
    for l in range(n_layers):
        p = f"decoder_transformer.layers.{l}."
        h = _bf(F.layer_norm(x, (C,), sd[p + "input_layernorm.weight"], sd[p + "input_layernorm.bias"], eps))
        sp = lambda t: t.view(B, T, n_heads, Dh).transpose(1, 2)  # noqa: E731
        q, k, v = (sp(F.linear(h, _bf(sd[p + f"self_attn.{n}_proj.weight"]))) for n in ("q", "k", "v"))
        q, k = rope(q, k)
        if attention == "tc":
            q, k, v = _bf(q), _bf(k), _bf(v)
            s = torch.matmul(q, k.transpose(2, 3)) * (1.0 / math.sqrt(Dh))
            s = s.masked_fill(~allowed, float("-inf"))
            pr = _bf(torch.exp(s - s.amax(dim=-1, keepdim=True)))  # probabilities are rounded BEFORE they are summed
            a = torch.matmul(pr, v) / pr.sum(dim=-1, keepdim=True)
        else:
            s = torch.matmul(q, k.transpose(2, 3)) * (1.0 / math.sqrt(Dh))
            a = torch.matmul(F.softmax(s.masked_fill(~allowed, float("-inf")), dim=-1), v)
        a = _bf(a).transpose(1, 2).contiguous().view(B, T, C)
        x = x + sd[p + "self_attn_layer_scale.scale"] * F.linear(a, _bf(sd[p + "self_attn.o_proj.weight"]))
        h = _bf(F.layer_norm(x, (C,), sd[p + "post_attention_layernorm.weight"], sd[p + "post_attention_layernorm.bias"], eps))
        h = _bf(F.gelu(F.linear(h, _bf(sd[p + "mlp.fc1.weight"]))))
        x = x + sd[p + "mlp_layer_scale.scale"] * F.linear(h, _bf(sd[p + "mlp.fc2.weight"]))
    return x


def seanet_decoder_bf16_operands(sd: SD, x: Tensor) -> Tensor:
    a = _bf(F.elu(conv1d_causal(_bf(x), _bf(sd["decoder.layers.0.conv.weight"]), sd["decoder.layers.0.conv.bias"])))
    li = 1
    for r in UPSAMPLING_RATIOS:
        z = conv_transpose_causal(a, _bf(sd[f"decoder.layers.{li + 1}.conv.weight"]), sd[f"decoder.layers.{li + 1}.conv.bias"], r)
        p = f"decoder.layers.{li + 2}.block."
        h = _bf(F.elu(conv1d_causal(_bf(F.elu(z)), _bf(sd[p + "1.conv.weight"]), sd[p + "1.conv.bias"])))
        a = _bf(F.elu(z + conv1d_causal(h, _bf(sd[p + "3.conv.weight"]), sd[p + "3.conv.bias"])))  # fp32 skip, bf16 operand out
        li += 3
    # the final conv keeps its fp32 weights; its input is the bf16 ELU'd activation above
    return conv1d_causal(a, sd[f"decoder.layers.{li + 1}.conv.weight"], sd[f"decoder.layers.{li + 1}.conv.bias"])


def mimi_decode_bf16_operands(sd: SD, codes_bqt: Tensor, attention: str = "tc") -> Tensor:
    """attention="tc" models the one-shot tensor-core decode, "fp32" the tensor-core stream (transformer_bf16_operands)."""
    x = upsample(sd, rvq_decode(sd, codes_bqt))  # fp32 in both modes of the product
    x = transformer_bf16_operands(sd, x, attention=attention)
    return seanet_decoder_bf16_operands(sd, x).transpose(1, 2)
