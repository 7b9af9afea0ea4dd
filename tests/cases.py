"""Seeded, platform-independent test cases shared by the golden generator
(tests/golden/make_golden.py, run against the reference), the CPU oracle tests
and the GPU parity tests.  Inputs come from integer hashing
(sopro_b200.weights.hash_uniform), never from torch's RNG, so every host
rebuilds identical bytes."""
from __future__ import annotations

import math
from typing import Dict, List

import numpy as np
import torch

from oracle.ar_oracle import ArSampling
from sopro_b200.config import SoproTTSConfig
from sopro_b200.weights import hash_uniform, round_through_bf16, synth_state_dict

SMALL_CFG = dict(
    num_codebooks=8, codebook_size=256, d_model=128, n_layers_ar=4, ar_kernel=5,
    ar_dilation_cycle=(1, 3), ar_text_attn_freq=2, min_gen_frames=4, max_frames=60,
)

# name -> spec
AR_CASES: Dict[str, dict] = {
    # BASELINE.json configs 2/3 shape: 401 steps, L=52, EOS never terminates
    "default_fp32": dict(cfg={}, L=52, max_frames=400, noise_seed=1234, head_gain=1.0, min_gen=10 ** 9, bf16=False, key=11),
    "default_bf16": dict(cfg={}, L=52, max_frames=400, noise_seed=1235, head_gain=1.0, min_gen=10 ** 9, bf16=True, key=12),
    # peaked logits: exercises repetition penalty, anti-loop recovery and EOS handling
    "peaked_fp32": dict(cfg={}, L=23, max_frames=200, noise_seed=77, head_gain=8.0, min_gen=None, bf16=False, key=13),
    "peaked_nostop": dict(cfg={}, L=9, max_frames=150, noise_seed=5, head_gain=12.0, min_gen=10 ** 9, bf16=False, key=14,
                          top_p=0.95, temperature=0.7),
    "noantiloop": dict(cfg={}, L=52, max_frames=100, noise_seed=9, head_gain=12.0, min_gen=10 ** 9, bf16=False, key=15,
                       anti_loop=False),
    # EOS made likely: sampled before min_gen_frames (fed back as table row 2048, SURVEY §7.2
    # quirk) and then terminating the stream once t+1 >= min_gen
    "eos_early": dict(cfg={}, L=17, max_frames=120, noise_seed=21, head_gain=2.0, min_gen=None, bf16=False, key=17,
                      eos_bias=4.5),
    "eos_mingen40": dict(cfg={}, L=17, max_frames=120, noise_seed=22, head_gain=2.0, min_gen=40, bf16=False, key=18,
                         eos_bias=3.0),
    # constant conditioning + near-greedy sampling: the n-gram loop detector and the
    # same-token streak both fire (model.py:274-279), recovery sampling breaks out
    "loopy_a": dict(cfg={}, L=9, max_frames=150, noise_seed=5, head_gain=8.0, min_gen=10 ** 9, bf16=False, key=19,
                    temperature=0.6, const_cond=True),
    "loopy_b": dict(cfg={}, L=9, max_frames=150, noise_seed=5, head_gain=10.0, min_gen=10 ** 9, bf16=False, key=19,
                    temperature=0.8, const_cond=True),
    # a non-default geometry: every dimension must come from cfg
    "small_fp32": dict(cfg=SMALL_CFG, L=7, max_frames=60, noise_seed=3, head_gain=4.0, min_gen=10 ** 9, bf16=False, key=16),
}


def _unit(n: int, key: int) -> torch.Tensor:
    return torch.from_numpy(hash_uniform(n, key) * np.float32(math.sqrt(3.0)))


_SD_CACHE: Dict[tuple, dict] = {}


def ar_weights(cfg: SoproTTSConfig, head_gain: float, bf16: bool, seed: int = 0, eos_bias: float = 0.0) -> dict:
    key = (cfg.to_json(), float(head_gain), bool(bf16), int(seed), float(eos_bias))
    if key not in _SD_CACHE:
        sd = synth_state_dict(cfg, text_vocab=64, seed=seed, only_prefix=("ar.", "cb_embed."), head_gain=head_gain)
        if eos_bias:
            sd["ar.head.bias"] = sd["ar.head.bias"].clone()
            sd["ar.head.bias"][int(cfg.codebook_size)] += float(eos_bias)
        if bf16:
            sd = round_through_bf16(sd, prefixes=("ar.", "cb_embed."))
        _SD_CACHE[key] = sd
    return _SD_CACHE[key]


def ar_case_inputs(spec: dict):
    cfg = SoproTTSConfig(**spec["cfg"])
    sd = ar_weights(cfg, spec["head_gain"], spec["bf16"], eos_bias=spec.get("eos_bias", 0.0))
    D, L, T = int(cfg.d_model), int(spec["L"]), int(spec["max_frames"]) + 1
    k = int(spec["key"]) * 1000
    cond_ar = _unit(T * D, k + 1).view(1, T, D)
    if spec.get("const_cond"):
        cond_ar = cond_ar[:, :1].expand(1, T, D).contiguous()
    txt_seq = _unit(L * D, k + 2).view(1, L, D)
    samp = ArSampling(
        top_p=spec.get("top_p", 0.9), temperature=spec.get("temperature", 1.05),
        anti_loop=spec.get("anti_loop", True), min_gen_frames=spec["min_gen"],
    )
    inp = dict(cond_ar=cond_ar, txt_seq=txt_seq, text_mask=torch.ones(1, L, dtype=torch.bool),
               max_frames=int(spec["max_frames"]), sampling=samp)
    return cfg, sd, inp


def ar_forced_batch(cfg: SoproTTSConfig, lens: List[int], steps: int, key: int, pad: float = 30.0):
    """A teacher-forced ragged batch: cond_ar [B, steps, D]; txt_seq [B, max(lens), D] whose rows past lens[b] are
    padding of pad x unit-variance values (pad = 0: zeros); forced ids [B, steps] int32 in [0, codebook_size), with
    EOS (= codebook_size) every 37th step from a per-utterance offset."""
    D, B, Lm, eos = int(cfg.d_model), len(lens), max(lens), int(cfg.codebook_size)
    k = int(key) * 1000
    cond = torch.stack([_unit(steps * D, k + b).view(steps, D) for b in range(B)])
    txt = (_unit(B * Lm * D, k + 500) * float(pad)).view(B, Lm, D)
    for b, L in enumerate(lens):
        txt[b, :L] = _unit(L * D, k + 600 + b).view(L, D)
    u = torch.from_numpy(hash_uniform(B * steps, k + 900)).double().view(B, steps) * 0.5 + 0.5
    forced = (u * eos).long().clamp(max=eos - 1)
    t = torch.arange(steps)[None, :]
    forced[(t + 11 * torch.arange(B)[:, None]) % 37 == 5] = eos
    return cond, txt, forced.to(torch.int32)


# ---------------------------------------------------------------------------
# sampler known-answer cases (reference: sampling.py:24-93)
# ---------------------------------------------------------------------------
def _hist(n: int, key: int, V: int, period: int = 0) -> List[int]:
    u = hash_uniform(max(n, 1), key)
    h = [int((x * 0.5 + 0.5) * V) % V for x in u[:n]]
    if period:
        h = [h[i % period] for i in range(n)]
    return h


SAMPLER_CASES: Dict[str, dict] = {}


def _add(name, **kw):
    SAMPLER_CASES[name] = kw


for _i in range(6):
    _add(f"flat{_i}", V=2049, scale=0.5, key=100 + _i, hist=0, seed=10 + _i)
    _add(f"mid{_i}", V=2049, scale=3.0, key=200 + _i, hist=30 + 10 * _i, seed=20 + _i)
    _add(f"peak{_i}", V=2049, scale=9.0, key=300 + _i, hist=80, seed=30 + _i, period=7 if _i % 2 else 0)
_add("recovery", V=2049, scale=3.0, key=400, hist=64, seed=40, top_p=0.85, temperature=1.2)
_add("temp1", V=2049, scale=2.0, key=401, hist=10, seed=41, temperature=1.0)
_add("norep", V=2049, scale=2.0, key=402, hist=10, seed=42, repetition_penalty=1.0)
_add("notopk", V=2049, scale=4.0, key=403, hist=10, seed=43, top_k=0)
_add("notopp", V=2049, scale=4.0, key=404, hist=10, seed=44, top_p=1.0)
_add("neither", V=2049, scale=4.0, key=405, hist=10, seed=45, top_p=1.0, top_k=0)
_add("spike", V=2049, scale=1.0, key=406, hist=5, seed=46, spike=(1000, 40.0))
_add("naninf", V=2049, scale=2.0, key=407, hist=5, seed=47, special=True)
_add("smallv", V=257, scale=3.0, key=408, hist=20, seed=48)
_add("topk_gt_v", V=33, scale=3.0, key=409, hist=3, seed=49)
_add("tiny_top_p", V=2049, scale=3.0, key=410, hist=12, seed=50, top_p=0.05)


def sampler_case_inputs(spec: dict):
    V = int(spec["V"])
    logits = torch.from_numpy(hash_uniform(V, spec["key"] * 7919) * np.float32(spec["scale"] * math.sqrt(3.0)))
    if "spike" in spec:
        logits[spec["spike"][0]] = spec["spike"][1]
    if spec.get("special"):
        logits[3] = float("nan")
        logits[5] = float("inf")
        logits[7] = float("-inf")
    hist = _hist(int(spec["hist"]), spec["key"] * 31 + 1, V, spec.get("period", 0))
    kw = dict(top_p=spec.get("top_p", 0.9), top_k=spec.get("top_k", 50),
              temperature=spec.get("temperature", 1.05), repetition_penalty=spec.get("repetition_penalty", 1.1))
    return logits, hist, kw, int(spec["seed"])


# ---------------------------------------------------------------------------
# whole-model case (prefill + AR + NAR): full synthetic checkpoint, small text vocabulary
# ---------------------------------------------------------------------------
E2E_CASE = dict(text_vocab=1000, L=52, ref_frames=38, max_frames=400, nar_T=50, style_strength=1.0, key=77)
_E2E_CACHE = {}


def e2e_inputs():
    if "v" not in _E2E_CACHE:
        cfg = SoproTTSConfig()
        sd = synth_state_dict(cfg, text_vocab=E2E_CASE["text_vocab"], seed=0)
        k = E2E_CASE["key"] * 1000
        def ints(n, key, hi):
            u = hash_uniform(n, key) * 0.5 + 0.5
            return torch.from_numpy(np.minimum((u * hi).astype(np.int64), hi - 1))
        text_ids = ints(E2E_CASE["L"], k + 1, E2E_CASE["text_vocab"])
        ref_tokens = ints(E2E_CASE["ref_frames"] * 32, k + 2, 2048).view(E2E_CASE["ref_frames"], 32)
        rvq1 = ints(E2E_CASE["nar_T"], k + 3, 2048)
        _E2E_CACHE["v"] = (cfg, sd, dict(text_ids=text_ids, ref_tokens_tq=ref_tokens, rvq1=rvq1, max_frames=E2E_CASE["max_frames"],
                                         nar_T=E2E_CASE["nar_T"], style_strength=E2E_CASE["style_strength"]))
    return _E2E_CACHE["v"]
