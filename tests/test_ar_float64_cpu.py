"""CPU: the float64 mode of the AR oracle, and the bound tests/test_ar_float64_gpu.py holds the AR step to.

The bound: for every utterance, each layer's residual, the logits and the text K / V, the error against the float64
oracle (max and RMS, relative to the utterance's own peak and RMS over all its steps) is at most KAPPA x the error of
the fp32 oracle on the same input (floor U).  The controls below prove the bound has teeth: each is a subtly wrong
fp32 step (monkeypatched here, never in the product), and each must exceed KAPPA on every utterance it touches."""
import pytest
import torch
import torch.nn.functional as F

from oracle import ar_oracle as O
from oracle.dense_probes import KAPPA, U
from tests.cases import AR_CASES, ar_case_inputs, ar_forced_batch

torch.set_grad_enabled(False)

LENS = [1, 52, 129, 2048, 7, 128]
STEPS = 60
_CACHE = {}


def _setup():
    """default config, bf16-rounded weights, ragged texts with zero padding (so that one extra key is a quiet one)"""
    if "s" not in _CACHE:
        cfg, sd, _ = ar_case_inputs(AR_CASES["default_bf16"])
        cond, txt, forced = ar_forced_batch(cfg, LENS, STEPS, key=41, pad=0.0)
        ref64 = O.ar_teacher_forced(sd, cfg, cond, txt, LENS, forced, torch.float64)
        ref32 = O.ar_teacher_forced(sd, cfg, cond, txt, LENS, forced, torch.float32)
        e32 = O.ar_trace_errors(ref32, ref64, LENS)
        _CACHE["s"] = (cfg, sd, cond, txt, forced, ref64, ref32, e32)
    return _CACHE["s"]


def _ratios(got, ref64, e32, lens):
    """[B, quantities, 2] error against float64 over the fp32 oracle's (floored at U)"""
    return O.ar_trace_errors(got, ref64, lens) / e32.clamp(min=U)


def test_float64_mode_keeps_float64():
    cfg, sd, cond, txt, forced, ref64, ref32, e32 = _setup()
    assert ref64.blocks.dtype == ref64.logits.dtype == torch.float64
    assert all(k.dtype == v.dtype == torch.float64 for k, v in ref64.kv.values())
    assert ref32.blocks.dtype == ref32.logits.dtype == torch.float32
    # the building blocks compute in float64 when handed float64: the result is the float64 formula, not an fp32 one
    g = torch.Generator().manual_seed(0)
    x, w = torch.randn(3, 1, 384, dtype=torch.float64, generator=g), torch.randn(384, dtype=torch.float64, generator=g)
    want = x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + 1e-6) * w
    assert torch.equal(O.rms_norm(x, w), want)
    p = "ar.x_attns.1."
    sd64 = {k: v.double() for k, v in sd.items()}
    k, v = O.text_kv_cache(sd64, p, txt[:2, :52].double(), cfg.AR_HEADS)
    keep = torch.ones(2, 52, dtype=torch.bool)
    y = O.xattn_step(sd64, p, x[:2], k, v, keep, cfg.AR_HEADS)
    y32 = O.xattn_step(sd, p, x[:2].float(), k.float(), v.float(), keep, cfg.AR_HEADS)
    assert y.dtype == torch.float64 and y32.dtype == torch.float32
    d = float((y - y32.double()).abs().max() / y.abs().max())
    assert 0 < d < 1e-5, d
    # the fp32 oracle sits at fp32 rounding from float64, and that error is not zero (the ratios below divide by it)
    assert float(e32.max()) < 1e-5 and float(e32.min()) > 0, e32


@pytest.mark.parametrize("name", ["default_bf16", "eos_mingen40", "small_fp32"])
def test_fp32_mode_is_ar_stream_bit_for_bit(name):
    """The batched driver's fp32 mode with ar_stream's own tokens forced: every step's logits bit-equal to ar_stream's
    (eos_mingen40 feeds EOS back as an embedding row; small_fp32 is a non-default geometry)."""
    spec = AR_CASES[name]
    cfg, sd, inp = ar_case_inputs(spec)
    tape = O.noise_tape(spec["noise_seed"], inp["max_frames"] + 1, cfg.ar_vocab())
    logits = []
    toks = O.ar_generate(sd, cfg, inp["cond_ar"], inp["txt_seq"], inp["text_mask"], max_frames=inp["max_frames"],
                         sampling=inp["sampling"], noise_tv=tape, logits_out=logits)
    n = len(toks)
    assert name != "eos_mingen40" or 2048 in toks[:-1]
    L = inp["txt_seq"].shape[1]
    got = O.ar_teacher_forced(sd, cfg, inp["cond_ar"][:, :n], inp["txt_seq"], [L], torch.tensor([toks]), torch.float32)
    assert torch.equal(got.logits[:, 0], torch.stack(logits))


def test_batched_row_equals_the_utterance_alone():
    """Row b of the ragged batch is utterance b run alone: in float64 to 1e-12, and the fp32 run alone within the
    bound of the batched fp32 run."""
    cfg, sd, cond, txt, forced, ref64, ref32, e32 = _setup()
    worst = 0.0
    for b, L in enumerate(LENS):
        args = (cond[b:b + 1], txt[b:b + 1, :L], [L], forced[b:b + 1])
        alone64 = O.ar_teacher_forced(sd, cfg, *args, torch.float64)
        row = O.ArTrace(ref64.blocks[:, :, b:b + 1], ref64.logits[:, b:b + 1],
                        {i: (k[b:b + 1, :, :L], v[b:b + 1, :, :L]) for i, (k, v) in ref64.kv.items()})
        assert float(O.ar_trace_errors(alone64, row, [L]).max()) < 1e-12, f"utterance {b} (L={L})"
        alone32 = O.ar_teacher_forced(sd, cfg, *args, torch.float32)
        r = float(_ratios(alone32, row, e32[b:b + 1], [L]).max())
        worst = max(worst, r)
        assert r <= KAPPA, f"utterance {b} (L={L}): {r:.2f} x the batched fp32 error"
    print(f"fp32 alone / fp32 batched: worst {worst:.2f}x")


def _keep_mutation(fn):
    """wrap ar_init_state so the keep-mask of every utterance is rewritten by fn(keep_row, length)"""
    orig = O.ar_init_state

    def init(sd, cfg, txt_seq, text_mask, batch=1):
        keep = text_mask.clone()
        for b in range(keep.size(0)):
            fn(keep[b], int(text_mask[b].sum()))
        return orig(sd, cfg, txt_seq, keep, batch)
    return init


def _layer_counter(cfg):
    """the layer of the n-th call of a once-per-layer building block (called in layer order, every step)"""
    n = {"calls": 0}

    def layer():
        i = n["calls"] % int(cfg.n_layers_ar)
        n["calls"] += 1
        return i
    return layer


def _extra_key(keep, L):  # attend one (zero) padding key past the text
    if L < keep.numel():
        keep[L] = True


def _drop_last_key(keep, L):
    if L > 1:
        keep[L - 1] = False


CONTROLS = ["extra_key", "drop_last_key", "eps_x10", "tanh_gelu", "bf16_glu_input", "dwconv_tap_off"]


@pytest.mark.parametrize("control", CONTROLS)
def test_controls_exceed_the_bound(control, monkeypatch):
    cfg, sd, cond, txt, forced, ref64, ref32, e32 = _setup()
    affected = list(range(len(LENS)))
    if control == "extra_key":
        monkeypatch.setattr(O, "ar_init_state", _keep_mutation(_extra_key))
        affected = [b for b, L in enumerate(LENS) if L < max(LENS)]
    elif control == "drop_last_key":
        monkeypatch.setattr(O, "ar_init_state", _keep_mutation(_drop_last_key))
        affected = [b for b, L in enumerate(LENS) if L > 1]
    elif control == "eps_x10":
        rms = O.rms_norm
        monkeypatch.setattr(O, "rms_norm", lambda x, w, eps=1e-6: rms(x, w, eps * 10))
    elif control == "tanh_gelu":
        gelu = F.gelu
        monkeypatch.setattr(O.F, "gelu", lambda x: gelu(x, approximate="tanh"))
    elif control == "bf16_glu_input":  # layer 2's GLU stage reads bf16-rounded activations
        glu, layer = O.glu, _layer_counter(cfg)
        monkeypatch.setattr(O, "glu", lambda x, w, b: glu(x.to(torch.bfloat16).float() if layer() == 2 else x, w, b))
    else:  # layer 3 (dilation 1) reads its dwconv window one frame late: the ring before this step's push
        dw, layer = O.dwconv_step, _layer_counter(cfg)

        def late(h, ring, w_dk, bias, dil):
            y, new = dw(h, ring, w_dk, bias, dil)
            if layer() == 3:
                taps = ring.index_select(1, torch.arange(0, int(w_dk.size(-1)) * dil, dil))
                y = ((taps.transpose(1, 2) * w_dk.unsqueeze(0)).sum(dim=-1) + bias.unsqueeze(0)).unsqueeze(1)
            return y, new
        monkeypatch.setattr(O, "dwconv_step", late)
    got = O.ar_teacher_forced(sd, cfg, cond, txt, LENS, forced, torch.float32)
    score = _ratios(got, ref64, e32, LENS).amax(dim=(1, 2))
    print(f"{control}: worst error / fp32 oracle's per utterance {[round(float(s), 1) for s in score]}")
    low = [(b, LENS[b], float(score[b])) for b in affected if not score[b] > KAPPA]
    assert not low, f"{control} stays within {KAPPA}x on (utterance, length, ratio) {low}"
