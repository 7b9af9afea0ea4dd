"""GPU: the AR step's warp task shape (sopro_ar_session_set_task_shape) decides which warp computes which outputs, never a
bit of them.  Every output keeps its two fp32 FMA chains over k = 4 * lane + 128 * i and the same lane-pairing tree in the
transposed reduction, so tokens, per-block residuals, logits and the exported attention weights must be bit-equal whether
every GEMV stage runs wide tasks (R rows x TU utterances), narrow ones (R x TU/2) or the shape the host picks per stage."""
import numpy as np
import pytest
import torch

from tests.cases import AR_CASES, _unit, ar_case_inputs

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

MODES = (0, 1, 2)  # host's choice, always wide, always narrow
GEMV = {"glu", "ffn1", "ffn2", "q", "o", "head"}
_ENG = {}


def _engine(wdtype):
    from sopro_b200.engine import ArEngine

    if wdtype not in _ENG:
        cfg, sd, _ = ar_case_inputs(AR_CASES["default_bf16" if wdtype == "bf16" else "default_fp32"])
        _ENG[wdtype] = (cfg, ArEngine(cfg, sd, device=0, weight_dtype=wdtype))
    return _ENG[wdtype]


def _inputs(cfg, B, steps, L):
    D = int(cfg.d_model)
    cond = torch.stack([_unit(steps * D, 8100 + i).view(steps, D) for i in range(B)])
    txt = torch.stack([_unit(L * D, 8300 + i).view(L, D) for i in range(B)])
    lens = [L - (b % 7) for b in range(B)]
    gen = torch.Generator().manual_seed(B)
    noise = torch.empty(B, steps, 50).exponential_(1.0, generator=gen)
    # teacher forcing with ids below EOS (= codebook_size): every utterance runs every step
    forced = torch.randint(0, int(cfg.codebook_size), (B, steps), generator=gen, dtype=torch.int32)
    return cond, txt, lens, noise, forced


def _run(eng, cfg, mode, B, steps, inputs, attn):
    from sopro_b200.engine import Sampling
    from sopro_b200.timestamps import trace_buffer

    cond, txt, lens, noise, forced = inputs
    ses = eng.session(B, steps, max(lens))
    ses.set_task_shape(mode)
    ses.set_forced(forced)
    tr_b = torch.zeros(steps, int(cfg.n_layers_ar), B, int(cfg.d_model), device="cuda")
    tr_l = torch.zeros(steps, B, cfg.ar_vocab(), device="cuda")
    ses.set_trace(tr_b, tr_l)
    tr_a = trace_buffer(cfg, steps, B, max(lens), "cuda:0") if attn else None
    if attn:
        ses.set_attn_trace(tr_a)
    ses.begin(cond, txt, lens, noise, Sampling(min_gen_frames=2 ** 31 - 1))
    ses.run()
    toks, n, _ = ses.read()
    sampled = ses.sampled().cpu().numpy()
    torch.cuda.synchronize()
    out = dict(toks=toks, n=n, sampled=sampled, blocks=tr_b.cpu(), logits=tr_l.cpu(),
               attn=tr_a.cpu() if attn else None, shapes=ses.stage_shapes())
    ses.set_attn_trace(None)
    ses.set_forced(None)
    ses.close()
    return out


def _check_modes(runs, B, attn):
    base = runs[0]
    assert (base["n"] == base["toks"].shape[1]).all()
    assert base["logits"].abs().sum() > 0 and base["blocks"].abs().sum() > 0
    for mode, r in zip(MODES[1:], runs[1:]):
        assert np.array_equal(r["toks"], base["toks"]), f"mode {mode}: tokens"
        assert np.array_equal(r["sampled"], base["sampled"]), f"mode {mode}: sampled tokens"
        assert torch.equal(r["blocks"], base["blocks"]), f"mode {mode}: block trace"
        assert torch.equal(r["logits"], base["logits"]), f"mode {mode}: logits trace"
        if attn:
            assert torch.equal(r["attn"], base["attn"]), f"mode {mode}: attention trace"
    # the forced modes run the shape they ask for; GLU and teams of one utterance have only the wide one
    assert all(s == "wide" for _k, s in runs[1]["shapes"])
    assert all(s == ("narrow" if k in GEMV and k != "glu" and B > 1 else "wide") for k, s in runs[2]["shapes"])


@pytest.mark.parametrize("B", [64, 12, 1])
@pytest.mark.parametrize("wdtype", ["bf16", "fp32"])
def test_outputs_bit_equal_across_task_shapes(wdtype, B):
    """B = 64: 8 teams of 8 (TU = 8); B = 12: 2 teams of 6 (TU = 4, a task straddles the team's end); B = 1: one
    shape only, the hook must leave it alone."""
    cfg, eng = _engine(wdtype)
    steps = 12
    inputs = _inputs(cfg, B, steps, 40)
    runs = [_run(eng, cfg, m, B, steps, inputs, attn=False) for m in MODES]
    _check_modes(runs, B, attn=False)
    # the host's rule at the bench geometry (DESIGN.md §3).  fp32 storage splits FFN2's 24-row slice into two ring tiles
    # (13 + 11 rows), where both shapes put 2 x 32 outputs on the busiest scheduler: that tie stays wide
    if B == 64 and wdtype == "bf16":
        by_kind = {}
        for k, s in runs[0]["shapes"]:
            by_kind.setdefault(k, set()).add(s)
        assert by_kind["ffn2"] == {"narrow"} and by_kind["o"] == {"narrow"} and by_kind["glu"] == {"wide"}, by_kind


@pytest.mark.parametrize("wdtype,B", [("bf16", 64), ("fp32", 12), ("fp32", 1)])
def test_word_timestamp_trace_bit_equal_across_task_shapes(wdtype, B):
    """The word-timestamp instantiation of the kernel (attention weights exported) under the three modes."""
    cfg, eng = _engine(wdtype)
    steps = 12
    inputs = _inputs(cfg, B, steps, 40)
    runs = [_run(eng, cfg, m, B, steps, inputs, attn=True) for m in MODES]
    _check_modes(runs, B, attn=True)
    assert runs[0]["attn"].abs().sum() > 0
