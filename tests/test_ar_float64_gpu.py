"""GPU: the persistent AR step against the float64 oracle, at every step, layer and utterance of ragged batched launches,
in every team geometry.

Every launch runs teacher-forced (random ids with EOS among them, min_gen_frames out of reach, so every utterance runs
every step) with the residual and logit traces on, and compares EVERY utterance at EVERY step: the residual after each
layer, all V logits, and the text K / V rows [:L] of every attention layer.  Text padding holds loud values, so a read
past an utterance's text cannot hide.  The bound (tests/test_ar_float64_cpu.py proves it has teeth): per utterance and
quantity, the max and RMS error against float64, relative to that utterance's own peak and RMS over its steps, is at most
KAPPA x the fp32 CPU oracle's error on the same input (floor U).  The oracle is computed once per input set."""
import pytest
import torch

from oracle import ar_oracle as O
from oracle.dense_probes import KAPPA, U
from tests.cases import AR_CASES, ar_case_inputs, ar_forced_batch

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

# name -> (weights case, text lengths, steps, session max_text_len, input key)
BENCH_LENS = [52] * 64
for _b, _L in zip((3, 17, 30, 44, 61), (1, 2, 3, 5, 51)):
    BENCH_LENS[_b] = _L
SWEEP_LENS = [52, 7, 129, 1, 128, 33, 2, 100, 17, 130, 5, 64, 127, 9, 52, 3, 81, 12, 119, 4,
              40, 1, 130, 23, 6, 96, 11, 128, 45, 8, 77, 2, 60, 129, 14, 30, 3, 110, 20, 50]
SETS = {
    "bench": ("default_bf16", BENCH_LENS, 401, 52, 51),
    "long": ("default_bf16", [1, 4, 5, 127, 128, 129, 255, 256, 257, 1000, 2048], 64, 2048, 52),
    "small": ("small_fp32", [7, 1, 23, 33, 2, 12, 5, 40, 17, 9, 52, 3, 28, 44, 4, 36, 11, 6, 50], 61, 52, 53),
    "sweep": ("default_bf16", SWEEP_LENS, 48, 130, 54),
}
_REF, _ENG, _RUNS = {}, {}, {}


def _set(name):
    """(cfg, sd, cond, txt, lens, forced, float64 oracle, fp32 oracle's errors [B, quantities, 2], steps, max_text_len)"""
    if name not in _REF:
        case, lens, steps, mtl, key = SETS[name]
        cfg, sd, _ = ar_case_inputs(AR_CASES[case])
        cond, txt, forced = ar_forced_batch(cfg, lens, steps, key)
        ref64 = O.ar_teacher_forced(sd, cfg, cond, txt, lens, forced, torch.float64)
        e32 = O.ar_trace_errors(O.ar_teacher_forced(sd, cfg, cond, txt, lens, forced, torch.float32), ref64, lens)
        _REF[name] = (cfg, sd, cond, txt, lens, forced, ref64, e32, steps, mtl)
    return _REF[name]


def _engine(name, wdtype):
    from sopro_b200.engine import ArEngine

    case = SETS[name][0]
    if (case, wdtype) not in _ENG:
        cfg, sd, _ = ar_case_inputs(AR_CASES[case])
        _ENG[case, wdtype] = ArEngine(cfg, sd, device=0, weight_dtype=wdtype)
    return _ENG[case, wdtype]


def _launch(name, wdtype, rows=None, team=0, task_shape=0, chunks=(), attn=False):
    """one teacher-forced launch over utterances `rows` of the set -> (ArTrace of the GPU, stage program)"""
    from sopro_b200.engine import Sampling
    from sopro_b200.timestamps import trace_buffer

    cfg, sd, cond, txt, lens, forced, ref64, e32, steps, mtl = _set(name)
    rows = list(range(len(lens))) if rows is None else list(rows)
    B, lens_r = len(rows), [lens[b] for b in rows]
    eng = _engine(name, wdtype)
    dev = eng.device
    ses = eng.session(B, steps, mtl)
    ses.set_team(team)
    ses.set_task_shape(task_shape)
    ses.set_forced(forced[rows])
    tr_b = torch.zeros(steps, int(cfg.n_layers_ar), B, int(cfg.d_model), device=dev)
    tr_l = torch.zeros(steps, B, cfg.ar_vocab(), device=dev)
    ses.set_trace(tr_b, tr_l)
    if attn:
        ses.set_attn_trace(trace_buffer(cfg, steps, B, max(lens_r), dev))
    noise = torch.empty(B, steps, 50).exponential_(1.0, generator=torch.Generator().manual_seed(B))
    ses.begin(cond[rows], txt[rows], lens_r, noise, Sampling(min_gen_frames=10 ** 9))
    for c in chunks:
        ses.run(c)
    ses.run()
    _toks, n, _done = ses.read()
    assert (n == steps).all(), n
    k, v = ses.kv()
    torch.cuda.synchronize()
    got = O.ArTrace(tr_b.cpu(), tr_l.cpu(), {li: (k[s].cpu(), v[s].cpu()) for s, li in enumerate(cfg.ar_attn_layers())})
    program = ses.stage_shapes()
    if attn:
        ses.set_attn_trace(None)
    ses.set_forced(None)
    ses.close()
    return got, program


def _attention_program(program):
    kinds = [k for k, _s in program]
    assert ("qatt" in kinds) != ("q" in kinds or "att" in kinds), kinds
    return "qatt" if "qatt" in kinds else "q+att"


def _check(label, name, got, program, rows=None):
    """the bound, per utterance and quantity; one report line per launch"""
    cfg, sd, cond, txt, lens, forced, ref64, e32, steps, mtl = _set(name)
    rows = list(range(len(lens))) if rows is None else list(rows)
    lens_r = [lens[b] for b in rows]
    ref = O.ArTrace(ref64.blocks[:, :, rows], ref64.logits[:, rows], {i: (k[rows], v[rows]) for i, (k, v) in ref64.kv.items()})
    ratio = O.ar_trace_errors(got, ref, lens_r) / e32[rows].clamp(min=U)  # [B, quantities, (max, rms)]
    labels = O.ar_trace_labels(cfg)
    worst = ratio.amax(dim=(0, 2))
    print(f"[ar-f64] {label}: B={len(rows)} program={_attention_program(program)} worst GPU/fp32 "
          + " ".join(f"{q}={float(w):.2f}" for q, w in zip(labels, worst)))
    bad = []
    for u, j, m in (ratio > KAPPA).nonzero().tolist():
        q, b = labels[j], rows[u]
        if j <= int(cfg.n_layers_ar):  # the step of the largest error
            z = got.blocks[:, j, u] if j < int(cfg.n_layers_ar) else got.logits[:, u]
            z64 = ref.blocks[:, j, u] if j < int(cfg.n_layers_ar) else ref.logits[:, u]
            step = int((z.double() - z64).abs().amax(dim=-1).argmax())
        else:
            step = -1
        bad.append(f"utterance {b} (L={lens[b]}) {q} {('max', 'rms')[m]}: {float(ratio[u, j, m]):.2f}x "
                   f"(err {float(ratio[u, j, m] * e32[b, j, m].clamp(min=U)):.3g}, step {step})")
    assert not bad, f"{label}: {len(bad)} over {KAPPA}x the fp32 oracle's error: " + "; ".join(bad[:12])
    return worst


def _bench_program(cfg):
    prog = []
    for i in range(int(cfg.n_layers_ar)):
        prog += ["glu", "ffn1", "ffn2"] + (["qatt", "o"] if i in cfg.ar_attn_layers() else [])
    return prog + ["head", "sample"]


def _bench_run(wdtype):
    if wdtype not in _RUNS:
        _RUNS[wdtype] = _launch("bench", wdtype)
    return _RUNS[wdtype]


@pytest.mark.parametrize("wdtype", ["bf16", "fp32"])
def test_bench_shape(wdtype):
    """64 utterances x 401 steps, session max_text_len 52, most texts 52 tokens and five ragged (1, 2, 3, 5, 51):
    the bench's stage program (fused q + attention, 8 utterances per team, LL exchange)."""
    cfg = _set("bench")[0]
    got, program = _bench_run(wdtype)
    assert [k for k, _s in program] == _bench_program(cfg)
    if wdtype == "bf16":  # the host's task-shape rule at the bench geometry (DESIGN.md §3)
        by_kind = {}
        for k, s in program:
            by_kind.setdefault(k, set()).add(s)
        assert by_kind["ffn2"] == {"narrow"} and by_kind["o"] == {"narrow"} and by_kind["glu"] == {"wide"}, by_kind
    _check(f"bench {wdtype}", "bench", got, program)


def test_bench_shape_resumed_launches_are_bit_equal():
    """run(1), run(6), then the rest: the same residual, logit and K / V traces as one launch, bit for bit."""
    got, program = _launch("bench", "bf16", chunks=(1, 6))
    one, _ = _bench_run("bf16")
    assert torch.equal(got.blocks, one.blocks) and torch.equal(got.logits, one.logits)
    assert all(torch.equal(got.kv[i][0], one.kv[i][0]) and torch.equal(got.kv[i][1], one.kv[i][1]) for i in one.kv)


def test_bench_shape_word_timestamp_kernel_is_bit_equal():
    """The word-timestamp instantiation (attention weights exported) computes the untraced kernel's numbers."""
    got, program = _launch("bench", "bf16", attn=True)
    one, prog1 = _bench_run("bf16")
    assert program == prog1
    assert torch.equal(got.blocks, one.blocks) and torch.equal(got.logits, one.logits)


@pytest.mark.parametrize("wdtype", ["bf16", "fp32"])
def test_long_and_ragged_texts_in_one_launch(wdtype):
    """Texts of 1 ... 2048 tokens (session max_text_len 2048) side by side: the long Lmax reshapes the shared-memory
    plan (smaller weight ring, the q + attention stages unfused) and mixes the resident and streaming attention paths."""
    got, program = _launch("long", wdtype)
    _check(f"long {wdtype}", "long", got, program)


def test_small_config():
    """D = 128, V = 257 (the EOS column alone in the head's last partial tile), Dh = 32, kernel 5, dilations (1, 3),
    19 ragged utterances."""
    got, program = _launch("small", "fp32")
    _check("small fp32", "small", got, program)


SWEEP = [dict(team=t) for t in (1, 2, 3, 4, 5, 7, 8, 16, 20)] + [
    dict(team=16, sync="ll"), dict(team=20, sync="ll"), dict(team=1, sync="barrier"), dict(team=2, sync="barrier"),
    dict(team=8, sync="barrier"),
    dict(max_p=3), dict(max_p=7), dict(max_p=3, team=4), dict(max_p=7, team=20),
    dict(task_shape=1), dict(task_shape=2), dict(task_shape=2, team=20),
    dict(rows=[2]), dict(rows=[3]),
]


def test_geometry_sweep(monkeypatch):
    """One ragged batch of 40 (texts of 1 ... 130 tokens, bf16 weights) under every team geometry: utterances per team
    1, 2, 3, 4, 5, 7, 8, 16, 20 (TU = 1, 2, 4, 8, partly filled groups, LL up to 8 and the barrier above, the 20-utterance
    cap); the LL exchange forced on large teams and the barrier on small ones; at most 3 or 7 CTAs per team (row
    slices with remainders; 3 < H turns the fused q + attention stage off); wide and narrow task shapes; batch 1."""
    from sopro_b200 import _lib

    programs, failures = set(), []
    for g in SWEEP:
        monkeypatch.delenv("SOPRO_AR_SYNC", raising=False)
        monkeypatch.delenv("SOPRO_AR_MAX_P", raising=False)
        if "sync" in g:
            monkeypatch.setenv("SOPRO_AR_SYNC", g["sync"])
        if "max_p" in g:
            monkeypatch.setenv("SOPRO_AR_MAX_P", str(g["max_p"]))
        label = "sweep " + " ".join(f"{k}={v}" for k, v in g.items())
        got, program = _launch("sweep", "bf16", rows=g.get("rows"), team=g.get("team", 0), task_shape=g.get("task_shape", 0))
        programs.add(_attention_program(program))
        try:
            _check(label, "sweep", got, program, rows=g.get("rows"))
        except AssertionError as e:
            failures.append(str(e))
    # one CTA per team would stream every weight matrix through one CTA: 272 weight tiles per step, more than the tile
    # table's 128, refused before the launch (so is P = 3 with 14-utterance teams: 129)
    monkeypatch.setenv("SOPRO_AR_MAX_P", "1")
    with pytest.raises(_lib.SoproError, match="weight tiles"):
        _launch("sweep", "bf16")
    assert not failures, "\n".join(failures)
    assert programs == {"qatt", "q+att"}, programs
