"""GPU parity of the CUDA NAR refiner (sopro_nar_refine, through the C-ABI) against the CPU oracle, which is pinned to
tokens written by the unmodified reference (tests/golden/e2e_prefill.npz)."""
import os

import numpy as np
import pytest
import torch

from oracle import dense_probes as P
from oracle import nar_oracle as N
from tests.cases import _unit, e2e_inputs

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
torch.set_grad_enabled(False)
_ENG = {}


def _engine():
    from sopro_b200.nar import NarEngine

    if "e" not in _ENG:
        cfg, sd, _ = e2e_inputs()
        _ENG["e"] = NarEngine(cfg, sd, 0)
    return _ENG["e"]


def _cond(B, T, D, key):
    return torch.stack([_unit(T * D, key + i).view(T, D) for i in range(B)])


def _check(eng, cfg, sd, cond, rvq1, lens=None):
    """ids identical to the oracle's; a differing id is accepted only if, teacher-forced on the oracle's codes, the
    oracle's own top-2 logits at that id are within 1e-5 (relative) of a tie.  Returns the accepted near-ties."""
    B, T, _ = cond.shape
    got = eng.refine(cond, rvq1, lens).cpu()
    want = torch.zeros_like(got)
    margin = torch.zeros(got.shape)
    for b in range(B):
        n = T if lens is None else int(lens[b])
        w, m = N.nar_refine(sd, cfg, cond[b:b + 1, :n], rvq1[b:b + 1, :n])
        want[b, :n], margin[b, :n] = w[0], m[0]
        got[b, n:] = 0
    if torch.equal(got, want):
        return []
    # classify through teacher forcing (so one flip cannot cascade into later stages)
    eng.set_forced(want)
    try:
        tf = eng.refine(cond, rvq1, lens).cpu()
    finally:
        eng.set_forced(None)
    for b in range(B):
        n = T if lens is None else int(lens[b])
        tf[b, n:] = 0
    bad = (tf != want).nonzero().tolist()
    ties = [(tuple(i), float(margin[tuple(i)])) for i in bad]
    assert all(m < 1e-5 for _i, m in ties), f"NAR ids differ away from a tie: {ties}"
    assert len(ties) <= max(2, got.numel() // 20000), ties
    return ties


def test_nar_ids_equal_the_reference_fixture():
    """The fixture's 50 x 32 tokens were written by the reference's own nar_refine; the kernel must reproduce them."""
    from sopro_b200 import prefill as P

    eng = _engine()
    cfg, sd, inp = e2e_inputs()
    g = np.load(os.path.join(GOLD, "e2e_prefill.npz"))
    dev = torch.device("cpu")
    pr = P.prepare_reference(sd, cfg, inp["ref_tokens_tq"], dev)
    tpos = P.sinusoid_table(int(cfg.max_text_len) + 8, int(cfg.d_model), dev)
    fpos = P.sinusoid_table(int(cfg.pos_emb_max) + 8, int(cfg.d_model), dev)
    prep = P.prepare_conditioning(sd, cfg, inp["text_ids"], pr, max_frames=inp["max_frames"], device=dev,
                                  style_strength=inp["style_strength"], text_pos=tpos, frame_pos=fpos)
    T = inp["nar_T"]
    got = eng.refine(prep["cond_ar"][:, :T], inp["rvq1"].unsqueeze(0))[0].cpu()
    gold = torch.from_numpy(g["nar_tokens"].astype(np.int64))
    diff = (got != gold).nonzero().tolist()
    if diff:
        _w, margin = N.nar_refine(sd, cfg, prep["cond_ar"][:, :T], inp["rvq1"].unsqueeze(0), forced=gold.unsqueeze(0))
        eng.set_forced(gold.unsqueeze(0))
        try:
            tf = eng.refine(prep["cond_ar"][:, :T], inp["rvq1"].unsqueeze(0))[0].cpu()
        finally:
            eng.set_forced(None)
        bad = [(tuple(i), float(margin[0][tuple(i)])) for i in (tf != gold).nonzero().tolist()]
        print("NAR ids differing from the reference fixture (teacher-forced) -> oracle top-2 margin:", bad)
        assert all(m < 1e-5 for _i, m in bad) and len(bad) <= 1, bad
    else:
        print("NAR ids identical to the reference fixture (50 x 32)")


@pytest.mark.parametrize("B,T", [(1, 1), (1, 6), (1, 16), (1, 17), (2, 40), (3, 129), (1, 401)])
def test_nar_matches_oracle_shapes(B, T):
    """Skinny kernel (B*T <= 16 rows), tile kernel, partial tiles, the full 401-frame length."""
    eng = _engine()
    cfg, sd, _ = e2e_inputs()
    cond = _cond(B, T, int(cfg.d_model), 9100 + 7 * T)
    rvq1 = torch.randint(0, 2048, (B, T), generator=torch.Generator().manual_seed(T))
    ties = _check(eng, cfg, sd, cond, rvq1)
    print(f"NAR B={B} T={T}: near-tie flips {ties}")


def test_nar_ragged_batch_equals_each_utterance_alone():
    """lens: utterance b of a padded batch equals the refiner run on its own frames (the refiner is not causal: padding
    rows must act as the convolutions' zero padding and never leak)."""
    eng = _engine()
    cfg, sd, _ = e2e_inputs()
    lens = torch.tensor([37, 5, 64, 1, 50])
    B, T = len(lens), 64
    cond = _cond(B, T, int(cfg.d_model), 9900)
    rvq1 = torch.randint(0, 2048, (B, T), generator=torch.Generator().manual_seed(3))
    got = eng.refine(cond, rvq1, lens).cpu()
    for b in range(B):
        n = int(lens[b])
        alone = eng.refine(cond[b:b + 1, :n].contiguous(), rvq1[b:b + 1, :n].contiguous()).cpu()
        assert torch.equal(got[b, :n], alone[0]), b
    _check(eng, cfg, sd, cond, rvq1, lens)


def test_nar_strided_conditioning_rows():
    """cond_ar[:, :T] of a longer prefill buffer: rows contiguous, batch stride larger than T*D (no copy)."""
    eng = _engine()
    cfg, sd, _ = e2e_inputs()
    D = int(cfg.d_model)
    full = _cond(2, 60, D, 9990).to("cuda:0")
    rvq1 = torch.randint(0, 2048, (2, 25), generator=torch.Generator().manual_seed(4))
    a = eng.refine(full[:, :25], rvq1)
    b = eng.refine(full[:, :25].contiguous(), rvq1)
    assert torch.equal(a, b)


def test_tensor_core_path_equals_the_fp32_path():
    """Above 16 rows the contractions run on the tensor cores with every fp32 operand split into three exact bf16 terms (six
    products, fp32 accumulation: the fp32 result up to summation order).  Same ids as the fp32 FMA kernels and as the CPU
    oracle on 4 x 300 frames; a differing id must be an oracle near-tie (the _check rule)."""
    eng = _engine()
    cfg, sd, _ = e2e_inputs()
    B, T = 4, 300
    cond = _cond(B, T, int(cfg.d_model), 9300)
    rvq1 = torch.randint(0, 2048, (B, T), generator=torch.Generator().manual_seed(31))
    eng.set_contraction(0)
    try:
        fp32_ids = eng.refine(cond, rvq1).cpu()
    finally:
        eng.set_contraction(-1)
    tc_ids = eng.refine(cond, rvq1).cpu()
    n_diff = int((fp32_ids != tc_ids).sum())
    print(f"tensor-core vs fp32 NAR ids: {n_diff} of {tc_ids.numel()} differ")
    ties = _check(eng, cfg, sd, cond[:2], rvq1[:2])  # tensor-core path (automatic) against the oracle
    assert n_diff <= 2 + len(ties)


@pytest.mark.parametrize("T", [6, 17, 187])
def test_streaming_windows_replay_from_graphs_identically(T):
    """Single-utterance windows are captured into a CUDA graph on first use and replayed afterwards (skinny fp32 path at 6
    frames, tensor-core path above 16): first call (eager + capture), replays and the plain launches give the same ids,
    also for a different window of the same length and for a strided conditioning slice."""
    eng = _engine()
    cfg, sd, _ = e2e_inputs()
    D = int(cfg.d_model)
    full = _cond(1, T + 9, D, 9700 + T).to("cuda:0")
    rv = torch.randint(0, 2048, (1, T + 9), generator=torch.Generator().manual_seed(T))
    eng.set_graphs(False)
    try:
        plain_a = eng.refine(full[:, :T], rv[:, :T]).cpu()
        plain_b = eng.refine(full[:, 9:T + 9], rv[:, 9:T + 9]).cpu()
    finally:
        eng.set_graphs(True)
    first = eng.refine(full[:, :T], rv[:, :T]).cpu()        # eager + capture
    replay_a = eng.refine(full[:, :T], rv[:, :T]).cpu()     # replay
    replay_b = eng.refine(full[:, 9:T + 9], rv[:, 9:T + 9]).cpu()
    assert torch.equal(first, plain_a) and torch.equal(replay_a, plain_a) and torch.equal(replay_b, plain_b)


# ---------------------------------------------------------------------------------------------------------------
# continuous values: each stage's pre-head activation z against the float64 oracle
# ---------------------------------------------------------------------------------------------------------------
def _stages(cfg):
    return [(n, idx) for n, idx in cfg.stage_indices().items() if len(idx) > 0]


def _traced(eng, cond, rvq1, lens, forced):
    """teacher-forced run with the z trace on -> (ids [B, T, Q], z [n_stages, B, T, Hn]) on the host"""
    B, T, _ = cond.shape
    z = torch.full((len(_stages(eng.cfg)), B, T, int(eng.cfg.nar_head_dim)), float("nan"), device=eng.device)
    eng.set_forced(forced)
    eng.set_trace(z)
    try:
        ids = eng.refine(cond, rvq1, lens).cpu()
    finally:
        eng.set_trace(None)
        eng.set_forced(None)
    return ids, z.cpu()


def _oracle_z(sd, cfg, cond, rvq1, forced, dtype):
    zs = []
    N.nar_refine(sd, cfg, cond, rvq1, forced=forced, dtype=dtype, z_out=zs)
    return [z[0] for z in zs]


def _z_errors(sd, cfg, cond, rvq1, lens, got_z, forced, utts):
    """per stage: (GPU max-rel, GPU rms-rel, fp32 oracle max-rel, fp32 oracle rms-rel), over the valid rows of `utts`"""
    per = [([], [], []) for _ in range(got_z.shape[0])]
    for b in utts:
        n = int(lens[b]) if lens is not None else cond.shape[1]
        args = (cond[b:b + 1, :n], rvq1[b:b + 1, :n], forced[b:b + 1, :n])
        z64 = _oracle_z(sd, cfg, *args, torch.float64)
        z32 = _oracle_z(sd, cfg, *args, torch.float32)
        for s in range(got_z.shape[0]):
            per[s][0].append(got_z[s, b, :n])
            per[s][1].append(z32[s])
            per[s][2].append(z64[s])
    out = []
    for g, f, r in per:
        g, f, r = torch.cat(g), torch.cat(f), torch.cat(r)
        out.append(P.rel_errors(g, r) + P.rel_errors(f, r))
    return out


def _assert_kappa(errs, label):
    for s, (eg, rg, ef, rf) in enumerate(errs):
        print(f"{label} stage {s}: GPU max {eg:.2e} rms {rg:.2e} | fp32 oracle max {ef:.2e} rms {rf:.2e} | ratio max {eg / ef:.2f} "
              f"rms {rg / rf:.2f}")
    for s, (eg, rg, ef, rf) in enumerate(errs):
        assert eg <= P.KAPPA * ef and rg <= P.KAPPA * rf, (label, s, eg / ef, rg / rf)


@pytest.mark.parametrize("mode", [0, -1])
@pytest.mark.parametrize("B,T", [(1, 6), (1, 16), (1, 17), (3, 129), (1, 401)])
def test_nar_stage_activations_against_float64(B, T, mode):
    """Teacher-forced on the oracle's codes, every stage's z (nar.pre's output) against the float64 oracle: the GPU's
    relative error, max and RMS, is at most KAPPA (oracle/dense_probes.py) times the fp32 CPU oracle's on the same input.
    mode 0 = fp32 FMA kernels, -1 = the default (tensor cores above 16 rows)."""
    eng = _engine()
    cfg, sd, _ = e2e_inputs()
    cond = _cond(B, T, int(cfg.d_model), 9400 + 3 * T)
    rvq1 = torch.randint(0, 2048, (B, T), generator=torch.Generator().manual_seed(T + 5))
    lens = torch.tensor([T, T // 2 + 1, 1][:B]) if B > 1 else None
    forced = torch.zeros((B, T, int(cfg.num_codebooks)), dtype=torch.long)
    for b in range(B):
        n = T if lens is None else int(lens[b])
        forced[b, :n] = N.nar_refine(sd, cfg, cond[b:b + 1, :n], rvq1[b:b + 1, :n])[0][0]
    eng.set_contraction(mode)
    try:
        _ids, z = _traced(eng, cond, rvq1, lens, forced)
    finally:
        eng.set_contraction(-1)
    _assert_kappa(_z_errors(sd, cfg, cond, rvq1, lens, z, forced, range(B)), f"B={B} T={T} mode={mode}")


def test_batch64_crosses_every_head_chunk():
    """synthesize_batch's geometry: 64 utterances x 401 frames = 25,664 rows on the default tensor-core path, where the head
    logits run in chunks of mc rows (nar_engine.cu: 256 MB of logits per chunk; 2048 rows for V = 2048 and 16 heads).  The
    utterances holding rows mc j - 1 and mc j of every chunk boundary, plus the first and the last, are checked: ids against
    the oracle (the _check near-tie rule, teacher-forced) and every stage's z against float64."""
    eng = _engine()
    cfg, sd, _ = e2e_inputs()
    B, T, D, V, Q = 64, 401, int(cfg.d_model), int(cfg.codebook_size), int(cfg.num_codebooks)
    M = B * T
    heads = max(len(idx) for _n, idx in _stages(cfg))
    mc = ((256 << 20) // (heads * V * 4)) // 128 * 128
    mc = max(128, min(mc, (M + 127) // 128 * 128))
    bounds = list(range(mc, M, mc))
    assert len(bounds) >= 12, (mc, len(bounds))  # 13 chunks at the default geometry
    rows = [r for m0 in bounds for r in (m0 - 1, m0)]
    sel = sorted({r // T for r in rows} | {0, B - 1})
    lens = torch.full((B,), T)
    short = [b for b in range(1, B - 1) if b not in sel][:5]
    for b, n in zip(short, (1, 17, 200, 399, 128)):
        lens[b] = n
    assert all(r % T < int(lens[r // T]) for r in rows), "every boundary row is a valid frame"
    cond = torch.stack([_unit(T * D, 12000 + b).view(T, D) for b in range(B)])
    rvq1 = torch.randint(0, V, (B, T), generator=torch.Generator().manual_seed(64))
    got = eng.refine(cond, rvq1, lens).cpu()
    want = got.clone()
    margin = torch.full(got.shape, float("inf"))
    for b in sel:
        n = int(lens[b])
        w, m = N.nar_refine(sd, cfg, cond[b:b + 1, :n], rvq1[b:b + 1, :n])
        want[b, :n], margin[b, :n] = w[0], m[0]
    tf, z = _traced(eng, cond, rvq1, lens, want)
    for b in range(B):
        got[b, int(lens[b]):] = 0
        tf[b, int(lens[b]):] = 0
        want[b, int(lens[b]):] = 0
    sel_t = torch.tensor(sel)
    n_diff = int((got[sel_t] != want[sel_t]).sum())
    bad = [(b, t, q) for b, t, q in (tf != want).nonzero().tolist() if b in sel]
    ties = [((b, t, q), float(margin[b, t, q])) for b, t, q in bad]
    print(f"batch 64 x 401: {len(bounds) + 1} head chunks of {mc} rows, {len(sel)} utterances checked, {n_diff} ids differ, "
          f"teacher-forced near-ties {ties}")
    assert all(m < 1e-5 for _i, m in ties), f"NAR ids differ away from a tie: {ties}"
    assert len(ties) <= max(2, len(sel) * T * Q // 20000), ties
    _assert_kappa(_z_errors(sd, cfg, cond, rvq1, lens, z, want, sel), "B=64 T=401")


def test_nar_engines_on_two_devices_in_one_process():
    """Function attributes (the skinny kernel's 96 KB of shared memory for FFN2, K = 1536) belong to each device's context: a
    second engine on another device must run the skinny path as the first does."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    from sopro_b200.nar import NarEngine

    eng0 = _engine()
    cfg, sd, _ = e2e_inputs()
    cond = _cond(1, 9, int(cfg.d_model), 9555)
    rvq1 = torch.randint(0, 2048, (1, 9), generator=torch.Generator().manual_seed(9))
    a = eng0.refine(cond, rvq1).cpu()
    eng1 = NarEngine(cfg, sd, 1)
    try:
        b = eng1.refine(cond, rvq1).cpu()
    finally:
        eng1.close()
    assert torch.equal(a, b)
