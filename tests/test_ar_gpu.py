"""GPU parity tests of the persistent AR kernel, through the C-ABI, against
(a) the golden fixtures written from the reference and (b) the CPU oracle."""
import os

import numpy as np
import pytest
import torch

from oracle import ar_oracle as O
from tests.cases import AR_CASES, _unit, ar_case_inputs

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
torch.set_grad_enabled(False)

_ENGINES = {}


def _engine(cfg, sd, wdtype, key):
    from sopro_b200.engine import ArEngine

    k = (key, wdtype)
    if k not in _ENGINES:
        _ENGINES[k] = ArEngine(cfg, sd, device=0, weight_dtype=wdtype)
    return _ENGINES[k]


def _wkey(spec):
    return (str(sorted(spec["cfg"].items())), spec["head_gain"], spec["bf16"], spec.get("eos_bias", 0.0))


def _sampling(samp, cfg, **over):
    from sopro_b200.engine import Sampling

    mg = samp.min_gen_frames if samp.min_gen_frames is not None else cfg.min_gen_frames
    d = dict(top_p=samp.top_p, temperature=samp.temperature, recovery_top_p=samp.recovery_top_p,
             recovery_temp=samp.recovery_temp, repetition_penalty=samp.repetition_penalty, top_k=samp.top_k,
             anti_loop=samp.anti_loop, loop_streak=samp.loop_streak, min_gen_frames=int(min(mg, 2 ** 31 - 1)),
             stop_on_first_eos=False)
    d.update(over)
    return Sampling(**d)


def _case(name):
    spec = AR_CASES[name]
    cfg, sd, inp = ar_case_inputs(spec)
    g = np.load(os.path.join(GOLD, f"ar_{name}.npz"))
    eng = _engine(cfg, sd, "bf16" if spec["bf16"] else "fp32", _wkey(spec))
    steps = inp["max_frames"] + 1
    tape = O.noise_tape(spec["noise_seed"], steps, cfg.ar_vocab())[:, :50].contiguous()
    return spec, cfg, sd, inp, g, eng, steps, tape


def _run_case(name, **samp_over):
    spec, cfg, sd, inp, g, eng, steps, tape = _case(name)
    ses = eng.session(1, steps, inp["txt_seq"].shape[1])
    ses.begin(inp["cond_ar"], inp["txt_seq"], [inp["txt_seq"].shape[1]], tape.unsqueeze(0), _sampling(inp["sampling"], cfg, **samp_over))
    ses.run()
    toks, n, done = ses.read()
    return toks[0, : n[0]].tolist(), g, ses


@pytest.mark.parametrize("name", list(AR_CASES))
def test_free_running_tokens_match_reference(name):
    """Sampled ids are bit-identical to the reference's ar_stream under the same seed."""
    toks, g, _ = _run_case(name)
    gold = g["tokens"].tolist()
    if toks != gold:
        first = next((i for i, (a, b) in enumerate(zip(toks, gold)) if a != b), min(len(toks), len(gold)))
        pytest.fail(f"{name}: diverges at step {first}: got {toks[first:first+4]} want {gold[first:first+4]} (len {len(toks)} vs {len(gold)})")


@pytest.mark.parametrize("name", ["default_fp32", "default_bf16", "peaked_fp32", "small_fp32"])
def test_teacher_forced_logits_and_blocks(name):
    """With the reference's tokens forced, every step's logits and the per-block residual
    stream match the reference within fp32 round-off (tolerance stated below)."""
    spec, cfg, sd, inp, g, eng, steps, tape = _case(name)
    gold = torch.from_numpy(g["tokens"].astype(np.int32))
    n = gold.numel()
    forced = torch.zeros(1, steps, dtype=torch.int32)
    forced[0, :n] = gold
    dev = eng.device
    tr_b = torch.zeros(steps, int(cfg.n_layers_ar), 1, int(cfg.d_model), device=dev)
    tr_l = torch.zeros(steps, 1, cfg.ar_vocab(), device=dev)
    ses = eng.session(1, steps, inp["txt_seq"].shape[1])
    ses.set_forced(forced)
    ses.set_trace(tr_b, tr_l)
    ses.begin(inp["cond_ar"], inp["txt_seq"], [inp["txt_seq"].shape[1]], tape.unsqueeze(0), _sampling(inp["sampling"], cfg))
    ses.run()
    toks, nn, done = ses.read()
    sampled = ses.sampled().cpu()[0, :n].tolist()
    torch.cuda.synchronize()
    # block traces at steps 0 and 1: |err| <= 2e-5 * max|ref| (fp32 accumulation-order noise)
    bt = g["block_trace"]  # [2, n_layers, D]
    got = tr_b[:2, :, 0].cpu().numpy()
    for t in range(2):
        for i in range(bt.shape[1]):
            tol = 2e-5 * max(1.0, float(np.abs(bt[t, i]).max()))
            np.testing.assert_allclose(got[t, i], bt[t, i], rtol=0, atol=tol, err_msg=f"step {t} block {i}")
    # logits at the fixture's steps
    lg = tr_l[:, 0].cpu().numpy()
    for row, t in zip(g["logits"], g["logit_steps"].tolist()):
        tol = 3e-5 * max(1.0, float(np.abs(row).max()))
        np.testing.assert_allclose(lg[t], row, rtol=0, atol=tol, err_msg=f"logits step {t}")
    # the token sampled at every step (given the reference history) is the reference's
    assert sampled == gold.tolist()


def test_batched_bf16_reference_case_over_a_team_of_eight():
    """The reference fixture default_bf16 replicated over a team of 8 utterances: teacher-forced logits and per-block
    residuals within the fixture tolerances (3e-5 / 2e-5 of the peak, fp32 accumulation-order noise), and every sampled
    token is the reference's."""
    spec, cfg, sd, inp, g, eng, steps, tape = _case("default_bf16")
    B, L = 8, inp["txt_seq"].shape[1]
    gold = torch.from_numpy(g["tokens"].astype(np.int32))
    n = gold.numel()
    forced = torch.zeros(B, steps, dtype=torch.int32)
    forced[:, :n] = gold
    dev = eng.device
    tr_b = torch.zeros(steps, int(cfg.n_layers_ar), B, int(cfg.d_model), device=dev)
    tr_l = torch.zeros(steps, B, cfg.ar_vocab(), device=dev)
    ses = eng.session(B, steps, L)
    ses.set_forced(forced)
    ses.set_trace(tr_b, tr_l)
    ses.begin(inp["cond_ar"].expand(B, -1, -1).contiguous(), inp["txt_seq"].expand(B, -1, -1).contiguous(), [L] * B,
              tape.unsqueeze(0).expand(B, -1, -1).contiguous(), _sampling(inp["sampling"], cfg))
    ses.run()
    sampled = ses.sampled().cpu()[:, :n]
    torch.cuda.synchronize()
    bt = g["block_trace"]
    for u in range(B):
        got = tr_b[:2, :, u].cpu().numpy()
        for t in range(2):
            for i in range(bt.shape[1]):
                tol = 2e-5 * max(1.0, float(np.abs(bt[t, i]).max()))
                np.testing.assert_allclose(got[t, i], bt[t, i], rtol=0, atol=tol, err_msg=f"utt {u} step {t} block {i}")
        lg = tr_l[:, u].cpu().numpy()
        for row, t in zip(g["logits"], g["logit_steps"].tolist()):
            tol = 3e-5 * max(1.0, float(np.abs(row).max()))
            np.testing.assert_allclose(lg[t], row, rtol=0, atol=tol, err_msg=f"utt {u} logits step {t}")
        assert sampled[u].tolist() == gold.tolist(), f"utterance {u}"
    ses.set_forced(None)
    ses.close()


@pytest.mark.parametrize("n_utts", [8, 19, 5])
def test_bf16_ragged_teams_match_the_oracle(n_utts):
    """bf16 weight storage, ragged texts, full and partially filled teams (19 -> 7 + 7 + 5 utterances), a resumed
    launch: every utterance equals the CPU oracle run alone on it."""
    spec = AR_CASES["default_bf16"]
    cfg, sd, _ = ar_case_inputs(spec)
    eng = _engine(cfg, sd, "bf16", _wkey(spec))
    lens = [52, 7, 23, 33, 1, 12, 5, 40, 17, 9, 52, 3, 28, 44, 2, 36, 11, 6, 50][:n_utts]
    n, steps = len(lens), 32
    cond, txt, tapes = _batch_inputs(cfg, n, steps, lens)
    samp = O.ArSampling(min_gen_frames=10 ** 9)
    want = _oracle_batch(sd, cfg, cond, txt, tapes, lens, samp, steps)
    ses = eng.session(n, steps, max(lens))
    ses.begin(cond, txt, lens, tapes[:, :, :50].contiguous(), _sampling(samp, cfg))
    ses.run(11)
    ses.run()
    toks, nn, done = ses.read()
    bad = [i for i in range(n) if toks[i, : nn[i]].tolist() != want[i]]
    assert not bad, f"utterances {bad} differ from the oracle"
    ses.close()


def test_sampler_known_answers_on_the_device_sampler():
    """The 29 sampler known-answer cases of the reference (tests/golden/sampler_kat.json, written by the reference's
    sample_token) through the kernel's sampler IN ISOLATION (sopro_debug_sample): flat / mid / peaked rows, history
    lengths 0..80 with periodic histories, recovery parameters, temperature 1, no repetition penalty, top_p = 1 (the
    unsorted multinomial branch, noise indexed by token id), a spike, NaN / +-inf logits, small vocabularies, top_k
    larger than the vocabulary, a tiny top_p.  Skipped: the two top_k = 0 cases (ar_stream always passes top_k = 50,
    reference model.py:283-292; the C-ABI rejects top_k = 0)."""
    import ctypes as C
    import json

    from sopro_b200 import _lib
    from tests.cases import SAMPLER_CASES, sampler_case_inputs

    lib = _lib.load()
    with open(os.path.join(GOLD, "sampler_kat.json")) as f:
        kat = json.load(f)
    ran = 0
    for name, spec in SAMPLER_CASES.items():
        logits, hist, kw, seed = sampler_case_inputs(spec)
        if int(kw["top_k"]) < 1:
            continue
        V = int(logits.numel())
        tape = O.noise_tape(seed, 1, V)[0].contiguous()
        top_k = min(int(kw["top_k"]), 64)
        q = _lib.ArSampling(float(kw["top_p"]), float(kw["temperature"]), float(kw["top_p"]), float(kw["temperature"]),
                            float(kw["repetition_penalty"]), top_k, 0, 8, 2 ** 31 - 1, 0)
        lg = logits.to(torch.float32).contiguous()
        h = np.asarray(hist, dtype=np.int32)
        out = C.c_int32(-1)
        nk = V if float(kw["top_p"]) >= 1.0 else min(top_k, V)
        _lib.check(lib.sopro_debug_sample(lg.data_ptr(), V, h.ctypes.data if len(hist) else None, len(hist), tape.data_ptr(), nk,
                                          C.byref(q), 0, 0, C.byref(out)))
        assert out.value == kat[name], f"{name}: device sampler {out.value}, reference {kat[name]}"
        ran += 1
    assert ran == len(SAMPLER_CASES) - 2


def test_kv_cache_matches_oracle():
    spec, cfg, sd, inp, g, eng, steps, tape = _case("default_fp32")
    L = inp["txt_seq"].shape[1]
    ses = eng.session(1, steps, L)
    ses.begin(inp["cond_ar"], inp["txt_seq"], [L], tape.unsqueeze(0), _sampling(inp["sampling"], cfg))
    k, v = ses.kv()
    torch.cuda.synchronize()
    for slot, li in enumerate(cfg.ar_attn_layers()):
        ko, vo = O.text_kv_cache(sd, f"ar.x_attns.{li}.", inp["txt_seq"], cfg.AR_HEADS)
        np.testing.assert_allclose(k[slot, 0, :, :L].cpu().numpy(), ko[0].numpy(), rtol=0, atol=2e-5)
        np.testing.assert_allclose(v[slot, 0, :, :L].cpu().numpy(), vo[0].numpy(), rtol=0, atol=2e-5)


def _batch_inputs(cfg, n, steps, lens):
    D = int(cfg.d_model)
    Ls = max(lens)
    cond = torch.stack([_unit(steps * D, 9000 + i).view(steps, D) for i in range(n)])
    txt = torch.zeros(n, Ls, D)
    for i, L in enumerate(lens):
        txt[i, :L] = _unit(L * D, 9500 + i).view(L, D)
    tapes = torch.stack([O.noise_tape(100 + i, steps, cfg.ar_vocab()) for i in range(n)])
    return cond, txt, tapes


def _oracle_batch(sd, cfg, cond, txt, tapes, lens, samp, steps):
    out = []
    for i, L in enumerate(lens):
        out.append(O.ar_generate(sd, cfg, cond[i:i + 1], txt[i:i + 1, :L], torch.ones(1, L, dtype=torch.bool),
                                 max_frames=steps - 1, sampling=samp, noise_tv=tapes[i]))
    return out


@pytest.mark.parametrize("n_utts", [8, 19])
def test_teams_of_eight_utterances_match_the_oracle(n_utts):
    """The bench geometry: teams of 8 utterances (8-utterance x 4-row register tile, LL exchange), full and
    partially filled teams, against the oracle run alone on every utterance."""
    spec = AR_CASES["peaked_fp32"]
    cfg, sd, _ = ar_case_inputs(spec)
    eng = _engine(cfg, sd, "fp32", _wkey(spec))
    lens = [52, 7, 23, 33, 1, 12, 5, 40, 17, 9, 52, 3, 28, 44, 2, 36, 11, 6, 50][:n_utts]
    n, steps = len(lens), 24
    cond, txt, tapes = _batch_inputs(cfg, n, steps, lens)
    samp = O.ArSampling(min_gen_frames=10 ** 9)
    want = _oracle_batch(sd, cfg, cond, txt, tapes, lens, samp, steps)
    ses = eng.session(n, steps, max(lens))
    ses.begin(cond, txt, lens, tapes[:, :, :50].contiguous(), _sampling(samp, cfg))
    ses.run()
    toks, nn, done = ses.read()
    bad = [i for i in range(n) if toks[i, : nn[i]].tolist() != want[i]]
    assert not bad, f"utterances {bad} differ from the oracle"


def test_teams_of_sixteen_utterances_barrier_mode():
    """Non-default geometry (sopro_ar_session_set_team(16)): two 8-utterance groups per team, team barrier instead of
    the LL exchange."""
    spec = AR_CASES["peaked_fp32"]
    cfg, sd, _ = ar_case_inputs(spec)
    eng = _engine(cfg, sd, "fp32", _wkey(spec))
    lens = [52, 7, 23, 33, 1, 12, 5, 40, 17, 9, 52, 3, 28, 44, 2, 36, 11, 6, 50]
    n, steps = len(lens), 16
    cond, txt, tapes = _batch_inputs(cfg, n, steps, lens)
    samp = O.ArSampling(min_gen_frames=10 ** 9)
    want = _oracle_batch(sd, cfg, cond, txt, tapes, lens, samp, steps)
    ses = eng.session(n, steps, max(lens))
    ses.set_team(16)
    ses.begin(cond, txt, lens, tapes[:, :, :50].contiguous(), _sampling(samp, cfg))
    ses.run()
    toks, nn, done = ses.read()
    bad = [i for i in range(n) if toks[i, : nn[i]].tolist() != want[i]]
    assert not bad, f"utterances {bad} differ from the oracle"


@pytest.mark.parametrize("team", [0, 1, 2, 3])
def test_batch_equals_each_utterance_alone(team):
    """Utterance i of a ragged batch == the oracle run alone on utterance i (SURVEY.md §0.3),
    for every team geometry (1 team, several teams, uneven last team)."""
    spec = AR_CASES["peaked_fp32"]
    cfg, sd, _ = ar_case_inputs(spec)
    eng = _engine(cfg, sd, "fp32", _wkey(spec))
    lens = [52, 7, 23, 33, 1, 12, 5]
    n, steps = len(lens), 40
    cond, txt, tapes = _batch_inputs(cfg, n, steps, lens)
    samp = O.ArSampling(min_gen_frames=10 ** 9)
    want = _oracle_batch(sd, cfg, cond, txt, tapes, lens, samp, steps)
    ses = eng.session(n, steps, max(lens))
    ses.set_team(team)
    ses.begin(cond, txt, lens, tapes[:, :, :50].contiguous(), _sampling(samp, cfg))
    ses.run()
    toks, nn, done = ses.read()
    for i in range(n):
        assert toks[i, : nn[i]].tolist() == want[i], f"utterance {i} (L={lens[i]})"


_WORKER_CACHE = {}


def _oracle_tokens_worker(args):
    """One utterance of the full-size case on the CPU oracle (runs in a worker process: 64 of them are ~1 CPU-minute)."""
    i, steps, L = args
    torch.set_num_threads(2)
    torch.set_grad_enabled(False)
    if "full" not in _WORKER_CACHE:
        _WORKER_CACHE["full"] = ar_case_inputs(AR_CASES["default_bf16"])[:2]
    cfg, sd = _WORKER_CACHE["full"]
    D = int(cfg.d_model)
    cond = _unit(steps * D, 7000 + i).view(1, steps, D)
    txt = _unit(L * D, 7500 + i).view(1, L, D)
    return i, O.ar_generate(sd, cfg, cond, txt, torch.ones(1, L, dtype=torch.bool), max_frames=steps - 1,
                            sampling=O.ArSampling(min_gen_frames=10 ** 9), noise_tv=O.noise_tape(300 + i, steps, cfg.ar_vocab()))


def _near_tie_margin(sd, cfg, cond_i, txt_i, samp, tape, want, t):
    """Relative distance to the nearest decision boundary of the oracle's sampler at step `t` (oracle history):
    the two best ratios p_sorted[j] / q[j] of the draw, the top-p cut (cum[j] vs top_p), and the order of the sorted
    probabilities around the winning rank (the noise is assigned by RANK, sampling.py:83-84: two candidates whose
    probabilities differ by an ulp-scale amount swap ranks, and with them their noise, under any fp32 reordering)."""
    logits, rec = [], []
    gen = O.ar_stream(sd, cfg, cond_i, txt_i, torch.ones(1, txt_i.size(1), dtype=torch.bool), max_frames=t, sampling=samp,
                      noise_tv=tape, logits_out=logits, recovery_out=rec)
    for _ in gen:
        pass
    top_p, temp = (samp.recovery_top_p, samp.recovery_temp) if t in rec else (samp.top_p, samp.temperature)
    tr = {}
    O.sample_token(logits[t].view(1, 1, -1), want[:t], top_p=top_p, top_k=samp.top_k, temperature=temp,
                   repetition_penalty=samp.repetition_penalty, noise_v=tape[t], trace=tr)
    sp = tr["sorted_probs"][:50].double()
    r = (sp / tape[t][:50].double()).sort(descending=True).values
    draw = float((r[0] - r[1]) / r[0])
    cut = float((tr["cum"][:50].double() - top_p).abs().min())
    cum = tr["cum"][:51].double()
    raw = torch.diff(cum, prepend=torch.zeros(1, dtype=torch.double))  # sorted probabilities before the top-p cut
    win = int((sp / tape[t][:50].double()).argmax())
    lo, hi = max(win - 1, 0), min(win + 1, 50)
    order = float(((raw[lo:hi] - raw[lo + 1:hi + 1]) / raw[lo:hi]).min())
    return min(draw, cut, order)


def test_full_size_batch64_properties():
    """BASELINE.json's batch-64 configuration at full size (64 utterances x 401 steps, L=52, bf16 weight storage),
    EVERY utterance against the CPU oracle:
    (1) the launch is deterministic and every utterance runs its full length;
    (2) with the oracle's tokens teacher-forced, the token the kernel samples at each of the 64 x 401 steps is the
        oracle's.  The sampler is discontinuous in the logits, so a flip is tolerated only when the oracle itself sits
        within 1e-5 (relative) of a decision boundary at that step (two candidates' p/q ratios, or the top-p cut), and
        at most 2 such flips in the whole batch;
    (3) free-running, every utterance equals the oracle for all 401 frames unless its first divergence is one of the
        near-tie steps of (2)."""
    spec = AR_CASES["default_bf16"]
    cfg, sd, _ = ar_case_inputs(spec)
    eng = _engine(cfg, sd, "bf16", _wkey(spec))
    n, steps, L = 64, 401, 52
    D = int(cfg.d_model)
    cond = torch.stack([_unit(steps * D, 7000 + i).view(steps, D) for i in range(n)])
    txt = torch.stack([_unit(L * D, 7500 + i).view(L, D) for i in range(n)])
    full_tapes = [O.noise_tape(300 + i, steps, cfg.ar_vocab()) for i in range(n)]
    tapes = torch.stack([t[:, :50] for t in full_tapes]).contiguous()
    samp = O.ArSampling(min_gen_frames=10 ** 9)
    ses = eng.session(n, steps, L)
    out = []
    for _ in range(2):
        ses.begin(cond, txt, [L] * n, tapes, _sampling(samp, cfg))
        ses.run()
        toks, nn, _ = ses.read()
        out.append(toks.copy())
        assert (nn == steps).all()
    assert np.array_equal(out[0], out[1])
    assert len({tuple(r) for r in out[0].tolist()}) == n  # 64 different utterances
    import multiprocessing as mp
    from concurrent.futures import ProcessPoolExecutor

    workers = max(1, min(16, (os.cpu_count() or 2) // 2))
    with ProcessPoolExecutor(max_workers=workers, mp_context=mp.get_context("spawn")) as ex:
        want = [toks for _i, toks in sorted(ex.map(_oracle_tokens_worker, [(i, steps, L) for i in range(n)]))]
    forced = torch.tensor(want, dtype=torch.int32)
    ses.set_forced(forced)
    ses.begin(cond, txt, [L] * n, tapes, _sampling(samp, cfg))
    ses.run()
    sampled = ses.sampled().cpu().numpy()
    ses.set_forced(None)
    flips = [(i, t) for i in range(n) for t in range(steps) if int(sampled[i, t]) != want[i][t]]
    margins = {(i, t): _near_tie_margin(sd, cfg, cond[i:i + 1], txt[i:i + 1], samp, full_tapes[i], want[i], t) for i, t in flips}
    print("full-size report: teacher-forced flips (utterance, step) -> oracle boundary margin:", margins)
    assert len(flips) <= 2, margins
    assert all(m < 1e-5 for m in margins.values()), margins
    for i in range(n):
        first = next((t for t in range(steps) if int(out[0][i, t]) != want[i][t]), None)
        assert first is None or (i, first) in margins, f"utterance {i} diverges free-running at step {first} without a near-tie"


def test_long_text_takes_the_streaming_attention_path():
    """Texts longer than the shared-memory K/V capacity (128 keys) use the cold attention path; a ragged batch
    mixes both paths in one launch."""
    spec = AR_CASES["peaked_fp32"]
    cfg, sd, _ = ar_case_inputs(spec)
    eng = _engine(cfg, sd, "fp32", _wkey(spec))
    lens = [200, 40, 131]
    n, steps = len(lens), 12
    cond, txt, tapes = _batch_inputs(cfg, n, steps, lens)
    samp = O.ArSampling(min_gen_frames=10 ** 9)
    want = _oracle_batch(sd, cfg, cond, txt, tapes, lens, samp, steps)
    ses = eng.session(n, steps, max(lens))
    ses.begin(cond, txt, lens, tapes[:, :, :50].contiguous(), _sampling(samp, cfg))
    ses.run()
    toks, nn, done = ses.read()
    for i in range(n):
        assert toks[i, : nn[i]].tolist() == want[i], f"utterance {i} (L={lens[i]})"


def test_resume_in_chunks_equals_one_launch():
    """Streaming drives the kernel chunk by chunk (stream(): 6 frames); state lives in HBM."""
    spec, cfg, sd, inp, g, eng, steps, tape = _case("peaked_fp32")
    L = inp["txt_seq"].shape[1]
    ses = eng.session(1, steps, L)
    ses.begin(inp["cond_ar"], inp["txt_seq"], [L], tape.unsqueeze(0), _sampling(inp["sampling"], cfg))
    while ses.position < steps:
        ses.run(6)
    toks, n, done = ses.read()
    assert toks[0, : n[0]].tolist() == g["tokens"].tolist()


def test_host_buffer_path():
    spec, cfg, sd, inp, g, eng, steps, tape = _case("eos_mingen40")
    L = inp["txt_seq"].shape[1]
    ses = eng.session(1, steps, L)
    toks, n = ses.generate_host(inp["cond_ar"].numpy(), inp["txt_seq"].numpy(), [L], tape.unsqueeze(0).numpy(),
                                _sampling(inp["sampling"], cfg))
    assert toks[0, : n[0]].tolist() == g["tokens"].tolist()


def test_stop_on_first_eos_mode():
    """generate_tokens()/stream() consumers break at the first EOS (model.py:382-383)."""
    toks, g, _ = _run_case("eos_mingen40", stop_on_first_eos=True)
    gold = g["tokens"].tolist()
    eos = 2048
    first = gold.index(eos)
    assert toks == gold[: first + 1]


def test_errors_are_loud():
    from sopro_b200 import _lib
    from sopro_b200.engine import Sampling

    spec, cfg, sd, inp, g, eng, steps, tape = _case("default_fp32")
    ses = eng.session(1, 8, 8)
    with pytest.raises(_lib.SoproError):
        ses.run(1)  # before begin
    with pytest.raises(_lib.SoproError):
        ses.begin(inp["cond_ar"][:, :8], inp["txt_seq"][:, :8], [0], tape[:8].unsqueeze(0), Sampling())  # text_len 0
    with pytest.raises(_lib.SoproError):
        ses.begin(inp["cond_ar"][:, :8], inp["txt_seq"][:, :8], [8], tape[:8].unsqueeze(0), Sampling(top_k=0))
    with pytest.raises(_lib.SoproError):
        ses.begin(inp["cond_ar"][:, :8], inp["txt_seq"][:, :8], [8], tape[:8, :10].unsqueeze(0).contiguous(), Sampling())
