"""Best-of-N synthesis on the host (sopro_b200/rerank.py and its use in sopro_b200/model.py), and the float64 Token2SV
restatement its GPU tests measure the kernels against (oracle/speaker_oracle.py).  No GPU: the engines are the
oracle-backed fakes of tests/test_host_pipeline_cpu.py."""
import numpy as np
import pytest
import torch

from oracle import speaker_oracle as SO
from sopro_b200 import prefill as P
from sopro_b200 import rerank
from sopro_b200.config import SoproTTSConfig
from sopro_b200.sampling import TapeFeed, noise_tape
from sopro_b200.weights import synth_state_dict
from tests.test_host_pipeline_cpu import tts  # noqa: F401  (the fixture)

torch.set_grad_enabled(False)


# ---- the choice rule
def test_choose_prefers_eligible_takes_by_cosine():
    # all eligible: highest cosine
    assert rerank.choose([30, 40, 35], [True, True, True], 10, [0.1, 0.5, 0.3]) == 1
    # the best cosine ran out of frames (no EOS): not eligible
    assert rerank.choose([30, 40, 35], [True, False, True], 10, [0.1, 0.9, 0.3]) == 2
    # the best cosine has fewer frames than text tokens: not eligible
    assert rerank.choose([30, 8, 35], [True, True, True], 10, [0.1, 0.9, 0.3]) == 2
    # T = text_len is eligible
    assert rerank.choose([10, 9], [True, True], 10, [0.1, 0.9]) == 0
    # the best cosine has no frames: never chosen
    assert rerank.choose([0, 12], [True, True], 10, [0.9, 0.2]) == 1


def test_choose_falls_back_to_live_takes_then_to_zero():
    # nothing eligible: highest cosine among T > 0, whatever the stop flag or length
    assert rerank.choose([5, 7, 0], [True, False, True], 10, [0.2, 0.4, 0.9]) == 1
    assert rerank.choose([50, 60], [False, False], 10, [0.7, 0.1]) == 0
    # every T = 0: candidate 0, cosines ignored (None allowed)
    assert rerank.choose([0, 0, 0], [True, True, False], 10, [0.1, 0.9, 0.5]) == 0
    assert rerank.choose([0, 0], [True, True], 3, None) == 0


def test_choose_ties_go_to_the_lowest_index():
    assert rerank.choose([20, 20, 20], [True, True, True], 5, [0.5, 0.5, 0.5]) == 0
    assert rerank.choose([20, 20, 20], [False, True, True], 5, [0.9, 0.5, 0.5]) == 1
    assert rerank.choose([3, 3, 3], [True, True, True], 5, [0.1, 0.6, 0.6]) == 1
    assert rerank.choose([7], [True], 5, [0.0]) == 0


def test_choose_refuses_mismatched_lists():
    with pytest.raises(ValueError):
        rerank.choose([1, 2], [True], 1, [0.0, 0.0])
    with pytest.raises(ValueError):
        rerank.choose([], [], 1, [])


@pytest.mark.parametrize("bad", [0, 17, 2.0, True, False, -1, "2", None])
def test_check_best_of_refuses(bad):
    with pytest.raises(ValueError):
        rerank.check_best_of(bad)


def test_check_best_of_accepts_its_range():
    assert [rerank.check_best_of(n) for n in (1, 2, 16)] == [1, 2, 16]
    rerank.check_rows(64, 64)
    rerank.check_rows(10 ** 6, None)
    with pytest.raises(ValueError):
        rerank.check_rows(65, 64)


# ---- the seed mapping, on the host tape feed
def test_candidate_seeds_feed_row_i_n_plus_k_with_seed_s_i_plus_k():
    seeds, N, steps, V, keep = [5, 40, 7], 3, 6, 97, 11
    rows = rerank.candidate_seeds(seeds, N)
    assert rows == [5, 6, 7, 40, 41, 42, 7, 8, 9]
    assert rerank.candidate_seeds(None, N) is None
    with TapeFeed(len(rows), steps, V, keep, "cpu", rows) as feed:
        feed.fill(steps)
        got = feed.host.clone()
    for i, s in enumerate(seeds):
        for k in range(N):
            assert torch.equal(got[i * N + k], noise_tape(steps, V, seed=s + k, keep=keep)), (i, k)


def test_unseeded_candidates_draw_the_global_generator_row_after_row():
    N, B, steps, V, keep = 2, 3, 5, 53, 7
    torch.manual_seed(123)
    with TapeFeed(B * N, steps, V, keep, "cpu", rerank.candidate_seeds(None, N)) as feed:
        feed.fill(steps)
        got = feed.host.clone()
    torch.manual_seed(123)
    for r in range(B * N):  # row i*N + k, in order: synthesize_batch of the B*N rows
        assert torch.equal(got[r], noise_tape(steps, V, keep=keep)), r


# ---- refusals come before any random draw
def test_bad_best_of_is_refused_before_any_draw(tts, monkeypatch):  # noqa: F811
    torch.manual_seed(9)
    state = torch.get_rng_state()
    for bad in (0, 17, 2.0, True):
        with pytest.raises(ValueError):
            tts.synthesize("3 14", ref=tts.ref, max_frames=8, best_of=bad)
        with pytest.raises(ValueError):
            tts.synthesize_batch(["3 14", "8 9"], ref=tts.ref, max_frames=8, best_of=bad)
        with pytest.raises(ValueError):
            tts.synthesize_long("3 14. 8 9.", ref=tts.ref, max_frames=8, best_of=bad)
    monkeypatch.setattr(tts, "_batch_limit", lambda: 4)
    with pytest.raises(ValueError):
        tts.synthesize_batch(["3 14", "8 9", "27"], ref=tts.ref, max_frames=8, best_of=2)
    with pytest.raises(ValueError):
        tts.synthesize("3 14", ref=tts.ref, max_frames=8, best_of=5)
    assert torch.equal(torch.get_rng_state(), state)


def _oracle_speaker_vectors(tts):
    """RefPrepEngine.speaker_vectors through the float64 restatement, rounded to fp32."""
    sd, V = tts.model.sd, int(tts.cfg.codebook_size)

    def fake(codes, lens, ref_sv=None):
        sv, cos = SO.speaker_vectors(sd, V, codes, lens, ref_sv)
        return sv.float(), None if cos is None else cos.float()

    return fake


def test_best_of_equals_the_picked_single_take(tts, monkeypatch):  # noqa: F811
    """Through the host pipeline: best_of=N returns synthesize(seed=s + k*), k* = choose over the N single takes, and
    decodes one row."""
    monkeypatch.setattr(tts.model.refprep, "speaker_vectors", _oracle_speaker_vectors(tts), raising=False)
    text, s, N, kw = "3 14 15 92 65 35", 4, 3, dict(max_frames=20, min_gen_frames=3)
    n_text = int(tts.encode_text(text).numel())
    Ts, stopped, cos = [], [], []
    for k in range(N):
        tok = tts.model.generate_tokens(tts.encode_text(text), tts.ref, style_strength=tts.cfg.style_strength, seed=s + k, **kw)
        Ts.append(int(tok.shape[0]))
        stopped.append(Ts[-1] < kw["max_frames"] + 1)
        if Ts[-1]:
            cos.append(float(SO.speaker_vectors(tts.model.sd, 2048, tok.unsqueeze(0), [Ts[-1]], tts.ref.sv_ref)[1][0]))
        else:
            cos.append(0.0)
    k = rerank.choose(Ts, stopped, n_text, cos)
    calls = len(tts.codec.engine.calls)
    got = tts.synthesize(text, ref=tts.ref, seed=s, best_of=N, **kw)
    assert len(tts.codec.engine.calls) == calls + 1 and tts.codec.engine.calls[-1][0] == 1
    want = tts.synthesize(text, ref=tts.ref, seed=s + k, **kw)
    np.testing.assert_allclose(got.numpy(), want.numpy(), rtol=0, atol=1e-5)
    assert got.shape == want.shape


# ---- the float64 restatement against the torch one
@pytest.mark.parametrize("lens", [[1], [2, 7, 40], [6, 5, 1, 23]])
def test_speaker_oracle_matches_prefill_token2sv_row_by_row(lens):
    cfg = SoproTTSConfig()
    sd = synth_state_dict(cfg, text_vocab=1000, seed=3)
    g = torch.Generator().manual_seed(len(lens))
    codes = torch.randint(0, int(cfg.codebook_size), (len(lens), max(lens), int(cfg.num_codebooks)), generator=g)
    ref = torch.nn.functional.normalize(torch.randn(192, generator=g), dim=0)
    sv, cos = SO.speaker_vectors(sd, int(cfg.codebook_size), codes, lens, ref)
    for b, n in enumerate(lens):
        want = P.token2sv(sd, cfg, codes[b: b + 1, :n], torch.tensor([n]))[0].double()
        # unit vectors of 192 fp32 terms: the fp32 chain's round-off stays far below 1e-5 per component
        assert float((sv[b] - want).abs().max()) < 1e-5, (b, n)
        assert abs(float(cos[b]) - float(sv[b] @ ref.double())) < 1e-12
