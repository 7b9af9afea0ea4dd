"""How the host drives the AR step, without a GPU: the noise tape each launch reads, where the caller's generator is
left, and the launch schedule of every path (single-utterance chunks, one-launch batches, growing-block batches).

The AR, prefill, NAR and Mimi engines are the oracle-backed fakes of tests/test_host_pipeline_cpu.py; the schedule
tests use a session that only records what it is asked to run.
"""
import copy
import threading

import numpy as np
import pytest
import torch

from sopro_b200.engine import Generation
from tests.test_host_pipeline_cpu import SEEDS, TEXTS, _FakeArEngine, tts  # noqa: F401

torch.set_grad_enabled(False)
KW = dict(max_frames=20, min_gen_frames=3)


@pytest.fixture(scope="module")
def long_tts(tts):  # noqa: F811
    """The pipeline of `tts` with EOS made less likely (bias +1.5 instead of +2.5): seeds 1-4 give utterances of
    about 4 to 60 frames, so a batch at max_frames=70 runs past the first noise block."""
    cfg = tts.cfg
    sd = dict(tts.model.engine.sd)
    bias = sd["ar.head.bias"].clone()
    bias[int(cfg.codebook_size)] -= 1.0
    sd["ar.head.bias"] = bias
    t = copy.copy(tts)
    t.model = copy.copy(tts.model)
    t.model.engine = _FakeArEngine(cfg, sd)
    t.model._sessions, t.model._sessions_busy, t.model._sessions_lock = {}, set(), threading.Lock()
    return t


def test_batch_equals_single_across_noise_blocks(long_tts):
    """A seeded batch of 71 steps draws its tapes and launches in blocks of 24 and 47 frames; each utterance still
    equals synthesize(text, seed=s)."""
    kw = dict(max_frames=70, min_gen_frames=3)
    wavs = long_tts.synthesize_batch(TEXTS, ref=long_tts.ref, seeds=SEEDS, **kw)
    lens = [w.shape[-1] // 1920 for w in wavs]
    assert len(set(lens)) >= 2 and max(lens) > 24, f"the case must be ragged and run past the first block, got {lens}"
    for text, seed, w in zip(TEXTS, SEEDS, wavs):
        single = long_tts.synthesize(text, ref=long_tts.ref, seed=seed, **kw)
        assert single.shape == w.shape, (single.shape, w.shape)
        np.testing.assert_allclose(w.numpy(), single.numpy(), rtol=0, atol=1e-5)


def test_batch_without_seeds_consumes_the_global_generator_utterance_after_utterance(tts, monkeypatch):  # noqa: F811
    got = {}
    real = tts.model.ar_generate_tensors

    def spy(*a, **k):
        got["toks"], got["n"] = real(*a, **k)
        return got["toks"], got["n"]

    monkeypatch.setattr(tts.model, "ar_generate_tensors", spy)
    torch.manual_seed(21)
    tts.synthesize_batch(TEXTS, ref=tts.ref, seeds=None, **KW)
    after = torch.get_rng_state()
    steps, V = KW["max_frames"] + 1, tts.cfg.ar_vocab()
    torch.manual_seed(21)
    states = []
    for _ in TEXTS:
        states.append(torch.get_rng_state())
        torch.empty(steps, V).exponential_(1.0)
    assert torch.equal(torch.get_rng_state(), after)
    for i, text in enumerate(TEXTS):
        g = torch.Generator()
        g.set_state(states[i])
        prep = tts.model.prepare_conditioning(tts.encode_text(text), tts.ref, max_frames=KW["max_frames"],
                                              style_strength=tts.cfg.style_strength)
        single = [tok for _t, tok, _e in tts.model.ar_stream(prep, generator=g, **KW)]
        n = int(got["n"][i])
        assert n > 0 and got["toks"][i, :n].tolist() == single[:n], i


def test_synthesize_settles_the_generator_and_a_batch_of_one_does_not(tts):  # noqa: F811
    """synthesize(t) leaves the global generator after the draws of its frames and the EOS step, as the reference
    does; synthesize_batch([t]) draws every tape in full, as it does for any number of texts."""
    text, V, steps = TEXTS[1], tts.cfg.ar_vocab(), KW["max_frames"] + 1
    torch.manual_seed(17)
    one = tts.synthesize(text, ref=tts.ref, **KW)
    after_one = torch.get_rng_state()
    torch.manual_seed(17)
    (batch,) = tts.synthesize_batch([text], ref=tts.ref, **KW)
    after_batch = torch.get_rng_state()
    assert torch.equal(one, batch)
    T = one.shape[-1] // 1920
    assert T + 1 < steps, f"the case must stop at an EOS before max_frames, got {T} frames"
    for drawn, state in ((T + 1, after_one), (steps, after_batch)):
        torch.manual_seed(17)
        torch.empty(drawn, V).exponential_(1.0)
        assert torch.equal(torch.get_rng_state(), state), drawn


def test_ar_stream_settles_the_passed_generator_to_the_consumed_frames(tts):  # noqa: F811
    prep = tts.model.prepare_conditioning(tts.encode_text(TEXTS[1]), tts.ref, max_frames=20,
                                          style_strength=tts.cfg.style_strength)
    kw = dict(max_frames=20, min_gen_frames=10 ** 9, launch_frames=6)
    g = torch.Generator().manual_seed(9)
    before = torch.get_rng_state()
    it = tts.model.ar_stream(prep, generator=g, **kw)
    toks = [next(it)[1] for _ in range(8)]  # 12 rows drawn for two launches, 8 consumed
    it.close()
    assert torch.equal(torch.get_rng_state(), before)
    want = torch.Generator().manual_seed(9)
    torch.empty(8, tts.cfg.ar_vocab()).exponential_(1.0, generator=want)
    assert torch.equal(g.get_state(), want.get_state())
    assert toks == [tok for _t, tok, _e in tts.model.ar_stream(prep, seed=9, **kw)][:8]


class _SpySession:
    """Records `begin` and the frames each run(n) launches (the library clamps n to the steps left)."""

    def __init__(self, log):
        self.log = log

    def begin(self, cond, txt, lens, noise, samp):
        self.B, self.steps, self.pos = int(cond.shape[0]), int(cond.shape[1]), 0
        self.log.append("begin")

    def run(self, n_steps=None):
        end = min(self.steps, self.pos + (self.steps if n_steps is None else int(n_steps)))
        if end > self.pos:
            self.log.append(end - self.pos)
        self.pos = end

    def read(self):
        return np.zeros((self.B, self.steps), np.int32), np.full(self.B, self.pos, np.int32), np.zeros(self.B, np.int32)

    def set_attn_trace(self, probs):
        pass

    def close(self):
        pass


@pytest.fixture
def launches(tts, monkeypatch):  # noqa: F811
    log = []
    eng = type("SpyEngine", (), {"session": lambda self, B, steps, L: _SpySession(log)})()
    monkeypatch.setattr(tts.model, "engine", eng)
    monkeypatch.setattr(tts.model, "_sessions", {})
    return log


@pytest.mark.parametrize("chunk_frames, want", [(6, [6, 6, 6, 3]), (0, [21]), (25, [21])])
def test_ar_stream_launch_schedule(tts, launches, chunk_frames, want):  # noqa: F811
    prep = {"cond_ar": torch.zeros(1, 21, 8), "txt_seq": torch.zeros(1, 4, 8)}
    list(tts.model.ar_stream(prep, max_frames=20, launch_frames=chunk_frames, seed=1))
    assert launches == ["begin"] + want


@pytest.mark.parametrize("max_frames, seeds, want", [
    (400, [1, 2], [24, 36, 54, 81, 121, 85]),  # growing blocks
    (62, [1, 2], [63]),  # under 64 steps: one launch
    (63, [1, 2], [24, 40]),
    (70, [1, 2], [24, 47]),
    (400, None, [401]),  # the global generator: one launch
])
def test_batch_launch_schedule_from_resolved_settings(tts, launches, max_frames, seeds, want):  # noqa: F811
    steps = max_frames + 1
    gen = Generation.resolve(tts.cfg, max_frames=max_frames, top_p=0.9, temperature=1.05, anti_loop=True,
                             style_strength=None, min_gen_frames=None)
    toks, n = tts.model.ar_generate_tensors(torch.zeros(2, steps, 8), torch.zeros(2, 4, 8), [4, 3], gen=gen, seeds=seeds)
    assert launches == ["begin"] + want and n.tolist() == [steps, steps]
