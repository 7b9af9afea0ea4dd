"""GPU: the chunk-stream contract every streaming output stage shares (csrc/chunk_stream.cuh), on each stage's stream:
an oversized push is refused and leaves the state as it was, a finished stream takes no call until a reset, and a reset
stream gives the one-shot result again bit for bit."""
import pytest
import torch

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
CHUNK = 1920  # the streams' max_chunk


def _resampler():
    from sopro_b200.resample import Resampler

    rs = Resampler(24000, 44100, "cuda:0")
    return (lambda: rs.stream(CHUNK)), (), rs


def _stretch():
    from sopro_b200.stretch import StretchStream, stretch

    return (lambda: StretchStream(CHUNK, 0, 1.25)), (1.25,), (lambda x: stretch(x, 1.25))


def _watermark():
    from sopro_b200.watermark import WatermarkStream, embed_watermark

    return (lambda: WatermarkStream(CHUNK, 0, 7)), (7,), (lambda x: embed_watermark(x, 7))


STAGES = {"resampler": _resampler, "stretch": _stretch, "watermark": _watermark}


@pytest.fixture(params=sorted(STAGES))
def stage(request):
    """(a new stream of max_chunk CHUNK, the arguments of its reset, the one-shot function it streams)"""
    return STAGES[request.param]()


def _signal(n):
    return (0.3 * torch.randn(n, generator=torch.Generator().manual_seed(n))).cuda()


def _run(st, x):
    parts = [st.push(x[i: i + CHUNK]) for i in range(0, x.numel(), CHUNK)]
    return torch.cat(parts + [st.finish()])


def test_oversized_push_is_refused_and_the_stream_still_gives_the_one_shot_result(stage):
    make, _args, one_shot = stage
    x = _signal(5 * CHUNK + 17)
    st = make()
    parts = [st.push(x[:CHUNK])]
    with pytest.raises(ValueError):
        st.push(x[CHUNK: 3 * CHUNK + 1])
    parts += [st.push(x[i: i + CHUNK]) for i in range(CHUNK, x.numel(), CHUNK)]
    assert torch.equal(torch.cat(parts + [st.finish()]), one_shot(x))
    st.close()


def test_finished_stream_refuses_push_finish_and_ready_until_a_reset(stage):
    from sopro_b200 import _lib

    make, args, one_shot = stage
    x = _signal(3 * CHUNK + 5)
    want = one_shot(x)
    st = make()
    assert torch.equal(_run(st, x), want)
    for call in (lambda: st.push(x[:10]), lambda: st.push(x[:0]), st.finish, lambda: st.ready(10)):
        with pytest.raises(_lib.SoproError):
            call()
    st.reset(*args)
    assert torch.equal(_run(st, x), want)
    st.close()


def test_reset_mid_utterance_starts_a_new_one(stage):
    make, args, one_shot = stage
    x = _signal(4 * CHUNK + 1)
    st = make()
    st.push(_signal(CHUNK))
    st.push(_signal(CHUNK - 7))
    st.reset(*args)
    assert torch.equal(_run(st, x), one_shot(x))
    st.close()
