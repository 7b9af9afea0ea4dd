"""GPU: timed synthesis -- the CUDA mix (longform.mix) against the oracle's sequential fp32 sum at deep overlaps, tile
edges, empty items, the timeline's ends and 10k items over 10 M samples; one cue equals synthesize_long followed by
zeros, with and without the output chain; a two-voice WebVTT track equals each cue's synthesize_long, stretched at the
oracle's S and summed by the oracle's mix, with CueFit equal to the oracle's fit; best_of picks synthesize_long's
takes.  All bit for bit (oracle/timed_oracle.py)."""
import numpy as np
import pytest
import torch

from oracle import timed_oracle as TO

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

FRAMES = 40
KW = dict(max_frames=FRAMES, min_gen_frames=3, max_tokens=7)


def _api():
    from tests.test_stream_batch_gpu import _tts

    return _tts()


def _bits(t):
    return t.reshape(-1).cpu().numpy().view(np.uint32)


def _check_mix(rows, offs, length):
    from sopro_b200.longform import mix

    got = mix(rows, offs, length)
    assert got.shape == (1, 1, length)
    want = TO.mix([r.cpu().numpy() for r in rows], offs, length)
    assert np.array_equal(_bits(got), want.view(np.uint32))
    return got.reshape(-1)


def test_mix_equals_the_sequential_sum():
    g = np.random.default_rng(1)
    L = 200_000
    # ~40 deep: 40 items over one 5000-sample window, plus scattered ones, every edge off the 4096 tiles
    offs = [int(v) for v in g.integers(60_000, 61_000, 40)] + [int(v) for v in g.integers(0, L - 9000, 60)]
    lens = [int(v) for v in g.integers(4000, 9000, 100)]
    offs += [0, 4095, 8192, 12_287, L - 4097, 100, 5]
    lens += [4096, 2, 4096, 0, 4097, 0, 1]  # an item at 0, one ending at y_len, empty items, tile edges
    rows = [torch.from_numpy(g.standard_normal(n).astype(np.float32)).cuda() for n in lens]
    y = _check_mix(rows, offs, L)
    depth = np.zeros(L, np.int64)
    for o, n in zip(offs, lens):
        depth[o: o + n] += 1
    assert depth.max() >= 40 and depth[L - 1] == 1 and depth[0] == 1 and (depth == 0).any()
    # singly covered samples are their source's, and uncovered ones are +0.0
    yc = y.cpu().numpy()
    for o, r in zip(offs, rows):
        one = np.nonzero(depth[o: o + r.numel()] == 1)[0]
        assert np.array_equal(yc[o + one].view(np.uint32), r.cpu().numpy()[one].view(np.uint32))
    assert not yc[depth == 0].view(np.uint32).any()
    # a negative zero covered once keeps its sign; covered by +0.0 after it, it sums to +0.0
    z = torch.tensor([-0.0, -0.0], device="cuda")
    assert _bits(_check_mix([z, torch.zeros(1, device="cuda")], [3, 4], 6)).tolist() == [0, 0, 0, 0x80000000, 0, 0]
    # no item: zeros, every sample written
    assert not _bits(_check_mix([], [], 5000)).any()


def test_mix_of_10k_items_over_10m_samples():
    g = np.random.default_rng(2)
    L, n = 10_000_000, 10_000
    lens = [int(v) for v in g.integers(0, 60_000, n)]
    offs = [int(g.integers(0, L - k + 1)) for k in lens]
    base = torch.from_numpy(g.standard_normal(70_000).astype(np.float32)).cuda()
    rows = [base[int(s): int(s) + k] for s, k in zip(g.integers(0, 10_000, n), lens)]  # views, read in place
    _check_mix(rows, offs, L)


def test_one_cue_equals_synthesize_long_then_zeros():
    from sopro_b200 import Cue
    from sopro_b200.output import OutputChain

    tts, refs = _api()
    text = "3 7 11 15. 5 9 13 17 21! 4 8?"
    long = tts.synthesize_long(text, ref=refs[0], seed=40, **KW)
    n = long.shape[-1]
    assert n > 0
    end = (n + 24_000 + 17) / 24000  # a slot a second longer than the speech
    pad = torch.cat([long.reshape(-1), torch.zeros(round(end * 24000) - n, device="cuda")]).reshape(1, 1, -1)
    for chain in (dict(), dict(sample_rate=16000), dict(loudness=-16.0), dict(watermark=0xC0FFEE),
                  dict(sample_rate=48000, loudness=-20.0, watermark=7)):
        got, fits = tts.synthesize_timed([Cue(0.0, end, text)], ref=refs[0], seed=40, **KW, **chain)
        want, _ = OutputChain(tts, chain.get("sample_rate"), None, chain.get("loudness"), chain.get("watermark"))(pad)
        assert got.shape == want.shape and torch.equal(got, want), chain
        assert fits == [type(fits[0])(0, 1.0, n / 24000, 0.0)]
    got, _ = tts.synthesize_timed([Cue(0.0, end, text)], ref=refs[0], seed=40, **KW)
    assert torch.equal(got[..., :n], long) and not got[..., n:].any()


def _ms(t):
    h, r = divmod(int(round(t * 1000)), 3_600_000)
    m, r = divmod(r, 60_000)
    return f"{h:02d}:{m:02d}:{r // 1000:02d}.{r % 1000:03d}"


def _track(n_cues, texts, times, voices):
    out = ["WEBVTT", ""]
    for k in range(n_cues):
        v = "" if voices[k] is None else f"<v {voices[k]}>"
        out += [f"cue-{k}", f"{_ms(times[k][0])} --> {_ms(times[k][1])} line:0", v + texts[k], ""]
    return "\n".join(out)


def test_two_voice_webvtt_track_equals_its_cues():
    from sopro_b200.cues import parse
    from sopro_b200.longform import SEGMENT_GROUP, split_text
    from sopro_b200.stretch import stretch_rows

    tts, refs = _api()
    seed = 90
    names = {"anna": refs[1], "ben": refs[2]}
    g = np.random.default_rng(5)
    n_cues = 30
    texts = [" ".join(str(int(v)) for v in g.integers(1, 900, int(g.integers(8, 22)))) + "." for _ in range(n_cues)]
    texts[7] = "<i></i>"  # an empty cue
    voices = [[None, "anna", "ben"][k % 3] for k in range(n_cues)]
    plain = ["" if k == 7 else x for k, x in enumerate(texts)]  # the cues' text after the reader
    segs = [split_text(t, tts.tokenizer, KW["max_tokens"]) for t in plain]
    assert sum(len(s) for s in segs) > SEGMENT_GROUP and segs[7] == []
    # each cue alone, through synthesize_long with its first segment's seed
    rows, first = [], 0
    for t, v, s in zip(plain, voices, segs):
        voice = refs[0] if v is None else names[v]
        rows.append(tts.synthesize_long(t, ref=voice, seed=seed + first, **KW).reshape(-1) if s
                    else torch.zeros(0, device="cuda"))
        first += len(s)
    n = [r.numel() for r in rows]
    # slots from the speech: cue k % 4 == 0 fits with room, 1 and 2 need a speed-up, 3 needs more than the cap
    times, t = [], 0.5
    for k in range(n_cues):
        d = max(n[k], 2400) / 24000 * [1.3, 1 / 1.15, 1 / 1.6, 1 / 3][k % 4]
        times.append((round(t, 3), round(t + d, 3)))
        t += d + 0.25
    times[12] = (times[11][0] + 0.1, times[11][0] + 0.1 + times[12][1] - times[12][0])  # overlaps cue 11's speech
    track = _track(n_cues, texts, times, voices)
    cues = parse(track)
    assert [c.text for c in cues] == plain and [c.voice for c in cues] == voices
    got, fits = tts.synthesize_timed(track, ref=refs[0], voices=names, seed=seed, max_rate=1.7, **KW)
    S, M, over, offs, N = TO.fit(n, [c.start for c in cues], [c.end for c in cues], 1.7)
    cap = round(1.7 * 65536)
    assert S[0] == 65536 and 65536 < S[1] < cap and 65536 < S[2] < cap and S[3] == cap and over[3] > 0
    assert n[7] == 0 and S[7] == 65536 and M[7] == 0 and offs[12] < offs[11] + M[11]
    stretched = [r if k == 65536 or r.numel() == 0 else stretch_rows(r.reshape(1, -1), [k / 65536]).reshape(-1)
                 for r, k in zip(rows, S)]
    assert [r.numel() for r in stretched] == M
    order = sorted(range(n_cues), key=lambda k: (offs[k], k))
    want = TO.mix([stretched[k].cpu().numpy() for k in order], [offs[k] for k in order], N)
    assert got.shape == (1, 1, N) and np.array_equal(_bits(got), want.view(np.uint32))
    assert [(f.index, f.rate, f.spoken, f.overrun) for f in fits] == \
        [(k, S[k] / 65536, M[k] / 24000, over[k] / 24000) for k in range(n_cues)]


def test_best_of_picks_synthesize_long_takes():
    from sopro_b200 import Cue

    tts, refs = _api()
    text = "3 7 11 15. 5 9 13 17 21! 4 8?\n\n6 2 10 12 14 16 18 20 22 24, 26 28 30. 1"
    long = tts.synthesize_long(text, ref=refs[1], seed=5, best_of=2, **KW)
    got, _ = tts.synthesize_timed([Cue(0.25, 0.25 + long.shape[-1] / 24000 + 0.5, text)], ref=refs[1], seed=5,
                                  best_of=2, **KW)
    assert torch.equal(got[..., 6000: 6000 + long.shape[-1]], long) and not got[..., :6000].any()
    assert not got[..., 6000 + long.shape[-1]:].any()
