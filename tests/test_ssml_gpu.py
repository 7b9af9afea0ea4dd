"""GPU: speech markup (SoproTTS.synthesize_ssml) -- plain text in <speak> equals synthesize_long, a two-voice script
equals synthesize_dialogue, a script with rates, volumes, breaks and a silent span equals its chain of public stages
with the oracle's gaps and gains (oracle/ssml_oracle.py), breaks stay absolute under `speed`, and best_of picks
synthesize_long's takes; all bit for bit."""
import numpy as np
import pytest
import torch

from oracle import ssml_oracle as SO

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

TEXT = "3 7 11 15. 5 9 13 17 21! 4 8?\n\n6 2 10 12 14 16 18 20 22 24, 26 28 30. 1"
FRAMES = 40
KW = dict(max_frames=FRAMES, min_gen_frames=3, max_tokens=7)


def _api():
    from tests.test_stream_batch_gpu import _tts

    return _tts()


def _bits(t):
    return t.reshape(-1).cpu().numpy().view(np.uint32)


@pytest.mark.parametrize("chain", (dict(), dict(sample_rate=16000), dict(loudness=-16.0), dict(watermark=0xC0FFEE),
                                   dict(sample_rate=48000, loudness=-20.0, watermark=7)))
def test_plain_text_equals_synthesize_long(chain):
    tts, refs = _api()
    got = tts.synthesize_ssml("<speak>" + TEXT + "</speak>", ref=refs[0], seed=40, **KW, **chain)
    want = tts.synthesize_long(TEXT, ref=refs[0], seed=40, **KW, **chain)
    assert got.shape == want.shape and torch.equal(got, want)


def test_two_voices_equal_synthesize_dialogue():
    tts, refs = _api()
    turns = [(refs[0], "3 7 11 15. 5 9 13 17 21!"), (refs[1], "4 8? 6 2 10 12 14."), (refs[0], "16 18 20."),
             (refs[1], "22 24, 26 28 30. 1 5.")]
    names = {"a": refs[0], "b": refs[1]}
    ssml = "<speak>" + "".join(f'<voice name="{"a" if v is refs[0] else "b"}">{t}</voice> ' for v, t in turns) + "</speak>"
    got = tts.synthesize_ssml(ssml, ref=refs[2], voices=names, seed=11, pause_ms=300, **KW)
    want = tts.synthesize_dialogue(turns, seed=11, pause_ms=300, turn_pause_ms=300, **KW)
    assert got.shape == want.shape and torch.equal(got, want)


MIXED = ('<speak><break time="120ms"/>3 7 11. <prosody rate="slow" volume="-6dB">5 9 13 17.</prosody>'
         '<break time="2.5s"/><voice name="b"><prosody rate="150%">4 8 6 2.</prosody> 10 12</voice>'
         '<prosody volume="silent"> 14 16 18.</prosody><p><prosody rate="x-fast" volume="+3dB">20 22, 24 26 28 30.</prosody>'
         '</p><s>1 5 <prosody rate="0.5">9</prosody></s><break strength="strong"/></speak>')


@pytest.mark.parametrize("chain", (dict(), dict(speed=1.25, sample_rate=16000, watermark=5), dict(speed=0.8, loudness=-18.0)))
def test_mixed_script_equals_its_chain_of_stages(chain):
    from sopro_b200 import ssml as M
    from sopro_b200.longform import join_gaps, speech_extents, split_text
    from sopro_b200.output import OutputChain
    from sopro_b200.stretch import stretch

    tts, refs = _api()
    names = {"b": refs[1]}
    seed = 70
    got = tts.synthesize_ssml(MIXED, ref=refs[0], voices=names, seed=seed, **KW, **chain)
    speed = chain.get("speed")
    plan = M.parse(MIXED, names, refs[0], 250, 500, speed, KW["max_tokens"], tts.tokenizer)
    o_segs, o_gaps, o_lead, o_trail = SO.plan(MIXED, names, refs[0], 250, 500, speed,
                                              lambda t: split_text(t, tts.tokenizer, KW["max_tokens"]))
    assert [s.text for s in plan.segments] == [s[0] for s in o_segs] and plan.gaps == o_gaps
    assert (plan.lead, plan.trail) == (o_lead, o_trail) and plan.lead == 2880 and 60000 in plan.gaps
    assert any(s.gain == 0.0 for s in plan.segments) and len({s.rate for s in plan.segments}) >= 4
    rows, dbs = [], []
    for k, (text, voice, rate, db) in enumerate(o_segs):
        w = tts.synthesize(text, ref=voice, seed=seed + k, max_frames=FRAMES, min_gen_frames=3).reshape(1, -1)
        dbs.append(db)
        if w.numel() == 0:
            rows.append(torch.zeros(0, device="cuda"))
            continue
        s, e = speech_extents(w).cpu().numpy()[0]
        span = w[0, int(s): int(e)]
        rows.append(span if round(rate * 65536) == 65536 else stretch(span, rate).reshape(-1))
    spoken = [r.numel() > 0 for r in rows]
    assert sum(spoken) >= 5
    pauses = SO.merged_pauses(o_gaps, spoken)
    gains = torch.tensor([SO.gain(d) for d in dbs], dtype=torch.float32, device="cuda")
    idx = [k for k in range(len(rows)) if spoken[k]]
    # the kernel join takes gaps up to 2 s: join around the 2.5 s break and lay its zeros between
    parts, a = [torch.zeros(o_lead, device="cuda")], 0
    for m, p in enumerate(pauses + [None]):
        if p is None or p > 48000:
            sub = idx[a: m + 1]
            parts.append(join_gaps([rows[k] for k in sub], [(0, rows[k].numel()) for k in sub], pauses[a: m],
                                   gains[sub]).reshape(-1))
            if p is not None:
                parts.append(torch.zeros(p, device="cuda"))
            a = m + 1
    parts.append(torch.zeros(o_trail, device="cuda"))
    joined = torch.cat(parts).reshape(1, 1, -1)
    # the float64 restatement of the assembly agrees with the kernel join
    o = SO.assemble([r.cpu().numpy() for r in rows], o_gaps, dbs, o_lead, o_trail)
    assert np.array_equal(o.view(np.uint32), _bits(joined))
    want, _ = OutputChain(tts, chain.get("sample_rate"), None, chain.get("loudness"), chain.get("watermark"))(joined)
    assert got.shape == want.shape and torch.equal(got, want)


def test_breaks_stay_absolute_under_speed():
    tts, refs = _api()
    ssml = '<speak>3 7 11 15. <break time="1s"/> 5 9 13 17.</speak>'
    for speed in (None, 2.0):
        wav = tts.synthesize_ssml(ssml, ref=refs[0], seed=3, speed=speed, **KW).reshape(-1).cpu().numpy()
        from sopro_b200 import ssml as M
        from sopro_b200.longform import speech_extents
        from sopro_b200.stretch import stretched_length

        plan = M.parse(ssml, None, refs[0], 250, 500, speed, KW["max_tokens"], tts.tokenizer)
        assert plan.gaps == [24000]
        first = tts.synthesize(plan.segments[0].text, ref=refs[0], seed=3, max_frames=FRAMES, min_gen_frames=3)
        s, e = speech_extents(first.reshape(1, -1)).cpu().numpy()[0]
        n0 = stretched_length(speed or 1.0, int(e - s))
        assert n0 > 0 and not wav[n0: n0 + 24000].any() and wav.size > n0 + 24000
        assert wav[n0 - 241: n0].any() and wav[n0 + 24000: n0 + 24241].any()  # the zeros are exactly the break


def test_best_of_picks_synthesize_long_takes():
    tts, refs = _api()
    got = tts.synthesize_ssml("<speak>" + TEXT + "</speak>", ref=refs[1], seed=5, best_of=2, **KW)
    want = tts.synthesize_long(TEXT, ref=refs[1], seed=5, best_of=2, **KW)
    assert got.shape == want.shape and torch.equal(got, want)
