"""GPU: the FLAC encoder (csrc/flac.cu through sopro_b200/flac.py) against the oracle (oracle/flac_oracle.py) byte for
byte -- signals, lengths, rates, a Mimi decode, a 19.2 M-sample row, ragged batches, the stream -- and through the public
API (synthesize_batch, stream)."""
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import flac_oracle as F
from oracle import mimi_oracle as MO
from sopro_b200 import wire

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
RATES = tuple(F.RATE_CODES) + (11025, 4000)
LENGTHS = (0, 1, 15, 16, 4095, 4096, 4097, 12 * 4096 + 17)
_CACHE = {}


def _mimi_wav():
    """A real Mimi decode (synthetic checkpoint, seeded codes): 41 frames = 78,720 samples at its own level."""
    if "mimi" not in _CACHE:
        from sopro_b200.codec import MimiEngine

        codes = torch.randint(0, 2048, (1, 32, 41), generator=torch.Generator().manual_seed(7))
        eng = MimiEngine(MO.synth_mimi_state_dict(), 0, 32)
        _CACHE["mimi"] = eng.decode(codes).reshape(-1).float().cuda()
    return _CACHE["mimi"]


def signal(kind, N, sr=24000, seed=0):
    """fp32 numpy [N]."""
    g = np.random.default_rng(1000 * seed + N % 997)
    t = np.arange(N, dtype=np.float64) / sr
    if kind == "silence":
        return np.zeros(N, dtype=np.float32)
    if kind == "noise":
        return g.uniform(-1, 1, N).astype(np.float32)
    if kind == "clipped":  # past full scale, with +-inf and NaN sprinkled in
        x = 1.7 * np.sin(2 * np.pi * 300 * t)
        x[::97] = np.inf
        x[5::101] = -np.inf
        x[7::89] = np.nan
        return x.astype(np.float32)
    if kind == "sine":
        return (0.5 * np.sin(2 * np.pi * 440 * t)).astype(np.float32)
    if kind == "chirp":
        return (0.6 * np.sin(2 * np.pi * (50 * t + 0.45 * sr * t * t / max(2 * N / sr, 1e-9)))).astype(np.float32)
    if kind == "speech":  # harmonics of a gliding 110-180 Hz pitch with a syllable-rate envelope and a little breath
        f0 = 145 + 35 * np.sin(2 * np.pi * 1.3 * t)
        ph = 2 * np.pi * np.cumsum(f0) / sr
        x = sum(0.25 / k * np.sin(k * ph) for k in range(1, 12)) * (0.55 + 0.45 * np.sin(2 * np.pi * 4 * t))
        return (x + 0.003 * g.standard_normal(N)).astype(np.float32)
    if kind == "mimi":
        w = _mimi_wav().cpu().numpy()
        return np.resize(w, N).astype(np.float32)
    raise ValueError(kind)


def gpu(x, sr, **kw):
    from sopro_b200.flac import encode_flac

    return encode_flac(torch.from_numpy(np.ascontiguousarray(x)).cuda(), sr, **kw)


@pytest.mark.parametrize("kind", ("silence", "noise", "clipped", "sine", "chirp", "speech", "mimi"))
@pytest.mark.parametrize("N", LENGTHS)
def test_bytes_equal_the_oracle(kind, N):
    x = signal(kind, N)
    want = F.encode(x, 24000)
    got = gpu(x, 24000)
    assert got == want
    _, s, _ = F.decode(got)
    assert np.array_equal(s, F.to_pcm16(x).astype(np.int16))


@pytest.mark.parametrize("sr", RATES)
def test_every_rate_code(sr):
    x = signal("speech", 5000, sr)
    assert gpu(x, sr) == F.encode(x, sr)


def test_a_19_2M_sample_row():
    """4688 frames (two- and three-byte frame numbers) over a palette of 8 distinct blocks in a scrambled order; the
    oracle memoises each distinct block's subframe."""
    N = 19_200_000
    pal = [signal(k, 4096, seed=i) for i, k in enumerate(("speech", "noise", "sine", "chirp", "silence", "mimi",
                                                           "clipped", "speech"))]
    order = np.random.default_rng(3).integers(0, len(pal), (N + 4095) // 4096)
    x = np.concatenate([pal[i] for i in order])[:N]
    memo = {}

    def sub(s):
        key = s.tobytes()
        if key not in memo:
            memo[key] = F.encode_subframe(s)
        return memo[key]

    assert gpu(x, 24000) == F.encode(x, 24000, subframe=sub)


def test_ragged_rows_equal_single_rows():
    from sopro_b200.flac import encode_flac

    kinds = ("speech", "noise", "silence", "mimi", "chirp", "sine")
    lens = [4097, 0, 1, 12 * 4096 + 17, 4096, 15]
    L = max(lens) + 33
    rows = [signal(k, L, seed=i) for i, k in enumerate(kinds)]
    alone = [gpu(r[:n], 24000) for r, n in zip(rows, lens)]
    X = torch.from_numpy(np.stack(rows)).cuda()
    X[:, max(lens):] = float("nan")  # past every row's length: never read
    assert encode_flac(X, 24000, lens=lens) == alone
    perm = [3, 0, 5, 1, 4, 2]
    assert encode_flac(X[perm].contiguous(), 24000, lens=[lens[i] for i in perm]) == [alone[i] for i in perm]
    assert encode_flac([X[i: i + 1, : lens[i]].reshape(1, 1, -1) for i in range(6)], 24000) == alone
    # more rows than one launch holds
    many = [X[i % 6, : lens[i % 6]] for i in range(131)]
    assert encode_flac(many, 24000) == [alone[i % 6] for i in range(131)]


def test_stream_frames_equal_the_oracle():
    from sopro_b200.flac import FlacStreamEncoder

    x = signal("speech", 3 * 4096 + 700)
    s = F.to_pcm16(x)
    enc = FlacStreamEncoder(24000)
    assert enc.header() == F.stream_header(24000)
    cuts = [0, 5000, 5003, 5010, 5030, 9000, 9000, 13000, len(x)]  # 3-, 7- and 20-sample pushes, an empty one
    got = []
    for a, b in zip(cuts, cuts[1:]):
        got.append(enc.push(torch.from_numpy(x[a:b]).cuda()))
        assert 0 <= enc.carried <= 15
    got.append(enc.finish())
    # rebuild the expected frames from the same cut rule
    want, carry, num = [], 0, 0
    for a, b in zip(cuts, cuts[1:]):
        tot = carry + (b - a)
        keep = tot % 4096 if tot % 4096 < 16 else 0
        seg = s[num: num + tot - keep]
        want.append(b"".join(F.stream_frames(seg, num, 24000)))
        num += tot - keep
        carry = keep
    want.append(b"".join(F.stream_frames(s[num: num + carry], num, 24000)))
    assert got == want
    info, dec, frames = F.decode(F.stream_header(24000) + b"".join(got))
    assert np.array_equal(dec, s.astype(np.int16)) and all(f["variable"] for f in frames)


def test_short_pushes_are_carried():
    from sopro_b200.flac import FlacStreamEncoder

    x = signal("sine", 40)
    enc = FlacStreamEncoder(48000)
    assert enc.push(torch.from_numpy(x[:7]).cuda()) == b"" and enc.carried == 7
    assert enc.push(torch.from_numpy(x[7:15]).cuda()) == b"" and enc.carried == 15
    out = enc.push(torch.from_numpy(x[15:40]).cuda())
    assert enc.carried == 0 and out == F.encode_frame(F.to_pcm16(x), 0, True, 48000)
    assert enc.finish() == b""


def test_refusals_raise_before_any_launch():
    from sopro_b200 import _lib
    from sopro_b200.flac import FlacStreamEncoder, encode_flac

    x = torch.zeros(100, device="cuda")
    for sr in (3999, 192001, 24000.5, True):
        with pytest.raises(ValueError):
            encode_flac(x, sr)
        with pytest.raises(ValueError):
            FlacStreamEncoder(sr)
    with pytest.raises(ValueError):
        encode_flac(x.view(2, 50), 24000, lens=[10, 51])
    with pytest.raises(_lib.SoproError):
        encode_flac(torch.zeros(100), 24000)
    with pytest.raises(_lib.SoproError):
        FlacStreamEncoder(24000).push(torch.zeros(100))


# ---- through the public API (the e2e fixture of test_e2e_gpu.py)

def _api():
    from tests.cases import e2e_inputs
    from tests.test_e2e_gpu import TEXT, _tts

    tts, _ = _tts()
    _cfg, _sd, inp = e2e_inputs()
    return tts, tts.prepare_reference(ref_tokens_tq=inp["ref_tokens_tq"]), TEXT


def _pcm(w):
    return np.frombuffer(wire.float_to_pcm16le(w.reshape(1, -1)), dtype=np.int16)


@pytest.mark.parametrize("kw", (dict(), dict(sample_rate=48000), dict(speed=1.25), dict(loudness=-16.0)))
def test_synthesize_batch_round_trip(kw):
    from sopro_b200.flac import encode_flac

    tts, ref, text = _api()
    texts = [text, " ".join(str(i) for i in range(3, 40, 3)), "5 9"]
    wavs = tts.synthesize_batch(texts, ref=ref, max_frames=16, min_gen_frames=10 ** 9, seeds=[1, 2, 3], **kw)
    streams = encode_flac(wavs, kw.get("sample_rate", 24000))
    ratio = []
    for w, b in zip(wavs, streams):
        info, s, _ = F.decode(b)
        assert info["sample_rate"] == kw.get("sample_rate", 24000)
        assert np.array_equal(s, _pcm(w))
        assert b == F.encode(w.reshape(-1).cpu().numpy(), info["sample_rate"])
        ratio.append(len(b) / max(2 * w.numel(), 1))
    print(f"{kw}: compressed / PCM16 = {[round(r, 3) for r in ratio]} (synthetic checkpoint: random weights, not speech)")


def test_save_flac(tmp_path):
    tts, ref, text = _api()
    w = tts.synthesize(text, ref=ref, max_frames=12, seed=5, min_gen_frames=10 ** 9)
    p = tmp_path / "a.flac"
    tts.save_flac(str(p), w)
    _, s, _ = F.decode(p.read_bytes())
    assert np.array_equal(s, _pcm(w))


@pytest.mark.parametrize("chunk_frames", (64, 6))
def test_stream_equals_one_shot(chunk_frames):
    """One chunk covering the utterance (fp32 Mimi): the stream's audio is synthesize()'s, so the FLAC stream decodes to
    the one-shot encoding's PCM16.  Six-frame chunks: the NAR refiner sees chunk windows (test_e2e_gpu), so the reference
    is the one-shot encoding of the concatenated chunks."""
    from sopro_b200.flac import encode_flac, encode_stream_flac

    tts, ref, text = _api()
    kw = dict(ref=ref, max_frames=25, seed=9, min_gen_frames=10 ** 9)
    tts.codec.engine.set_precision("fp32")
    try:
        one = tts.synthesize(text, **kw)
        chunks = list(tts.stream(text, chunk_frames=chunk_frames, **kw))
    finally:
        tts.codec.engine.set_precision("bf16_tc")
    whole = one if chunk_frames == 64 else torch.cat(chunks, dim=-1)
    if chunk_frames == 64:
        assert len(chunks) == 1
    data = b"".join(encode_stream_flac(iter(chunks), 24000))
    info, s, frames = F.decode(data)
    _, s1, _ = F.decode(encode_flac(whole, 24000))
    assert np.array_equal(s, s1) and np.array_equal(s, _pcm(whole))
    assert info["min_block"] == 16 and info["max_block"] == 4096 and info["total"] == 0
    # every frame is the oracle's encoding of its block
    pcm = _pcm(whole).astype(np.int64)
    for f in frames:
        blk = pcm[f["number"]: f["number"] + f["n"]]
        assert data[f["offset"]: f["offset"] + f["bytes"]] == F.encode_frame(blk, f["number"], True, 24000)


def test_an_installed_decoder_agrees(tmp_path):
    """Optional: a libFLAC-based decoder, if one is installed, reads the GPU's bytes back to the same PCM16."""
    x = signal("speech", 30000)
    data = gpu(x, 24000)
    want = F.to_pcm16(x).astype(np.int16)
    try:
        import soundfile as sf  # noqa: F401
    except ImportError:
        sf = None
    if sf is not None:
        p = tmp_path / "a.flac"
        p.write_bytes(data)
        got, sr = sf.read(str(p), dtype="int16")
        assert sr == 24000 and np.array_equal(got, want)
        return
    if shutil.which("flac"):
        r = subprocess.run(["flac", "-d", "-c", "--force-raw-format", "--endian=little", "--sign=signed", "-"], input=data,
                           capture_output=True, check=True)
        assert np.array_equal(np.frombuffer(r.stdout, dtype="<i2"), want)
        return
    pytest.skip("no soundfile module or flac binary here")
