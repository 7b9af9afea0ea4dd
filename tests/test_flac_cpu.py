"""CPU: the FLAC oracle (oracle/flac_oracle.py) -- CRC check values, the UTF-8 number coding, known-answer frames built
field by field here, round trips through the strict decoder over signals, lengths and rates, and the decoder's
rejection of damaged streams."""
import numpy as np
import pytest

from oracle import flac_oracle as F
from tests.test_flac_gpu import signal

LENGTHS = (0, 1, 15, 16, 4095, 4096, 4097, 12 * 4096 + 17)


def bits(v, w):
    return format(v & ((1 << w) - 1), f"0{w}b")


def to_bytes(b):
    b += "0" * (-len(b) % 8)
    return bytes(int(b[i: i + 8], 2) for i in range(0, len(b), 8))


def exact(v):
    """fp32 samples that quantise to the integers v: (v +- 0.5) / 32767 truncates back to v."""
    v = np.asarray(v, dtype=np.float64)
    return ((v + 0.5 * np.sign(v)) / 32767.0).astype(np.float32)


def one_frame_stream(n, sub_bits, sr=24000):
    """A one-shot stream of a single fixed-blocking frame 0 of n samples (n <= 256), built field by field."""
    head = bytes([0xFF, 0xF8, (0b0110 << 4) | F.RATE_CODES[sr], 0b0000_100_0, 0x00, n - 1])
    head += bytes([F.crc8(head)])
    body = head + to_bytes(sub_bits)
    fr = body + F.crc16(body).to_bytes(2, "big")
    info = (b"fLaC" + bytes([0x80, 0, 0, 34]) + (4096).to_bytes(2, "big") * 2 + len(fr).to_bytes(3, "big") * 2
            + ((sr << 44) | (15 << 36) | n).to_bytes(8, "big") + bytes(16))
    return info + fr


def test_crc_check_values():
    assert F.crc8(b"123456789") == 0xF4
    assert F.crc16(b"123456789") == 0xFEE8


@pytest.mark.parametrize("v,want", ((127, "7f"), (128, "c280"), (2047, "dfbf"), (2048, "e0a080"), (65535, "efbfbf"),
                                    (65536, "f0908080"), (2 ** 31 - 1, "fdbfbfbfbfbf"), (2 ** 36 - 1, "febfbfbfbfbfbf")))
def test_utf8_numbers(v, want):
    assert F.utf8_number(v).hex() == want


def test_c_round_and_the_input_rule():
    assert [F.c_round(v) for v in (0.5, 1.5, 2.5, -0.5, -1.5, 0.49999999999999994, -2.4)] == [1, 2, 3, -1, -2, 0, -2]
    x = np.array([0.0, 1.0, -1.0, 2.0, -np.inf, np.inf, np.nan, 0.5, -0.5, 1e-5], dtype=np.float32)
    assert F.to_pcm16(x).tolist() == [0, 32767, -32767, 32767, -32767, 32767, 0, 16383, -16383, 0]


def test_known_answer_constant_block():
    x = exact([5] * 20)
    sub = "0" + "000000" + "0" + bits(5, 16)
    want = one_frame_stream(20, sub)
    assert F.encode(x, 24000) == want
    info, s, frames = F.decode(want)
    assert s.tolist() == [5] * 20 and frames[0]["type"] == 0 and info["total"] == 20


def test_known_answer_one_sample_block():
    # CONSTANT costs 8 + 16 = 24 bits; FIXED 0 costs 8 + 2 + 4 + 4 + 1 = 19 (u = 0, k = 0: a lone "1")
    sub = "0" + "001000" + "0" + "00" + "0000" + "0000" + "1"
    want = one_frame_stream(1, sub)
    assert F.encode(np.zeros(1, dtype=np.float32), 24000) == want
    assert F.decode(want)[1].tolist() == [0]


def test_known_answer_fixed_order2_ramp():
    # s = 1000 + 3 i + (i odd): second differences alternate -2 (i even, u = 3) and +2 (i odd, u = 4), 7 of each.
    # Rice cost over the 14 residuals: k = 0: 14 + 49 = 63; k = 1: 28 + 21 = 49; k = 2: 42 + 7 = 49; k = 3: 56.
    # The tie goes to k = 1; codes "0" "1" "1" (u = 3) and "00" "1" "0" (u = 4); one partition (two cost 4 bits more).
    s = [1000 + 3 * i + (i % 2) for i in range(16)]
    res = [s[i] - 2 * s[i - 1] + s[i - 2] for i in range(2, 16)]
    assert res == [-2, 2] * 7
    codes = "".join("011" if e < 0 else "0010" for e in res)
    sub = "0" + "001010" + "0" + bits(s[0], 16) + bits(s[1], 16) + "00" + "0000" + bits(1, 4) + codes
    assert len(sub) == 99
    want = one_frame_stream(16, sub)
    assert F.encode(exact(s), 24000) == want
    assert F.decode(want)[1].tolist() == s


def test_known_answer_lpc_block():
    # a 16-sample-period sine, 48 samples: order-2 LPC wins with q = [1853, -982], shift 10 (precision 12)
    x = (np.float32(0.5) * np.sin(2 * np.pi * np.arange(48) / 16).astype(np.float32))
    s = F.to_pcm16(x).tolist()
    assert s[:5] == [0, 6269, 11584, 15136, 16383]
    q, shift = [1853, -982], 10
    res = [s[i] - ((q[0] * s[i - 1] + q[1] * s[i - 2]) >> shift) for i in range(2, 48)]
    assert res[:16] == [240, 186, 103, 5, -94, -177, -235, -257, -239, -185, -102, -4, 95, 178, 236, 258]
    assert res[16:32] == res[:16] and res[32:] == res[:14]
    k = 8  # |e| <= 258: u <= 516; per residual k + 1 + (u >> 8), cheapest at k = 8 (an unpartitioned block)
    codes = ""
    for e in res:
        u = 2 * e if e >= 0 else -2 * e - 1
        codes += "0" * (u >> k) + "1" + bits(u, k)
    sub = ("0" + "100001" + "0" + bits(s[0], 16) + bits(s[1], 16) + bits(11, 4) + bits(shift, 5) + bits(q[0], 12)
           + bits(q[1], 12) + "00" + "0000" + bits(k, 4) + codes)
    want = one_frame_stream(48, sub)
    assert F.encode(x, 24000) == want
    assert F.decode(want)[1].tolist() == s


def _round_trip(x, sr):
    data = F.encode(x, sr)
    info, s, frames = F.decode(data)
    assert np.array_equal(s, F.to_pcm16(x).astype(np.int16))
    assert info["sample_rate"] == sr and info["total"] == len(x)
    assert all(f["n"] == 4096 for f in frames[:-1])
    return data


@pytest.mark.parametrize("kind", ("silence", "clipped", "noise", "sine", "chirp", "speech"))
@pytest.mark.parametrize("N", LENGTHS)
def test_round_trip(kind, N):
    _round_trip(signal(kind, N), 24000)


@pytest.mark.parametrize("sr", tuple(F.RATE_CODES) + (11025,))
def test_round_trip_every_rate(sr):
    data = _round_trip(signal("speech", 5000, sr), sr)
    assert data[42 + 2] & 0x0F == F.RATE_CODES.get(sr, 0)


def test_compression_of_speech_like_signals():
    x = signal("speech", 10 * 24000)
    ratio = len(F.encode(x, 24000)) / (2 * len(x))
    print(f"speech-like test signal: FLAC / PCM16 = {ratio:.3f}")
    assert ratio < 0.7, ratio  # its breath noise is about 100 LSB rms, so about 7 bits a sample stay incompressible


def test_stream_frames_decode():
    s = F.to_pcm16(signal("speech", 9000))
    data = F.stream_header(24000) + b"".join(F.stream_frames(s[:5000], 0, 24000) + F.stream_frames(s[5000:], 5000, 24000))
    info, got, frames = F.decode(data)
    assert np.array_equal(got, s.astype(np.int16))
    assert [f["number"] for f in frames] == [0, 4096, 5000] and all(f["variable"] for f in frames)
    assert (info["min_block"], info["max_block"], info["min_frame"], info["max_frame"], info["total"]) == (16, 4096, 0, 0, 0)


def _damaged(data, byte, bit):
    b = bytearray(data)
    b[byte] ^= 1 << bit
    return bytes(b)


def test_decoder_rejects_damage():
    data = F.encode(signal("speech", 6000), 24000)
    _, _, frames = F.decode(data)
    f = frames[1]
    for where in (f["offset"] + 1, f["offset"] + 3, f["offset"] + 4):  # blocking bit, reserved bit, frame number
        for bit in (0, 1):
            with pytest.raises(F.FlacError):
                F.decode(_damaged(data, where, bit))
    mid = f["offset"] + f["bytes"] // 2  # inside the subframe
    for bit in range(8):
        with pytest.raises(F.FlacError):
            F.decode(_damaged(data, mid, bit))
    end = f["offset"] + f["bytes"] - 1  # the CRC-16 itself
    with pytest.raises(F.FlacError):
        F.decode(_damaged(data, end, 0))
    with pytest.raises(F.FlacError):  # STREAMINFO's total
        F.decode(_damaged(data, 8 + 17, 0))
    with pytest.raises(F.FlacError):  # a dropped frame breaks the numbering
        F.decode(data[: f["offset"]] + data[f["offset"] + f["bytes"]:])


def test_decoder_checks_lpc_fields():
    x = (np.float32(0.5) * np.sin(2 * np.pi * np.arange(48) / 16).astype(np.float32))
    s = F.to_pcm16(x).tolist()
    for pc, shift in ((0b1111, 10), (11, -3)):
        sub = ("0" + "100001" + "0" + bits(s[0], 16) + bits(s[1], 16) + bits(pc, 4) + bits(shift, 5) + "0" * 24
               + "00" + "0000" + bits(0, 4) + "1" * 46)
        with pytest.raises(F.FlacError):
            F.decode(one_frame_stream(48, sub))
    # a partition order the block does not allow: 48 = 16 * 3, order 5 needs 48 % 32 = 0
    sub = "0" + "001000" + "0" + "00" + bits(5, 4) + "0000" * 32 + "1" * 48
    with pytest.raises(F.FlacError):
        F.decode(one_frame_stream(48, sub))
