"""FLAC (RFC 9639) oracle for sopro_b200/csrc/flac.cu: an encoder that follows the contract of include/sopro_b200.h
literally, in numpy and Python integers and Python float scalars (no GPU), and a strict decoder written separately from
it.

Encoder: mono, 16 bits, fp32 -> trunc(clamp(x, -1, 1) * 32767.0f) (NaN -> 0); subframe candidates CONSTANT, FIXED 0-4,
LPC 1-12 (Levinson-Durbin in double, one rounding per operation; precision 12, error-feedback quantisation), VERBATIM,
each sized exactly, the smallest winning with ties to the earlier; partitioned Rice with exact per-partition parameters.

Decoder: checks the sync, every reserved bit, both CRCs, the UTF-8 frame / sample numbers and their continuity, the
STREAMINFO fields against the frames, the LPC shift and precision, and the partition constraints.  It is the only
independent reading of the format on machines without libFLAC."""
from __future__ import annotations

import math
from typing import Callable, Dict, List, Optional, Tuple

import numpy as np

BLOCK = 4096
PRECISION = 12
MAX_LPC = 12
MAX_FIXED = 4
STREAM_MIN_BLOCK = 16
RATE_CODES = {8000: 0b0100, 16000: 0b0101, 22050: 0b0110, 24000: 0b0111, 32000: 0b1000, 44100: 0b1001, 48000: 0b1010,
              96000: 0b1011, 88200: 0b0001, 176400: 0b0010, 192000: 0b0011}
FIXED_COEFS = {0: [], 1: [1], 2: [2, -1], 3: [3, -3, 1], 4: [4, -6, 4, -1]}


# ---------------------------------------------------------------------------------------------- shared primitives

def crc8(data: bytes) -> int:
    """CRC-8, polynomial x^8 + x^2 + x + 1 (0x07), init 0, MSB first, no final xor."""
    c = 0
    for b in data:
        c ^= b
        for _ in range(8):
            c = ((c << 1) ^ 0x07) & 0xFF if c & 0x80 else (c << 1) & 0xFF
    return c


def crc16(data: bytes) -> int:
    """CRC-16, polynomial x^16 + x^15 + x^2 + 1 (0x8005), init 0, MSB first, no final xor."""
    c = 0
    for b in data:
        c ^= b << 8
        for _ in range(8):
            c = ((c << 1) ^ 0x8005) & 0xFFFF if c & 0x8000 else (c << 1) & 0xFFFF
    return c


def utf8_number(v: int) -> bytes:
    """FLAC's UTF-8-style coding of a frame or sample number, v < 2^36: 1 to 7 bytes."""
    if v < 0 or v >= 1 << 36:
        raise ValueError(f"frame/sample number {v} out of range")
    if v < 0x80:
        return bytes([v])
    for nb in range(2, 8):
        if v < 1 << (5 * nb + 1):  # nb bytes carry 6 (nb - 1) bits plus 7 - nb in the lead byte
            break
    out = []
    for _ in range(nb - 1):
        out.append(0x80 | (v & 0x3F))
        v >>= 6
    lead = (0xFF00 >> nb) & 0xFF
    return bytes([lead | v] + out[::-1])


def to_pcm16(x) -> np.ndarray:
    """wire.float_to_pcm16le's rule: clamp to [-1, 1], multiply by 32767 in fp32, truncate toward zero; NaN -> 0.
    -> int64 [N]."""
    x = np.asarray(x, dtype=np.float32).reshape(-1)
    x = np.where(np.isnan(x), np.float32(0.0), x)
    y = np.clip(x, np.float32(-1.0), np.float32(1.0)) * np.float32(32767.0)
    return np.trunc(y).astype(np.int64)


def c_round(v: float) -> int:
    """C's round(): halves away from zero (Python's round and np.round round halves to even)."""
    if v >= 0:
        f = math.floor(v)
        return int(f) + (1 if v - f >= 0.5 else 0)
    c = math.ceil(v)
    return int(c) - (1 if c - v >= 0.5 else 0)


class _Writer:
    def __init__(self):
        self.parts: List[str] = []

    def put(self, value: int, width: int) -> None:
        if width:
            self.parts.append(format(value & ((1 << width) - 1), f"0{width}b"))

    def bits(self) -> str:
        return "".join(self.parts)


def _bytes(bits: str) -> bytes:
    bits = bits + "0" * (-len(bits) % 8)
    return int(bits, 2).to_bytes(len(bits) // 8, "big") if bits else b""


# ---------------------------------------------------------------------------------------------- encoder

def autocorrelation(s: np.ndarray, lags: int = MAX_LPC) -> List[int]:
    n = len(s)
    return [int(np.dot(s[l:], s[: n - l])) if l < n else 0 for l in range(lags + 1)]


def levinson(R: List[int]) -> List[List[float]]:
    """Levinson-Durbin in double, one IEEE rounding per operation: -> a for orders 1 .. (at most 12), a[0] multiplying
    the most recent sample.  Stops before an order where err <= 0 or a value is not finite."""
    err = float(R[0])
    a: List[float] = []
    out = []
    for p in range(1, MAX_LPC + 1):
        if not (err > 0.0 and math.isfinite(err)):
            break
        acc = float(R[p])
        for j in range(p - 1):
            acc = acc - a[j] * float(R[p - 1 - j])
        k = acc / err
        new = [a[j] - k * a[p - 2 - j] for j in range(p - 1)] + [k]
        if not all(math.isfinite(v) for v in new):
            break
        a = new
        out.append(list(a))
        t = k * k
        t = 1.0 - t
        err = err * t
    return out


def quantize(a: List[float], precision: int = PRECISION) -> Optional[Tuple[List[int], int]]:
    """-> (q, shift), or None when the order is skipped (max|a| = 0 or a negative shift)."""
    cmax = max(abs(v) for v in a)
    if cmax == 0.0:
        return None
    e = math.frexp(cmax)[1]
    shift = min(precision - 1 - e, 15)
    if shift < 0:
        return None
    lim = 1 << (precision - 1)
    scale = float(1 << shift)
    err, q = 0.0, []
    for v in a:
        err = err + v * scale
        qi = max(-lim, min(lim - 1, c_round(err)))
        q.append(qi)
        err = err - float(qi)
    return q, shift


def fixed_residual(s: np.ndarray, p: int) -> np.ndarray:
    n = len(s)
    r = s[p:].copy()
    for j, c in enumerate(FIXED_COEFS[p]):
        r -= c * s[p - 1 - j: n - 1 - j]
    return r


def lpc_residual(s: np.ndarray, q: List[int], shift: int) -> np.ndarray:
    n, p = len(s), len(q)
    pred = np.zeros(n - p, dtype=np.int64)
    for j, c in enumerate(q):
        pred += c * s[p - 1 - j: n - 1 - j]
    return s[p:] - (pred >> shift)


def zigzag(r: np.ndarray) -> np.ndarray:
    return np.where(r >= 0, 2 * r, -2 * r - 1)


def rice_plan(r: np.ndarray, n: int, p: int) -> Tuple[int, int, int, List[int]]:
    """Exact partitioned-Rice choice for the n - p residuals of a block of n samples, predictor order p ->
    (bits of the whole residual section, method, partition order, parameter per partition)."""
    omax = 0
    while omax < 8 and n % (1 << (omax + 1)) == 0 and (n >> (omax + 1)) >= p:
        omax += 1
    full = np.zeros(n, dtype=np.int64)
    full[p:] = zigzag(r)
    parts = 1 << omax
    S = np.stack([(full >> k).reshape(parts, -1).sum(1) for k in range(31)])  # [31, parts]
    cnt = np.full(parts, n >> omax, dtype=np.int64)
    cnt[0] -= p
    ks = np.arange(31, dtype=np.int64)[:, None]
    plans = {}
    for o in range(omax, -1, -1):
        cost = cnt[None, :] * (ks + 1) + S  # [31, parts]
        best = []
        for method, kmax, pbits in ((0, 14, 4), (1, 30, 5)):
            c = cost[: kmax + 1]
            arg = c.argmin(0)  # the first minimum: ties go to the smaller k
            best.append((int(c.min(0).sum()) + pbits * (1 << o), method, [int(v) for v in arg]))
        plans[o] = best[0] if best[0][0] <= best[1][0] else best[1]
        if o:
            S = S[:, 0::2] + S[:, 1::2]
            cnt = cnt[0::2] + cnt[1::2]
    o_best = min(range(omax + 1), key=lambda o: (plans[o][0], o))
    bits, method, kp = plans[o_best]
    return 6 + bits, method, o_best, kp


def _put_residual(w: _Writer, r: np.ndarray, n: int, p: int, method: int, order: int, kp: List[int]) -> None:
    w.put(method, 2)
    w.put(order, 4)
    u = zigzag(r)
    psize = n >> order
    pos = 0
    for j, k in enumerate(kp):
        m = psize - (p if j == 0 else 0)
        w.put(k, 5 if method else 4)
        for v in u[pos: pos + m].tolist():
            w.parts.append("0" * (v >> k) + "1")
            w.put(v, k)
        pos += m


def encode_subframe(s: np.ndarray) -> str:
    """One block's subframe (no wasted bits) as a bit string: the smallest candidate, ties to the earlier."""
    s = np.asarray(s, dtype=np.int64)
    n = len(s)
    cands = []  # (bits, kind, payload) in candidate order
    if n and (s == s[0]).all():
        cands.append((8 + 16, "const", None))
    for p in range(MAX_FIXED + 1):
        if p <= n:
            r = fixed_residual(s, p)
            plan = rice_plan(r, n, p)
            cands.append((8 + 16 * p + plan[0], "fixed", (p, r, plan)))
    R = autocorrelation(s)
    if R[0] != 0:
        for a in levinson(R):
            p = len(a)
            qs = quantize(a)
            if p > n or qs is None:
                continue
            q, shift = qs
            r = lpc_residual(s, q, shift)
            plan = rice_plan(r, n, p)
            cands.append((8 + 16 * p + 4 + 5 + PRECISION * p + plan[0], "lpc", (q, shift, r, plan)))
    cands.append((8 + 16 * n, "verbatim", None))
    bits, kind, pay = min(enumerate(cands), key=lambda t: (t[1][0], t[0]))[1]
    w = _Writer()
    if kind == "const":
        w.put(0b0000000, 7)
        w.put(0, 1)
        w.put(int(s[0]), 16)
    elif kind == "verbatim":
        w.put(0b0000001, 7)
        w.put(0, 1)
        for v in s.tolist():
            w.put(v, 16)
    elif kind == "fixed":
        p, r, (_, method, order, kp) = pay
        w.put(0b0001000 | p, 7)
        w.put(0, 1)
        for v in s[:p].tolist():
            w.put(v, 16)
        _put_residual(w, r, n, p, method, order, kp)
    else:
        q, shift, r, (_, method, order, kp) = pay
        p = len(q)
        w.put(0b0100000 | (p - 1), 7)
        w.put(0, 1)
        for v in s[:p].tolist():
            w.put(v, 16)
        w.put(PRECISION - 1, 4)
        w.put(shift, 5)
        for c in q:
            w.put(c, PRECISION)
        _put_residual(w, r, n, p, method, order, kp)
    out = w.bits()
    assert len(out) == bits, (kind, len(out), bits)
    return out


def frame_header(n: int, number: int, variable: bool, sr: int) -> bytes:
    if n == BLOCK:
        bcode, extra = 0b1100, b""
    elif n <= 256:
        bcode, extra = 0b0110, bytes([n - 1])
    else:
        bcode, extra = 0b0111, (n - 1).to_bytes(2, "big")
    h = bytes([0xFF, 0xF9 if variable else 0xF8, (bcode << 4) | RATE_CODES.get(sr, 0), 0b0000_100_0])
    h += utf8_number(number) + extra
    return h + bytes([crc8(h)])


def frame(sub_bits: str, n: int, number: int, variable: bool, sr: int) -> bytes:
    """A frame around one subframe's bits: header, subframe, zero pad, CRC-16."""
    body = frame_header(n, number, variable, sr) + _bytes(sub_bits)
    return body + crc16(body).to_bytes(2, "big")


def encode_frame(s: np.ndarray, number: int, variable: bool, sr: int) -> bytes:
    return frame(encode_subframe(s), len(s), number, variable, sr)


def streaminfo(sr: int, min_block: int, max_block: int, min_frame: int, max_frame: int, total: int) -> bytes:
    """`fLaC`, one last-block metadata header (type 0, length 34) and STREAMINFO with a zero MD5."""
    v = (((sr << 3) | 0) << 5 | 15) << 36 | total
    body = (min_block.to_bytes(2, "big") + max_block.to_bytes(2, "big") + min_frame.to_bytes(3, "big")
            + max_frame.to_bytes(3, "big") + v.to_bytes(8, "big") + bytes(16))
    return b"fLaC" + bytes([0x80, 0, 0, 34]) + body


def stream_header(sr: int) -> bytes:
    """The streaming encoder's STREAMINFO: blocks of 16 .. 4096 samples, frame sizes and total unknown (0)."""
    return streaminfo(sr, STREAM_MIN_BLOCK, BLOCK, 0, 0, 0)


def encode(x, sr: int, subframe: Optional[Callable[[np.ndarray], str]] = None) -> bytes:
    """One-shot stream of one row of fp32 samples: fixed blocking, 4096-sample blocks (the last may be shorter), exact
    STREAMINFO.  `subframe` (a test hook) replaces encode_subframe, e.g. to memoise repeated blocks."""
    s = to_pcm16(x)
    sub = subframe or encode_subframe
    frames = [frame(sub(s[i: i + BLOCK]), len(s[i: i + BLOCK]), i // BLOCK, False, sr) for i in range(0, len(s), BLOCK)]
    sizes = [len(f) for f in frames]
    head = streaminfo(sr, BLOCK, BLOCK, min(sizes, default=0), max(sizes, default=0), len(s))
    return head + b"".join(frames)


def stream_frames(s: np.ndarray, first_sample: int, sr: int) -> List[bytes]:
    """The streaming encoder's frames for samples s (int) starting at sample number first_sample: variable blocking,
    4096-sample frames, then one remainder frame."""
    return [encode_frame(s[i: i + BLOCK], first_sample + i, True, sr) for i in range(0, len(s), BLOCK)]


# ---------------------------------------------------------------------------------------------- strict decoder

class FlacError(ValueError):
    pass


class _Reader:
    """MSB-first bit reader over a '0'/'1' string."""

    def __init__(self, data: bytes):
        self.bits = "".join(f"{b:08b}" for b in data)
        self.pos = 0

    def u(self, w: int) -> int:
        if w == 0:
            return 0
        if self.pos + w > len(self.bits):
            raise FlacError("unexpected end of stream")
        v = int(self.bits[self.pos: self.pos + w], 2)
        self.pos += w
        return v

    def s(self, w: int) -> int:
        v = self.u(w)
        return v - (1 << w) if w and v >> (w - 1) else v

    def unary(self) -> int:
        i = self.bits.find("1", self.pos)
        if i < 0:
            raise FlacError("unterminated unary code")
        q = i - self.pos
        self.pos = i + 1
        return q

    def byte_pos(self) -> int:
        return self.pos // 8


_DEC_RATES = {v: k for k, v in RATE_CODES.items()}


def _read_utf8(rd: _Reader) -> int:
    lead = rd.u(8)
    if lead < 0x80:
        return lead
    nb = 0
    while nb < 8 and lead & (0x80 >> nb):
        nb += 1
    if nb < 2 or nb > 7:
        raise FlacError(f"bad UTF-8 lead byte {lead:#x}")
    v = lead & (0x7F >> nb)
    for _ in range(nb - 1):
        c = rd.u(8)
        if c >> 6 != 0b10:
            raise FlacError(f"bad UTF-8 continuation byte {c:#x}")
        v = (v << 6) | (c & 0x3F)
    if v < (0x80 if nb == 2 else 1 << (5 * (nb - 1) + 1)):
        raise FlacError("overlong UTF-8 number")
    return v


def _decode_residual(rd: _Reader, n: int, p: int) -> List[int]:
    method = rd.u(2)
    if method > 1:
        raise FlacError(f"reserved residual coding method {method}")
    order = rd.u(4)
    if n % (1 << order) or (n >> order) < p:
        raise FlacError(f"partition order {order} does not fit a block of {n} with predictor order {p}")
    pbits, esc = (4, 15) if method == 0 else (5, 31)
    out: List[int] = []
    for j in range(1 << order):
        m = (n >> order) - (p if j == 0 else 0)
        k = rd.u(pbits)
        if k == esc:
            w = rd.u(5)
            out.extend(rd.s(w) for _ in range(m))
            continue
        for _ in range(m):
            u = (rd.unary() << k) | rd.u(k)
            out.append(u >> 1 if not u & 1 else -(u >> 1) - 1)
    return out


def _decode_subframe(rd: _Reader, n: int) -> List[int]:
    if rd.u(1):
        raise FlacError("subframe zero bit is set")
    t = rd.u(6)
    wasted = 0
    if rd.u(1):
        wasted = rd.unary() + 1
    bps = 16 - wasted
    if t == 0:
        s = [rd.s(bps)] * n
    elif t == 1:
        s = [rd.s(bps) for _ in range(n)]
    elif 8 <= t <= 12:
        p = t - 8
        if p > n:
            raise FlacError("FIXED order exceeds the block")
        s = [rd.s(bps) for _ in range(p)]
        res = _decode_residual(rd, n, p)
        c = FIXED_COEFS[p]
        for e in res:
            s.append(e + sum(c[j] * s[-1 - j] for j in range(p)))
    elif t >= 32:
        p = t - 31
        if p > n:
            raise FlacError("LPC order exceeds the block")
        s = [rd.s(bps) for _ in range(p)]
        pc = rd.u(4)
        if pc == 0b1111:
            raise FlacError("LPC precision code 1111 is invalid")
        shift = rd.s(5)
        if shift < 0:
            raise FlacError(f"negative LPC shift {shift}")
        q = [rd.s(pc + 1) for _ in range(p)]
        res = _decode_residual(rd, n, p)
        for e in res:
            s.append(e + (sum(q[j] * s[-1 - j] for j in range(p)) >> shift))
    else:
        raise FlacError(f"reserved subframe type {t}")
    s = [v << wasted for v in s]
    if any(v < -32768 or v > 32767 for v in s):
        raise FlacError("decoded sample outside 16 bits")
    return s


def decode(data: bytes) -> Tuple[Dict[str, int], np.ndarray, List[Dict[str, int]]]:
    """-> (STREAMINFO fields, int16 samples, one dict per frame: number, n, variable, offset, bytes, type).  Raises
    FlacError at the first violation."""
    data = bytes(data)
    if data[:4] != b"fLaC":
        raise FlacError("missing fLaC marker")
    pos, info = 4, None
    while True:
        if pos + 4 > len(data):
            raise FlacError("truncated metadata")
        last, typ, ln = data[pos] >> 7, data[pos] & 0x7F, int.from_bytes(data[pos + 1: pos + 4], "big")
        if info is None:
            if typ != 0 or ln != 34:
                raise FlacError("the first metadata block must be a 34-byte STREAMINFO")
            rd = _Reader(data[pos + 4: pos + 38])
            info = dict(min_block=rd.u(16), max_block=rd.u(16), min_frame=rd.u(24), max_frame=rd.u(24), sample_rate=rd.u(20),
                        channels=rd.u(3) + 1, bits=rd.u(5) + 1, total=rd.u(36))
            info["md5"] = rd.u(128)
        elif typ == 127:
            raise FlacError("invalid metadata block type 127")
        pos += 4 + ln
        if last:
            break
    if info["channels"] != 1 or info["bits"] != 16:
        raise FlacError("only mono 16-bit streams are read")
    if info["min_block"] < 16 or info["max_block"] < info["min_block"] or info["sample_rate"] == 0:
        raise FlacError("bad STREAMINFO block sizes or rate")
    samples: List[int] = []
    frames: List[Dict[str, int]] = []
    rd = _Reader(data)
    while pos < len(data):
        start = pos
        rd.pos = 8 * pos
        sync = rd.u(15)
        if sync != 0b111111111111100:
            raise FlacError(f"bad frame sync at byte {pos}")
        variable = rd.u(1)
        bcode, rcode = rd.u(4), rd.u(4)
        ch, ss, res = rd.u(4), rd.u(3), rd.u(1)
        if ch != 0:
            raise FlacError("not a mono frame")
        if ss not in (0b000, 0b100):
            raise FlacError(f"sample size code {ss:03b} is not 16 bits")
        if res:
            raise FlacError("frame header reserved bit is set")
        number = _read_utf8(rd)
        if bcode == 0:
            raise FlacError("reserved block size code 0000")
        n = (192 if bcode == 1 else 576 << (bcode - 2) if bcode <= 5 else rd.u(8) + 1 if bcode == 6
             else rd.u(16) + 1 if bcode == 7 else 256 << (bcode - 8))
        if rcode == 0b1111:
            raise FlacError("invalid sample rate code 1111")
        rate = (info["sample_rate"] if rcode == 0 else rd.u(8) * 1000 if rcode == 12 else rd.u(16) if rcode == 13
                else rd.u(16) * 10 if rcode == 14 else _DEC_RATES[rcode])
        if rate != info["sample_rate"]:
            raise FlacError(f"frame rate {rate} differs from STREAMINFO's {info['sample_rate']}")
        hlen = rd.byte_pos() - start
        if rd.u(8) != crc8(data[start: start + hlen]):
            raise FlacError(f"frame header CRC-8 mismatch at byte {start}")
        t = int(rd.bits[rd.pos + 1: rd.pos + 7], 2) if rd.pos + 7 <= len(rd.bits) else -1
        s = _decode_subframe(rd, n)
        if rd.pos % 8:
            if int(rd.bits[rd.pos: rd.pos + (8 - rd.pos % 8)], 2):
                raise FlacError("nonzero frame padding")
            rd.pos += 8 - rd.pos % 8
        end = rd.byte_pos()
        if rd.u(16) != crc16(data[start: end]):
            raise FlacError(f"frame CRC-16 mismatch at byte {start}")
        if frames and variable != frames[0]["variable"]:
            raise FlacError("blocking strategy changes mid-stream")
        want = len(samples) if variable else len(frames)
        if number != want:
            raise FlacError(f"frame number {number}, expected {want}")
        frames.append(dict(number=number, n=n, variable=variable, offset=start, bytes=end + 2 - start, type=t))
        samples.extend(s)
        pos = end + 2
    for i, f in enumerate(frames):
        lastf = i == len(frames) - 1
        if f["n"] > info["max_block"] or (not lastf and f["n"] < info["min_block"]):
            raise FlacError(f"frame {i} has {f['n']} samples, outside STREAMINFO's block sizes")
        if not f["variable"] and not lastf and f["n"] != info["max_block"]:
            raise FlacError("a fixed-blocking frame before the last is not the full block size")
        if info["min_frame"] and f["bytes"] < info["min_frame"] or info["max_frame"] and f["bytes"] > info["max_frame"]:
            raise FlacError(f"frame {i} is {f['bytes']} bytes, outside STREAMINFO's frame sizes")
    if info["total"] and info["total"] != len(samples):
        raise FlacError(f"STREAMINFO says {info['total']} samples, the frames hold {len(samples)}")
    if frames and info["min_frame"] and info["min_frame"] != min(f["bytes"] for f in frames):
        raise FlacError("STREAMINFO min frame size is not the smallest frame")
    if frames and info["max_frame"] and info["max_frame"] != max(f["bytes"] for f in frames):
        raise FlacError("STREAMINFO max frame size is not the largest frame")
    return info, np.asarray(samples, dtype=np.int16), frames
