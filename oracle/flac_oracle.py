"""FLAC (RFC 9639) encoder and strict decoder for mono 16-bit streams, in numpy: the oracle of ``ev_flac_encode`` /
``format_audio(encoding="flac")``.  Restated from the RFC's text; shares no code with ``emotivoice_b200``.

Stream (RFC 9639 section 6): ``fLaC``, one STREAMINFO block with the last-metadata flag set (section 8.1: block sizes 4096 and
4096, the real minimum and maximum frame sizes, the rate, one channel, 16 bits, the total sample count, an all-zero MD5 meaning
"unknown"), then one frame per 4096 samples, the last one shorter.

Frame (section 9.1): sync code 0xFFF8 (fixed block size), block size code 1100 for 4096, else 0110 (8-bit n - 1) for n <= 256 or
0111 (16-bit n - 1); the sample rate code of ``rate_code``; channels 0000; sample size 100; the frame number UTF-8 coded;
CRC-8 (poly 0x07, init 0) of the header, then one subframe, zero padding to a byte and CRC-16 (poly 0x8005, init 0) of the
frame.

Subframe (section 9.2): the candidate with the fewest bits, ties to the first of CONSTANT, FIXED 0-4, LPC 1-12, VERBATIM; the
wasted-bits flag is 0.  Residuals (section 9.2.7) use coding method 00 (4-bit Rice parameters, no escape).  Each partition
takes the k in 0..14 with the fewest bits m (k + 1) + sum(u >> k), u the zig-zag folded residual, ties to the smaller k; the
partition order is the one in 0..8 with the fewest bits, ties to the smaller order, among the orders o with n % 2^o == 0 and
(n >> o) > predictor order.  A FIXED or LPC order must be below the block's sample count.

LPC analysis, every rounding fixed:
- Welch window in integers: y[i] = trunc(x[i] ((n + 1)^2 - (2i - n + 1)^2) / (n + 1)^2), int64.
- Autocorrelation of y at lags 0..min(12, n - 1), exact in int64.
- Levinson-Durbin in float64 with every product, sum and quotient rounded on its own (no fused multiply-add):
      err = r[0]; for i = 1..P: acc = r[i] - a[1] r[i-1] - ... - a[i-1] r[1] (left to right); k = acc / err;
      a'[j] = a[j] - k a[i-j] (j < i), a'[i] = k; err = err (1 - k k).
  Order i is a candidate while err > 0 after it; the first order whose err is <= 0 (or NaN) ends the recursion, and with
  r[0] == 0 there is no LPC candidate at all.
- Precision of order p: min(15, 16 - ceil(log2 p)), so that every prediction sum stays inside int32.
- shift = clamp(prec - 1 - e, 0, 15), e the exponent of frexp(max |a|); q = clamp(rint(a 2^shift), -2^(prec-1), 2^(prec-1) - 1).
- Prediction (sum_j q[j] x[t-1-j]) >> shift (arithmetic); a candidate whose residual leaves int32 is skipped.
"""
import math
import operator

import numpy as np

BLOCK = 4096
MAX_LPC = 12
MAX_FIXED = 4
MAX_PORDER = 8
MAX_RICE = 14
CONSTANT, VERBATIM, FIXED, LPC = "CONSTANT", "VERBATIM", "FIXED", "LPC"

# RFC 9639 section 9.1.2: the rates with a code of their own
STANDARD_RATES = {88200: 1, 176400: 2, 192000: 3, 8000: 4, 16000: 5, 22050: 6, 24000: 7, 32000: 8, 44100: 9, 48000: 10, 96000: 11}


def rate_code(rate):
    """Frame-header sample rate field -> (code, value of the trailing field, its bits)."""
    if rate in STANDARD_RATES:
        return STANDARD_RATES[rate], 0, 0
    if rate % 1000 == 0 and rate // 1000 <= 255:
        return 12, rate // 1000, 8
    if rate <= 65535:
        return 13, rate, 16
    if rate % 10 == 0:
        return 14, rate // 10, 16
    return 0, 0, 0


def _crc_table(poly, width):
    top, mask = 1 << (width - 1), (1 << width) - 1
    t = []
    for b in range(256):
        c = b << (width - 8)
        for _ in range(8):
            c = ((c << 1) ^ poly) if c & top else (c << 1)
        t.append(c & mask)
    return t


_CRC8 = _crc_table(0x07, 8)
_CRC16 = _crc_table(0x8005, 16)


def crc8(data):
    """RFC 9639 section 9.1.8: CRC-8, polynomial x^8 + x^2 + x + 1, initial value 0."""
    c = 0
    for b in bytes(data):
        c = _CRC8[c ^ b]
    return c


def crc16(data):
    """RFC 9639 section 9.3: CRC-16, polynomial x^16 + x^15 + x^2 + 1, initial value 0."""
    c = 0
    for b in bytes(data):
        c = ((c << 8) & 0xFFFF) ^ _CRC16[(c >> 8) ^ b]
    return c


def _bits(v, n):
    """v as n bits, most significant first (two's complement for negative v)."""
    return ((int(v) >> np.arange(n - 1, -1, -1)) & 1).astype(np.uint8)


def utf8_number(v):
    """RFC 9639 section 9.1.5: the frame number in the extended UTF-8 coding (up to 36 bits)."""
    if v < 0x80:
        return bytes([v])
    for nb, lead in ((2, 0xC0), (3, 0xE0), (4, 0xF0), (5, 0xF8), (6, 0xFC), (7, 0xFE)):
        if v < (1 << (5 * nb + 1)) or nb == 7:
            break
    out = [lead | (v >> (6 * (nb - 1)))]
    out += [0x80 | ((v >> (6 * i)) & 0x3F) for i in range(nb - 2, -1, -1)]
    return bytes(out)


def frame_header(index, n, rate):
    """Frame header bytes including its CRC-8 (RFC 9639 section 9.1)."""
    if n == BLOCK:
        bcode, bext = 12, b""
    elif n <= 256:
        bcode, bext = 6, bytes([n - 1])
    else:
        bcode, bext = 7, (n - 1).to_bytes(2, "big")
    rcode, rval, rbits = rate_code(rate)
    h = bytes([0xFF, 0xF8, (bcode << 4) | rcode, 0x08]) + utf8_number(index) + bext + (rval.to_bytes(rbits // 8, "big") if rbits else b"")
    return h + bytes([crc8(h)])


# ---- analysis --------------------------------------------------------------------------------------------------------

def zigzag(r):
    return np.where(r >= 0, 2 * r, -2 * r - 1)


def rice(r, order, n):
    """Fewest residual bits of a predictor of ``order`` on an n-sample block, residuals r (n - order,) int64 ->
    (bits incl. the 2-bit method and 4-bit order, partition order, Rice parameters)."""
    u = np.concatenate([np.zeros(order, np.int64), zigzag(r)])
    of = max(o for o in range(MAX_PORDER + 1) if n % (1 << o) == 0 and (n >> o) > order)
    ks = np.arange(MAX_RICE + 1, dtype=np.int64)
    S = (u[None, :] >> ks[:, None]).reshape(MAX_RICE + 1, 1 << of, n >> of).sum(-1)
    best = None
    for o in range(of, -1, -1):
        m = np.full(1 << o, n >> o, np.int64)
        m[0] -= order
        cost = m[None, :] * (ks[:, None] + 1) + S
        k = np.argmin(cost, axis=0)
        bits = int(4 * (1 << o) + cost[k, np.arange(1 << o)].sum())
        if best is None or bits <= best[0]:
            best = (bits, o, k)
        if o:
            S = S.reshape(MAX_RICE + 1, 1 << (o - 1), 2).sum(-1)
    return 6 + best[0], best[1], best[2]


def fixed_residual(x, p):
    """RFC 9639 section 9.2.5: the fixed predictors of orders 0..4."""
    c = {0: [], 1: [1], 2: [2, -1], 3: [3, -3, 1], 4: [4, -6, 4, -1]}[p]
    n = len(x)
    pred = np.zeros(n - p, np.int64)
    for j, cj in enumerate(c):
        pred += cj * x[p - 1 - j:n - 1 - j]
    return x[p:] - pred


def precision(p):
    return min(15, 16 - (p - 1).bit_length())


def lpc_orders(x):
    """Welch-windowed autocorrelation and Levinson-Durbin -> [(order, q (int64), shift, precision)] of the candidate orders."""
    n = len(x)
    P = min(MAX_LPC, n - 1)
    if P < 1:
        return []
    i = np.arange(n, dtype=np.int64)
    d = np.int64(n + 1) ** 2
    num = x * (d - (2 * i - n + 1) ** 2)
    y = np.sign(num) * (np.abs(num) // d)
    r = [int(np.dot(y[l:], y[:n - l])) for l in range(P + 1)]
    if r[0] == 0:
        return []
    out = []
    a = [0.0] * (P + 1)
    err = float(r[0])
    for i in range(1, P + 1):
        acc = float(r[i])
        for j in range(1, i):
            acc = acc - a[j] * float(r[i - j])
        k = acc / err
        new = list(a)
        new[i] = k
        for j in range(1, i):
            new[j] = a[j] - k * a[i - j]
        a = new
        err = err * (1.0 - k * k)
        if not err > 0.0:
            break
        prec = precision(i)
        c = np.array(a[1:i + 1], np.float64)
        e = math.frexp(float(np.abs(c).max()))[1]
        shift = min(max(prec - 1 - e, 0), 15)
        q = np.clip(np.rint(c * (2.0 ** shift)), -(1 << (prec - 1)), (1 << (prec - 1)) - 1).astype(np.int64)
        out.append((i, q, shift, prec))
    return out


def lpc_residual(x, q, shift):
    p, n = len(q), len(x)
    s = np.zeros(n - p, np.int64)
    for j in range(p):
        s += q[j] * x[p - 1 - j:n - 1 - j]
    return x[p:] - (s >> shift)


def choose(x):
    """The subframe of one block: (kind, order, bits, detail).  detail: for FIXED / LPC (residual, porder, params[, q, shift,
    prec])."""
    n = len(x)
    cands = []
    if np.all(x == x[0]):
        cands.append((CONSTANT, 0, 24, None))
    for p in range(min(MAX_FIXED, n - 1) + 1):
        r = fixed_residual(x, p)
        bits, o, k = rice(r, p, n)
        cands.append((FIXED, p, 8 + 16 * p + bits, (r, o, k)))
    for p, q, shift, prec in lpc_orders(x):
        r = lpc_residual(x, q, shift)
        if r.min() < -2 ** 31 or r.max() > 2 ** 31 - 1:
            continue
        bits, o, k = rice(r, p, n)
        cands.append((LPC, p, 8 + 16 * p + 9 + p * prec + bits, (r, o, k, q, shift, prec)))
    cands.append((VERBATIM, 0, 8 + 16 * n, None))
    return min(cands, key=lambda c: c[2])       # min keeps the first of equal costs


def _residual_bits(r, order, n, porder, params):
    """Coding method 00, partition order, then each partition's 4-bit parameter and Rice codes, as a bit array."""
    u = zigzag(r)
    psize = n >> porder
    out = [_bits(0, 2), _bits(porder, 4)]
    start = 0
    for j in range(1 << porder):
        m = psize - (order if j == 0 else 0)
        k = int(params[j])
        uj = u[start:start + m]
        start += m
        q = uj >> k
        lens = q + 1 + k
        pos = np.concatenate([[0], np.cumsum(lens)[:-1]])
        b = np.zeros(int(lens.sum()), np.uint8)
        b[pos + q] = 1
        for t in range(k):
            b[pos + q + 1 + t] = (uj >> (k - 1 - t)) & 1
        out += [_bits(k, 4), b]
    return out


def encode_frame(x, index, rate):
    n = len(x)
    kind, order, bits, det = choose(x)
    hdr = frame_header(index, n, rate)
    parts = []
    if kind == CONSTANT:
        parts = [_bits(0, 8), _bits(x[0], 16)]
    elif kind == VERBATIM:
        parts = [_bits(1 << 1, 8)] + [_bits(v, 16) for v in x]
    elif kind == FIXED:
        r, o, k = det
        parts = [_bits((8 | order) << 1, 8)] + [_bits(v, 16) for v in x[:order]] + _residual_bits(r, order, n, o, k)
    else:
        r, o, k, q, shift, prec = det
        parts = ([_bits((32 | (order - 1)) << 1, 8)] + [_bits(v, 16) for v in x[:order]] + [_bits(prec - 1, 4), _bits(shift, 5)]
                 + [_bits(v, prec) for v in q] + _residual_bits(r, order, n, o, k))
    b = np.concatenate(parts)
    assert len(b) == bits, (kind, order, len(b), bits)
    body = hdr + np.packbits(np.concatenate([b, np.zeros(-len(b) % 8, np.uint8)])).tobytes()
    return body + crc16(body).to_bytes(2, "big"), kind, order


def streaminfo(rate, total, fmin, fmax):
    """RFC 9639 sections 8.1 / 8.2: metadata block header (last flag, type 0, length 34) and STREAMINFO."""
    b = np.concatenate([_bits(BLOCK, 16), _bits(BLOCK, 16), _bits(fmin, 24), _bits(fmax, 24), _bits(rate, 20), _bits(0, 3),
                        _bits(15, 5), _bits(total, 36), np.zeros(128, np.uint8)])
    return bytes([0x80, 0, 0, 34]) + np.packbits(b).tobytes()


def encode(pcm16, rate):
    """int16 samples of one item at ``rate`` Hz -> the .flac file image (bytes)."""
    x = np.asarray(pcm16)
    if x.ndim != 1 or x.dtype != np.int16 or len(x) == 0:
        raise ValueError("expected a non-empty 1-D int16 array")
    if not 1 <= rate < 1 << 20:
        raise ValueError("rate %r does not fit STREAMINFO" % (rate,))
    x = x.astype(np.int64)
    frames = [encode_frame(x[s:s + BLOCK], i, rate)[0] for i, s in enumerate(range(0, len(x), BLOCK))]
    sizes = [len(f) for f in frames]
    return b"fLaC" + streaminfo(rate, len(x), min(sizes), max(sizes)) + b"".join(frames)


# ---- strict decoder ----------------------------------------------------------------------------------------------------

class FlacError(ValueError):
    pass


class _Reader:
    def __init__(self, data):
        self.s = np.unpackbits(np.frombuffer(data, np.uint8)).tobytes().translate(bytes.maketrans(b"\0\1", b"01")).decode()
        self.p = 0

    def u(self, n):
        if self.p + n > len(self.s):
            raise FlacError("truncated stream")
        v = int(self.s[self.p:self.p + n], 2) if n else 0
        self.p += n
        return v

    def s_(self, n):
        v = self.u(n)
        return v - (1 << n) if v >> (n - 1) else v

    def unary(self):
        z = self.s.find("1", self.p)
        if z < 0:
            raise FlacError("truncated Rice code")
        q = z - self.p
        self.p = z + 1
        return q


def _utf8(rd):
    b0 = rd.u(8)
    if b0 < 0x80:
        return b0
    nb = 0
    while nb < 8 and b0 & (0x80 >> nb):
        nb += 1
    if nb < 2 or nb > 7:
        raise FlacError("invalid coded number")
    v = b0 & (0x7F >> nb)
    for _ in range(nb - 1):
        c = rd.u(8)
        if c & 0xC0 != 0x80:
            raise FlacError("invalid coded number continuation")
        v = (v << 6) | (c & 0x3F)
    return v


def _decode_residual(rd, n, order):
    if rd.u(2) != 0:
        raise FlacError("residual coding method other than 00")
    o = rd.u(4)
    if n % (1 << o) or (n >> o) <= order:
        raise FlacError("partition order %d not allowed for %d samples at predictor order %d" % (o, n, order))
    out = []
    for j in range(1 << o):
        k = rd.u(4)
        if k == 15:
            raise FlacError("escaped partition")
        for _ in range((n >> o) - (order if j == 0 else 0)):
            q = rd.unary()
            u = (q << k) | rd.u(k)
            out.append((u >> 1) ^ -(u & 1))
    return np.array(out, np.int64), o


def decode(data):
    """.flac image -> (rate, int16 samples, per-frame stats [{"type", "order", "porder", "bytes", "samples"}]).  Raises
    FlacError on anything outside the stream format above: sync, reserved bits, CRCs, STREAMINFO fields, partition rules."""
    data = bytes(data)
    if data[:4] != b"fLaC":
        raise FlacError("no fLaC marker")
    if len(data) < 42 or data[4] != 0x80 or data[5:8] != b"\0\0\x22":
        raise FlacError("expected one STREAMINFO block of 34 bytes flagged last")
    rd = _Reader(data)
    rd.p = 8 * 8
    bmin, bmax, fmin, fmax, rate, ch, bps, total = rd.u(16), rd.u(16), rd.u(24), rd.u(24), rd.u(20), rd.u(3), rd.u(5), rd.u(36)
    md5 = rd.u(128)
    if (bmin, bmax, ch, bps, md5) != (BLOCK, BLOCK, 0, 15, 0):
        raise FlacError("STREAMINFO block sizes / channels / bits / MD5 differ from this stream format")
    pos, samples, stats = 42, [], []
    while pos < len(data):
        rd.p = 8 * pos
        if rd.u(14) != 0x3FFE or rd.u(1) != 0 or rd.u(1) != 0:
            raise FlacError("frame %d: bad sync code or reserved / blocking bits" % len(stats))
        bcode, rcode, chan, ss, res = rd.u(4), rd.u(4), rd.u(4), rd.u(3), rd.u(1)
        if chan != 0 or ss != 4 or res != 0:
            raise FlacError("frame %d: channels / sample size / reserved bit" % len(stats))
        if _utf8(rd) != len(stats):
            raise FlacError("frame %d: frame number" % len(stats))
        if bcode == 12:
            n = BLOCK
        elif bcode == 6:
            n = rd.u(8) + 1
        elif bcode == 7:
            n = rd.u(16) + 1
        else:
            raise FlacError("frame %d: block size code %d not produced by this format" % (len(stats), bcode))
        want = rate_code(rate)
        if rcode != want[0] or (want[2] and rd.u(want[2]) != want[1]):
            raise FlacError("frame %d: sample rate code does not match STREAMINFO" % len(stats))
        hlen = rd.p // 8 - pos
        if rd.u(8) != crc8(data[pos:pos + hlen]):
            raise FlacError("frame %d: header CRC-8" % len(stats))
        if rd.u(1) != 0:
            raise FlacError("frame %d: subframe padding bit" % len(stats))
        t = rd.u(6)
        if rd.u(1) != 0:
            raise FlacError("frame %d: wasted bits" % len(stats))
        porder = None
        if t == 0:
            kind, order, x = CONSTANT, 0, np.full(n, rd.s_(16), np.int64)
        elif t == 1:
            kind, order, x = VERBATIM, 0, np.array([rd.s_(16) for _ in range(n)], np.int64)
        elif 8 <= t <= 12 or t >= 32:
            kind, order = (FIXED, t - 8) if t < 32 else (LPC, t - 31)
            if order >= n:
                raise FlacError("frame %d: predictor order %d for %d samples" % (len(stats), order, n))
            warm = [rd.s_(16) for _ in range(order)]
            if kind == LPC:
                prec = rd.u(4) + 1
                if prec == 16:
                    raise FlacError("frame %d: invalid coefficient precision" % len(stats))
                shift = rd.s_(5)
                if shift < 0:
                    raise FlacError("frame %d: negative shift" % len(stats))
                q = [rd.s_(prec) for _ in range(order)]
            r, porder = _decode_residual(rd, n, order)
            c = {0: [], 1: [1], 2: [2, -1], 3: [3, -3, 1], 4: [4, -6, 4, -1]}[order] if kind == FIXED else q
            sh = shift if kind == LPC else 0
            cr = [int(v) for v in c[::-1]]            # aligned with the last `order` samples, oldest first
            x = list(warm)
            for e in r.tolist():
                v = e + (sum(map(operator.mul, cr, x[len(x) - order:])) >> sh) if order else e
                if not -32768 <= v <= 32767:
                    raise FlacError("frame %d: sample outside 16 bits" % len(stats))
                x.append(v)
            x = np.array(x, np.int64)
        else:
            raise FlacError("frame %d: reserved subframe type %d" % (len(stats), t))
        pad = (-rd.p) % 8
        if rd.u(pad) != 0:
            raise FlacError("frame %d: nonzero padding" % len(stats))
        end = rd.p // 8
        if rd.u(16) != crc16(data[pos:end]):
            raise FlacError("frame %d: CRC-16" % len(stats))
        if x.min() < -32768 or x.max() > 32767:
            raise FlacError("frame %d: sample outside 16 bits" % len(stats))
        samples.append(x)
        stats.append({"type": kind, "order": order, "porder": porder, "bytes": end + 2 - pos, "samples": n})
        pos = end + 2
    if not stats:
        raise FlacError("no frames")
    sizes = [s["bytes"] for s in stats]
    if any(s["samples"] != BLOCK for s in stats[:-1]) or stats[-1]["samples"] > BLOCK:
        raise FlacError("block sizes differ from a fixed 4096")
    x = np.concatenate(samples)
    if total != len(x) or (fmin, fmax) != (min(sizes), max(sizes)):
        raise FlacError("STREAMINFO total samples / frame sizes differ from the frames")
    return rate, x.astype(np.int16), stats
