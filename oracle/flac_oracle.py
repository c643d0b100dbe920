"""Integer restatement of the FLAC stage (faster_qwen3_tts/flac.py, csrc/fq3_flac.cu) and a FLAC decoder written from
RFC 9639: test infrastructure only, the product never imports it.

``Stream(rate)`` is the encoder: each ``push(samples, flush)`` returns the bytes that push releases, making every
decision the module docstring of ``faster_qwen3_tts/flac.py`` fixes (blocking, subframe type, predictor order, partition
order, Rice parameters, ties).  ``encode(x, rate)`` is one push with flush.  ``decode(data)`` parses a whole stream --
every subframe type (CONSTANT, VERBATIM, FIXED, LPC), both Rice methods and escaped partitions, wasted bits -- checks
the CRC-8 of every frame header and the CRC-16 of every frame, and returns (samples int16, rate, frames).
"""
import numpy as np

RATES = (8000, 16000, 22050, 24000, 32000, 44100, 48000)
RATE_CODES = {88200: 1, 176400: 2, 192000: 3, 8000: 4, 16000: 5, 22050: 6, 24000: 7, 32000: 8, 44100: 9, 48000: 10,
              96000: 11}
BLOCK = 4096        # the largest block
GRAIN = 16          # blocks before the flush are multiples of this
MAX_ORDER = 4
MAX_PARTITION_ORDER = 8
MAX_K = 30
HEAD_BYTES = 42     # "fLaC" + STREAMINFO


def crc8(data, crc=0):
    for b in bytes(data):
        crc ^= b
        for _ in range(8):
            crc = ((crc << 1) ^ 0x07) & 0xFF if crc & 0x80 else (crc << 1) & 0xFF
    return crc


def _crc16_table():
    t = []
    for i in range(256):
        c = i << 8
        for _ in range(8):
            c = ((c << 1) ^ 0x8005) & 0xFFFF if c & 0x8000 else (c << 1) & 0xFFFF
        t.append(c)
    return t


_T16 = _crc16_table()


def crc16(data, crc=0):
    for b in bytes(data):
        crc = ((crc << 8) & 0xFFFF) ^ _T16[(crc >> 8) ^ b]
    return crc


class BitWriter:
    def __init__(self):
        self.out, self.acc, self.n = bytearray(), 0, 0

    def put(self, value, bits):
        self.acc = (self.acc << bits) | (int(value) & ((1 << bits) - 1))
        self.n += bits
        if self.n >= 64:
            keep = self.n % 8
            self.out += (self.acc >> keep).to_bytes((self.n - keep) // 8, "big")
            self.acc &= (1 << keep) - 1
            self.n = keep

    def bytes(self):
        pad = -self.n % 8
        return bytes(self.out) + (self.acc << pad).to_bytes((self.n + pad) // 8, "big")


def stream_header(rate, total=0):
    """'fLaC' and one STREAMINFO block (the last metadata block): block sizes 16 .. 4096, frame sizes unknown, mono,
    16 bits, ``total`` samples (0: unknown), MD5 unset"""
    w = BitWriter()
    for v, b in ((GRAIN, 16), (BLOCK, 16), (0, 24), (0, 24), (rate, 20), (0, 3), (15, 5), (total, 36)):
        w.put(v, b)
    return b"fLaC" + bytes([0x80, 0, 0, 34]) + w.bytes() + bytes(16)


def coded_number(v):
    """the UTF-8-like coding of a frame's first sample index (up to 36 bits)"""
    if v < 0x80:
        return bytes([v])
    for nb, lim in ((2, 1 << 11), (3, 1 << 16), (4, 1 << 21), (5, 1 << 26), (6, 1 << 31), (7, 1 << 36)):
        if v < lim:
            break
    out = []
    for _ in range(nb - 1):
        out.append(0x80 | (v & 0x3F))
        v >>= 6
    lead = 0xFE if nb == 7 else ((0xFF << (8 - nb)) & 0xFF) | v
    return bytes([lead] + out[::-1])


def frame_header(n, first, rate):
    """variable blocking: the header codes the index of the block's first sample"""
    bs = 12 if n == BLOCK else 6 if n <= 256 else 7
    h = bytes([0xFF, 0xF9, (bs << 4) | RATE_CODES[rate], 0x08]) + coded_number(first)
    if bs == 6:
        h += bytes([n - 1])
    elif bs == 7:
        h += (n - 1).to_bytes(2, "big")
    return h + bytes([crc8(h)])


def fixed_residual(x, order):
    """residuals x[order:] of the FIXED predictor of that order (int64)"""
    r = x.astype(np.int64)
    for _ in range(order):
        r = r[1:] - r[:-1]
    return r


def zigzag(r):
    return np.where(r >= 0, 2 * r, -2 * r - 1)


def partition_orders(n, order):
    """the partition orders allowed for a block of n samples and a predictor of that order: n divisible by 2^p and more
    than ``order`` samples in each partition"""
    return [p for p in range(MAX_PARTITION_ORDER + 1) if n % (1 << p) == 0 and (n >> p) > order]


def rice_sums(u, n, order):
    """S[k, j] = sum of (u >> k) over the residuals of the finest partition j (n >> pmax samples, pmax the largest
    partition order n allows), k = 0 .. 30"""
    pmax = max(partition_orders(n, 0))
    full = np.concatenate([np.zeros(order, np.int64), u])
    return (full[None, :] >> np.arange(MAX_K + 1)[:, None]).reshape(MAX_K + 1, 1 << pmax, -1).sum(-1)


def best_rice(S, n, order, p):
    """(bits of the residual section, method, parameters) for partition order p: per partition the lowest k with the
    fewest bits sum((u >> k) + 1 + k)"""
    sums = S.reshape(MAX_K + 1, 1 << p, -1).sum(-1)
    cnt = np.full(1 << p, n >> p, np.int64)
    cnt[0] -= order
    costs = sums + cnt[None, :] * (np.arange(MAX_K + 1)[:, None] + 1)
    ks = costs.argmin(0)
    method = 1 if ks.max() > 14 else 0
    return 2 + 4 + (4 + method) * len(ks) + int(costs.min(0).sum()), method, [int(k) for k in ks]


def choose(x):
    """the subframe of a block: ('constant',), ('verbatim',) or ('fixed', order, p, method, ks), and its bits"""
    n = len(x)
    if (x == x[0]).all():
        return ("constant",), 8 + 16
    verbatim = 8 + 16 * n
    best, best_bits = None, None
    for order in range(min(MAX_ORDER, n - 1) + 1):
        S = rice_sums(zigzag(fixed_residual(x, order)), n, order)
        for p in partition_orders(n, order):
            bits, method, ks = best_rice(S, n, order, p)
            bits += 8 + 16 * order
            if best_bits is None or bits < best_bits:
                best, best_bits = ("fixed", order, p, method, ks), bits
    if best is None or best_bits >= verbatim:
        return ("verbatim",), verbatim
    return best, best_bits


def encode_frame(x, first, rate):
    x = np.asarray(x, dtype=np.int64)
    n = len(x)
    head = frame_header(n, first, rate)
    sub, _ = choose(x)
    w = BitWriter()
    if sub[0] == "constant":
        w.put(0x00, 8)
        w.put(x[0], 16)
    elif sub[0] == "verbatim":
        w.put(0x02, 8)
        for v in x:
            w.put(v, 16)
    else:
        _, order, p, method, ks = sub
        w.put((0x08 | order) << 1, 8)
        for v in x[:order]:
            w.put(v, 16)
        w.put(method, 2)
        w.put(p, 4)
        u = zigzag(fixed_residual(x, order))
        size = n >> p
        for j, k in enumerate(ks):
            w.put(k, 4 + method)
            a = j * size - (order if j else 0)
            for v in u[a:a + size - (order if j == 0 else 0)]:
                v = int(v)
                w.put(1, (v >> k) + 1)
                w.put(v & ((1 << k) - 1), k)
    body = head + w.bytes()
    return body + crc16(body).to_bytes(2, "big")


class Stream:
    """one stream pushed in pieces: a push of m samples after c carried ones encodes 16 * floor((c + m) / 16) of them
    (all at flush) as blocks of 4096 and one block of the remainder, and carries the rest"""

    def __init__(self, rate):
        assert rate in RATES
        self.rate, self.carry, self.index, self.started, self.flushed = rate, np.zeros(0, np.int64), 0, False, False

    def push(self, x, flush=False):
        assert not self.flushed
        seq = np.concatenate([self.carry, np.asarray(x, dtype=np.int64)])
        take = len(seq) if flush else len(seq) // GRAIN * GRAIN
        out = b""
        if not self.started:
            out += stream_header(self.rate, len(seq) + self.index if flush else 0)
            self.started = True
        for a in range(0, take, BLOCK):
            blk = seq[a:min(a + BLOCK, take)]
            out += encode_frame(blk, self.index, self.rate)
            self.index += len(blk)
        self.carry = seq[take:]
        self.flushed = flush
        return out


def encode(x, rate):
    return Stream(rate).push(x, True)


def max_bytes(carried, n, flush):
    """a bound on the bytes one push releases: the stream header, and per block 16 header bytes, the subframe header,
    two bytes a sample and the CRC-16"""
    ready = carried + n
    take = ready if flush else ready // GRAIN * GRAIN
    full, rest = divmod(take, BLOCK)
    return HEAD_BYTES + full * (2 * BLOCK + 19) + (2 * rest + 19 if rest else 0)


# ---- decoder (RFC 9639) --------------------------------------------------------------------------------------------
class _Bits:
    def __init__(self, data, pos=0):
        self.b, self.p = bytes(data) + bytes(16), pos * 8

    def read(self, k):
        if k == 0:
            return 0
        i = self.p >> 3
        w = int.from_bytes(self.b[i:i + 8], "big")
        s = 64 - (self.p & 7) - k
        if s >= 0:
            v = (w >> s) & ((1 << k) - 1)
        else:
            v = ((w << -s) | (self.b[i + 8] >> (8 + s))) & ((1 << k) - 1)
        self.p += k
        return v

    def sread(self, k):
        v = self.read(k)
        return v - (1 << k) if k and v >> (k - 1) else v

    def unary(self):
        q = 0
        while True:
            i = self.p >> 3
            w = int.from_bytes(self.b[i:i + 8], "big") & ((1 << (64 - (self.p & 7))) - 1)
            if w:
                z = 64 - (self.p & 7) - w.bit_length()
                self.p += z + 1
                return q + z
            q += 64 - (self.p & 7)
            self.p += 64 - (self.p & 7)

    def align(self):
        self.p = (self.p + 7) // 8 * 8


def _utf8(bits):
    b = bits.read(8)
    if b < 0x80:
        return b
    nb = 7 if b == 0xFE else 8 - (~b & 0xFF).bit_length()
    assert 2 <= nb <= 7, "bad coded number"
    v = b & (0x3F >> (nb - 1)) if nb < 7 else 0
    for _ in range(nb - 1):
        c = bits.read(8)
        assert c >> 6 == 2, "bad coded number"
        v = (v << 6) | (c & 0x3F)
    return v


def _residual(bits, n, order):
    method, p = bits.read(2), bits.read(4)
    assert method in (0, 1), "reserved residual coding method"
    width, esc = (4, 15) if method == 0 else (5, 31)
    out = []
    size = n >> p
    assert size << p == n and size >= order, "bad partition order"
    for j in range(1 << p):
        cnt = size - (order if j == 0 else 0)
        k = bits.read(width)
        if k == esc:
            w = bits.read(5)
            out.extend(bits.sread(w) for _ in range(cnt))
        else:
            for _ in range(cnt):
                u = (bits.unary() << k) | bits.read(k)
                out.append((u >> 1) ^ -(u & 1))
    return out


_FIXED = {0: [], 1: [1], 2: [2, -1], 3: [3, -3, 1], 4: [4, -6, 4, -1]}


def _subframe(bits, n, bps):
    assert bits.read(1) == 0, "subframe padding bit set"
    t = bits.read(6)
    wasted = 0
    if bits.read(1):
        wasted = bits.unary() + 1
    bps -= wasted
    if t == 0:
        x = [bits.sread(bps)] * n
    elif t == 1:
        x = [bits.sread(bps) for _ in range(n)]
    elif 8 <= t <= 12 or t >= 32:
        if t < 32:
            order, coefs, shift = t - 8, _FIXED[t - 8], 0
        else:
            order = t - 31
        x = [bits.sread(bps) for _ in range(order)]
        if t >= 32:
            prec = bits.read(4) + 1
            assert prec != 16, "reserved LPC precision"
            shift = bits.sread(5)
            coefs = [bits.sread(prec) for _ in range(order)]
        res = _residual(bits, n, order)
        for r in res:
            acc = sum(c * x[-1 - i] for i, c in enumerate(coefs))
            x.append((acc >> shift) + r)
    else:
        raise AssertionError(f"reserved subframe type {t}")
    return [v << wasted for v in x]


def decode(data):
    """-> (int16 samples, rate, [(first sample, block size, byte offset, byte length)]) of a whole mono 16-bit stream,
    every CRC checked"""
    data = bytes(data)
    assert data[:4] == b"fLaC", "not a FLAC stream"
    pos, last, rate = 4, False, None
    while not last:
        last, typ, size = data[pos] >> 7, data[pos] & 0x7F, int.from_bytes(data[pos + 1:pos + 4], "big")
        if typ == 0:
            si = _Bits(data, pos + 4)
            si.read(16), si.read(16), si.read(24), si.read(24)
            rate, ch, bps, total = si.read(20), si.read(3) + 1, si.read(5) + 1, si.read(36)
            assert ch == 1 and bps == 16, "only mono 16-bit streams"
        pos += 4 + size
    out, frames = [], []
    while pos < len(data):
        bits = _Bits(data, pos)
        assert bits.read(15) == 0x7FFC, "lost frame sync"
        variable = bits.read(1)
        bs, rc, chan, ss = bits.read(4), bits.read(4), bits.read(4), bits.read(3)
        assert bits.read(1) == 0 and chan == 0 and ss in (0, 4), "unsupported frame"
        num = _utf8(bits)
        if bs == 6:
            n = bits.read(8) + 1
        elif bs == 7:
            n = bits.read(16) + 1
        elif bs == 1:
            n = 192
        elif 2 <= bs <= 5:
            n = 576 << (bs - 2)
        else:
            assert bs >= 8, "reserved block size"
            n = 256 << (bs - 8)
        if rc == 12:
            frate = bits.read(8) * 1000
        elif rc in (13, 14):
            frate = bits.read(16) * (10 if rc == 14 else 1)
        else:
            frate = {v: k for k, v in RATE_CODES.items()}.get(rc, rate)
        hlen = (bits.p >> 3) - pos
        assert crc8(data[pos:pos + hlen]) == bits.read(8), "frame header CRC-8 mismatch"
        assert frate == rate, "frame rate differs from STREAMINFO"
        first = num if variable else num * n
        out.extend(_subframe(bits, n, 16))
        bits.align()
        end = bits.p >> 3
        assert crc16(data[pos:end]) == int.from_bytes(data[end:end + 2], "big"), "frame CRC-16 mismatch"
        frames.append((first, n, pos, end + 2 - pos))
        pos = end + 2
    return np.asarray(out, dtype=np.int64).astype(np.int16), rate, frames
