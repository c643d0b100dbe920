"""Float64 restatement of the output-rate and encoding stage (faster_qwen3_tts/resample.py, csrc/fq3_resample.cu),
written from the definition and not from the kernel: test infrastructure only, the product never imports it.

``design(rate)`` is the filter, ``resample(x, rate)`` the closed form over a whole (flushed) stream, ``Stream(rate)`` the
same stream pushed in pieces: each push computes, from the input it has seen so far only, the outputs whose newest input
exists (checked output by output, not by the closed form of ``resample.emitted``).  ``lin2ulaw`` / ``lin2alaw`` are
ITU-T G.711 of 16-bit samples, ``to_s16`` the fp32 rule of ``serving.to_pcm16``.
"""
import math

import numpy as np

IN_RATE = 24000
RATES = (8000, 16000, 22050, 24000, 32000, 44100, 48000)
HALF_PER_M = 32
CUTOFF = 0.9
BETA = 8.6


def ratio(rate):
    """(L, M, half); 24000 is the encode-only identity filter"""
    if rate == IN_RATE:
        return 1, 1, 0
    g = math.gcd(rate, IN_RATE)
    L, M = rate // g, IN_RATE // g
    return L, M, HALF_PER_M * max(L, M)


def design(rate):
    """h: a Kaiser-windowed sinc of 2 half + 1 taps, cutoff 0.9 / m of the up-sampled Nyquist, unit DC gain"""
    L, M, half = ratio(rate)
    if half == 0:
        return np.ones(1)
    m = max(L, M)
    fc = CUTOFF / m
    t = np.arange(-half, half + 1, dtype=np.float64)
    w = np.i0(BETA * np.sqrt(1.0 - (t / half) ** 2)) / np.i0(BETA)
    h = fc * np.sinc(fc * t) * w
    return h / h.sum()


def _outputs(x, rate, n_lo, n_hi, h=None):
    """y[n_lo, n_hi) of the closed form, x zero outside [0, len(x)): output n sums h[j] x[(t - j) / L], t = n M + half,
    over the j = p, p + L, ... (p = t mod L) with 0 <= t - j and j <= 2 half"""
    L, M, half = ratio(rate)
    h = design(rate) if h is None else h
    x = np.asarray(x, dtype=np.float64)
    t = np.arange(n_lo, n_hi, dtype=np.int64)[:, None] * M + half
    j = t % L + L * np.arange(2 * half // L + 1, dtype=np.int64)[None, :]
    i = (t - j) // L
    ok = (j <= 2 * half) & (j <= t) & (i < len(x))
    terms = np.where(ok, h[np.minimum(j, 2 * half)] * x[np.clip(i, 0, max(len(x) - 1, 0))] if len(x) else 0.0, 0.0)
    return L * terms.sum(axis=1)


def out_len(n_in, rate):
    L, M, _ = ratio(rate)
    return -(-n_in * L // M)


def resample(x, rate):
    """the whole stream, flushed: ceil(N L / M) samples"""
    return _outputs(x, rate, 0, out_len(len(x), rate))


def magnitude(x, rate):
    """sum_j |L h[j] x[i]| of every output of the flushed stream: the scale of an fp32 accumulation bound"""
    return _outputs(np.abs(np.asarray(x, dtype=np.float64)), rate, 0, out_len(len(x), rate), np.abs(design(rate)))


def reads(n, rate):
    """the input indices output n reads (before clipping to the stream), newest first"""
    L, M, half = ratio(rate)
    t = n * M + half
    return [(t - j) // L for j in range(t % L, min(2 * half, t) + 1, L)]


class Stream:
    """a stream pushed in pieces: ``push(x, final)`` returns the outputs that push releases"""

    def __init__(self, rate):
        self.rate, self.x, self.done = rate, np.zeros(0), 0

    def push(self, x, final=False):
        self.x = np.concatenate([self.x, np.asarray(x, dtype=np.float64)])
        if final:
            hi = out_len(len(self.x), self.rate)
        else:
            hi = self.done
            L, M, half = ratio(self.rate)
            while (hi * M + half) // L < len(self.x):   # its newest input exists
                hi += 1
        y = _outputs(self.x, self.rate, self.done, hi)
        self.done = hi
        return y


def to_s16(y):
    """serving.to_pcm16's rule: clip(x * 32768, -32768, 32767) in fp32, truncated toward zero"""
    return np.clip(np.asarray(y, dtype=np.float32) * np.float32(32768), -32768, 32767).astype(np.int16)


def _segment(v, ends):
    seg = np.zeros(v.shape, dtype=np.int64)
    for e in ends:
        seg += v > e
    return seg


def lin2ulaw(s16):
    """G.711 mu-law: 14-bit magnitude, clipped to 8159, biased by 33, 8 segments of 16 steps, all bits inverted"""
    v = np.asarray(s16, dtype=np.int64) >> 2
    mask = np.where(v < 0, 0x7F, 0xFF)
    v = np.minimum(np.abs(v), 8159) + 33
    seg = _segment(v, [0x3F, 0x7F, 0xFF, 0x1FF, 0x3FF, 0x7FF, 0xFFF, 0x1FFF])
    code = np.where(seg >= 8, 0x7F, (np.minimum(seg, 7) << 4) | ((v >> (np.minimum(seg, 7) + 1)) & 0xF))
    return (code ^ mask).astype(np.uint8)


def lin2alaw(s16):
    """G.711 A-law: 13-bit magnitude (one's complement below zero), 8 segments of 16 steps, even bits inverted"""
    v = np.asarray(s16, dtype=np.int64) >> 3
    mask = np.where(v >= 0, 0xD5, 0x55)
    v = np.where(v >= 0, v, -v - 1)
    seg = _segment(v, [0x1F, 0x3F, 0x7F, 0xFF, 0x1FF, 0x3FF, 0x7FF, 0xFFF])
    q = np.where(seg < 2, v >> 1, v >> np.minimum(seg, 7)) & 0xF
    code = np.where(seg >= 8, 0x7F, (np.minimum(seg, 7) << 4) | q)
    return (code ^ mask).astype(np.uint8)


def encode(y, encoding):
    """float output -> the encoded array (f32 rounds the float64 value to float32)"""
    if encoding == "f32":
        return np.asarray(y, dtype=np.float32)
    s = to_s16(y)
    return {"s16": s, "ulaw": lin2ulaw(s), "alaw": lin2alaw(s)}[encoding]
