"""Float64 restatement of the resampler at a pitch (faster_qwen3_tts/resample.py, csrc/fq3_resample.cu): the output rate
R and the pitch rho together, written from the definition and not from the kernel.  At rho 256 it is
``oracle/resample_oracle.py`` exactly (a CPU test checks it); the encodings are that module's.

(L, M) = (256 R, 24000 rho) / gcd, half = 32 max(L, M) (L == M: the one-tap filter), h = firwin(2 half + 1, 0.9 / m,
Kaiser 8.6) at unit DC gain, y[n] = L sum_j h[j] x[(n M + half - j) / L].  ``tempo_q`` / ``rho_of`` / ``gain_of`` are
the request's mapping.
"""
import math

import numpy as np

from oracle.resample_oracle import BETA, CUTOFF, HALF_PER_M, IN_RATE, encode  # noqa: F401

PITCH_ONE = 256


def rho_of(pitch):
    return round(PITCH_ONE * 2.0 ** (pitch / 12.0))


def tempo_q(speed, pitch):
    return round(speed * 2 ** 18 / rho_of(pitch))


def gain_of(gain_db):
    return np.float32(10.0 ** (gain_db / 20.0))


def ratio(rate, rho):
    g = math.gcd(rate * PITCH_ONE, IN_RATE * rho)
    L, M = rate * PITCH_ONE // g, IN_RATE * rho // g
    return (1, 1, 0) if L == M else (L, M, HALF_PER_M * max(L, M))


def design(rate, rho):
    L, M, half = ratio(rate, rho)
    if half == 0:
        return np.ones(1)
    fc = CUTOFF / max(L, M)
    t = np.arange(-half, half + 1, dtype=np.float64)
    w = np.i0(BETA * np.sqrt(1.0 - (t / half) ** 2)) / np.i0(BETA)
    h = fc * np.sinc(fc * t) * w
    return h / h.sum()


def out_len(n_in, rate, rho):
    L, M, _ = ratio(rate, rho)
    return -(-n_in * L // M)


def outputs(x, rate, rho, n_lo, n_hi, h=None):
    """y[n_lo, n_hi) of the closed form, x zero outside [0, len(x)), in blocks of outputs to bound the memory"""
    L, M, half = ratio(rate, rho)
    h = design(rate, rho) if h is None else h
    x = np.asarray(x, dtype=np.float64)
    K = 2 * half // L + 1
    out = np.zeros(max(n_hi - n_lo, 0))
    step = max(1, 4_000_000 // K)
    for a in range(n_lo, n_hi, step):
        b = min(n_hi, a + step)
        t = np.arange(a, b, dtype=np.int64)[:, None] * M + half
        j = t % L + L * np.arange(K, dtype=np.int64)[None, :]
        i = (t - j) // L
        ok = (j <= 2 * half) & (j <= t) & (i < len(x))
        terms = np.where(ok, h[np.minimum(j, 2 * half)] * x[np.clip(i, 0, max(len(x) - 1, 0))] if len(x) else 0.0, 0.0)
        out[a - n_lo:b - n_lo] = L * terms.sum(axis=1)
    return out


def resample(x, rate, rho):
    """the whole stream, flushed: ceil(N L / M) samples"""
    return outputs(x, rate, rho, 0, out_len(len(x), rate, rho))


def magnitude(x, rate, rho):
    """sum_j |L h[j] x[i]| of every output: the scale of an fp32 accumulation bound"""
    return outputs(np.abs(np.asarray(x, dtype=np.float64)), rate, rho, 0, out_len(len(x), rate, rho),
                   np.abs(design(rate, rho)))


class Stream:
    """a stream pushed in pieces: each push returns the outputs whose newest input exists (all of them at flush)"""

    def __init__(self, rate, rho):
        self.rate, self.rho, self.x, self.done = rate, rho, np.zeros(0), 0

    def push(self, x, final=False):
        self.x = np.concatenate([self.x, np.asarray(x, dtype=np.float64)])
        L, M, half = ratio(self.rate, self.rho)
        if final:
            hi = out_len(len(self.x), self.rate, self.rho)
        else:
            hi = self.done
            while (hi * M + half) // L < len(self.x):
                hi += 1
        y = outputs(self.x, self.rate, self.rho, self.done, hi)
        self.done = hi
        return y
