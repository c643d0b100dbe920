"""Float64 restatement of the speaking-rate stage (WSOLA, faster_qwen3_tts/tempo.py, csrc/fq3_tempo.cu), written from
the definition and not from the kernel: test infrastructure only, the product never imports it.

``Wsola(speed)`` is a stream: ``push(x, final)`` returns the samples that push releases.  Frames run as soon as every
sample they can read exists (checked frame by frame, not by the closed form of ``tempo.ready_frames``); output is
released once no later frame can add to it.  ``forced`` replays given positions p_k instead of the argmax; every frame
records its candidates and their scores either way, so a caller can check a position chosen elsewhere against them.
"""
import numpy as np

N = 480          # window (20 ms at 24 kHz), periodic Hann
H = N // 2       # synthesis hop
D = 240          # search half-width
EPS = 1e-6
Q_ONE = 1024


def quantize(speed):
    q = round(float(speed) * 1024)
    if not 256 <= q <= 4096:
        raise ValueError(f"speed must be in [0.25, 4.0], got {speed!r}")
    return q


def hann():
    n = np.arange(N, dtype=np.float64)
    return 0.5 - 0.5 * np.cos(2 * np.pi * n / N)


class Wsola:
    def __init__(self, speed, forced=None):
        self.q = quantize(speed)
        self.forced = None if forced is None else [int(p) for p in forced]
        self.x = np.zeros(H)              # x~: H zeros, then the input
        self.L = 0
        self.final = False
        self.p = []                       # p_k of every frame run
        self.scores = []                  # per frame k >= 1: (candidate positions, their scores)
        self.acc = np.zeros(0)            # y~
        self.out = 0                      # output samples released so far
        self.w = hann()

    def a(self, k):
        return (k * H * self.q) >> 10

    def _reads_to(self, k):
        """one past the last x~ index frame k can read"""
        if k == 0:
            return N
        return max(self.a(k) + D + N, self.a(k - 1) + D + H + N)

    def _xt(self, lo, hi):
        """x~[lo, hi), zeros after the end"""
        seg = self.x[lo:hi]
        return np.concatenate([seg, np.zeros(hi - lo - len(seg))]) if len(seg) < hi - lo else seg

    def _frame(self, k):
        if k == 0:
            p = 0
        else:
            a = self.a(k)
            lo, hi = max(0, a - D), a + D
            t = self._xt(self.p[-1] + H, self.p[-1] + H + N)
            span = self._xt(lo, hi + N)
            win = np.lib.stride_tricks.sliding_window_view(span, N)[:hi - lo + 1]
            c = (win @ t) / np.sqrt(EPS + (win * win).sum(axis=1))
            cand = np.arange(lo, hi + 1)
            self.scores.append((cand, c))
            best = np.flatnonzero(c == c.max())
            p = int(cand[best[np.lexsort((cand[best], np.abs(cand[best] - a)))[0]]])
            if self.forced is not None:
                p = self.forced[k]
        self.p.append(p)
        end = k * H + N
        if len(self.acc) < end:
            self.acc = np.concatenate([self.acc, np.zeros(end - len(self.acc))])
        self.acc[k * H:end] += self.w * self._xt(p, p + N)

    def push(self, x, final=False):
        if self.final:
            raise RuntimeError("stream already flushed")
        x = np.asarray(x, dtype=np.float64).reshape(-1)
        if self.q == Q_ONE:
            return x.copy()
        self.x = np.concatenate([self.x, x])
        self.L += len(x)
        self.final = final
        if final:
            total = (self.L * 1024 + self.q // 2) // self.q
            while (len(self.p) - 1) * H < total:     # y[m] is final once frame floor((m + H) / H) has run
                self._frame(len(self.p))
        else:
            while self._reads_to(len(self.p)) <= H + self.L:
                self._frame(len(self.p))
            total = max(0, len(self.p) - 1) * H
        y = self.acc[H + self.out:H + total]
        self.out = total
        return y.copy()


def stretch(x, speed, forced=None):
    """(output of one push with flush, the stream) -- the stream holds p and the per-frame scores"""
    s = Wsola(speed, forced)
    return s.push(x, final=True), s
