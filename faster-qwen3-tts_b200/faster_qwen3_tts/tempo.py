"""Speaking-rate control: a pitch-preserving time-stretch of the 24 kHz PCM, on the device, after the codec.

The algorithm is waveform-similarity overlap-add (WSOLA), fixed exactly so that this module's counts, the float64
oracle (``oracle/tempo_oracle.py``) and the kernel (``csrc/fq3_tempo.cu``) agree:

* window ``N = 480`` (20 ms), periodic Hann ``w[n] = 0.5 - 0.5 cos(2 pi n / N)``; synthesis hop ``H = N / 2 = 240``;
  search half-width ``D = 240`` (+-10 ms, a whole pitch period down to 50 Hz).
* ``q = round(speed * 1024)``, refused outside [256, 4096] (speed 0.25 - 4.0).  ``q == 1024`` is the identity: nothing
  is created or launched and the PCM is passed through untouched.
* ``x~`` is the input with H zeros in front (and, at flush only, zeros after its end).  Frame k has the nominal position
  ``a_k = (k H q) >> 10``; ``p_0 = 0``; for k >= 1 the target is ``t[n] = x~[p_{k-1} + H + n]``, the candidates are
  ``p = a_k + d`` with ``|d| <= D`` and ``p >= 0``, scored ``c(p) = sum t[n] x~[p+n] / sqrt(eps + sum x~[p+n]^2)``;
  ``p_k`` is the argmax, ties to the smallest ``|d|``, then the smaller ``p``.  The kernel sums in fp32.
* Overlap-add ``y~[kH + n] += w[n] x~[p_k + n]`` (the earlier frame's term first); the output is ``y[m] = y~[m + H]``.
* A frame runs as soon as every sample it can read exists; output is released as soon as no later frame can add to it.
  At flush, with L input samples in all, the output has ``L_out = (L * 1024 + q // 2) // q`` samples.

So the output depends on the input samples and the flush point only: splitting the input into pushes changes no
sample, and the number of samples a push releases (``released``) is known on the host before the launch.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Optional, Sequence

import torch

# one place for the constants (include/fq3_engine.h FQ3_TEMPO_*; a CPU test checks that they agree)
WINDOW = 480
HOP = WINDOW // 2
SEARCH = 240
EPS = 1e-6
Q_ONE, Q_MIN, Q_MAX = 1024, 256, 4096
SAMPLE_RATE = 24000


def quantize(speed) -> int:
    """speed -> q = round(speed * 1024); ValueError outside [0.25, 4.0]"""
    try:
        s = float(speed)
    except (TypeError, ValueError):
        raise ValueError(f"speed must be a number in [0.25, 4.0], got {speed!r}") from None
    q = round(s * 1024) if math.isfinite(s) else -1
    if not Q_MIN <= q <= Q_MAX:
        raise ValueError(f"speed must be in [0.25, 4.0], got {speed!r}")
    return q


def nominal(k: int, q: int) -> int:
    """a_k, the nominal analysis position of frame k"""
    return (k * HOP * q) >> 10


def ready_frames(total_in: int, q: int) -> int:
    """frames that can run once ``total_in`` samples exist (no flush).  Frame 0 reads x~[0, N); frame k >= 1 reads up to
    max(a_k, a_{k-1} + H) + D + N (exclusive): its candidates, and its target, since p_{k-1} <= a_{k-1} + D."""
    lim = HOP + total_in
    if lim < WINDOW:
        return 0
    m = lim - SEARCH - WINDOW          # frame k >= 1 runs iff a_k <= m and a_{k-1} <= m - H
    if m - HOP < 0:
        return 1
    k1 = ((m + 1) * 1024 - 1) // (HOP * q)
    k2 = ((m - HOP + 1) * 1024 - 1) // (HOP * q) + 1
    return min(k1, k2) + 1


def out_len(total_in: int, q: int) -> int:
    """L_out: the samples of a flushed stream of ``total_in`` input samples"""
    return (total_in * 1024 + q // 2) // q


def emitted(total_in: int, q: int, final: bool) -> int:
    """output samples released once ``total_in`` samples have been pushed (and flushed, when ``final``)"""
    if q == Q_ONE:
        return total_in
    if final:
        return out_len(total_in, q)
    return max(0, ready_frames(total_in, q) - 1) * HOP


def released(total_in: int, n: int, q: int, final: bool) -> int:
    """samples a push of ``n`` samples releases after ``total_in`` samples of the stream, with or without flush"""
    return emitted(total_in + n, q, final) - emitted(total_in, q, False)


def frames_run(total_in: int, n: int, q: int, final: bool) -> int:
    """frames such a push runs (the length of its p_k record)"""
    before = ready_frames(total_in, q)
    if final:
        return max(before, -(-out_len(total_in + n, q) // HOP) + 1) - before
    return ready_frames(total_in + n, q) - before


class Tempo:
    """Device state of one time-stretched stream (C ABI ``fq3_tempo_*``): the input tail later frames can still reach,
    the pending overlap and p_{k-1}.  Push its PCM with ``process``; ``close`` hands the handle back to a pool of its
    speed, so a new request reuses one instead of allocating."""

    _pool = {}   # (device, q) -> released handles

    def __init__(self, speed, device=None):
        self.q = quantize(speed)
        if self.q == Q_ONE:
            raise ValueError("speed 1 is the identity: use tempo_for(), which returns None for it")
        from .engine import load_library
        self._lib = load_library()
        dev = torch.device(device if device is not None else "cuda")
        self.device = torch.device("cuda", dev.index if dev.index is not None else torch.cuda.current_device())
        pool = Tempo._pool.get((self.device.index, self.q))
        if pool:
            self._h = pool.pop()
            self._lib.fq3_tempo_reset(self._h)
        else:
            h = C.c_void_p()
            if self._lib.fq3_tempo_create(self.device.index, C.c_double(self.q / 1024), C.byref(h)):
                raise RuntimeError(self._lib.fq3_tempo_last_error().decode())
            self._h = h
        self.total_in, self.final = 0, False

    def released(self, n: int, final: bool) -> int:
        return released(self.total_in, n, self.q, final)

    def close(self) -> None:
        if self._h is not None:
            Tempo._pool.setdefault((self.device.index, self.q), []).append(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def tempo_for(speed, device=None) -> Optional[Tempo]:
    """A ``Tempo`` for ``speed``, or None at speed 1 (the identity: nothing to create or launch)"""
    return None if quantize(speed) == Q_ONE else Tempo(speed, device)


def process(tempos: Sequence[Tempo], pcms: Sequence[torch.Tensor], final, positions: bool = False):
    """One launch for every stream: ``pcms[i]`` (float32, 1-D, on the tempos' device) is pushed to ``tempos[i]``;
    ``final`` (a bool, or one per stream) flushes.  Returns the released PCM per stream (device tensors, views of one
    buffer), and with ``positions`` also the p_k of every frame run per stream (int32 device tensors).  No host
    synchronisation: every size comes from ``released`` / ``frames_run``."""
    n = len(tempos)
    finals = [bool(final)] * n if isinstance(final, bool) else [bool(f) for f in final]
    if not (len(pcms) == n == len(finals)):
        raise ValueError("one PCM tensor and one flush flag per tempo")
    if n == 0:
        return ([], []) if positions else []
    if len({id(t) for t in tempos}) != n:
        raise ValueError("tempo listed twice")
    for t in tempos:
        if t._h is None or t.final:
            raise ValueError("tempo is closed or already flushed")
    dev = tempos[0].device
    pcms = [p.reshape(-1) for p in pcms]
    for p in pcms:
        if p.dtype != torch.float32 or p.device != dev:
            raise ValueError(f"tempo input must be float32 on {dev}")
    lens = [int(p.numel()) for p in pcms]
    outs = [t.released(m, f) for t, m, f in zip(tempos, lens, finals)]
    nks = [frames_run(t.total_in, m, t.q, f) for t, m, f in zip(tempos, lens, finals)]
    out = torch.empty(sum(outs), dtype=torch.float32, device=dev)
    pk = torch.empty(sum(nks), dtype=torch.int32, device=dev) if positions else None
    if sum(outs) or sum(nks) or any(lens):
        inp = pcms[0].contiguous() if n == 1 else torch.cat(pcms)
        arr = (C.c_void_p * n)(*[t._h for t in tempos])
        lib = tempos[0]._lib
        with torch.cuda.device(dev):
            rc = lib.fq3_tempo_process(
                arr, n, C.c_void_p(inp.data_ptr() if inp.numel() else None), (C.c_int64 * n)(*lens),
                (C.c_int32 * n)(*[int(f) for f in finals]), C.c_void_p(out.data_ptr() if out.numel() else None),
                out.numel(), C.c_void_p(pk.data_ptr() if positions and pk.numel() else None),
                pk.numel() if positions else 0, C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
        if rc:
            raise RuntimeError(lib.fq3_tempo_last_error().decode())
    for t, m, f in zip(tempos, lens, finals):
        t.total_in += m
        t.final = f
    res = list(torch.split(out, outs))
    return (res, list(torch.split(pk, nks))) if positions else res


def stretch(pcm: torch.Tensor, speed, positions: bool = False):
    """The whole of ``pcm`` (1-D float32 on a CUDA device) at ``speed`` in one push with flush; speed 1 returns it."""
    t = tempo_for(speed, pcm.device)
    if t is None:
        return (pcm, None) if positions else pcm
    try:
        r = process([t], [pcm], True, positions=positions)
        return (r[0][0], r[1][0]) if positions else r[0]
    finally:
        t.close()
