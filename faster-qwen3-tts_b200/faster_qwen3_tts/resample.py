"""Output sample rate and encoding: polyphase resampling of the 24 kHz PCM on the device, after the codec (and the tempo),
with the encoding applied in the kernel's store so that only the encoded bytes leave the device.

The algorithm is fixed exactly so that this module's counts, the float64 oracle (``oracle/resample_oracle.py``) and the
kernel (``csrc/fq3_resample.cu``) agree:

* output rates ``R`` in ``RATES``; ``g = gcd(R, 24000)``, ``L = R / g``, ``M = 24000 / g``, ``m = max(L, M)``,
  ``half = 32 m``.
* ``h = scipy.signal.firwin(2 half + 1, 0.9 / m, window=("kaiser", 8.6))`` (unit DC gain), designed in double.
* ``y[n] = L * sum_j h[j] x[(n M + half - j) / L]`` over the j where ``n M + half - j`` is a non-negative multiple of L
  and the index lies in [0, N); x is zero outside.  A flushed stream of N samples has ``ceil(N L / M)`` outputs.  The
  kernel sums in fp32, taps in a fixed order.
* before flush, output n is released once input ``(n M + half) // L`` exists (``emitted``), so a push releases a count
  known on the host before the launch, and any chunking of the input gives the same bits.
* encodings ``f32``; ``s16`` (``serving.to_pcm16``: ``clip(x * 32768, -32768, 32767)`` truncated toward zero, in fp32);
  ``ulaw`` / ``alaw`` (ITU-T G.711 of that s16, as ``audioop.lin2ulaw`` / ``lin2alaw``).
* 24000 with a non-f32 encoding is encode-only: ``h = [1]``, ``half = 0``.  24000 with ``f32`` is the identity: nothing
  is created or launched (``resampler_for`` returns None).
"""
from __future__ import annotations

import ctypes as C
import math
import numbers
from typing import Optional, Sequence

import torch

# one place for the constants (include/fq3_engine.h FQ3_RESAMPLE_* / FQ3_ENC_*; a CPU test checks that they agree)
IN_RATE = 24000
RATES = (8000, 16000, 22050, 24000, 32000, 44100, 48000)
HALF_PER_M = 32
CUTOFF = 0.9
BETA = 8.6
ALIGN = 16
ENCODINGS = {"f32": 0, "s16": 1, "ulaw": 2, "alaw": 3}
DTYPES = {"f32": torch.float32, "s16": torch.int16, "ulaw": torch.uint8, "alaw": torch.uint8}
SAMPLE_BYTES = {"f32": 4, "s16": 2, "ulaw": 1, "alaw": 1}


def check_rate(rate) -> int:
    """``rate`` (None = 24000) -> the output rate as an int; ValueError outside ``RATES``"""
    if rate is None:
        return IN_RATE
    if isinstance(rate, bool) or not isinstance(rate, numbers.Real) or not float(rate).is_integer() \
            or int(rate) not in RATES:
        raise ValueError(f"sample_rate must be one of {', '.join(map(str, RATES))}, got {rate!r}")
    return int(rate)


def check_encoding(encoding) -> str:
    if encoding not in ENCODINGS:
        raise ValueError(f"encoding must be one of {', '.join(ENCODINGS)}, got {encoding!r}")
    return encoding


def ratio(rate: int):
    """(L, M, half) of an output rate; 24000 is the encode-only identity filter (1, 1, 0)"""
    if rate == IN_RATE:
        return 1, 1, 0
    g = math.gcd(rate, IN_RATE)
    L, M = rate // g, IN_RATE // g
    return L, M, HALF_PER_M * max(L, M)


def emitted(total_in: int, rate: int, final: bool) -> int:
    """output samples released once ``total_in`` samples have been pushed (and flushed, when ``final``)"""
    L, M, half = ratio(rate)
    every = -(-total_in * L // M)
    if final:
        return every
    return min(every, max(0, -(-(total_in * L - half) // M)))


def released(total_in: int, n: int, rate: int, final: bool) -> int:
    """samples a push of ``n`` samples releases after ``total_in`` samples of the stream, with or without flush"""
    return emitted(total_in + n, rate, final) - emitted(total_in, rate, False)


class Resampler:
    """Device state of one resampled stream (C ABI ``fq3_resample_*``): the last ceil(2 half / L) input samples.  Push
    its PCM with ``process``; ``close`` hands the handle back to a pool of its (device, rate, encoding), so a new
    request reuses one instead of allocating."""

    _pool = {}   # (device, rate, encoding) -> released handles

    def __init__(self, rate, encoding: str = "f32", device=None):
        self.rate, self.encoding = check_rate(rate), check_encoding(encoding)
        if self.rate == IN_RATE and self.encoding == "f32":
            raise ValueError("24000 Hz f32 is the identity: use resampler_for(), which returns None for it")
        from .engine import load_library
        self._lib = load_library()
        dev = torch.device(device if device is not None else "cuda")
        self.device = torch.device("cuda", dev.index if dev.index is not None else torch.cuda.current_device())
        self._key = (self.device.index, self.rate, self.encoding)
        pool = Resampler._pool.get(self._key)
        if pool:
            self._h = pool.pop()
            self._lib.fq3_resample_reset(self._h)
        else:
            h = C.c_void_p()
            if self._lib.fq3_resample_create(self.device.index, self.rate, ENCODINGS[self.encoding], C.byref(h)):
                raise RuntimeError(self._lib.fq3_resample_last_error().decode())
            self._h = h
        self.total_in, self.final = 0, False

    def released(self, n: int, final: bool) -> int:
        return released(self.total_in, n, self.rate, final)

    def close(self) -> None:
        if self._h is not None:
            Resampler._pool.setdefault(self._key, []).append(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def resampler_for(rate, encoding: str = "f32", device=None) -> Optional[Resampler]:
    """A ``Resampler`` for ``rate`` / ``encoding``, or None for 24000 Hz f32 (the identity: nothing to create or launch)"""
    rate, encoding = check_rate(rate), check_encoding(encoding)
    return None if (rate, encoding) == (IN_RATE, "f32") else Resampler(rate, encoding, device)


def process(resamplers: Sequence[Resampler], pcms: Sequence[torch.Tensor], final):
    """One launch for every stream: ``pcms[i]`` (float32, 1-D, on the resamplers' device) is pushed to
    ``resamplers[i]``; ``final`` (a bool, or one per stream) flushes.  Returns the released samples per stream in its
    encoding (float32, int16 or uint8 device tensors, views of one buffer).  No host synchronisation: every size comes
    from ``released``."""
    n = len(resamplers)
    finals = [bool(final)] * n if isinstance(final, bool) else [bool(f) for f in final]
    if not (len(pcms) == n == len(finals)):
        raise ValueError("one PCM tensor and one flush flag per resampler")
    if n == 0:
        return []
    if len({id(r) for r in resamplers}) != n:
        raise ValueError("resampler listed twice")
    for r in resamplers:
        if r._h is None or r.final:
            raise ValueError("resampler is closed or already flushed")
    dev = resamplers[0].device
    pcms = [p.reshape(-1) for p in pcms]
    for p in pcms:
        if p.dtype != torch.float32 or p.device != dev:
            raise ValueError(f"resampler input must be float32 on {dev}")
    lens = [int(p.numel()) for p in pcms]
    counts = [r.released(m, f) for r, m, f in zip(resamplers, lens, finals)]
    offs, end = [], 0
    for r, c in zip(resamplers, counts):
        off = -(-end // ALIGN) * ALIGN
        offs.append(off)
        end = off + c * SAMPLE_BYTES[r.encoding]
    out = torch.empty(end, dtype=torch.uint8, device=dev)
    if end or any(lens):
        inp = pcms[0].contiguous() if n == 1 else torch.cat(pcms)
        arr = (C.c_void_p * n)(*[r._h for r in resamplers])
        lib = resamplers[0]._lib
        with torch.cuda.device(dev):
            rc = lib.fq3_resample_process(
                arr, n, C.c_void_p(inp.data_ptr() if inp.numel() else None), (C.c_int64 * n)(*lens),
                (C.c_int32 * n)(*[int(f) for f in finals]), C.c_void_p(out.data_ptr() if out.numel() else None),
                out.numel(), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
        if rc:
            raise RuntimeError(lib.fq3_resample_last_error().decode())
    for r, m, f in zip(resamplers, lens, finals):
        r.total_in += m
        r.final = f
    return [out[o:o + c * SAMPLE_BYTES[r.encoding]].view(DTYPES[r.encoding])
            for r, o, c in zip(resamplers, offs, counts)]


def convert(pcm: torch.Tensor, rate, encoding: str = "f32") -> torch.Tensor:
    """The whole of ``pcm`` (1-D float32 on a CUDA device) at ``rate`` / ``encoding`` in one push with flush; 24000 Hz
    f32 returns it."""
    r = resampler_for(rate, encoding, pcm.device)
    if r is None:
        return pcm
    try:
        return process([r], [pcm], True)[0]
    finally:
        r.close()
