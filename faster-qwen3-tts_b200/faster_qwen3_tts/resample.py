"""Output sample rate, pitch, gain and encoding: polyphase resampling of the 24 kHz PCM on the device, after the codec
(and the tempo), with the gain and the encoding applied in the kernel's store so that only the encoded bytes leave the
device.

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

Pitch and gain (DESIGN.md §4, "Pitch and gain"):

* ``pitch``: semitones, a finite real in [-12, 12] -> ``rho = round(256 * 2 ** (pitch / 12))`` in [128, 512]; the pitch
  ratio is ``rho / 256`` (at most 6.8 cents off the request).  A shift by ``r`` is a time-stretch by ``1 / r`` followed
  by resampling by ``r``: the tempo runs at ``q = round(speed * 2 ** 18 / rho)`` (``tempo.Tempo(q / 1024)``, which
  quantises back to q), refused unless 256 <= q <= 4096; q == 1024 creates no tempo.  At rho 256 q is the plain speed's.
* the resampler at (R, rho): ``(L, M) = (256 R, 24000 rho) / gcd``, ``half = 32 max(L, M)``, and everything above
  unchanged; ``L == M`` is the one-tap encode-only filter.  At rho 256 every table, count and bit is the plain rate's.
* ``gain_db``: a finite real in [-96, 16] -> ``g = float32(10 ** (gain_db / 20))``; each output is ``fl(acc * g)``
  before the encoding, so s16 / G.711 clip by the s16 rule.  At 0 dB the bits are the ungained ones.
* a delivery lasts ``2 ** 18 / (q rho)`` times the 24 kHz speed-1 audio (under 0.2 % from ``1 / speed``).
* pitch 0 at 0 dB is the identity of both: every call is made exactly as without them.
"""
from __future__ import annotations

import collections
import ctypes as C
import math
import numbers
import threading
from typing import Optional, Sequence

import numpy as np
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
PITCH_ONE, PITCH_MIN, PITCH_MAX = 256, 128, 512
SEMITONES = 12.0          # |pitch| limit
GAIN_DB_MIN, GAIN_DB_MAX = -96.0, 16.0
TABLE_CACHE = 8           # unreferenced pitched tables a device keeps; also the pitched handle pools kept here


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


def _real(value, name, lo, hi) -> float:
    if isinstance(value, bool) or not isinstance(value, numbers.Real) or not math.isfinite(float(value)) \
            or not lo <= float(value) <= hi:
        raise ValueError(f"{name} must be a finite number in [{lo:g}, {hi:g}], got {value!r}")
    return float(value)


def pitch_rho(pitch) -> int:
    """semitones in [-12, 12] -> rho = round(256 * 2 ** (pitch / 12)); ValueError otherwise"""
    return round(PITCH_ONE * 2.0 ** (_real(pitch, "pitch (semitones)", -SEMITONES, SEMITONES) / 12.0))


def gain_of(gain_db) -> float:
    """dB in [-96, 16] -> the float32 gain 10 ** (gain_db / 20), as a Python float; ValueError otherwise"""
    return float(np.float32(10.0 ** (_real(gain_db, "gain_db", GAIN_DB_MIN, GAIN_DB_MAX) / 20.0)))


def tempo_q(speed, pitch) -> int:
    """the tempo's q for a speaking rate and a pitch: round(speed * 2 ** 18 / rho); ValueError outside [256, 4096]"""
    from .tempo import Q_MAX, Q_MIN, quantize
    quantize(speed)
    q = round(float(speed) * 2 ** 18 / pitch_rho(pitch))
    if not Q_MIN <= q <= Q_MAX:
        raise ValueError(f"speed {speed!r} with pitch {pitch!r} needs a time-stretch by q / 1024 = {q} / 1024, outside "
                         f"[{Q_MIN / 1024:g}, {Q_MAX / 1024:g}]")
    return q


def check_prosody(speed, pitch, gain_db):
    """(q, rho, g) of a request; every refusal (ValueError) happens here, before anything is tokenized"""
    gain = gain_of(gain_db)
    return tempo_q(speed, pitch), pitch_rho(pitch), gain


def tempo_speed(speed, pitch):
    """the speed to build the request's tempo with: ``speed`` itself at pitch 0, else q / 1024"""
    return speed if pitch == 0 else tempo_q(speed, pitch) / 1024


def ratio(rate: int, rho: int = PITCH_ONE):
    """(L, M, half) of an output rate at pitch rho; L == M (24000 at rho 256) is the encode-only filter (1, 1, 0)"""
    g = math.gcd(rate * PITCH_ONE, IN_RATE * rho)
    L, M = rate * PITCH_ONE // g, IN_RATE * rho // g
    if L == M:
        return 1, 1, 0
    return L, M, HALF_PER_M * max(L, M)


def emitted(total_in: int, rate: int, final: bool, rho: int = PITCH_ONE) -> int:
    """output samples released once ``total_in`` samples have been pushed (and flushed, when ``final``)"""
    L, M, half = ratio(rate, rho)
    every = -(-total_in * L // M)
    if final:
        return every
    return min(every, max(0, -(-(total_in * L - half) // M)))


def released(total_in: int, n: int, rate: int, final: bool, rho: int = PITCH_ONE) -> int:
    """samples a push of ``n`` samples releases after ``total_in`` samples of the stream, with or without flush"""
    return emitted(total_in + n, rate, final, rho) - emitted(total_in, rate, False, rho)


class Resampler:
    """Device state of one resampled stream (C ABI ``fq3_resample_*``): the last ceil(2 half / L) input samples, and
    the stream's gain.  Push its PCM with ``process``; ``close`` hands the handle back to a pool of its (device, rate,
    rho, encoding), so a new request reuses one instead of allocating.  A pooled handle holds its phase table, so only
    the ``TABLE_CACHE`` most recently used pitched keys keep their handles: the others' are destroyed, which lets the
    extension free their tables (``fq3_resample_table_bytes``)."""

    _pool = {}                          # (device, rate, rho, encoding) -> released handles
    _pitched = collections.OrderedDict()   # pitched pool keys, least recently used first
    _lock = threading.Lock()

    def __init__(self, rate, encoding: str = "f32", device=None, pitch=0, gain_db=0):
        self.rate, self.encoding = check_rate(rate), check_encoding(encoding)
        self.rho, self.gain = pitch_rho(pitch), gain_of(gain_db)
        if (self.rate, self.encoding, self.rho, self.gain) == (IN_RATE, "f32", PITCH_ONE, 1.0):
            raise ValueError("24000 Hz f32 is the identity: use resampler_for(), which returns None for it")
        from .engine import load_library
        self._lib = load_library()
        dev = torch.device(device if device is not None else "cuda")
        self.device = torch.device("cuda", dev.index if dev.index is not None else torch.cuda.current_device())
        self._key = (self.device.index, self.rate, self.rho, self.encoding)
        with Resampler._lock:
            pool = Resampler._pool.get(self._key)
            h = pool.pop() if pool else None
            if self.rho != PITCH_ONE and self._key in Resampler._pitched:
                Resampler._pitched.move_to_end(self._key)
        if h is not None:
            self._h = h
            self._lib.fq3_resample_reset(self._h)
        else:
            h = C.c_void_p()
            if self._lib.fq3_resample_create_pitch(self.device.index, self.rate, self.rho, ENCODINGS[self.encoding],
                                                   C.byref(h)):
                raise RuntimeError(self._lib.fq3_resample_last_error().decode())
            self._h = h
        if self._lib.fq3_resample_set_gain(self._h, C.c_float(self.gain)):
            raise RuntimeError(self._lib.fq3_resample_last_error().decode())
        self.total_in, self.final = 0, False

    def released(self, n: int, final: bool) -> int:
        return released(self.total_in, n, self.rate, final, self.rho)

    def close(self) -> None:
        if self._h is None:
            return
        h, self._h, drop = self._h, None, []
        with Resampler._lock:
            Resampler._pool.setdefault(self._key, []).append(h)
            if self.rho != PITCH_ONE:
                Resampler._pitched[self._key] = None
                Resampler._pitched.move_to_end(self._key)
                while len(Resampler._pitched) > TABLE_CACHE:
                    old, _ = Resampler._pitched.popitem(last=False)
                    drop += Resampler._pool.pop(old, [])
        for d in drop:
            self._lib.fq3_resample_destroy(d)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def resampler_for(rate, encoding: str = "f32", device=None, pitch=0, gain_db=0) -> Optional[Resampler]:
    """A ``Resampler`` for ``rate`` / ``encoding`` / ``pitch`` / ``gain_db``, or None for 24000 Hz f32 at pitch 0 and
    0 dB (the identity: nothing to create or launch)"""
    rate, encoding = check_rate(rate), check_encoding(encoding)
    if (rate, encoding, pitch_rho(pitch), gain_of(gain_db)) == (IN_RATE, "f32", PITCH_ONE, 1.0):
        return None
    return Resampler(rate, encoding, device, pitch, gain_db)


def warm(rate, encoding: str, device, pitch) -> None:
    """Design and upload the (rate, rho) table of a pitch on the calling thread, by pooling one handle for it, so that
    a request's resampler is later taken from the pool without designing anything (``ContinuousBatcher.submit``)"""
    if pitch_rho(pitch) == PITCH_ONE:
        return
    key = (torch.device(device).index, check_rate(rate), pitch_rho(pitch), check_encoding(encoding))
    with Resampler._lock:
        if Resampler._pool.get(key):
            return
    Resampler(rate, encoding, device, pitch).close()


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


def convert(pcm: torch.Tensor, rate, encoding: str = "f32", pitch=0, gain_db=0) -> torch.Tensor:
    """The whole of ``pcm`` (1-D float32 on a CUDA device) at ``rate`` / ``encoding`` in one push with flush, resampled
    at the pitch's rho and scaled by the gain; 24000 Hz f32 at pitch 0 and 0 dB returns it.  A delivery at a pitch
    equals ``convert(tempo.stretch(pcm, tempo_q(speed, pitch) / 1024), rate, encoding, pitch, gain_db)`` of the speed-1
    24 kHz PCM."""
    r = resampler_for(rate, encoding, pcm.device, pitch, gain_db)
    if r is None:
        return pcm
    try:
        return process([r], [pcm], True)[0]
    finally:
        r.close()
