"""FLAC output: lossless compression of the s16 PCM on the device, after the resampler's s16 store, so that only the
compressed bytes leave the device.

The format and every encoder decision are fixed exactly, so that the kernel (``csrc/fq3_flac.cu``) and the numpy oracle
(``oracle/flac_oracle.py``) produce the same bytes:

* A FLAC stream (RFC 9639), mono, 16 bits per sample, at a rate in ``resample.RATES``.  It starts with ``fLaC`` and one
  STREAMINFO block, the last metadata block: min / max block size 16 / 4096, min / max frame size 0 (unknown), the rate,
  1 channel, 16 bits, total samples 0 -- or the true count when the push that releases the header also flushes (a
  one-shot ``convert``) -- and an all-zero MD5 (unset).  The first bytes a stream releases carry this header.
* Variable blocking (blocking-strategy bit 1; a frame header codes its first sample's index).  A push of m samples after
  c carried ones encodes ``16 * ((c + m) // 16)`` of them, or all of them at flush, as blocks of 4096 and one block of
  the remainder; the rest (fewer than 16 samples) carries to the next push.  So the encoder never holds audio back
  waiting for a fixed block to fill.
* Frame header: sync ``0xFFF9``; block-size code 12 for 4096, else 6 (8-bit n - 1) when n <= 256, else 7 (16-bit n - 1);
  the rate's own code (all seven rates have one); mono; 16 bits; the UTF-8-coded first sample index; CRC-8 (poly 0x07).
* Subframe: CONSTANT when all samples are equal.  Otherwise the choice with the fewest bits among FIXED orders 0 ..
  min(4, n - 1), every partition order p in 0 .. 8 with n divisible by 2^p and more than ``order`` samples per
  partition, and per partition the Rice parameter k in 0 .. 30 minimising ``sum((u >> k) + 1 + k)`` over its residuals
  (u the zig-zag of the residual).  Coding method 0 when every k <= 14, else method 1 (5-bit parameters).  No escape
  partitions, no wasted bits.  Ties go to the lowest order, then the lowest p, then the lowest k.  VERBATIM when the best
  choice is not smaller than it.
* Frame: header, subframe, zero bits to a byte boundary, CRC-16 (poly 0x8005) of all of it.

The bytes are a pure function of (samples, push sizes, flush); the decoded samples depend on the samples alone.

The stage's output size depends on the data, so ``process`` reads one int32 byte count per stream back to the host:
that copy is the stage's one host synchronisation per step.
"""
from __future__ import annotations

import ctypes as C
from typing import Sequence

import torch

from .resample import ENCODINGS as PCM_ENCODINGS, check_rate

# one place for the constants (include/fq3_engine.h FQ3_FLAC_*; a CPU test checks that they agree)
BLOCK = 4096
GRAIN = 16
MAX_ORDER = 4
MAX_PARTITION_ORDER = 8
MAX_K = 30
HEAD_BYTES = 42
ALIGN = 16
ENCODINGS = tuple(PCM_ENCODINGS) + ("flac",)   # what a serving ticket may carry


def check_encoding(encoding) -> str:
    """a ticket's encoding: one of the resampler's (``f32 | s16 | ulaw | alaw``) or ``flac``; ValueError otherwise"""
    if encoding not in ENCODINGS:
        raise ValueError(f"encoding must be one of {', '.join(ENCODINGS)}, got {encoding!r}")
    return encoding


def max_bytes(carried: int, n: int, flush: bool) -> int:
    """a bound on the bytes a push of ``n`` samples after ``carried`` ones releases: the stream header, and per block of
    b samples 2 b + 19 bytes (frame header <= 16, subframe header, the samples verbatim, CRC-16)"""
    ready = carried + n
    take = ready if flush else ready // GRAIN * GRAIN
    full, rest = divmod(take, BLOCK)
    return HEAD_BYTES + full * (2 * BLOCK + 19) + (2 * rest + 19 if rest else 0)


class Encoder:
    """Device state of one FLAC stream (C ABI ``fq3_flac_*``): up to 15 carried samples, the next sample index and
    whether the header has been released.  Push its s16 PCM with ``process``; ``close`` hands the handle back to a pool
    of its (device, rate), so a new request reuses one instead of allocating."""

    _pool = {}   # (device, rate) -> released handles

    def __init__(self, rate, device=None):
        self.rate = check_rate(rate)
        from .engine import load_library
        self._lib = load_library()
        dev = torch.device(device if device is not None else "cuda")
        self.device = torch.device("cuda", dev.index if dev.index is not None else torch.cuda.current_device())
        self._key = (self.device.index, self.rate)
        pool = Encoder._pool.get(self._key)
        if pool:
            self._h = pool.pop()
            self._lib.fq3_flac_reset(self._h)
        else:
            h = C.c_void_p()
            if self._lib.fq3_flac_create(self.device.index, self.rate, C.byref(h)):
                raise RuntimeError(self._lib.fq3_flac_last_error().decode())
            self._h = h
        self.carried, self.final = 0, False

    def close(self) -> None:
        if self._h is not None:
            Encoder._pool.setdefault(self._key, []).append(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def process(encoders: Sequence[Encoder], pcms: Sequence[torch.Tensor], final):
    """One encoding launch and one packing launch for every stream: ``pcms[i]`` (int16, 1-D, on the encoders' device)
    is pushed to ``encoders[i]``; ``final`` (a bool, or one per stream) flushes.  Returns the released bytes per stream
    as uint8 device tensors (views of one buffer).  Reads the byte counts back: one device-to-host copy."""
    n = len(encoders)
    finals = [bool(final)] * n if isinstance(final, bool) else [bool(f) for f in final]
    if not (len(pcms) == n == len(finals)):
        raise ValueError("one PCM tensor and one flush flag per encoder")
    if n == 0:
        return []
    if len({id(e) for e in encoders}) != n:
        raise ValueError("FLAC encoder listed twice")
    for e in encoders:
        if e._h is None or e.final:
            raise ValueError("FLAC encoder is closed or already flushed")
    dev = encoders[0].device
    pcms = [p.reshape(-1) for p in pcms]
    for p in pcms:
        if p.dtype != torch.int16 or p.device != dev:
            raise ValueError(f"FLAC encoder input must be int16 on {dev}")
    lens = [int(p.numel()) for p in pcms]
    offs, end = [], 0
    for e, m, f in zip(encoders, lens, finals):
        off = -(-end // ALIGN) * ALIGN
        offs.append(off)
        end = off + max_bytes(e.carried, m, f)
    out = torch.empty(end, dtype=torch.uint8, device=dev)
    out_lens = torch.empty(n, dtype=torch.int32, device=dev)
    inp = pcms[0].contiguous() if n == 1 else torch.cat(pcms)
    arr = (C.c_void_p * n)(*[e._h for e in encoders])
    lib = encoders[0]._lib
    with torch.cuda.device(dev):
        rc = lib.fq3_flac_process(
            arr, n, C.c_void_p(inp.data_ptr() if inp.numel() else None), (C.c_int64 * n)(*lens),
            (C.c_int32 * n)(*[int(f) for f in finals]), C.c_void_p(out.data_ptr()), out.numel(),
            C.c_void_p(out_lens.data_ptr()), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
    if rc:
        raise RuntimeError(lib.fq3_flac_last_error().decode())
    for e, m, f in zip(encoders, lens, finals):
        ready = e.carried + m
        e.carried = 0 if f else ready % GRAIN
        e.final = f
    sizes = out_lens.tolist()   # the stage's one host synchronisation
    return [out[o:o + s] for o, s in zip(offs, sizes)]


def convert(pcm: torch.Tensor, rate) -> torch.Tensor:
    """The whole of ``pcm`` (1-D int16 on a CUDA device) as one FLAC file at ``rate``: one push with flush, so the
    header carries the total sample count"""
    e = Encoder(rate, pcm.device)
    try:
        return process([e], [pcm], True)[0]
    finally:
        e.close()
