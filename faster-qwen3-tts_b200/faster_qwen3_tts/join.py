"""Long inputs: the join of a segmented request's rows into one stream, on the device, before the post-codec stages.

A segmented request (``segment.split_text``) speaks S segments; each is decoded as its own row, with its own codec
window, and the rows finish in any order.  The join (``csrc/fq3_join.cu``; ``tests/join_oracle.py`` restates it) makes
their 24 kHz float32 PCM one stream, in segment order:

* ``seg_0``, ``P`` zeros, ``seg_1``, ..., ``seg_{S-1}`` with ``P = 24 * pause_ms``, ``pause_ms`` an integer in [0, 2000].
* Or, with a pause per boundary (``pauses``, SSML breaks): ``P_0`` zeros, ``seg_0``, ``P_1`` zeros, ..., ``seg_{S-1}``,
  ``P_S`` zeros with ``P_k = 24 * pauses[k]``, each an integer in [0, 10000].  The leading zeros are released with
  segment 0's first push, the trailing ones in the call that completes the stream.  ``pause_ms`` is the plan
  ``[0, P, ..., P, 0]``, bit for bit.
* Every inner boundary is faded, also at pause 0: sample n of segment k (length L) becomes ``x * a * b`` in fp32, in that
  order, with ``a = w[n]`` for k > 0 and n < F and ``b = w[L - 1 - n]`` for k < S - 1 and L - 1 - n < F (1 otherwise),
  ``F = 120`` (5 ms) and ``w[i] = float32(0.5 - 0.5 cos(pi (i + 0.5) / F))`` (``fade_table``).
* The segment being played is released as its samples arrive, but for its last F while it has not ended; a later
  segment's samples stay on the device until every earlier segment has ended.  The counts a call releases depend on the
  pushed lengths and end flags alone (``Join.released``), so nothing is read back, and the joined stream does not depend
  on how the segments were pushed.

The request's tempo, resampler and FLAC encoder run once on the joined stream, so they stay continuous across segments.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch

# one place for the constants (include/fq3_engine.h FQ3_JOIN_*; a CPU test checks that they agree)
RATE = 24000
FADE = 120
PAUSE_MAX_MS = 2000
BREAK_MAX_MS = 10000            # one boundary of a pause plan (an SSML document's breaks)


def check_pause(pause_ms) -> int:
    """``pause_ms`` as an int; ValueError unless it is an integer in [0, 2000]"""
    if isinstance(pause_ms, bool) or not isinstance(pause_ms, (int, np.integer)) or not 0 <= pause_ms <= PAUSE_MAX_MS:
        raise ValueError(f"pause_ms must be an integer in [0, {PAUSE_MAX_MS}], got {pause_ms!r}")
    return int(pause_ms)


def check_pauses(pauses, n_segments: int) -> List[int]:
    """a pause plan (``n_segments + 1`` integers in [0, 10000] ms) as a list; ValueError otherwise"""
    pauses = list(pauses)
    if len(pauses) != n_segments + 1:
        raise ValueError(f"a pause plan has one entry per boundary: {n_segments + 1}, got {len(pauses)}")
    for p in pauses:
        if isinstance(p, bool) or not isinstance(p, (int, np.integer)) or not 0 <= p <= BREAK_MAX_MS:
            raise ValueError(f"every pause must be an integer in [0, {BREAK_MAX_MS}] ms, got {p!r}")
    return [int(p) for p in pauses]


def pause_samples(pause_ms: int) -> int:
    return check_pause(pause_ms) * (RATE // 1000)


def fade_table() -> np.ndarray:
    """w[i] = float32(0.5 - 0.5 cos(pi (i + 0.5) / F)), i < F: the raised-cosine fade-in; its reverse fades out"""
    return (0.5 - 0.5 * np.cos(np.pi * (np.arange(FADE) + 0.5) / FADE)).astype(np.float32)


class Join:
    """Device state of one segmented request (C ABI ``fq3_join_*``): the held tail of the segment being played and the
    samples of later segments.  ``pauses``: a pause per boundary (module docstring) instead of ``pause_ms``.  ``close``
    hands the handle back to a per-device pool."""

    _pool = {}   # device index -> released handles

    def __init__(self, n_segments: int, pause_ms: int = 0, device=None, pauses=None):
        if int(n_segments) < 1:
            raise ValueError("a join needs at least one segment")
        self.n_segments, self.pause_ms = int(n_segments), check_pause(pause_ms)
        self.pauses = None if pauses is None else check_pauses(pauses, self.n_segments)
        from .engine import load_library
        self._lib = load_library()
        dev = torch.device(device if device is not None else "cuda")
        self.device = torch.device("cuda", dev.index if dev.index is not None else torch.cuda.current_device())
        plan = None if self.pauses is None else (C.c_int32 * len(self.pauses))(*self.pauses)
        pool = Join._pool.get(self.device.index)
        if pool:
            self._h = pool.pop()
            if plan is None:
                self._lib.fq3_join_reset(self._h, self.n_segments, self.pause_ms)
            else:
                self._lib.fq3_join_reset_pauses(self._h, self.n_segments, plan)
        else:
            h = C.c_void_p()
            rc = (self._lib.fq3_join_create(self.device.index, self.n_segments, self.pause_ms, C.byref(h)) if plan is None
                  else self._lib.fq3_join_create_pauses(self.device.index, self.n_segments, plan, C.byref(h)))
            if rc:
                raise RuntimeError(self._lib.fq3_join_last_error().decode())
            self._h = h
        self.ended = [False] * self.n_segments

    @property
    def done(self) -> bool:
        """every segment has ended: the joined stream is complete"""
        return all(self.ended)

    def close(self) -> None:
        if self._h is not None:
            self._lib.fq3_join_reset(self._h, 1, 0)   # frees what a cancelled request still held
            Join._pool.setdefault(self.device.index, []).append(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _args(joins, pushes):
    index = {id(j): i for i, j in enumerate(joins)}
    if len(index) != len(joins):
        raise ValueError("join listed twice")
    n = len(pushes)
    join_of = (C.c_int32 * max(n, 1))(*[index[id(j)] for j, _, _, _ in pushes])
    seg = (C.c_int32 * max(n, 1))(*[int(k) for _, k, _, _ in pushes])
    lens = (C.c_int64 * max(n, 1))(*[int(p.numel()) for _, _, p, _ in pushes])
    ends = (C.c_int32 * max(n, 1))(*[int(bool(e)) for _, _, _, e in pushes])
    return n, join_of, seg, lens, ends


def released(joins: Sequence[Join], pushes) -> List[int]:
    """the samples ``process(joins, pushes)`` would release per join (host arithmetic, no state changes)"""
    lib = joins[0]._lib
    n, join_of, seg, lens, ends = _args(joins, pushes)
    arr = (C.c_void_p * len(joins))(*[j._h for j in joins])
    out = (C.c_int64 * len(joins))()
    if lib.fq3_join_released(arr, len(joins), n, join_of, seg, lens, ends, out):
        raise ValueError(lib.fq3_join_last_error().decode())
    return list(out)


def process(joins: Sequence[Join], pushes: Sequence[Tuple[Join, int, torch.Tensor, bool]]) -> List[torch.Tensor]:
    """One launch for every join: ``pushes`` are (join, segment, new float32 PCM on the joins' device, whether the
    segment ends with it), at most one per (join, segment).  Returns the released PCM per join (device tensors, views of
    one buffer), in the order of ``joins``.  No host synchronisation: every size comes from ``released``."""
    if not joins:
        return []
    for j in joins:
        if j._h is None:
            raise ValueError("join is closed")
    dev = joins[0].device
    pcms = [p.reshape(-1) for _, _, p, _ in pushes]
    for p in pcms:
        if p.dtype != torch.float32 or p.device != dev:
            raise ValueError(f"join input must be float32 on {dev}")
    pushes = [(j, k, p, e) for (j, k, _, e), p in zip(pushes, pcms)]
    counts = released(joins, pushes)
    out = torch.empty(sum(counts), dtype=torch.float32, device=dev)
    inp = torch.cat(pcms) if len(pcms) > 1 else (pcms[0].contiguous() if pcms else out[:0])
    lib = joins[0]._lib
    n, join_of, seg, lens, ends = _args(joins, pushes)
    arr = (C.c_void_p * len(joins))(*[j._h for j in joins])
    with torch.cuda.device(dev):
        rc = lib.fq3_join_process(arr, len(joins), n, join_of, seg, lens, ends,
                                  C.c_void_p(inp.data_ptr() if inp.numel() else None),
                                  C.c_void_p(out.data_ptr() if out.numel() else None), out.numel(),
                                  C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
    if rc:
        raise RuntimeError(lib.fq3_join_last_error().decode())
    for j, k, _, e in pushes:
        if e:
            j.ended[k] = True
    return list(torch.split(out, counts))


def join(pcms: Sequence[torch.Tensor], pause_ms: int = 0, pauses=None) -> torch.Tensor:
    """The whole join of complete segments (1-D float32 on one CUDA device), each pushed once with its end."""
    j = Join(len(pcms), pause_ms, pcms[0].device, pauses)
    try:
        return process([j], [(j, k, p, True) for k, p in enumerate(pcms)])[0]
    finally:
        j.close()
