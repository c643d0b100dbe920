"""Serving more listeners than a launch has columns, without a GPU: ``BatchScheduler`` on a fake engine that records its
calls, and ``ContinuousBatcher`` on a fake clock.  What is checked: which requests a step launches when more are ready than
``max_batch`` (smallest lead first), that nobody starves, when underruns are counted, the watermark, per-request chunk
sizes, that unpaced traffic makes exactly the calls it made before, and the ctypes mirror of ``fq3_config``."""
import os
import subprocess
import threading
import types

import pytest
import torch

from oracle import prompt_cases  # noqa: F401  (puts the package on sys.path)
from faster_qwen3_tts import batching, engine as E
from faster_qwen3_tts.batching import BatchScheduler, SlotRequest
from faster_qwen3_tts.serving import ContinuousBatcher

FRAME_S = 0.08


class _Engine:
    """Request slots that emit frames numbered from 0; records every decode call."""

    def __init__(self, max_batch, max_slots=None, total=1000):
        self.max_batch, self.max_seq_len, self.eos = max_batch, 64, -1
        if max_slots is not None:
            self.max_slots = max_slots
        self.gen_step0, self.total, self.done, self.calls, self.text = {}, {}, {}, [], {}
        self.default_total = total

    def begin(self, slot, total):
        self.gen_step0[slot], self.total[slot], self.done[slot] = 0, total, 0

    def set_text_rows(self, slot, n, open):
        self.text[slot] = (n, open)

    def _emit(self, slot, budget):
        k = min(budget, self.total[slot] - self.done[slot])
        if slot in self.text and self.text[slot][1]:
            k = min(k, self.text[slot][0] - self.done[slot])
        codes = torch.arange(self.done[slot], self.done[slot] + k)[:, None].repeat(1, 16) + 1000 * slot
        self.done[slot] += k
        return codes, types.SimpleNamespace(frames_emitted=k, finished=int(self.done[slot] >= self.total[slot]),
                                            next_token=0)

    def decode_chunk(self, n_frames, slot=0):
        self.calls.append(("one", slot, n_frames))
        return self._emit(slot, n_frames)

    def decode_chunk_batch(self, slots, n_frames):
        self.calls.append(("batch", list(slots), n_frames if isinstance(n_frames, int) else list(n_frames)))
        budgets = [n_frames] * len(slots) if isinstance(n_frames, int) else n_frames
        outs = [self._emit(s, b) for s, b in zip(slots, budgets)]
        F = max(budgets)
        buf = torch.zeros(len(slots), F, 16, dtype=torch.long)
        for j, (c, _) in enumerate(outs):
            buf[j, : c.shape[0]] = c
        return buf, [r for _, r in outs]


@pytest.fixture
def sched_for(monkeypatch):
    """BatchScheduler over a fake engine; the prefill is replaced by the fake's latch"""
    def make(max_batch, max_slots=None):
        eng = _Engine(max_batch, max_slots)

        def begin_batch(engine, talker, rows, config, pg, tg, slots, logprob=False):
            for s, r in zip(slots, rows):
                engine.begin(s, r["max_new_tokens"])

        def begin_one(engine, talker, tie, tam, tth, tpe, config, pg, tg, *, slot, max_new_tokens, **kw):
            engine.begin(slot, max_new_tokens)

        monkeypatch.setattr(batching, "begin_fused_batch", begin_batch)
        monkeypatch.setattr(batching, "begin_fused", begin_one)
        return BatchScheduler(eng, None, None, None, None), eng
    return make


def _req(tag, n=1000, **kw):
    return dict(tie=None, tam=None, tth=None, tpe=None, tag=tag, max_new_tokens=n, **kw)


def test_more_ready_than_columns_launches_the_32_with_the_smallest_due(sched_for):
    sched, eng = sched_for(32, 80)
    assert sched.capacity() == 80
    rqs = sched.submit_many([_req(i) for i in range(32)]) + sched.submit_many([_req(32 + i) for i in range(32)]) + \
        sched.submit_many([_req(64 + i) for i in range(16)])
    assert not sched.has_capacity() and [rq.slot for rq in rqs] == list(range(80))
    for rq in rqs:
        rq.due = float((rq.tag * 37) % 80)          # a permutation of 0..79
    out = sched.step(8)
    want = sorted(rq.slot for rq in rqs if rq.due < 32)
    assert eng.calls == [("batch", want, 8)] and sorted(rq.slot for rq, _ in out) == want
    # ties: the request admitted first; a request on hold is passed over
    eng.calls.clear()
    for rq in rqs:
        rq.due = 0.0
    rqs[3].hold = True
    before = dict(eng.done)
    sched.step(8)
    assert eng.calls == [("batch", [s for s in range(33) if s != 3], 8)]
    # the others kept their slots and state: nothing was emitted for them
    assert all(eng.done[s] == before[s] for s in [3] + list(range(33, 80)))


def test_at_most_max_batch_active_makes_the_calls_made_without_max_slots(sched_for):
    """same submissions and steps on an engine with spare resident slots and on one without: identical engine calls"""
    logs = []
    for max_slots in (None, 64):
        sched, eng = sched_for(4, max_slots)
        sched.submit_many([_req(0, 9), _req(1, 20)])
        sched.submit(None, None, None, None, tag=2, max_new_tokens=5)
        got = {}
        while len(sched):
            for rq, codes in sched.step(4):
                got.setdefault(rq.tag, []).append(codes)
            if len(sched) == 2 and 3 not in got:
                sched.submit_many([_req(3, 6)])
                got[3] = []
        logs.append((eng.calls, {k: torch.cat(v).tolist() for k, v in got.items()}))
    assert logs[0] == logs[1]
    assert logs[0][0][0] == ("batch", [0, 1, 2], 4) and logs[0][0][-1][0] == "one"   # int n_frames, single-slot call at the end


def test_chunk_size_and_first_chunk_per_request(sched_for):
    sched, eng = sched_for(8, 16)
    a, b, c = sched.submit_many([_req(0, 30, chunk_size=4), _req(1, 30, first_chunk=2), _req(2, 30)])
    assert (a.budget(8), b.budget(8), c.budget(8)) == (4, 2, 8)
    sched.step(8)
    sched.step(8)
    assert eng.calls == [("batch", [0, 1, 2], [4, 2, 8]), ("batch", [0, 1, 2], [4, 8, 8])]
    assert (a.frames, b.frames, c.frames) == (8, 10, 16)
    sched.cancel(a)
    sched.step(8)
    assert eng.calls[-1] == ("batch", [1, 2], 8)      # equal budgets: the call of a scheduler without the option
    sched.cancel(c)
    d = sched.submit(None, None, None, None, tag=3, max_new_tokens=30, chunk_size=3, first_chunk=1)
    sched.cancel(b)
    sched.step(8)
    sched.step(8)
    assert eng.calls[-2:] == [("one", d.slot, 1), ("one", d.slot, 3)]
    for bad in (dict(chunk_size=0), dict(first_chunk=-1)):
        with pytest.raises(ValueError, match="at least 1 frame"):
            sched.submit_many([_req(9, **bad)])
    assert sched.capacity() == 15


class _Feed:
    def __init__(self):
        self.n_rows, self.closed = 0, False

    def update(self):
        return self.n_rows


def test_text_fed_requests_get_full_chunks_when_budgets_differ(sched_for):
    """rows_ahead is the request's own chunk size: a text-fed slot is launched only when a full chunk of its rows exists,
    next to a slot with another budget"""
    sched, eng = sched_for(4, 8)
    feed = _Feed()
    a, b = sched.submit_many([_req(0, 40, chunk_size=4, feed=feed, rows_ahead=4), _req(1, 100, chunk_size=8)])
    emitted = []
    for rows in (2, 3, 4, 6, 9, 12, 12):
        feed.n_rows = rows
        for rq, codes in sched.step(8):
            if rq is a:
                emitted.append(int(codes.shape[0]))
    assert emitted == [4, 4, 4]                       # at 4, 9 and 12 rows; never a short chunk
    assert [c for c in eng.calls if c[0] == "batch"][0] == ("batch", [0, 1], [4, 8])
    assert b.frames == 7 * 8


# ---- the worker on a fake clock -----------------------------------------------------------------------------------------
class _Clock:
    def __init__(self):
        self.t, self.lock = 0.0, threading.Lock()

    def __call__(self):
        return self.t

    def sleep(self, dt):
        with self.lock:
            self.t += dt


class _PacedSched:
    """max_slots requests, max_batch per step by (due, seq) as BatchScheduler does; a step costs ``step_s`` of the fake
    clock.  Admits nothing before ``go`` is set and starts stepping once ``expect`` requests are in, so that the run does
    not depend on thread timing: only the worker thread moves the fake clock."""

    def __init__(self, clock, max_batch, max_slots, step_s, expect):
        self.clock, self.max_batch, self.max_slots, self.step_s, self.expect = clock, max_batch, max_slots, step_s, expect
        self.active, self.launched, self.seq, self.started = {}, [], 0, False
        self.max_prompts = max_batch
        self.admitted, self.go = [], threading.Event()

    def __len__(self):
        self.started = self.started or self.seq >= self.expect
        return len(self.active) if self.started else 0

    def capacity(self):
        return self.max_slots - len(self.active) if self.go.is_set() else 0

    def has_capacity(self):
        return self.capacity() > 0

    def submit_many(self, reqs):
        assert len(reqs) <= self.max_prompts
        self.admitted.append(len(reqs))
        out = []
        for r in reqs:
            self.seq += 1
            rq = SlotRequest(slot=self.seq, tag=r["tag"], max_new_tokens=r["max_new_tokens"], seq=self.seq,
                             chunk_size=r.get("chunk_size"), first_chunk=r.get("first_chunk"))
            self.active[rq.tag] = rq
            out.append(rq)
        return out

    def cancel(self, rq):
        self.active.pop(rq.tag, None)

    def step(self, n):
        ready = sorted((rq for rq in self.active.values() if rq.ready()), key=lambda rq: (rq.due, rq.seq))[: self.max_batch]
        if not ready:
            return []
        self.launched.append([(rq.tag, rq.due) for rq in ready])
        self.t_first = self.clock() if len(self.launched) == 1 else self.t_first
        self.clock.sleep(self.step_s)
        self.t_last = self.clock()
        out = []
        for rq in ready:
            k = min(rq.budget(n), rq.max_new_tokens - rq.frames)
            rq.frames += k
            rq.finished = int(rq.frames >= rq.max_new_tokens)
            if rq.finished:
                del self.active[rq.tag]
            out.append((rq, torch.zeros(k, 16, dtype=torch.long)))
        return out


class _Win:
    any_chunking = True

    def __init__(self, ref, chunk=None):
        pass

    def push(self, codes):
        return codes[:, 0].numpy(), 24000


def _serve(n_listeners, step_s, frames=200, max_batch=32, pace=1.0, lead_high_s=2.0, **gen):
    clock = _Clock()
    sched = _PacedSched(clock, max_batch, n_listeners, step_s, expect=n_listeners)
    b = ContinuousBatcher(sched, _Win, chunk_size=8, idle_sleep=0.01, lead_high_s=lead_high_s, frame_s=FRAME_S,
                          clock=clock, sleep=clock.sleep)
    try:
        tickets = [b.submit(lambda: (torch.zeros(1, 4, 8), 0, 0, 0, None), pace=pace, max_new_tokens=frames, **gen)
                   for _ in range(n_listeners)]
        sched.go.set()
        chunks = [[c[2]["chunk_steps"] for c in t] for t in tickets]
    finally:
        b.close()
    return tickets, chunks, sched, sched.t_last - sched.t_first   # ... and the fake time from first to last launch


def test_paced_listeners_with_headroom_never_run_dry_and_none_starves():
    # 96 listeners, 3 launches of 32 serve everyone once: 0.3 s per 0.64 s of audio each
    tickets, chunks, sched, took = _serve(96, step_s=0.1)
    assert sched.admitted == [32, 32, 32]                              # one submit_many per 32 prompts
    assert all(sum(c) == 200 for c in chunks)                           # every listener got all its audio
    assert [t.underruns for t in tickets] == [0] * 96
    assert all(len(l) <= 32 for l in sched.launched) and max(len(l) for l in sched.launched) == 32
    # who ran was whoever had the smallest lead: nobody left out of a launch was more urgent than somebody in it
    # (the first launches are all -inf: no audio yet, oldest first)
    assert [tag for tag, _ in sched.launched[0]] == [t.rid for t in tickets[:32]]
    assert {tag for l in sched.launched[:3] for tag, _ in l} == {t.rid for t in tickets}
    # the engine was not kept busy making audio nobody would hear for seconds: the run took about as long as the audio
    assert took > 200 * FRAME_S - 2.0 - 1.0
    assert max(t.lead_s for t in tickets) < 2.0 + 8 * FRAME_S + 1e-9


def test_underruns_are_counted_when_the_steps_are_too_slow():
    # 96 listeners but a launch takes 0.3 s: a round of 3 launches makes 0.64 s of audio per listener in 0.9 s
    tickets, chunks, sched, _ = _serve(96, step_s=0.3, frames=120)
    assert all(sum(c) == 120 for c in chunks)
    assert all(t.underruns > 0 for t in tickets)
    # and still nobody starves: the deliveries are spread evenly (lead order = round robin under overload)
    n = [len(c) for c in chunks]
    assert max(n) - min(n) <= 1


def test_a_listener_at_the_watermark_is_skipped_and_comes_back():
    tickets, chunks, sched, took = _serve(2, step_s=0.05, frames=80, max_batch=2, lead_high_s=1.0)
    assert [t.underruns for t in tickets] == [0, 0] and all(sum(c) == 80 for c in chunks)
    # leads at launch stay below the watermark; with 0.64 s per chunk against 0.05 s per step the worker idled
    assert all(due < 1.0 for l in sched.launched for _, due in l)
    assert len(sched.launched) == 10 and took >= 80 * FRAME_S - 1.0 - 0.64 - 0.05


def test_unpaced_tickets_are_never_held_and_keep_due_zero():
    tickets, chunks, sched, took = _serve(40, step_s=0.1, frames=40, pace=None)
    assert all(due == 0.0 for l in sched.launched for _, due in l)
    assert [t.underruns for t in tickets] == [0] * 40 and all(t.lead_s == 0.0 for t in tickets)
    # as fast as possible and first come first served (equal due: admission order): the first 32 take their 5 launches,
    # then the other 8 theirs; the worker never idles
    assert len(sched.launched) == 10 and abs(took - 1.0) < 1e-6
    assert [len(l) for l in sched.launched] == [32] * 5 + [8] * 5
    with pytest.raises(ValueError, match="pace must be positive"):
        ContinuousBatcher.__dict__["_pace"].__func__(0)


def test_first_chunk_needs_a_window_that_allows_any_chunking():
    clock = _Clock()
    sched = _PacedSched(clock, 4, 8, 0.01, expect=2)

    class Window(_Win):
        any_chunking = False

    b = ContinuousBatcher(sched, Window, chunk_size=8, idle_sleep=0.01, clock=clock, sleep=clock.sleep)
    try:
        bad = b.submit(lambda: (torch.zeros(1, 4, 8), 0, 0, 0, None), max_new_tokens=8, first_chunk=2)
        sched.go.set()
        with pytest.raises(ValueError, match="first_chunk needs"):
            list(bad)
    finally:
        b.close()
    tickets, chunks, _, _ = _serve(3, step_s=0.01, frames=20, max_batch=4, first_chunk=2, chunk_size=6)
    assert chunks == [[2, 6, 6, 6]] * 3


# ---- the engine's config struct and slot arithmetic ---------------------------------------------------------------------
def test_ctypes_config_mirrors_the_c_struct(tmp_path):
    """size and offset of every fq3_config field, as the C compiler lays the header's struct out"""
    names = [n for n, _ in E.Config._fields_]
    assert names[-2:] == ["max_batch", "max_slots"]
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "fq3_engine.h"\nint main(void) {\n'
                   '  printf("%zu\\n", sizeof(fq3_config));\n'
                   + "".join(f'  printf("%zu\\n", offsetof(fq3_config, {n}));\n' for n in names)
                   + '  printf("%d\\n", FQ3_MAX_SLOTS);\n  return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.run([os.environ.get("CC", "cc"), "-I", E.INCLUDE, "-o", str(exe), str(src)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got[0] == E.C.sizeof(E.Config)
    assert got[1:-1] == [getattr(E.Config, n).offset for n in names]
    assert got[-1] == 256


def test_slot_bytes_arithmetic():
    """what max_slots multiplies: 2 x (talker + predictor) KV + loop state + past hidden + penalty bitmap"""
    t17 = dict(hidden_size=2048, intermediate_size=6144, num_hidden_layers=28, num_attention_heads=16,
               num_key_value_heads=8, vocab_size=3072)
    p17 = dict(hidden_size=1024, intermediate_size=3072, num_hidden_layers=5, num_attention_heads=16,
               num_key_value_heads=8, vocab_size=2048)
    try:
        E.load_library()
    except RuntimeError:
        pytest.skip("engine library not built")
    b = E.slot_bytes(t17, p17, torch.bfloat16, 2048)
    tkv = 2 * 28 * 8 * 2048 * 128 * 2
    pkv = 2 * 5 * 8 * 32 * 128 * 2
    assert 0 < b - tkv - pkv < 64 * 1024   # loop state, past hidden, penalty bitmap
    assert tkv == 234_881_024 and 0 < b - tkv < 4 * 2 ** 20                          # "234 MB of talker KV per slot"
    assert E.slot_bytes(t17, p17, torch.float32, 2048) - b == tkv + pkv               # fp32 doubles the caches only
    assert E.slot_bytes(t17, p17, torch.bfloat16, 1024) < b / 2 + 2 ** 20
    assert 128 * b < 32 * 2 ** 30 and 256 * b > 56 * 2 ** 30                          # 128 slots: 30 GB; 256: 60 GB


# ---- the worker over the real BatchScheduler ----------------------------------------------------------------------------
def test_worker_over_batch_scheduler_serves_96_listeners_on_32_columns(sched_for):
    """ContinuousBatcher -> BatchScheduler -> recording fake engine whose launches cost fake time: the scheduler's own
    selection by (due, admission order), fed the worker's leads, serves everyone without underruns and nobody starves"""
    clock = _Clock()
    sched, eng = sched_for(32, 96)
    real_batch, capacity, go = eng.decode_chunk_batch, sched.capacity, threading.Event()

    def timed_batch(slots, n_frames):
        clock.sleep(0.1)
        return real_batch(slots, n_frames)

    eng.decode_chunk_batch = timed_batch
    sched.capacity = lambda: capacity() if go.is_set() else 0      # admit once every ticket is in: no thread timing
    b = ContinuousBatcher(sched, _Win, chunk_size=8, idle_sleep=0.01, frame_s=FRAME_S, clock=clock, sleep=clock.sleep)
    try:
        tickets = [b.submit(lambda: (torch.zeros(1, 4, 8), 0, 0, 0, None), pace=1.0, max_new_tokens=200)
                   for _ in range(96)]
        go.set()
        chunks = [[c[2]["chunk_steps"] for c in t] for t in tickets]
    finally:
        b.close()
    assert all(sum(c) == 200 for c in chunks) and [t.underruns for t in tickets] == [0] * 96
    launches = [c for c in eng.calls if c[0] == "batch"]
    assert max(len(c[1]) for c in launches) == 32 and all(len(c[1]) <= 32 for c in launches)
    assert launches[:3] == [("batch", list(range(i, i + 32)), 8) for i in (0, 32, 64)]   # no audio yet: oldest first
    assert {s for c in eng.calls for s in (c[1] if c[0] == "batch" else [c[1]])} == set(range(96))
    assert b.max_concurrent == 96 and len(sched) == 0


def test_window_factory_gets_the_tickets_own_chunk_size():
    clock, seen = _Clock(), []
    sched = _PacedSched(clock, 4, 8, 0.01, expect=2)

    def factory(ref, chunk=None):
        seen.append(chunk)
        return _Win(ref)

    b = ContinuousBatcher(sched, factory, chunk_size=8, idle_sleep=0.01, clock=clock, sleep=clock.sleep)
    try:
        tickets = [b.submit(lambda: (torch.zeros(1, 4, 8), 0, 0, 0, None), max_new_tokens=60, **kw)
                   for kw in ({}, {"chunk_size": 28})]
        sched.go.set()
        chunks = [[c[2]["chunk_steps"] for c in t] for t in tickets]
    finally:
        b.close()
    assert seen == [None, 28] and chunks == [[8] * 7 + [4], [28, 28, 4]]
