"""Batched admission without a GPU: the continuous batcher hands every ready request that fits the free slots to ONE
``submit_many`` call (one batched prefill), fails a request whose prompt cannot be built or is too long on its own, and
still serves a scheduler that only has ``submit`` one request at a time; ``BatchScheduler.submit_many`` latches what
consecutive ``submit`` calls latch, text-fed requests included; ``begin_fused_batch`` latches every row as
``begin_fused`` does, from one batched prefill."""
import threading
import time
import types

import numpy as np
import pytest
import torch

from oracle import prompt_cases  # noqa: F401  (puts the package on sys.path)
from faster_qwen3_tts import batching, generate
from faster_qwen3_tts.serving import ContinuousBatcher


class _Gated(ContinuousBatcher):
    """the worker admits nothing until ``gate`` is set: a burst submitted before that is one admission round"""

    def __init__(self, *a, **kw):
        self.gate = threading.Event()
        super().__init__(*a, **kw)

    def _admit(self):
        self.gate.wait()
        super()._admit()


class _Req:
    def __init__(self, tag, total):
        self.tag, self.total, self.done, self.finished = tag, total, 0, 0


class _Sched:
    """max_batch slots, prompts up to max_seq_len rows; every step emits min(n, remaining) frames per request."""

    def __init__(self, max_batch, max_seq_len=100, many=True):
        self.max_batch, self.max_seq_len, self.active = max_batch, max_seq_len, {}
        self.many_calls, self.submit_calls = [], []
        if many:
            self.submit_many = self._submit_many

    def __len__(self):
        return len(self.active)

    def has_capacity(self):
        return len(self.active) < self.max_batch

    def capacity(self):
        return self.max_batch - len(self.active)

    def _add(self, tag, max_new_tokens):
        assert len(self.active) < self.max_batch
        rq = self.active[tag] = _Req(tag, max_new_tokens)
        return rq

    def submit(self, tie, tam, tth, tpe, tag=None, max_new_tokens=0, **kw):
        self.submit_calls.append(tag)
        return self._add(tag, max_new_tokens)

    def _submit_many(self, reqs):
        self.many_calls.append([r["tag"] for r in reqs])
        return [self._add(r["tag"], r["max_new_tokens"]) for r in reqs]

    def step(self, n):
        out = []
        for tag, rq in list(self.active.items()):
            k = min(n, rq.total - rq.done)
            codes = np.arange(rq.done, rq.done + k, dtype=np.int64)[:, None] + 1000 * tag
            rq.done += k
            if rq.done >= rq.total:
                rq.finished = 1
                del self.active[tag]
            out.append((rq, codes))
        time.sleep(0.001)
        return out


class _Win:
    def __init__(self, ref):
        pass

    def push(self, codes):
        return codes[:, 0].astype(np.float32), 24000


def _prompt(P):
    return lambda: (np.zeros((1, P, 4)), None, None, None, None)


def _serve(sched, prepares, totals):
    b = _Gated(sched, _Win, chunk_size=4, idle_sleep=0.0005)
    tickets = [b.submit(p, max_new_tokens=n) for p, n in zip(prepares, totals)]
    b.gate.set()
    try:
        got = []
        for t in tickets:
            try:
                got.append(t.audio())
            except Exception as ex:   # noqa: BLE001 -- the ticket's own failure is the result
                got.append(ex)
    finally:
        b.close()
    return tickets, got


def test_admit_groups_ready_tickets_into_one_submit_many_up_to_the_free_slots():
    sched = _Sched(max_batch=3)
    totals = [5, 9, 3, 7, 2]
    tickets, got = _serve(sched, [_prompt(10)] * 5, totals)
    rids = [t.rid for t in tickets]
    assert sched.many_calls[0] == rids[:3]                       # the burst fills every free slot in one call
    assert sorted(sum(sched.many_calls, [])) == rids and not sched.submit_calls
    for t, a, n in zip(tickets, got, totals):
        assert a.tolist() == [1000 * t.rid + k for k in range(n)]


def test_a_bad_prepare_or_an_over_long_prompt_fails_only_its_own_ticket():
    sched = _Sched(max_batch=4, max_seq_len=100)

    def broken():
        raise ValueError("bad prompt")
    tickets, got = _serve(sched, [_prompt(10), broken, _prompt(101), _prompt(100)], [4, 4, 4, 6])
    assert sched.many_calls == [[tickets[0].rid, tickets[3].rid]]
    assert isinstance(got[1], ValueError)
    assert isinstance(got[2], RuntimeError) and "Input is too long: prefill has 101 tokens but max_seq_len=100" in str(got[2])
    assert got[0].tolist() == [1000 * tickets[0].rid + k for k in range(4)]
    assert got[3].tolist() == [1000 * tickets[3].rid + k for k in range(6)]


def test_a_scheduler_without_submit_many_is_served_one_ticket_at_a_time():
    sched = _Sched(max_batch=2, many=False)
    tickets, got = _serve(sched, [_prompt(10)] * 3, [3, 5, 2])
    assert sched.submit_calls == [t.rid for t in tickets] and not sched.many_calls
    for t, a, n in zip(tickets, got, [3, 5, 2]):
        assert a.tolist() == [1000 * t.rid + k for k in range(n)]


# ---- BatchScheduler.submit_many against a fake engine --------------------------------------------------------------
class _Feed:
    def __init__(self, n_rows=0, closed=False):
        self.n_rows, self.closed = n_rows, closed

    def update(self):
        return self.n_rows


class _Engine:
    def __init__(self, max_batch):
        self.max_batch, self.max_seq_len = max_batch, 64
        self.gen_step0, self.rows, self.begun = {}, {}, {}

    def set_text_rows(self, slot, n, open):
        self.rows[slot] = (n, open)


def _fake_begin(engine, slot, trailing_len, kw):
    engine.gen_step0[slot] = 3 + slot
    engine.begun[slot] = (trailing_len, kw["max_new_tokens"], kw["do_sample"])


def _requests():
    z = torch.zeros(1)
    return [dict(tie=z, tam=z, tth=z, tpe=z, tag="plain", max_new_tokens=9),
            dict(tie=z, tam=z, tth=z, tpe=z, tag="a", feed=_Feed(0), rows_ahead=4, do_sample=False),
            dict(tie=z, tam=z, tth=z, tpe=z, tag="b", feed=_Feed(5, closed=True))]


def _state(sched, rqs):
    e = sched.engine
    return ([(r.slot, r.tag, r.max_new_tokens, r.gen0, r.rows_ahead, r.feed is not None) for r in rqs],
            dict(e.rows), dict(e.begun), list(sched.free))


def test_submit_many_latches_like_consecutive_submits(monkeypatch):
    def one(engine, *a, slot=None, trailing_len=None, **kw):
        _fake_begin(engine, slot, trailing_len, kw)

    def many(engine, talker, rows, config, pg, tg, slots):
        for r, s in zip(rows, slots):
            _fake_begin(engine, s, r["trailing_len"], r)
    monkeypatch.setattr(batching, "begin_fused", one)
    monkeypatch.setattr(batching, "begin_fused_batch", many)
    a = batching.BatchScheduler(_Engine(4), None, None, None, None)
    a.cancel(a.submit(torch.zeros(1), None, None, None))         # slot 0 goes to the back of the free list
    want = _state(a, [a.submit(**r) for r in _requests()])
    b = batching.BatchScheduler(_Engine(4), None, None, None, None)
    b.cancel(b.submit(torch.zeros(1), None, None, None))
    got = _state(b, b.submit_many(_requests()))
    assert got == want
    assert got[1] == {2: (0, True), 3: (5, False)}                # text-fed rows announced, open / closed
    assert got[2][2] == (0, 2048, False) and got[2][1] == (None, 9, True)
    with pytest.raises(RuntimeError, match="slots are free"):
        b.submit_many(_requests())
    assert b.free == [0]


def test_submit_many_releases_every_slot_when_the_prefill_fails(monkeypatch):
    def many(*a, **kw):
        raise RuntimeError("Input is too long")
    monkeypatch.setattr(batching, "begin_fused_batch", many)
    s = batching.BatchScheduler(_Engine(4), None, None, None, None)
    with pytest.raises(RuntimeError):
        s.submit_many(_requests())
    assert s.free == [0, 1, 2, 3] and not s.active


# ---- begin_fused_batch against begin_fused, on a fake K3 engine --------------------------------------------------
class _K3Engine:
    """records the latches; its 'prefill' is a function of the prompt alone, so batched and single calls agree"""
    has_prefill, device, H, V = True, torch.device("cpu"), 4, 6

    def __init__(self):
        self.log, self.prefills, self.gen_step0 = [], [], {}

    def _one(self, x, pad):
        lg = torch.arange(self.V, dtype=torch.float32) * float(x.sum()) + pad
        return lg, x[-1] * 2

    def prefill(self, x, pad, slot=0):
        self.prefills.append([slot])
        return self._one(x, pad)

    def prefill_batch(self, rows, pads, slots):
        self.prefills.append(list(slots))
        outs = [self._one(x, p) for x, p in zip(rows, pads)]
        return torch.stack([o[0] for o in outs]), torch.stack([o[1] for o in outs])

    def sample_logits(self, logits, sp, u=0.0, **kw):
        return (logits.reshape(-1).argmax() + int(u * 10)).view(1)

    def set_generation_state(self, pad, rope_delta, slot=0):
        self.log.append(("state", slot, pad, rope_delta))

    def begin_request(self, *, past_hidden, uniforms, **kw):
        self.log.append(("begin", kw["slot"], tuple(past_hidden.reshape(-1).tolist()),
                         None if uniforms is None else float(uniforms.reshape(-1)[0]),
                         tuple(sorted((k, v) for k, v in kw.items() if not isinstance(v, torch.Tensor) and k != "sp_predictor"))))


def test_begin_fused_batch_latches_every_row_as_begin_fused_does():
    pg = types.SimpleNamespace(do_sample=False, sampling=lambda: None)
    tg = types.SimpleNamespace(slot=0)
    cfg = types.SimpleNamespace(codec_eos_token_id=2)
    g = torch.Generator().manual_seed(0)
    rows = []
    for P, pad, ds in ((5, 0, True), (3, 1, False), (7, 4, True)):
        tam = torch.ones(1, P, dtype=torch.long)
        tam[0, :pad] = 0
        rows.append(dict(tie=torch.randn(1, P, 4, generator=g), tam=tam, tth=torch.zeros(1, 2, 4), tpe=torch.zeros(1, 1, 4),
                         max_new_tokens=5, min_new_tokens=2, temperature=0.9, top_k=50, top_p=1.0, do_sample=ds,
                         repetition_penalty=1.05, uniforms=torch.rand(6, 16, generator=g) if ds else None,
                         trailing_len=None))
    slots = [2, 0, 1]
    single = _K3Engine()
    want = [int(generate.begin_fused(single, None, r["tie"], r["tam"], r["tth"], r["tpe"], cfg, pg, tg, slot=s,
                                     **{k: v for k, v in r.items() if k not in ("tie", "tam", "tth", "tpe")}))
            for r, s in zip(rows, slots)]
    batched = _K3Engine()
    got = generate.begin_fused_batch(batched, None, rows, cfg, pg, tg, slots)
    assert got == want
    assert batched.prefills == [slots] and single.prefills == [[s] for s in slots]
    assert batched.log == single.log
