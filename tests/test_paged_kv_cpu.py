"""BatchScheduler's talker KV pages (batching.KvPager) without a GPU: a fake paged engine keeps page tables and a page
pool in which every frame writes its cache row and checks the rows before it, so a page lost, shared or restored wrong
shows up as a wrong row.  What is checked: page accounting after finish, cancel and cancel of a parked request;
admission when pages run out, also of a prompt of max_seq_len rows; that a request short of pages launches a whole
chunk or its last frames, never part of a chunk, so that a window decoding whole chunks gets the chunks it gets with
plenty of pages; the parking victim (largest ``due``, then the latest
admitted); that random arrivals on a pool of one full request plus a few pages always drain; and that an engine with
the default pool gets no page call at all."""
import numpy as np
import pytest
import torch

from oracle import prompt_cases  # noqa: F401  (puts the package on sys.path)
from faster_qwen3_tts import batching
from faster_qwen3_tts.batching import BatchScheduler
from faster_qwen3_tts.engine import KV_PAGE

S = 256   # max_seq_len: 4 pages


class _PagedEngine:
    """Request slots whose frame s writes cache row P + s (P = prompt rows) through the slot's page table; refuses what
    the real engine refuses (a page mapped twice or to two slots, work on unmapped rows)."""

    kv_page_bytes = KV_PAGE * 8

    def __init__(self, max_batch, max_slots, kv_pages, paged=True):
        self.max_batch, self.max_slots, self.max_seq_len, self.eos = max_batch, max_slots, S, -1
        self.paged, self.kv_pages = paged, kv_pages
        self.pool = torch.full((kv_pages, KV_PAGE), -1, dtype=torch.int64)
        self.table = {s: [] for s in range(max_slots)}
        self.gen_step0, self.P, self.total, self.done, self.page_calls, self.launches = {}, {}, {}, {}, [], []

    def _key(self, slot, row):
        return slot * 100000 + row * 10 + self.gen[slot]

    def _row(self, slot, row):
        return self.table[slot][row // KV_PAGE], row % KV_PAGE

    # ---- page ABI
    def map_kv_pages(self, slot, pages):
        self.page_calls.append(("map", slot, list(pages)))
        assert len(set(pages)) == len(pages) and len(pages) <= -(-self.max_seq_len // KV_PAGE)
        for s, t in self.table.items():
            assert s == slot or not set(t) & set(pages), "a page mapped to two slots"
        self.table[slot] = list(pages)

    def kv_pages_to(self, pages, dst):
        self.page_calls.append(("to", list(pages)))
        dst.view(torch.int64).view(len(pages), KV_PAGE).copy_(self.pool[list(pages)])

    def kv_pages_from(self, pages, src):
        self.page_calls.append(("from", list(pages)))
        self.pool[list(pages)] = src.view(torch.int64).view(len(pages), KV_PAGE)

    # ---- requests
    def begin(self, slot, P, total):
        self.gen = getattr(self, "gen", {})
        self.gen[slot] = self.gen.get(slot, 0) + 1   # a new request's rows differ from a former one's in the slot
        self.gen_step0[slot], self.P[slot], self.total[slot], self.done[slot] = 0, P, total, 0
        if self.paged:
            assert P <= KV_PAGE * len(self.table[slot]), "prefill into unmapped rows"
            for r in range(P):
                self.pool[self._row(slot, r)] = self._key(slot, r)

    def _emit(self, slot, budget):
        pos0 = self.P[slot] + self.done[slot]
        if self.paged:
            assert min(pos0 + budget, self.max_seq_len - 1) <= KV_PAGE * len(self.table[slot]), "budget past the mapped rows"
            for r in range(pos0):   # every row the next frame attends to is the one written
                assert self.pool[self._row(slot, r)] == self._key(slot, r), (slot, r)
        k, fin = 0, 0
        while k < budget:
            if self.done[slot] >= self.total[slot]:
                fin = 1
                break
            pos = self.P[slot] + self.done[slot]
            k += 1
            self.done[slot] += 1
            if pos >= self.max_seq_len - 1:
                fin = 3
                break
            if self.paged:
                self.pool[self._row(slot, pos)] = self._key(slot, pos)
        fin = fin or (1 if self.done[slot] >= self.total[slot] else 0)
        codes = torch.arange(self.done[slot] - k, self.done[slot])[:, None].repeat(1, 16) + 1000 * slot
        return codes, type("R", (), dict(frames_emitted=k, finished=fin, next_token=0))()

    def decode_chunk(self, n_frames, slot=0):
        self.launches.append({slot: n_frames})
        return self._emit(slot, n_frames)

    def decode_chunk_batch(self, slots, n_frames):
        budgets = [n_frames] * len(slots) if isinstance(n_frames, int) else list(n_frames)
        self.launches.append(dict(zip(slots, budgets)))
        outs = [self._emit(s, b) for s, b in zip(slots, budgets)]
        buf = torch.zeros(len(slots), max(budgets), 16, dtype=torch.long)
        for j, (c, _) in enumerate(outs):
            buf[j, : c.shape[0]] = c
        return buf, [r for _, r in outs]


@pytest.fixture
def make(monkeypatch):
    def mk(max_batch=4, max_slots=8, kv_pages=6, paged=True):
        eng = _PagedEngine(max_batch, max_slots, kv_pages, paged)

        def begin_batch(engine, talker, rows, config, pg, tg, slots, logprob=False):
            for s, r in zip(slots, rows):
                engine.begin(s, int(r["tie"].shape[1]), r["max_new_tokens"])

        def begin_one(engine, talker, tie, tam, tth, tpe, config, pg, tg, *, slot, max_new_tokens, **kw):
            engine.begin(slot, int(tie.shape[1]), max_new_tokens)

        monkeypatch.setattr(batching, "begin_fused_batch", begin_batch)
        monkeypatch.setattr(batching, "begin_fused", begin_one)
        return BatchScheduler(eng, None, None, None, None), eng
    return mk


def _req(P, n, tag=None, **kw):
    return dict(tie=torch.zeros(1, P, 1), tam=None, tth=None, tpe=None, tag=tag, max_new_tokens=n, **kw)


def _drain(sched, chunk, due=None, limit=10000):
    frames = {}
    for _ in range(limit):
        if not len(sched):
            return frames
        if due is not None:
            for rq in sched.active.values():
                rq.due = due(rq)
        for rq, c in sched.step(chunk):
            frames.setdefault(rq.tag, []).append(c)
    raise AssertionError("the scheduler did not drain")


def _no_leak(sched, eng):
    assert sorted(sched.pager.free) == list(range(eng.kv_pages)) and not sched.pager.mapped
    assert all(not t for t in eng.table.values())
    assert sorted(sched.free) == list(range(eng.max_slots))


def test_default_pool_makes_no_page_call(make):
    sched, eng = make(kv_pages=32, paged=False)
    assert sched.pager is None
    sched.submit_many([_req(30, 50, tag=i) for i in range(3)])
    rq = sched.submit(**_req(20, 40, tag=9))
    sched.step(8)
    sched.cancel(rq)
    got = _drain(sched, 8)
    assert eng.page_calls == [] and sorted(got) == [0, 1, 2]


def test_pages_come_back_after_finish_cancel_and_cancel_of_a_parked_request(make):
    sched, eng = make(max_batch=4, max_slots=8, kv_pages=5)
    a, b, c = sched.submit_many([_req(60, 150, tag="a"), _req(60, 150, tag="b"), _req(10, 20, tag="c")])
    assert sched.pager.in_use() == 3   # prompt + one frame: one page each
    a.due, b.due, c.due = 0.0, 5.0, 1.0
    for _ in range(100):   # a and b grow until neither can: then b, the larger due, is parked
        sched.step(8)
        if b.parked is not None:
            break
    assert "c" not in [rq.tag for rq in sched.active.values()]   # finished, its page is back
    assert b.parked is not None and sched.pager.parks == 1 and not sched.pager.mapped.get(b.slot)
    sched.cancel(b)                                              # a parked request
    assert b.parked is None and len(sched.pager.free) == 5 - len(sched.pager.mapped[a.slot])
    sched.cancel(a)
    _no_leak(sched, eng)


def test_admission_needs_pages_for_the_prompt_and_one_chunk(make):
    sched, eng = make(max_batch=4, max_slots=8, kv_pages=4)
    sched.step(16)                                               # the chunk admission reserves for: 16 frames
    assert sched.admits([_req(100, 50)]) and not sched.admits([_req(100, 50), _req(100, 50), _req(10, 5)])
    sched.submit_many([_req(100, 50, tag=0)])                    # 116 rows: 2 pages
    assert sched.pager.in_use() == 2 and sched.has_capacity()
    with pytest.raises(RuntimeError, match="KV pages"):
        sched.submit_many([_req(60, 50, tag=1), _req(120, 50, tag=2)])   # 2 + 3 pages
    assert sched.pager.in_use() == 2 and len(sched.free) == 7 and len(sched) == 1   # nothing taken
    sched.submit_many([_req(100, 50, tag=3, chunk_size=4)])      # its own chunk: 104 rows
    assert not sched.has_capacity() and not sched.admits([_req(1, 1)])
    with pytest.raises(RuntimeError, match="KV pages"):
        sched.submit(**_req(1, 1))
    _drain(sched, 16)
    _no_leak(sched, eng)


def test_short_of_pages_a_request_launches_a_whole_chunk_or_its_last_frames(make):
    sched, eng = make(max_batch=4, max_slots=4, kv_pages=5)
    x, y, z = sched.submit_many([_req(120, 200, tag="x"), _req(50, 14, tag="y"), _req(40, 40, tag="z")])
    assert sched.pager.in_use() == 4                             # 121, 51 and 41 rows: 2 + 1 + 1 pages of 5
    sched.step(12)     # x: rows to 132 -> its third page, the last free one; y to 62, z to 52
    assert eng.launches[-1] == {x.slot: 12, y.slot: 12, z.slot: 12} and not sched.pager.free
    sched.step(12)     # x fits 192 rows; y at 62 has 2 frames left and they fit 64 rows; z at 52 fits 12 frames
    assert eng.launches[-1] == {x.slot: 12, y.slot: 2, z.slot: 12}
    assert len(sched) == 2                                        # y is done: its page is free
    sched.pager.free, spare = [], sched.pager.free               # ... but not for z
    sched.step(12)     # z at 64: 12 frames do not fit, nor its 16 left, and part of a chunk is never launched
    assert eng.launches[-1] == {x.slot: 12} and z.parked is None
    sched.pager.free = spare
    _drain(sched, 12)
    _no_leak(sched, eng)


def test_admission_of_a_prompt_of_max_seq_len_rows(make):
    """max_seq_len % 64 == 1: the prompt's own rows need one page more than max_seq_len - 1 rows"""
    sched, eng = make(max_batch=2, max_slots=2, kv_pages=5)
    sched.max_seq_len = eng.max_seq_len = 257
    rq = sched.submit(**_req(257, 10, tag=0))
    assert sched.pager.rows(rq.slot) == 320
    _drain(sched, 8)
    _no_leak(sched, eng)


def test_a_window_that_decodes_whole_chunks_gets_the_chunks_of_plenty(make):
    """ContinuousBatcher on a pool where requests wait for pages and are parked: a window whose audio depends on the
    chunking receives every request's frames in the pushes it receives with plenty of pages, whole chunks of 8 and the
    remainder last"""
    from faster_qwen3_tts.serving import ContinuousBatcher
    sched, eng = make(max_batch=4, max_slots=6, kv_pages=6)
    pushes = {}

    class Window:
        any_chunking = False

        def __init__(self, tag, chunk=None):
            self.tag = tag

        def push(self, codes):
            pushes.setdefault(self.tag, []).append(int(codes.shape[0]))
            return np.zeros(int(codes.shape[0]), dtype=np.float32), 24000

    frames, prompts = [150, 61, 37, 90, 77, 45], [60, 10, 100, 30, 5, 120]
    b = ContinuousBatcher(sched, Window, chunk_size=8, idle_sleep=0.001)
    try:
        tickets = [b.submit((lambda P=P, i=i: (torch.zeros(1, P, 1), None, None, None, i)), max_new_tokens=n)
                   for i, (P, n) in enumerate(zip(prompts, frames))]
        audio = [t.audio() for t in tickets]
    finally:
        b.close()
    assert sched.pager.parks > 0
    for i, n in enumerate(frames):
        assert audio[i].shape[0] == n
        assert pushes[i] == [8] * (n // 8) + ([n % 8] if n % 8 else []), (i, pushes[i])
    _no_leak(sched, eng)


def test_victim_is_the_largest_due_then_the_latest_admitted(make):
    sched, eng = make(max_batch=4, max_slots=6, kv_pages=4)
    rqs = sched.submit_many([_req(63, 100, tag=i) for i in range(4)])   # prompt + one frame: one page each
    sched.step(1)                                                       # now every one is at row 64, no page free
    for rq, d in zip(rqs, (0.0, 3.0, 3.0, 1.0)):
        rq.due = d
    sched.step(4)   # nobody can advance: park 2 (due 3, admitted after 1); its page lets 0, the most urgent, go on
    assert [rq.tag for rq in rqs if rq.parked is not None] == [2]
    assert eng.launches[-1] == {rqs[0].slot: 4}
    rqs[2].due = -1.0      # now the most urgent: restored, into pages others gave up, once they cover it
    for _ in range(100):
        sched.step(4)
        if rqs[2].slot in eng.launches[-1]:
            break
    assert rqs[2].parked is None and rqs[2].slot in eng.launches[-1]
    assert [rq.tag for rq in rqs if rq.parked is not None] in ([1, 3], [1], [3])   # the victims after it
    _drain(sched, 4)
    _no_leak(sched, eng)


@pytest.mark.parametrize("seed", range(6))
def test_random_arrivals_on_one_full_request_plus_a_few_pages_drain(make, seed):
    rng = np.random.default_rng(seed)
    npt = -(-S // KV_PAGE)
    sched, eng = make(max_batch=4, max_slots=12, kv_pages=npt + int(rng.integers(0, 4)))
    want, arrivals, t = {}, [], 0
    for i in range(40):
        P = int(rng.integers(1, 120))
        arrivals.append((int(rng.integers(0, 3)) + t, i, P, int(rng.integers(1, S)), int(rng.integers(1, 20))))
        t = arrivals[-1][0]
    step, got = 0, {}
    while arrivals or len(sched):
        while arrivals and arrivals[0][0] <= step:
            _, i, P, n, chunk = arrivals[0]
            if not sched.admits([_req(P, n, chunk_size=chunk)]):
                break
            arrivals.pop(0)
            sched.submit(**_req(P, n, tag=i, chunk_size=chunk))
            want[i] = min(n, S - P)
        for rq in sched.active.values():
            rq.due = float(rng.normal())
        if rng.random() < 0.03 and len(sched):
            victim = list(sched.active.values())[int(rng.integers(0, len(sched)))]
            sched.cancel(victim)
            want.pop(victim.tag)
        for rq, c in sched.step(int(rng.integers(1, 24))):
            got[rq.tag] = got.get(rq.tag, 0) + int(c.shape[0])
        step += 1
        assert step < 20000, "no progress"
    assert all(got.get(i, 0) == n for i, n in want.items()), (want, got)
    _no_leak(sched, eng)
