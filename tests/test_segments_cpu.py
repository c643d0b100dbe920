"""Long inputs without a GPU: the splitter's rule, the numpy oracle of the join, and a segmented request through
``ContinuousBatcher`` on a fake scheduler, fake codec windows and a fake joiner (admission order, in-order delivery when
rows finish in reverse order, cancel, the ``due`` / ``hold`` of later segments), and the refusals."""
import os
import re
import threading
import time

import numpy as np
import pytest
import torch

from oracle import prompt_cases  # noqa: F401  (puts the package on sys.path)
from faster_qwen3_tts import join as J
from faster_qwen3_tts import segment as S
from faster_qwen3_tts.serving import ContinuousBatcher, Segments, segment_requests

import join_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- splitter -------------------------------------------------------------------------------------------------------
def _rejoins(text, segs):
    """text == w0 s0 w1 s1 ... with whitespace-only w"""
    pos = 0
    for s in segs:
        i = text.index(s, pos)
        assert text[pos:i].strip() == "", (text[pos:i], s)
        pos = i + len(s)
    assert text[pos:].strip() == ""


TEXTS = [
    "Hello there. How are you today? I am fine; thanks!  And you?\nNew line here",
    "今天天气很好。我们去公园吧！你觉得怎么样？好；走吧",
    "no punctuation at all " * 40,
    "x" * 1000,
    "   leading and trailing whitespace.   \n\n  ",
    "Mr. Smith paid 3.50 dollars. e.g. this. Done",
    "",
    "   \n ",
]


@pytest.mark.parametrize("max_chars", [1, 7, 40, 400])
@pytest.mark.parametrize("text", TEXTS)
def test_split_rejoins_and_respects_max_chars(text, max_chars):
    segs = S.split_text(text, max_chars)
    _rejoins(text, segs)
    assert all(1 <= len(s) <= max_chars for s in segs)
    assert all(s == s.strip() for s in segs)
    assert S.split_text(text, max_chars) == segs   # deterministic
    if not text.strip():
        assert segs == []


def test_split_sentences_cjk_and_merges():
    assert S.split_text("The first sentence is long enough. The second one is long enough too.", 400) == [
        "The first sentence is long enough.", "The second one is long enough too."]
    # short pieces merge into the next one
    assert S.split_text("Hi. Yes. This sentence is long enough by itself.", 400) == [
        "Hi. Yes. This sentence is long enough by itself."]
    assert S.split_text("今天天气很好，阳光明媚，适合出去走走。我们去公园吧，带上孩子们一起去玩！", 400, min_chars=1) == [
        "今天天气很好，阳光明媚，适合出去走走。", "我们去公园吧，带上孩子们一起去玩！"]
    # "3.50" and "e.g" do not end a sentence (no whitespace after the mark)
    assert S.split_text("It costs 3.50 dollars in total today. Done", 400, min_chars=1) == [
        "It costs 3.50 dollars in total today.", "Done"]
    assert S.split_text("line one\nline two", 400, min_chars=1) == ["line one", "line two"]


def test_split_hard_cuts_at_the_last_space():
    segs = S.split_text("aaaa bbbb cccc dddd", 10, min_chars=1)
    assert segs == ["aaaa bbbb", "cccc dddd"]
    assert S.split_text("abcdefghij" * 3, 10) == ["abcdefghij"] * 3
    assert S.split_text("ab,cdefghijkl", 5, min_chars=1) == ["ab,", "cdefg", "hijkl"]


def test_split_refusals_and_seeds():
    for bad in (0, -1, 2.5, True, "400"):
        with pytest.raises(ValueError):
            S.split_text("text", bad)
    assert S.segment_seed(7, 0) == 7
    assert S.segment_seed(7, 3) == (7 + 3 * 0x9E3779B97F4A7C15) % 2 ** 63
    assert len({S.segment_seed(1, k) for k in range(100)}) == 100


# ---- the join oracle ------------------------------------------------------------------------------------------------
def test_constants_agree_with_the_header():
    h = open(os.path.join(ROOT, "include", "fq3_engine.h")).read()
    val = dict(re.findall(r"#define FQ3_JOIN_(\w+) (\d+)", h))
    assert (int(val["RATE"]), int(val["FADE"]), int(val["PAUSE_MAX_MS"])) == (J.RATE, J.FADE, J.PAUSE_MAX_MS)
    assert O.F == J.FADE
    assert np.array_equal(O.fade(), J.fade_table())


@pytest.mark.parametrize("pause_ms", [0, 1, 37, 2000])
def test_oracle_pauses_and_fades(pause_ms):
    rng = np.random.default_rng(pause_ms)
    segs = [rng.standard_normal(n).astype(np.float32) for n in (1000, 300, 50, 2000)]
    y = O.join(segs, pause_ms)
    P, F = 24 * pause_ms, 120
    assert len(y) == sum(map(len, segs)) + 3 * P
    w = np.float64(0.5) - 0.5 * np.cos(np.pi * (np.arange(F) + 0.5) / F)
    pos = 0
    for k, s in enumerate(segs):
        L = len(s)
        g = np.ones(L)
        if k > 0:
            g[:min(F, L)] *= w[:min(F, L)]
        if k < 3:
            g[L - min(F, L):] *= w[:min(F, L)][::-1]
        np.testing.assert_allclose(y[pos:pos + L], s * g, rtol=1e-6, atol=1e-7)
        if k == 0:
            assert np.array_equal(y[:L - F], s[:L - F])   # untouched away from the boundaries
        pos += L
        if k < 3:
            assert not y[pos:pos + P].any()
            pos += P
    assert np.array_equal(O.join(segs[:1], pause_ms), segs[0])   # one segment: no fade at all


def test_check_pause():
    for ok in (0, 1, 2000):
        assert J.check_pause(ok) == ok
    for bad in (-1, 2001, 1.5, True, None, "5"):
        with pytest.raises(ValueError):
            J.check_pause(bad)


# ---- a segmented request through the batcher ------------------------------------------------------------------------
class _Req:
    def __init__(self, tag, total):
        self.tag, self.total, self.done, self.finished = tag, total, 0, False
        self.due, self.hold = 0.0, False


class _Sched:
    """slots for `max_slots` requests; each emits up to n frames per step until its max_new_tokens; records submissions"""

    def __init__(self, max_slots=8, max_batch=8, totals=None):
        self.totals = totals
        self.max_slots, self.max_batch, self.active, self.submitted, self.cancelled = max_slots, max_batch, [], [], []
        self.lock = threading.Lock()

    def capacity(self):
        return self.max_slots - len(self.active)

    def has_capacity(self):
        return self.capacity() > 0

    def submit_many(self, reqs):
        out = []
        for r in reqs:
            rq = _Req(r["tag"], self.totals[len(self.submitted)] if self.totals else r["max_new_tokens"])
            self.submitted.append(r)
            self.active.append(rq)
            out.append(rq)
        return out

    def cancel(self, rq):
        self.cancelled.append(rq.tag)
        self.active.remove(rq)

    def step(self, n):
        res = []
        go = sorted([rq for rq in self.active if not rq.hold], key=lambda rq: rq.due)[:self.max_batch]
        for rq in go:
            k = min(n, rq.total - rq.done)
            codes = torch.arange(rq.done, rq.done + k)[:, None].repeat(1, 16) + 1000 * rq.tag
            rq.done += k
            rq.finished = rq.done >= rq.total
            if rq.finished:
                self.active.remove(rq)
            res.append((rq, codes))
        return res

    def __len__(self):
        return len(self.active)


class _Win:
    def push(self, codes):
        return torch.repeat_interleave(codes[:, 0].float() * 1e-4, 4), 24000


def _window(ref_codes, *a, **kw):
    assert kw.get("segment")
    return _Win()


class _Joiner:
    """numpy join: a segment is released once it and every earlier one ended"""

    def __init__(self):
        self.opened = self.closed = 0

    def open(self, t, out_kw):
        self.opened += 1
        return dict(n=len(t.segments), pause=t.segments.pause_ms, segs=[[] for _ in t.segments],
                    ended=[False] * len(t.segments), next=0)

    def run(self, states, pushes):
        for st, k, pcm, ended in pushes:
            if pcm is not None:
                st["segs"][k].append(pcm.numpy())
            st["ended"][k] = st["ended"][k] or ended
        out = []
        for st in states:
            parts = []
            while st["next"] < st["n"] and st["ended"][st["next"]]:
                k = st["next"]
                x = np.concatenate(st["segs"][k]) if st["segs"][k] else np.zeros(0, np.float32)
                full = O.join([np.zeros(0, np.float32)] * k + [x] + [np.zeros(0, np.float32)] * (st["n"] - 1 - k),
                              st["pause"])
                start = 24 * st["pause"] * k   # this segment and the pause after it
                parts.append(full[start:start + len(x) + (24 * st["pause"] if k < st["n"] - 1 else 0)])
                st["next"] += 1
            a = np.concatenate(parts) if parts else np.zeros(0, np.float32)
            out.append((a, 24000, len(a)))
        return out

    def close(self, state):
        self.closed += 1


class _Clock:
    def __init__(self):
        self.t = 0.0

    def __call__(self):
        return self.t


def _segments(lengths, texts=None):
    texts = texts or [f"segment {k}" for k in range(len(lengths))]
    return Segments([(lambda: (torch.zeros(1, 3, 4), None, None, None, None)) for _ in lengths], texts)


def _batcher(sched, **kw):
    return ContinuousBatcher(sched, _window, chunk_size=4, joiner=_Joiner(), idle_sleep=0.0005, **kw)


def _wait(cond, timeout=10):
    t0 = time.time()
    while not cond():
        assert time.time() - t0 < timeout
        time.sleep(0.001)


def test_rows_in_segment_order_reverse_finish_delivered_in_order():
    lengths = [12, 8, 4, 2]   # the last row finishes first
    sched = _Sched(totals=lengths)
    b = _batcher(sched)
    try:
        t = b.submit(_segments(lengths), split=True, pause_ms=3, seed=11, max_new_tokens=12)
        chunks = list(t)
    finally:
        b.close()
    # admitted in segment order, one row per segment, each with max_new_tokens of its own
    assert [r["tag"] for r in sched.submitted] == sorted(r["tag"] for r in sched.submitted)
    assert len(sched.submitted) == 4 and all(r["max_new_tokens"] == 12 for r in sched.submitted)
    assert all(c[2]["n_segments"] == 4 for c in chunks) and chunks[-1][2]["is_final"]
    assert [c[2]["segment"] for c in chunks] == sorted(c[2]["segment"] for c in chunks)
    audio = np.concatenate([c[0] for c in chunks])
    tags = [r["tag"] for r in sched.submitted]
    want = [torch.repeat_interleave((torch.arange(n) + 1000 * tag).float() * 1e-4, 4).numpy()
            for n, tag in zip(lengths, tags)]
    assert np.array_equal(audio, O.join(want, 3))


def test_join_failure_ends_the_request_not_the_worker():
    """an error in the join fails the requests of that step and frees their rows; the worker serves the next one"""
    sched = _Sched()
    b = _batcher(sched)
    real = b.joiner.run
    fail = [True]

    def run(states, pushes):
        if fail[0]:
            fail[0] = False
            raise RuntimeError("join failed")
        return real(states, pushes)
    b.joiner.run = run
    try:
        t = b.submit(_segments([1, 1]), split=True, max_new_tokens=8)
        with pytest.raises(RuntimeError, match="join failed"):
            list(t)
        _wait(lambda: not sched.active and not b.segmented)
        u = b.submit(_segments([1, 1]), split=True, max_new_tokens=8)
        chunks = list(u)
    finally:
        b.close()
    assert chunks[-1][2]["is_final"] and b.joiner.closed == 2


def test_cancel_frees_every_row():
    sched = _Sched()
    sched_step = sched.step
    sched.step = lambda n: (time.sleep(0.002), sched_step(n))[1]
    b = _batcher(sched)
    try:
        t = b.submit(_segments([1, 1, 1]), split=True, max_new_tokens=100000)
        _wait(lambda: len(sched.submitted) == 3)
        t.cancel()
        _wait(lambda: len(sched.active) == 0)
        list(t)
        _wait(lambda: b.joiner.closed == 1)
    finally:
        b.close()
    assert sorted(sched.cancelled) == sorted(r["tag"] for r in sched.submitted)
    assert not b.segmented and not b.live


def test_due_and_hold_of_later_segments():
    """a paced request: the current segment gets the lead, a later one lead + the seconds before it starts, and a
    segment whose due reaches lead_high_s is neither admitted nor launched"""
    clock = _Clock()
    b = ContinuousBatcher(_Sched(), _window, chunk_size=4, joiner=_Joiner(), clock=clock, sleep=lambda s: None,
                          lead_high_s=2.0)
    b.close()   # drive the worker's methods by hand
    texts = ["a" * 14, "b" * 28, "c" * 42]
    segs = _segments([1, 1, 1], texts)
    t = b.submit(segs, split=True, pause_ms=500, pace=1.0)
    t.segments.state = b.joiner.open(t, {})
    b.segmented.append(t)
    # no audio yet: segment 0 is the most urgent; 1 starts after ~1 s of speech and the pause
    assert b._segment_due(t, 0, 0.0) == float("-inf")
    assert b._segment_due(t, 1, 0.0) == pytest.approx(1.0 + 0.5)
    assert b._segment_due(t, 2, 0.0) == pytest.approx(1.0 + 0.5 + 2.0 + 0.5)
    assert [r.seg for r in b._candidate_rows()] == [0, 1]   # segment 2 is due 4 s out: held back
    # audio arrives: 10 frames of segment 0 made, 0.5 s of joined audio delivered at t = 0
    t.first_chunk_at = 0.0
    segs.frames[0] = 10
    segs.joined = 12000
    clock.t = 0.25
    lead = 0.5 - 0.25
    assert b._segment_due(t, 0, clock.t) == pytest.approx(lead)
    assert b._segment_due(t, 1, clock.t) == pytest.approx(lead + (1.0 - 0.8) + 0.5)
    # segment 0 ends with 1.2 s; segment 1 is now current
    segs.ended[0], segs.frames[0] = True, 15
    assert b._segment_due(t, 1, clock.t) == pytest.approx(lead)
    assert b._segment_due(t, 2, clock.t) == pytest.approx(lead + 2.0 + 0.5)
    # unpaced: every segment may be admitted, in order
    u = b.submit(_segments([1, 1, 1], texts), split=True)
    u.segments.state = b.joiner.open(u, {})
    b.segmented = [u]
    assert [r.seg for r in b._candidate_rows()] == [0, 1, 2]


def test_refusals():
    b = ContinuousBatcher(_Sched(), _window, chunk_size=4, joiner=_Joiner())
    nojoin = ContinuousBatcher(_Sched(), _window, chunk_size=4)
    try:
        segs = _segments([1])
        with pytest.raises(ValueError):
            b.submit(lambda: None, split=True)
        with pytest.raises(ValueError):
            b.submit(segs)                          # Segments without split
        with pytest.raises(ValueError):
            b.submit(segs, split=True, pause_ms=2001)
        with pytest.raises(ValueError):
            b.submit(segs, split=True, uniforms=torch.zeros(1))
        with pytest.raises(ValueError):
            nojoin.submit(segs, split=True)
        with pytest.raises(ValueError, match="seed"):
            b.submit(lambda: None, seed=3)          # a seed without split would be silently ignored
        with pytest.raises(ValueError):
            b.submit_text(lambda f: None, split=True)
        with pytest.raises(ValueError):
            Segments([], [])
    finally:
        b.close()
        nojoin.close()
    assert len(segment_requests(lambda s: s, "One sentence here, long enough. Another sentence, also long.", 400)) == 2


def test_model_refuses_split_for_takes_and_text_streaming():
    from faster_qwen3_tts.model import FasterQwen3TTS
    m = object.__new__(FasterQwen3TTS)   # refused before anything about the model is read
    with pytest.raises(ValueError, match="split"):
        m.generate_custom_voice_takes("hi", "ryan", "English", split=True)
    with pytest.raises(ValueError, match="split"):
        m.generate_voice_design_takes("hi", "calm", "English", split=True)
    with pytest.raises(ValueError, match="split"):
        m.generate_voice_clone_takes("hi", "English", split=True)
    for gen in (m.generate_custom_voice_text_streaming(iter(["hi"]), "ryan", "English", split=True),
                m.generate_voice_design_text_streaming(iter(["hi"]), "calm", "English", split=True),
                m.generate_voice_clone_text_streaming(iter(["hi"]), "English", split=True)):
        with pytest.raises(ValueError, match="split"):
            next(gen)
    with pytest.raises(ValueError):
        FasterQwen3TTS._check_split(True, 0, 0)
    with pytest.raises(ValueError):
        FasterQwen3TTS._check_split(True, 400, 2001)
    with pytest.raises(ValueError, match="seed"):
        FasterQwen3TTS._check_split(False, 400, 0, seed=5)
    assert FasterQwen3TTS._check_split(True, 400, 0, seed=5) and not FasterQwen3TTS._check_split(False, 400, 0)


# ---- server plumbing ------------------------------------------------------------------------------------------------
def test_server_split_field_flag_and_pause_range():
    pytest.importorskip("fastapi")
    pytest.importorskip("httpx")
    import importlib.util
    from fastapi.testclient import TestClient
    spec = importlib.util.spec_from_file_location("openai_server", os.path.join(ROOT, "examples", "openai_server.py"))
    srv = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(srv)
    calls = []

    class _B:
        sched, max_concurrent = [], 0

        def submit(self, prepare, **kw):
            calls.append((prepare, kw))
            from faster_qwen3_tts.serving import Ticket
            t = Ticket(1, prepare, {})
            t.out.put(__import__("faster_qwen3_tts.serving", fromlist=["_DONE"])._DONE)
            return t

    model = object()
    import faster_qwen3_tts.serving as sv
    orig = sv.voice_clone_request
    sv.voice_clone_request = lambda m, text, lang, ref, rt="", split=False, **k: ("segs" if split else "one", text)
    try:
        voices = {"default": {"ref_audio": "r.wav"}}
        for split_default in (False, True):
            c = TestClient(srv.build_app(model, _B(), voices, "default", split_default=split_default))
            body = {"input": "Hello. World.", "voice": "default"}
            assert c.post("/v1/audio/speech", json=body).status_code == 200
            assert calls[-1][1]["split"] is split_default and calls[-1][0][0] == ("segs" if split_default else "one")
            assert c.post("/v1/audio/speech", json=dict(body, split=True, pause_ms=250)).status_code == 200
            assert calls[-1][1]["split"] is True and calls[-1][1]["pause_ms"] == 250
            assert c.post("/v1/audio/speech", json=dict(body, split=False)).status_code == 200
            assert calls[-1][1]["split"] is False
            assert c.post("/v1/audio/speech", json=dict(body, input="  ")).status_code == 400
            for bad in (-1, 2001):
                r = c.post("/v1/audio/speech", json=dict(body, split=True, pause_ms=bad))
                assert r.status_code == 400 and "pause_ms" in r.text
    finally:
        sv.voice_clone_request = orig
    src = open(os.path.join(ROOT, "examples", "openai_server.py")).read()
    assert '"--split"' in src and "split_default=args.split" in src
