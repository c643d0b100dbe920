"""Continuous batching for the serving callers (SURVEY.md section 8(f)3).

The reference's servers run one request at a time behind a global lock (``examples/openai_server.py:71,181`` --
``_model_lock``; ``cli.py serve`` likewise): a second client waits for the first one's last chunk.  Here requests JOIN
and LEAVE the engine's request slots between chunks: one worker thread owns the GPU, admits queued requests into free
slots (prompt assembly + prefill), advances every active slot by one chunk with ONE persistent-kernel launch
(``BatchScheduler.step``), runs each slot's streaming codec window (model.py:1052-1135) and hands the PCM to the
request's own queue.  Wire helpers keep the reference's formats (``examples/openai_server.py:91-118``): 16-bit
little-endian PCM, streaming WAV header with unknown length.
"""
from __future__ import annotations

import io
import queue
import struct
import threading
import time
from dataclasses import dataclass, field
from typing import Callable, Dict, Iterator, List, Optional

import numpy as np

_DONE = object()


def to_pcm16(pcm: np.ndarray) -> bytes:
    """float32 [-1,1] -> raw 16-bit little-endian PCM (examples/openai_server.py:91-93)."""
    return np.clip(np.asarray(pcm, dtype=np.float32) * 32768, -32768, 32767).astype(np.int16).tobytes()


def wav_header(sample_rate: int, data_len: int = 0xFFFFFFFF) -> bytes:
    """WAV header; data_len = 0xFFFFFFFF for a stream of unknown length (examples/openai_server.py:96-112)."""
    n_channels, bits = 1, 16
    byte_rate = sample_rate * n_channels * bits // 8
    block_align = n_channels * bits // 8
    riff_size = 0xFFFFFFFF if data_len == 0xFFFFFFFF else 36 + data_len
    buf = io.BytesIO()
    buf.write(b"RIFF")
    buf.write(struct.pack("<I", riff_size))
    buf.write(b"WAVE")
    buf.write(b"fmt ")
    buf.write(struct.pack("<IHHIIHH", 16, 1, n_channels, sample_rate, byte_rate, block_align, bits))
    buf.write(b"data")
    buf.write(struct.pack("<I", data_len))
    return buf.getvalue()


def to_wav_bytes(pcm: np.ndarray, sample_rate: int) -> bytes:
    raw = to_pcm16(pcm)
    return wav_header(sample_rate, len(raw)) + raw


@dataclass
class Ticket:
    """Handle of one submitted request: iterate it for (pcm float32, sample_rate, timing) chunks."""
    rid: int
    prepare: Callable[[], tuple]          # -> (tie, tam, tth, tpe, ref_codes); runs on the worker thread
    gen_kwargs: dict
    out: "queue.Queue" = field(default_factory=queue.Queue)
    submitted_at: float = field(default_factory=time.time)   # the batcher's clock, as first_chunk_at
    first_chunk_at: Optional[float] = None
    frames: int = 0
    cancelled: threading.Event = field(default_factory=threading.Event)
    pace: Optional[float] = None          # a listener playing at pace x real time; None: wants the audio as fast as possible
    lead_s: float = 0.0                   # paced: audio seconds handed over minus seconds played, as of the last step
    underruns: int = 0                    # paced: chunks delivered after the listener had run dry (lead < 0)
    prepared: Optional[tuple] = None      # (submit arguments, window) of a ticket waiting for KV pages
    speed: float = 1.0                    # speaking rate: the listener consumes model audio `speed` times as fast

    def cancel(self) -> None:
        """End the request: the worker frees its slot (or drops it from the queue) and closes the ticket."""
        self.cancelled.set()

    def __iter__(self) -> Iterator:
        while True:
            item = self.out.get()
            if item is _DONE:
                return
            if isinstance(item, BaseException):
                raise item
            yield item

    def audio(self) -> np.ndarray:
        parts = [c[0] for c in self]
        return np.concatenate(parts) if parts else np.zeros(0, dtype=np.float32)


@dataclass
class TextTicket(Ticket):
    """Ticket of a text-fed request: ``write`` text pieces as they arrive (an LLM's reply), ``close`` when the text is
    complete.  Both are safe to call from any thread; the worker commits, embeds and announces the rows.  A client that
    goes away before ``close`` must ``cancel``, or the request keeps its slot waiting for text."""
    feed: Optional[object] = None
    _pieces: List[str] = field(default_factory=list)
    _closed: bool = False
    _text_lock: threading.Lock = field(default_factory=threading.Lock)

    def write(self, piece: str) -> None:
        with self._text_lock:
            if self._closed:
                raise RuntimeError("text already closed")
            self._pieces.append(piece)

    def close(self) -> None:
        with self._text_lock:
            self._closed = True

    def _take(self):
        with self._text_lock:
            pieces, self._pieces = self._pieces, []
            return pieces, self._closed


class ContinuousBatcher:
    """One worker thread, many clients.  ``scheduler_factory()`` -> object with ``has_capacity()``,
    ``submit(tie, tam, tth, tpe, tag=..., **gen) -> request``, ``step(n) -> [(request, codes)]`` and ``__len__`` (the
    ``BatchScheduler`` of batching.py); with ``submit_many(list of submit arguments) -> [request]`` and ``capacity()``
    the ready requests that fit the free slots are admitted together (one batched prefill); ``window_factory(ref_codes)``
    -> object with ``push(codes) -> (pcm, sr)`` (``model._StreamWindow``); ``feed_factory(max_rows)`` -> ``text_stream.TextFeed`` (text-fed requests).

    Paced listeners.  The engine makes audio several times faster than it is played, and a scheduler may hold more
    requests than one launch carries (``BatchScheduler``: ``max_slots`` > ``max_batch``).  ``submit(..., pace=1.0)`` says
    that the client plays the audio at ``pace`` x real time.  Its *lead* is the audio handed to it minus what it has
    played: ``frames x frame_s - pace x (now - first_chunk_at)``.  Before every step the worker gives each paced request
    its lead as ``due`` -- so when more requests are ready than a launch has columns, those closest to running dry go
    -- and holds back (``hold``) those whose lead is at least ``lead_high_s``: audio nobody will hear for seconds is not
    made while someone else is about to run dry.  A request without audio yet is the most urgent of all, the oldest
    first.  ``pace=None`` (the default) is a client that wants everything at once: never held, ``due`` 0.
    No paced request starves: while it waits its lead only falls, by ``pace`` per second, and every request that is
    launched instead gains a chunk of lead; after finitely many steps the waiting one has the smallest lead of all and
    is launched.  (Requests with ``pace=None`` keep ``due`` 0, so a paced request waits behind them only while its own
    lead is positive.)  The argument covers paced tickets only: an unpaced ticket yields to every listener that has run
    dry (lead < 0), so while ``max_batch`` or more listeners stay in underrun -- an engine loaded beyond what it can
    serve in real time -- unpaced tickets are not launched until some of them recover or end.  A delivery with negative
    lead is counted in ``Ticket.underruns``.
    The worker launches as soon as one listener is below the watermark; at low load its launches therefore carry few
    slots, each costing a whole pass over the weights (no low watermark or minimum launch width is implemented).
    ``window_factory`` is called with the ticket's own ``chunk_size`` as a second argument when it has one, and with
    ``speed=`` when the ticket's speaking rate is not 1 (``submit(..., speed=)``): the window then time-stretches its
    PCM on the device, ``batch_decode`` gets a third argument (whether each request ends with this chunk: its tempo
    flushes), and the lead counts audio seconds at that rate, ``frames x frame_s / speed``.
    ``clock`` / ``sleep`` are the worker's time source, replaceable in tests."""

    def __init__(self, scheduler, window_factory: Callable, chunk_size: int = 8, idle_sleep: float = 0.002,
                 batch_decode: Optional[Callable] = None, feed_factory: Optional[Callable] = None,
                 lead_high_s: float = 2.0, frame_s: float = 0.08, clock: Callable[[], float] = time.monotonic,
                 sleep: Callable[[float], None] = time.sleep):
        self.sched, self.window_factory, self.chunk_size = scheduler, window_factory, chunk_size
        self.lead_high_s, self.frame_s, self.clock, self.sleep = lead_high_s, frame_s, clock, sleep
        self.batch_decode = batch_decode   # (windows, code chunks) -> [(pcm, sr)]: one codec batch per window length
        self.idle_sleep = idle_sleep
        self.pending: "queue.Queue[Ticket]" = queue.Queue()
        self.live: Dict[int, tuple] = {}     # rid -> (ticket, window)
        self.feed_factory = feed_factory
        self.waiting: List[TextTicket] = []  # text-fed tickets whose first text id is not committed yet
        self.requests: Dict[int, object] = {}   # rid -> scheduler request
        self._rid = 0
        self._lock = threading.Lock()
        self._stop = threading.Event()
        self._queued: List[Ticket] = []      # ordinary tickets taken from `pending`, waiting for a slot
        self.steps = 0
        self.max_concurrent = 0
        self._thread = threading.Thread(target=self._run, name="fq3-batcher", daemon=True)
        self._thread.start()

    # ---- client side ------------------------------------------------------------------------------------
    def submit(self, prepare: Callable[[], tuple], pace: Optional[float] = None, speed: float = 1.0,
               **gen_kwargs) -> Ticket:
        """``pace``: the client plays at ``pace`` x real time (class docstring); ``speed``: speaking rate in [0.25,
        4.0].  ``gen_kwargs`` are the scheduler's ``submit`` keywords, among them ``chunk_size`` / ``first_chunk`` for
        this request alone."""
        speed = self._speed(speed)
        with self._lock:
            self._rid += 1
            t = Ticket(self._rid, prepare, gen_kwargs, pace=self._pace(pace), submitted_at=self.clock(), speed=speed)
        self.pending.put(t)
        return t

    @staticmethod
    def _pace(pace):
        if pace is not None and not pace > 0:
            raise ValueError(f"pace must be positive (or None for an unpaced client), got {pace}")
        return None if pace is None else float(pace)

    @staticmethod
    def _speed(speed):
        from .tempo import quantize
        quantize(speed)
        return float(speed)

    def submit_text(self, prepare: Callable, pace: Optional[float] = None, speed: float = 1.0,
                    **gen_kwargs) -> TextTicket:
        """A text-fed request.  ``prepare(feed)`` -> (tie, tam, tpe, ref_codes) builds the prompt once the feed holds its
        first committed id (``text_stream.TextFeed.prompt_ids``); it runs on the worker thread."""
        if self.feed_factory is None:
            raise RuntimeError("this batcher has no text feed factory")
        speed = self._speed(speed)
        with self._lock:
            self._rid += 1
            t = TextTicket(self._rid, prepare, gen_kwargs, pace=self._pace(pace), submitted_at=self.clock(), speed=speed)
        t.feed = self.feed_factory(int(gen_kwargs.get("max_new_tokens", 2048)))
        self.pending.put(t)
        return t

    def close(self):
        self._stop.set()
        self._thread.join(timeout=10)

    # ---- worker -----------------------------------------------------------------------------------------
    @staticmethod
    def _fail(t: Ticket, ex: BaseException):
        t.out.put(ex)
        t.out.put(_DONE)

    def _drain_text(self):
        """commit the text written since the last step (rows are embedded and announced by the scheduler's step)"""
        for t in self.waiting + [t for t, _ in self.live.values() if isinstance(t, TextTicket)]:
            pieces, closed = t._take()
            try:
                if pieces:   # one commit per drained batch: each commit re-tokenizes the text received so far
                    t.feed.push("".join(pieces))
                if closed and not t.feed.closed:
                    t.feed.close()
            except BaseException as ex:
                t.cancel()
                self._fail(t, ex)

    def _reap_cancelled(self):
        for t in [t for t in self.waiting if t.cancelled.is_set()]:
            self.waiting.remove(t)
            t.out.put(_DONE)
        for rid, (t, win) in list(self.live.items()):
            if t.cancelled.is_set():
                self.sched.cancel(self.requests.pop(rid))
                del self.live[rid]
                self._drop_tempo(win)
                t.out.put(_DONE)

    def _prepare(self, t: Ticket):
        """-> (the ticket's ``submit`` arguments by name, its codec window); a prompt longer than the scheduler's
        ``max_seq_len`` is refused here, with the reference's message (talker_graph.py:163-167)"""
        chunk = t.gen_kwargs.get("chunk_size") or self.chunk_size
        if isinstance(t, TextTicket):
            tie, tam, tpe, ref_codes = t.prepare(t.feed)
            win = self._window(t, ref_codes)
            # a window whose audio depends on the chunking (the reference's window policy) must see the one-shot
            # chunking: the slot is launched only when a full chunk of text rows exists, so every launch emits a full
            # chunk or ends the request.  A stateful stream decodes to the same PCM in any chunking: one row suffices.
            ahead = 1 if getattr(win, "any_chunking", False) else chunk
            req = dict(tie=tie, tam=tam, tth=t.feed.rows[None], tpe=tpe, tag=t.rid, feed=t.feed, rows_ahead=ahead,
                       **t.gen_kwargs)
        else:
            tie, tam, tth, tpe, ref_codes = t.prepare()
            win = self._window(t, ref_codes)
            req = dict(tie=tie, tam=tam, tth=tth, tpe=tpe, tag=t.rid, **t.gen_kwargs)
        S = getattr(self.sched, "max_seq_len", None)
        if S is not None and tie.shape[1] > S:
            raise RuntimeError(f"Input is too long: prefill has {tie.shape[1]} tokens but max_seq_len={S}. "
                               "Use shorter text or shorter reference audio.")
        return req, win

    @staticmethod
    def _drop_tempo(win):
        tempo = getattr(win, "tempo", None)
        if tempo is not None:
            tempo.close()

    def _window(self, t: Ticket, ref_codes):
        """the request's codec window, built for the request's own chunk size where it has one (the window policy's
        calibration point depends on it); a short first chunk is for windows whose audio does not depend on the chunking"""
        own = t.gen_kwargs.get("chunk_size")
        kw = {} if t.speed == 1.0 else {"speed": t.speed}
        win = self.window_factory(ref_codes, **kw) if own is None else self.window_factory(ref_codes, own, **kw)
        if t.gen_kwargs.get("first_chunk") and not getattr(win, "any_chunking", False):
            raise ValueError("first_chunk needs a codec window whose audio does not depend on the chunking (the stateful "
                             "codec stream); under the window policy the audio of a request is defined by one chunk_size")
        return win

    def _live(self, t: Ticket, rq, win):
        self.requests[t.rid] = rq
        self.live[t.rid] = (t, win)

    def _admit(self):
        while True:
            try:
                t = self.pending.get_nowait()
            except queue.Empty:
                break
            if isinstance(t, TextTicket):
                self.waiting.append(t)
            else:
                self._queued.append(t)
        self._reap_cancelled()
        self._drain_text()
        for t in [t for t in self._queued if t.cancelled.is_set()]:
            self._queued.remove(t)
            t.out.put(_DONE)
        # text-fed requests enter once their first id is committed (the prompt holds it), in arrival order
        ready = sorted([t for t in self.waiting if t.feed.n_ids] + self._queued, key=lambda t: t.rid)
        many = hasattr(self.sched, "submit_many")
        admits = getattr(self.sched, "admits", None)   # a paged scheduler: do the prompts' KV pages fit as well
        batch = []   # (ticket, submit arguments, window) admitted together by one submit_many
        for t in ready:
            if (len(batch) >= self.sched.capacity()) if many else not self.sched.has_capacity():
                break
            queue_of = self.waiting if isinstance(t, TextTicket) else self._queued
            queue_of.remove(t)
            try:   # a bad request must not take the worker down, nor the requests admitted with it
                req, win = t.prepared or self._prepare(t)
                if many and admits is not None and not admits([r for _, r, _ in batch] + [req]):
                    t.prepared = (req, win)   # waits, prompt built, until finished requests free pages
                    queue_of.append(t)
                    break
                if many:
                    batch.append((t, req, win))
                else:
                    self._live(t, self.sched.submit(**req), win)
            except BaseException as ex:
                self._fail(t, ex)
        # one batched prefill takes as many prompts as a launch has columns; free slots may be more
        per_call = getattr(self.sched, "max_prompts", None) or len(batch) or 1
        for i in range(0, len(batch), per_call):
            part = batch[i:i + per_call]
            try:
                rqs = self.sched.submit_many([req for _, req, _ in part])
            except BaseException as ex:
                for t, _, _ in part:
                    self._fail(t, ex)
                continue
            for (t, _, win), rq in zip(part, rqs):
                self._live(t, rq, win)

    def _set_urgency(self):
        """hand every paced request's lead to the scheduler (class docstring)"""
        now = self.clock()
        for rid, (t, _) in self.live.items():
            if t.pace is None:
                continue
            rq = self.requests[rid]
            if t.first_chunk_at is None:
                rq.due, rq.hold = float("-inf"), False
            else:
                t.lead_s = t.frames * self.frame_s / t.speed - t.pace * (now - t.first_chunk_at)
                rq.due, rq.hold = t.lead_s, t.lead_s >= self.lead_high_s

    def _run(self):
        while not self._stop.is_set():
            self._admit()
            if not len(self.sched):
                self.sleep(self.idle_sleep)
                continue
            self.max_concurrent = max(self.max_concurrent, len(self.sched))
            self._set_urgency()
            try:
                results = self.sched.step(self.chunk_size)
            except BaseException as ex:
                for rid, (t, _) in list(self.live.items()):
                    t.out.put(ex)
                    t.out.put(_DONE)
                self.live.clear()
                continue
            if not results:   # every active request is waiting for text, or is a listener far enough ahead
                self.sleep(self.idle_sleep)
                continue
            self.steps += 1
            # a stretched request's last step flushes its tempo, even when that step made no frames
            live = [(rq, codes) for rq, codes in results
                    if int(codes.shape[0]) or (rq.finished and self.live[rq.tag][0].speed != 1.0)]
            stretched = any(self.live[rq.tag][0].speed != 1.0 for rq, _ in live)
            # windows of equal length of all requests are decoded as one batch when the window objects support it
            pcm_of = {}
            if live and self.batch_decode is not None:
                args = ([self.live[rq.tag][1] for rq, _ in live], [codes for _, codes in live])
                if stretched:
                    args += ([bool(rq.finished) for rq, _ in live],)
                for (rq, _), (pcm, sr) in zip(live, self.batch_decode(*args)):
                    pcm_of[rq.tag] = (pcm, sr)
            for rq, codes in results:
                t, win = self.live[rq.tag]
                n = int(codes.shape[0])
                if n or rq.tag in pcm_of:
                    if rq.tag in pcm_of:
                        pcm, sr = pcm_of[rq.tag]
                    else:
                        pcm, sr = win.push(codes) if t.speed == 1.0 else win.push(codes, final=bool(rq.finished))
                    now = self.clock()
                    if t.first_chunk_at is None:
                        t.first_chunk_at = now
                    elif t.pace is not None and t.frames * self.frame_s / t.speed - t.pace * (now - t.first_chunk_at) < 0:
                        t.underruns += 1      # what it had was played out before this chunk arrived
                    t.frames += n
                    if t.pace is not None:
                        t.lead_s = t.frames * self.frame_s / t.speed - t.pace * (now - t.first_chunk_at)
                    t.out.put((pcm, sr, {"chunk_steps": n, "total_steps_so_far": t.frames,
                                         "is_final": bool(rq.finished)}))
                if rq.finished:
                    t.out.put(_DONE)
                    del self.live[rq.tag]
                    self.requests.pop(rq.tag, None)
                    self._drop_tempo(win)


def batcher_for_model(model, chunk_size: int = 8, to_host: bool = True, **kw) -> ContinuousBatcher:
    """ContinuousBatcher over a ``FasterQwen3TTS`` whose engine was created with ``max_batch`` > 1 (and, to serve more
    paced listeners than that, ``max_slots`` > ``max_batch``); ``kw``: ``lead_high_s``, ``clock``, ``sleep``."""
    from .batching import BatchScheduler
    from .model import _StreamWindow, decode_windows_batched
    m = model.model.model
    sched = BatchScheduler(model.engine, m.talker, m.config.talker_config, model.predictor_graph, model.talker_graph)
    st = m.speech_tokenizer

    class _CodesOnly:
        def push(self, codes):
            return codes.cpu().numpy(), model.sample_rate

    def window(ref_codes, chunk=chunk_size, speed=1.0):
        if st is None:
            if speed != 1.0:
                raise ValueError("a speaking rate other than 1 needs the codec (PCM)")
            return _CodesOnly()
        return model._make_window(st, ref_codes, chunk, to_host, **({} if speed == 1.0 else {"speed": speed}))

    bd = (lambda wins, chunks, finals=None: decode_windows_batched(st, wins, chunks, finals)) if st is not None else None
    from .text_stream import TextFeed
    return ContinuousBatcher(sched, window, chunk_size=chunk_size, batch_decode=bd,
                             feed_factory=lambda max_rows: TextFeed(model, max_rows), **kw)


def custom_voice_text_request(model, speaker: str, language: str, instruct: Optional[str] = None):
    """``prepare`` callable for ``ContinuousBatcher.submit_text``: the prompt of a text-fed custom-voice request, built
    from the feed's first committed id exactly like ``generate_custom_voice_text_streaming`` builds it."""
    from .text_stream import build_prompt
    (instruct,), _ = model._custom_voice_rules([None], [language], [speaker], [instruct], None)   # text: from the feed

    def prepare(feed):
        ins = model.model._tokenize_texts([model.model._build_instruct_text(instruct)])[0] if instruct else None
        tie, tam, tpe = build_prompt(model, feed, language=language, speaker=speaker, instruct_ids=ins)
        return tie, tam, tpe, None
    return prepare


def voice_clone_request(model, text: str, language: str, ref_audio, ref_text: str = "", xvec_only: bool = False,
                        non_streaming_mode: bool = False, append_silence: bool = True):
    """``prepare`` callable for ``ContinuousBatcher.submit``: the voice-clone prompt path of the public API
    (model.py:465-543) up to the embeddings."""
    def prepare():
        _, _, _, tie, tam, tth, tpe, ref_codes = model._prepare_generation(
            text, ref_audio=ref_audio, ref_text=ref_text, language=language, xvec_only=xvec_only,
            non_streaming_mode=non_streaming_mode, append_silence=append_silence)
        return tie, tam, tth, tpe, ref_codes
    return prepare
