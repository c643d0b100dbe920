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
    """Handle of one submitted request: iterate it for (audio, sample_rate, timing) chunks; the audio is float32, or
    int16 / uint8 in the encodings ``s16`` / ``ulaw`` / ``alaw``, or uint8 FLAC bytes in ``flac`` (the chunks of a
    finished ticket concatenate to one complete .flac file)."""
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
    sample_rate: int = 24000              # output rate and encoding of the audio (resample.py)
    encoding: str = "f32"
    pitch: float = 0.0                    # semitones and dB, applied by the tempo and the resampler (resample.py)
    gain_db: float = 0.0
    segments: Optional["Segments"] = None   # a segmented request: its rows, join and post-codec chain (split=True)
    parent: Optional["Ticket"] = None     # a row of a segmented request: the request, and the row's segment index
    seg: int = -1

    @property
    def flushes(self) -> bool:
        """whether the request's window holds device stages (a tempo, a resampler, a FLAC encoder) that flush with its
        last chunk"""
        return (self.speed != 1.0 or (self.sample_rate, self.encoding) != (24000, "f32") or self.pitch != 0
                or self.gain_db != 0)

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
        empty = {"f32": np.float32, "s16": np.int16}.get(self.encoding, np.uint8)
        return np.concatenate(parts) if parts else np.zeros(0, dtype=empty)


class Segments(list):
    """The per-segment ``prepare`` callables of a segmented request, in order (what the ``*_request`` helpers return
    with ``split=True``, or ``ssml_request``), with the texts they speak; ``prosody``: each segment's (speed, pitch,
    gain_db), applied to its row before the join (None: all (1, 0, 0)); ``breaks``: the S + 1 boundaries' pauses in ms,
    None where the request's ``pause_ms`` applies (``ssml.parse``).  On the worker also the request's state: the pause
    plan, the next segment to admit, the frames each row has made, which rows have ended, and the join."""

    def __init__(self, prepares, texts, prosody=None, breaks=None):
        super().__init__(prepares)
        if not self:
            raise ValueError("the text has no segment to speak")
        self.texts = list(texts)
        self.prosody = [(1.0, 0.0, 0.0)] * len(self) if prosody is None else [tuple(map(float, p)) for p in prosody]
        self.breaks = [None] * (len(self) + 1) if breaks is None else list(breaks)
        if len(self.texts) != len(self) or len(self.prosody) != len(self) or len(self.breaks) != len(self) + 1:
            raise ValueError("Segments needs one text and one prosody per segment and one break per boundary")
        self.pauses = None                  # the filled pause plan (``plan``), set by ``submit``
        self.next = 0                       # rows [0, next) have been admitted
        self.frames = [0] * len(self)
        self.ended = [False] * len(self)
        self.rows = {}                      # segment -> its row ticket, once the worker made it
        self.joined = 0                     # 24 kHz samples of the joined stream released so far
        self.seed, self.pause_ms = 0, 0
        self.state = None                   # the joiner's per-request state

    def current(self) -> int:
        """the segment being played: the first that has not ended"""
        return next((k for k, e in enumerate(self.ended) if not e), len(self) - 1)

    def plan(self, pause_ms: int) -> List[int]:
        """the pause of every boundary in ms: the document's breaks, else ``pause_ms`` inside and 0 at the two ends"""
        S = len(self)
        return [b if b is not None else (pause_ms if 0 < k < S else 0) for k, b in enumerate(self.breaks)]


def segment_requests(make, text: str, max_segment_chars: int):
    """``Segments`` of ``make(segment_text)`` over the segments of ``text`` (``segment.split_text``)"""
    from .segment import split_text
    texts = split_text(text, max_segment_chars)
    return Segments([make(s) for s in texts], texts)


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
    flushes), and the lead counts audio seconds at that rate, ``frames x frame_s / speed``.  Likewise with
    ``sample_rate=`` / ``encoding=`` when the ticket asks for other than 24 kHz f32 (``submit(..., sample_rate=,
    encoding=)``): the window resamples and encodes on the device, its resampler flushes with the last chunk, and the
    lead, which counts audio seconds, is the same at every rate.  ``encoding="flac"`` adds a FLAC encoder after an s16
    resampler: the ticket's chunks are FLAC bytes, and its lead still counts audio seconds.  ``pitch=`` / ``gain_db=``
    (``submit(..., pitch=, gain_db=)``) reach the window likewise when not 0; the lead is still ``frames x frame_s /
    speed`` (a pitched delivery lasts within 0.2 % of that).  A pitch's filter table is designed and uploaded by
    ``submit`` on the caller's thread (``window_factory.warm``, when the factory has one), not by the worker.
    ``clock`` / ``sleep`` are the worker's time source, replaceable in tests.

    Long inputs (``submit(segments, split=True, pause_ms=)``, DESIGN.md "Long inputs").  A segmented request is one
    ticket made of N rows, one per segment of its text (``Segments``), each with its own prompt, slot and codec window
    (``window_factory(ref_codes, [chunk], segment=True)``: codec only, PCM left on the device).  Row k is admitted only
    after row k-1 (in ``submit_many`` order) and samples with the uniforms of ``segment.segment_seed(seed, k)``
    (``joiner.uniforms``); ``max_new_tokens`` is per row.  ``joiner`` runs the join (``join.py``): ``open(ticket)`` ->
    per-request state, ``run(states, pushes)`` with pushes (state, segment, pcm, ended) -> [(audio, sr, joined 24 kHz
    samples)] per state, after the request's own tempo, resampler and FLAC encoder, and ``close(state)``.  Paced: the
    segment being played gets the ticket's lead as ``due``; a later one ``lead + `` the seconds before it starts --
    real seconds for audio already made, ``segment.CHARS_PER_S`` characters per second for text not yet made, plus the
    pauses -- and is held (not admitted, not launched) while that is at least ``lead_high_s``.  The lead counts the
    joined audio.  ``cancel`` frees every row."""

    def __init__(self, scheduler, window_factory: Callable, chunk_size: int = 8, idle_sleep: float = 0.002,
                 batch_decode: Optional[Callable] = None, feed_factory: Optional[Callable] = None,
                 lead_high_s: float = 2.0, frame_s: float = 0.08, clock: Callable[[], float] = time.monotonic,
                 sleep: Callable[[float], None] = time.sleep, joiner=None):
        self.sched, self.window_factory, self.chunk_size = scheduler, window_factory, chunk_size
        self.lead_high_s, self.frame_s, self.clock, self.sleep = lead_high_s, frame_s, clock, sleep
        self.joiner = joiner
        self.segmented: List[Ticket] = []   # segmented requests on the worker, in arrival order
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
               sample_rate: Optional[int] = None, encoding: str = "f32", pitch: float = 0.0, gain_db: float = 0.0,
               split: bool = False, pause_ms: int = 0, seed: Optional[int] = None, **gen_kwargs) -> Ticket:
        """``pace``: the client plays at ``pace`` x real time (class docstring); ``speed``: speaking rate in [0.25,
        4.0]; ``sample_rate`` (None: 24000) and ``encoding`` (``f32 | s16 | ulaw | alaw | flac``): the audio the ticket
        carries; ``pitch``: semitones in [-12, 12]; ``gain_db``: in [-96, 16].
        ``split``: ``prepare`` is a ``Segments`` (a ``*_request`` helper with ``split=True``) and the request is spoken
        segment by segment, joined with ``pause_ms`` (integer in [0, 2000]) of silence; ``seed`` (None: drawn) is the
        request's seed, segment k uses ``segment.segment_seed(seed, k)``.  Streamed chunks then carry ``segment`` and
        ``n_segments`` in their timing dict.
        ``gen_kwargs`` are the scheduler's ``submit`` keywords, among them ``chunk_size`` / ``first_chunk`` for this
        request alone."""
        speed = self._speed(speed, pitch, gain_db)
        out = self._output(sample_rate, encoding, pitch, gain_db)
        segs = self._segments(prepare, split, pause_ms, seed, gen_kwargs)
        with self._lock:
            self._rid += 1
            t = Ticket(self._rid, prepare, gen_kwargs, pace=self._pace(pace), submitted_at=self.clock(), speed=speed,
                       segments=segs, **out)
        self.pending.put(t)
        return t

    def _segments(self, prepare, split, pause_ms, seed, gen_kwargs):
        """the checked ``Segments`` of a ``split`` submission (None without split)"""
        from .join import check_pause
        check_pause(pause_ms)
        if not split:
            if isinstance(prepare, Segments):
                raise ValueError("segmented prepare callables need split=True")
            if seed is not None:
                raise ValueError("seed= is the seed of a split request: it needs split=True")
            return None
        if not isinstance(prepare, Segments):
            raise ValueError("split=True needs the Segments of a *_request helper called with split=True")
        if self.joiner is None:
            raise ValueError("this batcher has no joiner: it cannot serve segmented requests")
        if "uniforms" in gen_kwargs:
            raise ValueError("a segmented request draws its rows' uniforms from its seed")
        if seed is None:
            import random
            seed = random.getrandbits(62)
        from .join import check_pauses
        prepare.seed, prepare.pause_ms = int(seed), pause_ms
        prepare.pauses = check_pauses(prepare.plan(pause_ms), len(prepare))
        for speed, pitch, gain_db in set(prepare.prosody):
            self._speed(speed, pitch, gain_db)
            self._output(None, "f32", pitch, gain_db)   # warms a pitched 24 kHz table on the caller's thread
        return prepare

    @staticmethod
    def _pace(pace):
        if pace is not None and not pace > 0:
            raise ValueError(f"pace must be positive (or None for an unpaced client), got {pace}")
        return None if pace is None else float(pace)

    @staticmethod
    def _speed(speed, pitch=0.0, gain_db=0.0):
        from .resample import check_prosody
        check_prosody(speed, pitch, gain_db)
        return float(speed)

    def _output(self, sample_rate, encoding, pitch=0.0, gain_db=0.0):
        from .flac import check_encoding
        from .resample import check_rate
        out = dict(sample_rate=check_rate(sample_rate), encoding=check_encoding(encoding))
        warm = getattr(self.window_factory, "warm", None)
        if pitch != 0 and warm is not None:
            warm(out["sample_rate"], "s16" if out["encoding"] == "flac" else out["encoding"], pitch)
        return dict(out, pitch=float(pitch), gain_db=float(gain_db))

    def submit_text(self, prepare: Callable, pace: Optional[float] = None, speed: float = 1.0,
                    sample_rate: Optional[int] = None, encoding: str = "f32", pitch: float = 0.0, gain_db: float = 0.0,
                    split: bool = False, **gen_kwargs) -> TextTicket:
        """A text-fed request.  ``prepare(feed)`` -> (tie, tam, tpe, ref_codes) builds the prompt once the feed holds its
        first committed id (``text_stream.TextFeed.prompt_ids``); it runs on the worker thread.  Text that arrives
        incrementally is not split (``split=True``: ValueError)."""
        if split:
            raise ValueError("split=True is not supported for text fed while it is spoken")
        if self.feed_factory is None:
            raise RuntimeError("this batcher has no text feed factory")
        speed = self._speed(speed, pitch, gain_db)
        out = self._output(sample_rate, encoding, pitch, gain_db)
        with self._lock:
            self._rid += 1
            t = TextTicket(self._rid, prepare, gen_kwargs, pace=self._pace(pace), submitted_at=self.clock(), speed=speed,
                           **out)
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
            if t.cancelled.is_set():   # a row shares its request's event: cancelling the request frees every row
                self.sched.cancel(self.requests.pop(rid))
                del self.live[rid]
                self._drop_stages(win)
                t.out.put(_DONE)
        for t in [t for t in self.segmented if t.cancelled.is_set()]:
            self._end_segmented(t)

    def _end_segmented(self, t: Ticket):
        self.segmented.remove(t)
        self.joiner.close(t.segments.state)
        t.out.put(_DONE)

    def _row(self, t: Ticket, k: int) -> Ticket:
        """the row of segment k of the segmented request t (made once; it shares t's cancel event)"""
        segs = t.segments
        row = segs.rows.get(k)
        if row is None:
            from .segment import segment_seed
            gen = dict(t.gen_kwargs)
            uniforms = getattr(self.joiner, "uniforms", None)
            if uniforms is not None:
                gen["uniforms"] = uniforms(segment_seed(segs.seed, k), int(gen.get("max_new_tokens", 2048)))
            speed, pitch, gain_db = segs.prosody[k]
            with self._lock:
                self._rid += 1
                row = Ticket(self._rid, segs[k], gen, submitted_at=t.submitted_at, cancelled=t.cancelled, parent=t,
                             seg=k, speed=speed, pitch=pitch, gain_db=gain_db)
            segs.rows[k] = row
        return row

    def _made_s(self, t: Ticket) -> float:
        """audio seconds handed to the listener: frames, or the joined samples of a segmented request"""
        if t.segments is not None:
            from .join import RATE
            return t.segments.joined / RATE / t.speed
        return t.frames * self.frame_s / t.speed

    def _segment_due(self, t: Ticket, k: int, now: float) -> float:
        """``due`` of segment k of a paced segmented request (class docstring)"""
        from .segment import CHARS_PER_S
        segs = t.segments
        cur = segs.current()
        if t.first_chunk_at is None:
            lead = float("-inf") if k <= cur else 0.0
        else:
            lead = self._made_s(t) - t.pace * (now - t.first_chunk_at)
        before = 0.0
        for j in range(cur, k):
            speed = t.speed * segs.prosody[j][0]   # the row's own rate, then the request's
            made = segs.frames[j] * self.frame_s / speed
            est = len(segs.texts[j]) / CHARS_PER_S / speed
            if j == cur:
                before += 0.0 if segs.ended[j] else max(0.0, est - made)
            else:
                before += made if segs.ended[j] else max(made, est)
            before += segs.pauses[j + 1] / 1000.0 / t.speed
        return lead + before

    def _candidate_rows(self) -> List[Ticket]:
        """the rows of segmented requests that may be admitted now: in segment order, and for a paced request only
        while the segment's due is below ``lead_high_s``"""
        now, rows = self.clock(), []
        for t in self.segmented:
            segs = t.segments
            for k in range(segs.next, len(segs)):
                if t.pace is not None and k > segs.current() and self._segment_due(t, k, now) >= self.lead_high_s:
                    break
                rows.append(self._row(t, k))
        return rows

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
    def _drop_stages(win):
        """hand the window's tempo, resampler and FLAC encoder state back to their pools"""
        for stage in (getattr(win, "tempo", None), getattr(win, "resampler", None), getattr(win, "flac", None)):
            if stage is not None:
                stage.close()

    def _window(self, t: Ticket, ref_codes):
        """the request's codec window, built for the request's own chunk size where it has one (the window policy's
        calibration point depends on it); a short first chunk is for windows whose audio does not depend on the chunking"""
        own = t.gen_kwargs.get("chunk_size")
        kw = self._row_kw(t) if t.parent is not None else self._out_kw(t)
        win = self.window_factory(ref_codes, **kw) if own is None else self.window_factory(ref_codes, own, **kw)
        if t.gen_kwargs.get("first_chunk") and not getattr(win, "any_chunking", False):
            raise ValueError("first_chunk needs a codec window whose audio does not depend on the chunking (the stateful "
                             "codec stream); under the window policy the audio of a request is defined by one chunk_size")
        return win

    @staticmethod
    def _row_kw(t: Ticket) -> dict:
        """a row's window keywords: codec only, or with its segment's prosody where that is not the identity"""
        if t.flushes:
            return {"segment": True, "speed": t.speed, "pitch": t.pitch, "gain_db": t.gain_db}
        return {"segment": True}

    @staticmethod
    def _out_kw(t: Ticket) -> dict:
        """the ticket's post-codec stages as window keywords, only where they are not the identity"""
        kw = {} if t.speed == 1.0 else {"speed": t.speed}
        if (t.sample_rate, t.encoding) != (24000, "f32"):
            kw.update(sample_rate=t.sample_rate, encoding=t.encoding)
        if t.pitch != 0:
            kw["pitch"] = t.pitch
        if t.gain_db != 0:
            kw["gain_db"] = t.gain_db
        return kw

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
            elif t.segments is not None:
                try:
                    t.segments.state = self.joiner.open(t, self._out_kw(t))
                    self.segmented.append(t)
                except BaseException as ex:
                    self._fail(t, ex)
            else:
                self._queued.append(t)
        self._reap_cancelled()
        self._drain_text()
        for t in [t for t in self._queued if t.cancelled.is_set()]:
            self._queued.remove(t)
            t.out.put(_DONE)
        # text-fed requests enter once their first id is committed (the prompt holds it), in arrival order; the rows of
        # a segmented request in segment order, at its place in that order
        ready = sorted([t for t in self.waiting if t.feed.n_ids] + self._queued + self._candidate_rows(),
                       key=lambda t: (t.parent.rid, t.seg) if t.parent is not None else (t.rid, -1))
        many = hasattr(self.sched, "submit_many")
        admits = getattr(self.sched, "admits", None)   # a paged scheduler: do the prompts' KV pages fit as well
        batch = []   # (ticket, submit arguments, window) admitted together by one submit_many
        for t in ready:
            if (len(batch) >= self.sched.capacity()) if many else not self.sched.has_capacity():
                break
            if t.parent is not None and (t.cancelled.is_set() or t.seg != t.parent.segments.next):
                continue   # its request failed, or an earlier row of it is still waiting
            queue_of = self.waiting if isinstance(t, TextTicket) else self._queued if t.parent is None else None
            if queue_of is not None:
                queue_of.remove(t)
            try:   # a bad request must not take the worker down, nor the requests admitted with it
                req, win = t.prepared or self._prepare(t)
                if many and admits is not None and not admits([r for _, r, _ in batch] + [req]):
                    t.prepared = (req, win)   # waits, prompt built, until finished requests free pages
                    if queue_of is not None:
                        queue_of.append(t)
                    break
                if t.parent is not None:
                    t.parent.segments.next += 1
                if many:
                    batch.append((t, req, win))
                else:
                    self._live(t, self.sched.submit(**req), win)
            except BaseException as ex:
                if t.parent is not None:   # a row that cannot be spoken fails its request
                    t.parent.cancel()
                    self._fail(t.parent, ex)
                else:
                    self._fail(t, ex)
        # one batched prefill takes as many prompts as a launch has columns; free slots may be more
        per_call = getattr(self.sched, "max_prompts", None) or len(batch) or 1
        for i in range(0, len(batch), per_call):
            part = batch[i:i + per_call]
            try:
                rqs = self.sched.submit_many([req for _, req, _ in part])
            except BaseException as ex:
                for t, _, _ in part:
                    if t.parent is not None:
                        t.parent.cancel()
                    self._fail(t.parent or t, ex)
                continue
            for (t, _, win), rq in zip(part, rqs):
                self._live(t, rq, win)

    def _set_urgency(self):
        """hand every paced request's lead to the scheduler (class docstring)"""
        now = self.clock()
        for rid, (t, _) in self.live.items():
            if t.parent is not None:
                if t.parent.pace is not None:
                    rq = self.requests[rid]
                    rq.due = self._segment_due(t.parent, t.seg, now)
                    rq.hold = rq.due >= self.lead_high_s
                continue
            if t.pace is None:
                continue
            rq = self.requests[rid]
            if t.first_chunk_at is None:
                rq.due, rq.hold = float("-inf"), False
            else:
                t.lead_s = self._made_s(t) - t.pace * (now - t.first_chunk_at)
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
                for t in list(self.segmented):
                    t.out.put(ex)
                    self._end_segmented(t)
                continue
            if not results:   # every active request is waiting for text, or is a listener far enough ahead
                self.sleep(self.idle_sleep)
                continue
            self.steps += 1
            # the last step of a request with device stages flushes them, even when that step made no frames
            live = [(rq, codes) for rq, codes in results
                    if int(codes.shape[0]) or (rq.finished and self.live[rq.tag][0].flushes)]
            stretched = any(self.live[rq.tag][0].flushes for rq, _ in live)
            # windows of equal length of all requests are decoded as one batch when the window objects support it
            pcm_of = {}
            if live and self.batch_decode is not None:
                args = ([self.live[rq.tag][1] for rq, _ in live], [codes for _, codes in live])
                if stretched:
                    args += ([bool(rq.finished) for rq, _ in live],)
                for (rq, _), (pcm, sr) in zip(live, self.batch_decode(*args)):
                    pcm_of[rq.tag] = (pcm, sr)
            pushes = []   # (row, frames, its new PCM or None, whether it ended) of segmented requests
            for rq, codes in results:
                t, win = self.live[rq.tag]
                n = int(codes.shape[0])
                if t.parent is not None:
                    if rq.tag in pcm_of:
                        pcm = pcm_of[rq.tag][0]
                    elif t.flushes and (n or rq.finished):
                        pcm = win.push(codes, final=bool(rq.finished))[0]
                    else:
                        pcm = win.push(codes)[0] if n else None
                    pushes.append((t, n, pcm, bool(rq.finished)))
                    if rq.finished:
                        del self.live[rq.tag]
                        self.requests.pop(rq.tag, None)
                        self._drop_stages(win)
                    continue
                if n or rq.tag in pcm_of:
                    if rq.tag in pcm_of:
                        pcm, sr = pcm_of[rq.tag]
                    else:
                        pcm, sr = win.push(codes, final=bool(rq.finished)) if t.flushes else win.push(codes)
                    now = self.clock()
                    if t.first_chunk_at is None:
                        t.first_chunk_at = now
                    elif t.pace is not None and t.frames * self.frame_s / t.speed - t.pace * (now - t.first_chunk_at) < 0:
                        t.underruns += 1      # what it had was played out before this chunk arrived
                    t.frames += n
                    if t.pace is not None:
                        t.lead_s = self._made_s(t) - t.pace * (now - t.first_chunk_at)
                    t.out.put((pcm, sr, {"chunk_steps": n, "total_steps_so_far": t.frames,
                                         "is_final": bool(rq.finished)}))
                if rq.finished:
                    t.out.put(_DONE)
                    del self.live[rq.tag]
                    self.requests.pop(rq.tag, None)
                    self._drop_stages(win)
            if pushes:
                self._join_step(pushes)

    def _join_step(self, pushes):
        """the rows' new PCM -> the join of every segmented request they belong to, in one ``joiner.run``; delivers
        what each request's join released, in order"""
        parents = []
        for row, n, _, ended in pushes:
            segs = row.parent.segments
            segs.frames[row.seg] += n
            segs.ended[row.seg] = segs.ended[row.seg] or ended
            if row.parent not in parents:
                parents.append(row.parent)
        try:
            outs = self.joiner.run([p.segments.state for p in parents],
                                   [(row.parent.segments.state, row.seg, pcm, ended) for row, _, pcm, ended in pushes])
        except BaseException as ex:   # the join failed: end these requests (their rows are freed), not the worker
            for p in parents:
                p.cancel()
                p.out.put(ex)
                self._end_segmented(p)
            return
        for p, (audio, sr, n24) in zip(parents, outs):
            segs, n = p.segments, sum(m for row, m, _, _ in pushes if row.parent is p)
            final = all(segs.ended)
            if len(audio) or final:
                now = self.clock()
                if p.first_chunk_at is None:
                    p.first_chunk_at = now
                elif p.pace is not None and self._made_s(p) - p.pace * (now - p.first_chunk_at) < 0:
                    p.underruns += 1
                p.frames += n
                segs.joined += n24
                if p.pace is not None:
                    p.lead_s = self._made_s(p) - p.pace * (now - p.first_chunk_at)
                p.out.put((audio, sr, {"chunk_steps": n, "total_steps_so_far": p.frames, "is_final": final,
                                       "segment": segs.current(), "n_segments": len(segs)}))
            else:
                p.frames += n
            if final:
                self._end_segmented(p)


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

    def window(ref_codes, chunk=chunk_size, speed=1.0, segment=False, **out):
        if segment:   # a row of a segmented request: its PCM stays on the device for the join, at 24 kHz f32
            if st is None:
                raise ValueError("split=True needs the codec (PCM)")
            return model._make_window(st, ref_codes, chunk, False, **({} if speed == 1.0 else {"speed": speed}), **out)
        if st is None:
            if speed != 1.0:
                raise ValueError("a speaking rate other than 1 needs the codec (PCM)")
            if out:
                raise ValueError("an output rate, encoding, pitch or gain other than 24 kHz f32, 0, 0 dB needs the codec "
                                 "(PCM)")
            return _CodesOnly()
        return model._make_window(st, ref_codes, chunk, to_host, **({} if speed == 1.0 else {"speed": speed}), **out)

    if st is not None:
        from .model import _pcm_device
        from .resample import warm as _warm
        window.warm = lambda rate, encoding, pitch: _warm(rate, encoding, _pcm_device(st), pitch)

    bd = (lambda wins, chunks, finals=None: decode_windows_batched(st, wins, chunks, finals)) if st is not None else None
    from .text_stream import TextFeed
    return ContinuousBatcher(sched, window, chunk_size=chunk_size, batch_decode=bd,
                             feed_factory=lambda max_rows: TextFeed(model, max_rows),
                             joiner=_Joiner(model, to_host) if st is not None else None, **kw)


class _Joiner:
    """The join of segmented requests on a model's device (``ContinuousBatcher`` class docstring): a ``join.Join`` and
    a ``model._Chain`` of the request's post-codec stages per request"""

    def __init__(self, model, to_host=True):
        from .model import _pcm_device
        self.model, self.to_host = model, to_host
        self.st = model.model.model.speech_tokenizer
        self.device = _pcm_device(self.st)

    def uniforms(self, seed, n):
        from .model import take_uniforms
        return take_uniforms(seed, n, self.model.engine.device)

    def open(self, t, out_kw):
        from .join import Join
        from .model import _Chain
        segs = t.segments
        return (Join(len(segs), segs.pause_ms, self.device, segs.pauses),
                _Chain(self.model, self.st, self.to_host, **out_kw))

    def run(self, states, pushes):
        import torch
        from . import join
        from .model import run_stages
        empty = torch.zeros(0, dtype=torch.float32, device=self.device)
        pcm = join.process([j for j, _ in states], [(s[0], k, empty if p is None else p, e) for s, k, p, e in pushes])
        outs = run_stages([c for _, c in states], pcm, [j.done for j, _ in states], 24000)
        return [(a, sr, int(p.numel())) for (a, sr), p in zip(outs, pcm)]

    def close(self, state):
        j, chain = state
        j.close()
        ContinuousBatcher._drop_stages(chain)


def custom_voice_text_request(model, speaker: str, language: str, instruct: Optional[str] = None, split: bool = False):
    """``prepare`` callable for ``ContinuousBatcher.submit_text``: the prompt of a text-fed custom-voice request, built
    from the feed's first committed id exactly like ``generate_custom_voice_text_streaming`` builds it.  Text that
    arrives incrementally is not split (``split=True``: ValueError)."""
    if split:
        raise ValueError("split=True is not supported for text fed while it is spoken")
    from .text_stream import build_prompt
    (instruct,), _ = model._custom_voice_rules([None], [language], [speaker], [instruct], None)   # text: from the feed

    def prepare(feed):
        ins = model.model._tokenize_texts([model.model._build_instruct_text(instruct)])[0] if instruct else None
        tie, tam, tpe = build_prompt(model, feed, language=language, speaker=speaker, instruct_ids=ins)
        return tie, tam, tpe, None
    return prepare


def voice_clone_request(model, text: str, language: str, ref_audio, ref_text: str = "", xvec_only: bool = False,
                        non_streaming_mode: bool = False, append_silence: bool = True, split: bool = False,
                        max_segment_chars: int = 400):
    """``prepare`` callable for ``ContinuousBatcher.submit``: the voice-clone prompt path of the public API
    (model.py:465-543) up to the embeddings.  ``split=True``: the ``Segments`` of ``text`` (``segment.split_text`` at
    ``max_segment_chars``), one prompt per segment in the same voice, for ``submit(..., split=True)``."""
    def make(text):
        def prepare():
            _, _, _, tie, tam, tth, tpe, ref_codes = model._prepare_generation(
                text, ref_audio=ref_audio, ref_text=ref_text, language=language, xvec_only=xvec_only,
                non_streaming_mode=non_streaming_mode, append_silence=append_silence)
            return tie, tam, tth, tpe, ref_codes
        return prepare
    return segment_requests(make, text, max_segment_chars) if split else make(text)


def custom_voice_request(model, text: str, speaker: Optional[str], language: str, instruct: Optional[str] = None,
                         non_streaming_mode: Optional[bool] = None, split: bool = False, max_segment_chars: int = 400):
    """``prepare`` callable for ``ContinuousBatcher.submit``: a custom-voice request (a voice-design one with speaker
    None and the design as ``instruct``), built like ``generate_custom_voice`` / ``generate_voice_design`` build it.
    ``split=True``: the ``Segments`` of ``text``, as in ``voice_clone_request``."""
    if speaker is None:
        nsm = model._voice_design_rules(language, non_streaming_mode)
    else:
        (instruct,), nsm = model._custom_voice_rules([text], [language], [speaker], [instruct], non_streaming_mode)

    def make(text):
        def prepare():
            _, _, _, tie, tam, tth, tpe = model._prepare_generation_custom(text, language, speaker, instruct, nsm)
            return tie, tam, tth, tpe, None
        return prepare
    return segment_requests(make, text, max_segment_chars) if split else make(text)


def ssml_request(model, ssml: str, voices, voice: Optional[str] = None, language: str = "Auto",
                 max_segment_chars: int = 400) -> Segments:
    """``Segments`` of an SSML document (``ssml.py``) for ``ContinuousBatcher.submit(..., split=True)``: each segment's
    prompt in its voice (``voices``: name -> voice spec, ``ssml.voice_request``; ``voice``: the name spoken outside every
    ``<voice>``) and language, its prosody and the document's breaks.  Every refusal is a ValueError."""
    from .ssml import parse, voice_request
    doc = parse(ssml, voices, voice, language, max_segment_chars)
    return Segments([voice_request(model, voices[s.voice], s.text, s.language) for s in doc.spans],
                    [s.text for s in doc.spans], [(s.speed, s.pitch, s.gain_db) for s in doc.spans], doc.breaks)
