"""Batched decode over the engine's request slots (BASELINE config 4: concurrent requests per GPU).

The reference batches only the prompt: ``_build_talker_inputs_local`` left-pads a list of requests and returns a
per-row attention mask (faster_qwen3_tts/model.py:774-787), ``TalkerGraph.set_generation_state`` takes per-row pad
counts and rope deltas (talker_graph.py:177-187); its decode loop itself is batch-1 (``token.item()``,
generate.py:150).  Here every row of such a batch becomes one request *slot* of the engine and all active slots
advance together: one persistent-kernel launch per chunk in which the slots share every pass over the weight tape
(``fq3_decode_chunk(slots[], n_slots, ...)``).  Slots finish independently and can be re-used between chunks
(``BatchScheduler.submit`` while others are mid-stream = continuous batching for the serving callers,
examples/openai_server.py:71 serialises requests behind a lock instead).

Per row the arithmetic -- and therefore the codes -- is identical to running that request alone (tests/test_gpu_batch.py).
"""
from __future__ import annotations

import time
from dataclasses import dataclass, field
from typing import Dict, Generator, List, Optional, Tuple

import torch

from .engine import FQ3_FIN_MAX_SEQ, KV_PAGE
from .generate import _sync, begin_fused, begin_fused_batch, shared_engine
from .logprobs import FrameLogprobs


@dataclass
class SlotRequest:
    slot: int
    tag: object
    max_new_tokens: int
    frames: int = 0
    finished: int = 0
    parts: List[torch.Tensor] = field(default_factory=list)
    feed: Optional[object] = None   # text_stream.TextFeed of a text-fed request (rows announced before every step)
    gen0: int = 0                   # generation_step at begin: the next frame reads trailing row gen0 + frames
    rows_ahead: int = 1             # text-fed: trailing rows that must exist beyond gen0 + frames before a launch
    lp: Optional[FrameLogprobs] = None        # submit_many(logprobs=True): host assembly of the per-frame log-probabilities
    chunk_logprobs: Optional[torch.Tensor] = None   # ... of the frames the last step returned, [n,16]
    eos_logprob: Optional[float] = None       # ... of the EOS draw that ended the request
    chunk_size: Optional[int] = None          # frames per launch of this request (default: the step's n_frames)
    first_chunk: Optional[int] = None         # ... of its first launch only: a shorter one brings the first audio sooner
    due: float = 0.0                          # urgency when more requests are ready than a launch has columns: smallest first
    hold: bool = False                        # set by the caller between steps: not launched (a listener far enough ahead)
    seq: int = 0                              # admission order, the tie-break of ``due``
    prompt_rows: int = 0                      # cache rows of the prompt: frame s writes row prompt_rows + s
    parked: Optional[torch.Tensor] = None     # paged engine: the request's KV pages while parked in host memory

    def budget(self, n_frames: int) -> int:
        """frames the next launch may emit for this request"""
        if self.frames == 0 and self.first_chunk:
            return self.first_chunk
        return self.chunk_size or n_frames

    def ready(self) -> bool:
        """A text-fed request is launched once the rows of its next ``rows_ahead`` frames exist (fewer where
        max_new_tokens ends it first), once its text is closed, or once it has reached max_new_tokens (the launch then
        reports it finished).  A request on ``hold`` is not launched."""
        if self.hold:
            return False
        if self.feed is None or self.feed.closed or self.frames >= self.max_new_tokens:
            return True
        need = min(self.gen0 + self.frames + self.rows_ahead, self.gen0 + self.max_new_tokens)
        return self.feed.n_rows >= need


# keyword defaults of BatchScheduler.submit, which submit_many applies to every request
_SUBMIT_DEFAULTS = dict(max_new_tokens=2048, min_new_tokens=2, temperature=0.9, top_k=50, top_p=1.0, do_sample=True,
                        repetition_penalty=1.05, uniforms=None)


class KvPager:
    """The talker KV pages of a paged engine (``Engine(kv_pages=N)``) as one scheduler hands them to its slots.  A slot
    maps the pages of the rows it has written and of its next launch; a parked request's pages wait in pinned host
    memory (``park`` / ``restore``), its slot keeping everything else.  ``peak``: most pages in use at once."""

    def __init__(self, engine):
        self.engine = engine
        self.free: List[int] = list(range(engine.kv_pages))
        self.mapped: Dict[int, List[int]] = {}
        self.peak = 0
        self.parks = 0

    @staticmethod
    def pages(rows: int) -> int:
        return -(-int(rows) // KV_PAGE)

    def in_use(self) -> int:
        return self.engine.kv_pages - len(self.free)

    def rows(self, slot: int) -> int:
        return KV_PAGE * len(self.mapped.get(slot, ()))

    def grow(self, slot: int, rows: int) -> int:
        """map pages for the slot's rows [0, rows) as far as free pages go; -> the rows it maps"""
        have = self.mapped.setdefault(slot, [])
        n = min(self.pages(rows) - len(have), len(self.free))
        if n > 0:
            self.engine.map_kv_pages(slot, have + self.free[:n])
            have += self.free[:n]
            del self.free[:n]
            self.peak = max(self.peak, self.in_use())
        return self.rows(slot)

    def release(self, slot: int) -> None:
        pages = self.mapped.pop(slot, [])
        if pages:
            self.engine.map_kv_pages(slot, [])
            self.free += pages

    def park(self, slot: int, rows: int) -> torch.Tensor:
        """copy the pages of the slot's rows [0, rows) to pinned host memory and free all its pages"""
        pages = self.mapped.get(slot, [])[: self.pages(rows)]
        host = torch.empty(len(pages), self.engine.kv_page_bytes, dtype=torch.uint8,
                           pin_memory=torch.cuda.is_available())
        self.engine.kv_pages_to(pages, host)
        self.release(slot)
        self.parks += 1
        return host

    def restore(self, slot: int, host: torch.Tensor, rows: int) -> bool:
        """once free pages cover rows [0, rows): map them and copy the parked pages back into the first ones"""
        if self.pages(rows) > len(self.free) or self.mapped.get(slot):
            return False
        n = int(host.shape[0])
        self.grow(slot, n * KV_PAGE)
        self.engine.kv_pages_from(self.mapped[slot], host)
        if torch.cuda.is_available():   # the host buffer is dropped after this
            torch.cuda.current_stream(getattr(self.engine, "device", None)).synchronize()
        return True


def _frames_arg(name: str, v) -> Optional[int]:
    if v is None:
        return None
    if int(v) < 1:
        raise ValueError(f"{name} must be at least 1 frame, got {v}")
    return int(v)


class BatchScheduler:
    """Owns the engine's slots: ``submit`` prefills one request into a free slot and latches it (``submit_many``:
    several, with one batched prefill), ``step`` advances the ready slots by up to ``n_frames`` frames with ONE launch
    and returns the new codes per request, ``cancel`` frees a slot.  A text-fed request (``feed``) is ready while its next trailing row exists or its text is closed; a
    slot that waits for text costs the others nothing.

    The engine holds ``max_slots`` requests and a launch carries ``max_batch`` of them.  While no more than that are
    ready, ``step`` launches all of them.  When more are, it launches the ``max_batch`` with the smallest ``due``
    (ties: the one admitted first); the others keep their slot and state and cost the launch nothing.  ``due`` and
    ``hold`` belong to the caller, which sets them between steps (serving.ContinuousBatcher: the listener's playback
    lead).  A request's ``chunk_size`` / ``first_chunk`` replace the step's ``n_frames`` for that request alone: its codes
    do not depend on them, only how many frames each launch hands back.

    Paged engines (``Engine(kv_pages=N)``, a pool smaller than ``max_slots x max_seq_len`` rows) get their talker KV
    pages through ``pager`` (``KvPager``); with the default pool it is None and the scheduler makes no page calls.
    Admission (``submit_many``) needs a free slot and free pages for each prompt plus one chunk (the frames of the last
    step), else ``has_capacity()`` is false and it raises as when slots run out.  Before each step every launched
    request maps pages for its position plus budget (at most ``max_seq_len`` rows).  One that cannot get them all is
    launched only if its pages hold all the frames it has left, for those; otherwise it is not launched, like a request
    waiting for text.  A launch thus never ends inside a chunk, so every request's chunks (and under the codec's window
    policy its audio) are those it gets when pages are plenty.  When no ready
    request can advance one frame, the resident request with the largest ``due`` (ties: the latest admitted) other
    than the most urgent ready one is *parked*: its pages go to pinned host memory and are freed, its slot and the rest
    of its state stay.  It is restored into whatever pages are free, before it is next launched, once they cover its
    rows plus one chunk.  Parking is exact: a page comes back with the bytes it left with.
    Progress: the pool holds at least one request of ``max_seq_len`` rows (the engine refuses a smaller one), so after
    parking every other resident request the most urgent ready one has all the pages it can use and advances.  A
    request parks only while another is launched instead, so, as for starvation above, it runs again once its
    ``due`` is the smallest.  Pages are freed when a request finishes or is cancelled, parked or not."""

    def __init__(self, engine, talker, config, predictor_graph, talker_graph, slots=None):
        """``slots``: the engine's request slots this scheduler hands out (default: all of them)."""
        self.engine, self.talker, self.config = engine, talker, config
        self.pg, self.tg = predictor_graph, talker_graph
        self.free: List[int] = list(range(getattr(engine, "max_slots", engine.max_batch))) if slots is None \
            else [int(s) for s in slots]
        self.max_slots = len(self.free)
        self.max_prompts = engine.max_batch   # prompts one submit_many takes (one batched prefill)
        self.active: Dict[int, SlotRequest] = {}
        self._seq = 0
        self.max_seq_len = getattr(engine, "max_seq_len", None)   # longest prompt a slot takes
        self.pager = KvPager(engine) if getattr(engine, "paged", False) else None
        self._chunk = 1   # frames of the last step: the chunk a paged admission reserves pages for

    def __len__(self) -> int:
        return len(self.active)

    def has_capacity(self) -> bool:
        return bool(self.free) and (self.pager is None or bool(self.pager.free))

    def _admit_rows(self, r: dict) -> int:
        """cache rows a request needs at admission: its prompt plus one chunk (a frame at row max_seq_len - 1 writes
        none)"""
        chunk = r.get("first_chunk") or r.get("chunk_size") or self._chunk
        P = int(r["tie"].shape[1])
        return max(P, min(P + int(chunk), self.max_seq_len - 1))

    def admits(self, requests: List[dict]) -> bool:
        """whether ``submit_many(requests)`` finds the slots and KV pages it needs"""
        if len(requests) > len(self.free):
            return False
        return self.pager is None or \
            sum(KvPager.pages(self._admit_rows(r)) for r in requests) <= len(self.pager.free)

    def capacity(self) -> int:
        """free request slots"""
        return len(self.free)

    @torch.inference_mode()
    def submit(self, tie, tam, tth, tpe, *, tag=None, max_new_tokens: int = 2048, min_new_tokens: int = 2,
               temperature: float = 0.9, top_k: int = 50, top_p: float = 1.0, do_sample: bool = True,
               repetition_penalty: float = 1.05, uniforms: Optional[torch.Tensor] = None, feed=None,
               rows_ahead: int = 1, chunk_size: Optional[int] = None, first_chunk: Optional[int] = None) -> SlotRequest:
        """One request: tie [1,P,H], tam [1,P] (zeros = left padding), tth [1,Tt,H], tpe [1,1,H].  ``feed``: a
        ``text_stream.TextFeed`` whose row buffer replaces ``tth``; ``rows_ahead``: rows it must hold beyond the next
        frame's before the slot is launched (``n_frames`` of the steps keeps every launch a full chunk).
        ``chunk_size`` / ``first_chunk``: this request's frames per launch / in its first launch."""
        return self.submit_many([dict(tie=tie, tam=tam, tth=tth, tpe=tpe, tag=tag, max_new_tokens=max_new_tokens,
                                      min_new_tokens=min_new_tokens, temperature=temperature, top_k=top_k, top_p=top_p,
                                      do_sample=do_sample, repetition_penalty=repetition_penalty, uniforms=uniforms,
                                      feed=feed, rows_ahead=rows_ahead, chunk_size=chunk_size,
                                      first_chunk=first_chunk)])[0]

    def _next_seq(self) -> int:
        self._seq += 1
        return self._seq

    @torch.inference_mode()
    def submit_many(self, requests: List[dict], logprobs: bool = False) -> List[SlotRequest]:
        """Several requests at once: ``requests[i]`` holds the arguments of one ``submit`` call by name (tie, tam, tth,
        tpe, tag, the sampling keywords, uniforms, feed, rows_ahead, chunk_size, first_chunk).  They take the slots consecutive ``submit`` calls
        would take and latch what those would latch, but on a K3 engine their prompts share ONE prefill launch chain
        (``generate.begin_fused_batch``).  All or none: on an error every slot is released.  ``logprobs``: every
        ``step`` also sets ``chunk_logprobs`` (and, at the end, ``eos_logprob``) of these requests (logprobs.py)."""
        n = len(requests)
        if n > len(self.free):
            raise RuntimeError(f"{n} requests but only {len(self.free)} of {self.max_slots} request slots are free")
        if not self.admits(requests):
            raise RuntimeError(f"{n} requests need more KV pages than the {len(self.pager.free)} of "
                               f"{self.engine.kv_pages} that are free")
        chunking = [(_frames_arg("chunk_size", r.get("chunk_size")), _frames_arg("first_chunk", r.get("first_chunk")))
                    for r in requests]
        slots, self.free = self.free[:n], self.free[n:]
        rows = []
        for r in requests:
            gen = dict(_SUBMIT_DEFAULTS)
            gen.update({k: v for k, v in r.items() if k not in ("tag", "feed", "rows_ahead", "chunk_size", "first_chunk")})
            gen["trailing_len"] = None if r.get("feed") is None else 0
            rows.append(gen)
        first_lps = [None] * n
        lkw = {"logprob": True} if logprobs else {}   # off: the calls of a scheduler without the option
        try:
            if self.pager is not None:
                for slot, r in zip(slots, requests):
                    self.pager.grow(slot, self._admit_rows(r))
            if n == 1:   # one request: ``begin_fused``, the one-row case of ``begin_fused_batch``
                r = rows[0]
                got = begin_fused(self.engine, self.talker, r["tie"], r["tam"], r["tth"], r["tpe"], self.config, self.pg,
                                  self.tg, slot=slots[0], **{k: v for k, v in r.items() if k not in ("tie", "tam", "tth", "tpe")},
                                  **lkw)
                first_lps = [got[1]] if logprobs else first_lps
            elif n:
                got = begin_fused_batch(self.engine, self.talker, rows, self.config, self.pg, self.tg, slots, **lkw)
                first_lps = got[1] if logprobs else first_lps
            for slot, r in zip(slots, requests):
                if r.get("feed") is not None:
                    self.engine.set_text_rows(slot, r["feed"].update(), open=not r["feed"].closed)
        except Exception:
            if self.pager is not None:
                for slot in slots:
                    self.pager.release(slot)
            self.free = slots + self.free
            raise
        out = []
        for slot, r, gen, flp, (chunk_size, first_chunk) in zip(slots, requests, rows, first_lps, chunking):
            tag = r.get("tag")
            rq = SlotRequest(slot=slot, tag=tag if tag is not None else slot, max_new_tokens=gen["max_new_tokens"],
                             feed=r.get("feed"), gen0=self.engine.gen_step0[slot], rows_ahead=max(1, int(r.get("rows_ahead", 1))),
                             lp=FrameLogprobs(flp) if logprobs else None, chunk_size=chunk_size, first_chunk=first_chunk,
                             seq=self._next_seq(),
                             prompt_rows=int(r["tie"].shape[1]) if self.pager is not None else 0)
            self.active[slot] = rq
            out.append(rq)
        return out

    @torch.inference_mode()
    def step(self, n_frames: int) -> List[Tuple[SlotRequest, torch.Tensor]]:
        """Advance the ready slots -- all of them, or the ``max_batch`` most urgent (class docstring); returns [(request,
        codes [n,16])] for every slot that was launched (n may be 0 for a slot that stopped before emitting).  Finished
        slots are released."""
        for rq in self.active.values():
            if rq.feed is not None:
                self.engine.set_text_rows(rq.slot, rq.feed.update(), open=not rq.feed.closed)
        ready = [rq for rq in self.active.values() if rq.ready()]
        self._chunk = n_frames
        if self.pager is not None:
            budget_of = self._page_budgets(ready, n_frames)
        else:
            if len(ready) > self.engine.max_batch:
                ready = sorted(ready, key=lambda rq: (rq.due, rq.seq))[: self.engine.max_batch]
            budget_of = {rq.slot: rq.budget(n_frames) for rq in ready}
        slots = sorted(budget_of)
        if not slots:
            return []
        budgets = [budget_of[s] for s in slots]
        if len(set(budgets)) > 1:
            n_frames = budgets              # one budget per slot (fq3_decode_chunk_n)
        else:
            n_frames = budgets[0]           # without per-request chunking: the step's n_frames, the calls made without it
        want_lp = any(self.active[s].lp is not None for s in slots)
        lps = [None] * len(slots)
        # off: the calls are exactly those of a scheduler without the option
        if len(slots) == 1 and want_lp:
            codes, lp, res = self.engine.decode_chunk(n_frames, slot=slots[0], logprobs=True)
            outs, lps, ress = [codes], [lp], [res]
        elif len(slots) == 1:
            codes, res = self.engine.decode_chunk(n_frames, slot=slots[0])
            outs, ress = [codes], [res]
        else:
            if want_lp:
                buf, lpb, ress = self.engine.decode_chunk_batch(slots, n_frames, logprobs=True)
                lps = [lpb[j, : ress[j].frames_emitted] for j in range(len(slots))]
            else:
                buf, ress = self.engine.decode_chunk_batch(slots, n_frames)
            outs = [buf[j, : ress[j].frames_emitted] for j in range(len(slots))]
        done = []
        for s, c, r, lp in zip(slots, outs, ress, lps):
            rq = self.active[s]
            rq.frames += int(r.frames_emitted)
            rq.finished = int(r.finished)
            if rq.lp is not None:
                rq.chunk_logprobs = rq.lp.push(lp)
                rq.eos_logprob = rq.lp.eos_logprob(r.next_token, self.engine.eos)
            done.append((rq, c.clone()))
            if r.finished:
                self._end(rq)
        return done

    def _end(self, rq: SlotRequest) -> None:
        del self.active[rq.slot]
        rq.parked = None
        if self.pager is not None:
            self.pager.release(rq.slot)
        self.free.append(rq.slot)

    def _fit(self, rq: SlotRequest, budget: int) -> int:
        """paged engine: restore a parked request and map pages for its next ``budget`` frames; -> the budget of its
        launch (0: not launched)"""
        pos = rq.prompt_rows + rq.frames                      # the row its next frame writes
        want = min(pos + budget, self.max_seq_len - 1)        # a frame at row max_seq_len - 1 writes nothing
        if rq.parked is not None:
            if not self.pager.restore(rq.slot, rq.parked, want):
                return 0
            rq.parked = None
        got = self.pager.grow(rq.slot, want)
        if got >= want:
            return budget
        # short of pages: only the frames the request has left, never part of a chunk, so that its launches end where
        # they end when pages are plenty (a window policy's audio depends on where its chunks end)
        left = rq.max_new_tokens - rq.frames
        return left if 0 < left and min(pos + left, self.max_seq_len - 1) <= got else 0

    def _page_budgets(self, ready: List[SlotRequest], n_frames: int) -> Dict[int, int]:
        """paged engine: {slot: budget} of the next launch, parking requests while none can advance (class docstring)"""
        order = sorted(ready, key=lambda rq: (rq.due, rq.seq))
        parked = set()   # parked by this step: not restored in it, or the pages would cycle
        while True:
            out = {}
            for rq in order:
                if len(out) == self.engine.max_batch:
                    break
                if rq.slot in parked:
                    continue
                b = self._fit(rq, rq.budget(n_frames))
                if b > 0:
                    out[rq.slot] = b
            if out or not order:
                return out
            victims = [rq for rq in self.active.values()
                       if rq is not order[0] and rq.parked is None and self.pager.rows(rq.slot)]
            if not victims:
                return out
            victim = max(victims, key=lambda rq: (rq.due, rq.seq))
            self.park(victim)
            parked.add(victim.slot)

    def park(self, rq: SlotRequest) -> None:
        """paged engine: move the request's KV pages to host memory; it is restored before it is next launched"""
        rq.parked = self.pager.park(rq.slot, min(rq.prompt_rows + rq.frames, self.max_seq_len))

    def cancel(self, rq: SlotRequest) -> None:
        """End a request now and free its slot (a client that went away)."""
        if self.active.get(rq.slot) is rq:
            self._end(rq)


def _single(engine, talker, config, predictor_graph, talker_graph, request: dict, logprobs: bool = False):
    """The one request of a single-request driver (``submit_many`` arguments), admitted to a scheduler that owns only
    the slot the graph handles drive.  -> (scheduler, request, prefill seconds)"""
    sched = BatchScheduler(engine, talker, config, predictor_graph, talker_graph,
                           slots=[getattr(talker_graph, "slot", 0)])
    t0 = time.time()
    rq = sched.submit_many([request], logprobs=logprobs)[0]
    _sync(request["tie"].device)
    return sched, rq, time.time() - t0


def _chunks(sched: BatchScheduler, chunk_size: int, t_prefill: float, before_step=None):
    """The launch loop of the fused drivers: ``sched.step(chunk_size)`` until no request is left.  Yields, per step that
    produced frames, [(request, codes [n,16], timing)] with the reference's per-chunk timing keys, "kernel_ms" when the
    engine times its kernels, and for a request admitted with log-probabilities "logprobs" [n,16] and, on its last
    chunk, "eos_logprob".  ``before_step`` runs before every step, inside its "decode_ms"."""
    engine, idx = sched.engine, 0
    while len(sched):
        t1 = time.time()
        if before_step is not None:
            before_step()
        out = sched.step(chunk_size)
        dt = time.time() - t1
        items = []
        for rq, codes in out:
            n = int(codes.shape[0])
            if not n:
                continue
            # the reference flags the trailing partial chunk -- and a full chunk cut off by the cache limit, which
            # leaves its loop before the "buffer full" check (streaming.py:130-132 vs :158-173)
            tm = {"chunk_index": idx, "chunk_steps": n, "prefill_ms": t_prefill * 1000 if idx == 0 else 0,
                  "decode_ms": dt * 1000, "total_steps_so_far": rq.frames,
                  "is_final": n < chunk_size or rq.finished == FQ3_FIN_MAX_SEQ}
            if engine.time_kernels:
                tm["kernel_ms"] = engine.last_kernel_ms
            if rq.lp is not None:
                tm["logprobs"] = rq.chunk_logprobs
                if rq.finished or rq.eos_logprob is not None:   # nothing follows this chunk
                    tm["eos_logprob"] = rq.eos_logprob
            items.append((rq, codes, tm))
        if items:
            yield items
            idx += 1


def _rows(x: torch.Tensor, b: int) -> torch.Tensor:
    return x[b:b + 1]


@torch.inference_mode()
def fast_generate_streaming_batch(
    talker,
    talker_input_embeds: torch.Tensor,     # [B,P,H] left-padded (model.py:774-787)
    attention_mask: torch.Tensor,          # [B,P]
    trailing_text_hiddens: torch.Tensor,   # [B,Tt,H] (rows padded with tts_pad_embed, model.py:789-803)
    tts_pad_embed: torch.Tensor,
    config,
    predictor_graph,
    talker_graph,
    max_new_tokens: int = 2048,
    min_new_tokens: int = 2,
    temperature: float = 0.9,
    top_k: int = 50,
    top_p: float = 1.0,
    do_sample: bool = True,
    repetition_penalty: float = 1.05,
    chunk_size: int = 12,
    uniforms: Optional[torch.Tensor] = None,   # [B, max_new_tokens+1, 16]
    return_logprobs: bool = False,
) -> Generator[List[Tuple[int, torch.Tensor, dict]], None, None]:
    """Batched counterpart of ``fast_generate_streaming`` (streaming.py:19-188): every yielded item is the list of
    (row, codes [n,16], timing) of the rows that produced frames in that chunk; timing keys are the reference's, plus
    with ``return_logprobs`` "logprobs" [n,16] and, on a row's last chunk, "eos_logprob" (as fast_generate_streaming)."""
    engine = shared_engine(predictor_graph, talker_graph)
    if engine is None:
        raise RuntimeError("batched decode needs graph handles backed by one loaded fq3 engine")
    B = talker_input_embeds.shape[0]
    if B > engine.max_batch:   # one prefill call and lock-step launches: the rows are columns, whatever max_slots is
        raise ValueError(f"batch of {B} rows exceeds the engine's max_batch={engine.max_batch}")
    sched = BatchScheduler(engine, talker, config, predictor_graph, talker_graph)
    device = talker_input_embeds.device
    t0 = time.time()
    sched.submit_many([dict(tie=_rows(talker_input_embeds, b), tam=_rows(attention_mask, b),
                            tth=_rows(trailing_text_hiddens, b), tpe=tts_pad_embed, tag=b, max_new_tokens=max_new_tokens,
                            min_new_tokens=min_new_tokens, temperature=temperature, top_k=top_k, top_p=top_p,
                            do_sample=do_sample, repetition_penalty=repetition_penalty,
                            uniforms=None if uniforms is None else uniforms[b]) for b in range(B)],
                      logprobs=return_logprobs)
    _sync(device)
    for items in _chunks(sched, chunk_size, time.time() - t0):
        yield [(rq.tag, codes, tm) for rq, codes, tm in items]


@torch.inference_mode()
def fast_generate_batch(talker, talker_input_embeds, attention_mask, trailing_text_hiddens, tts_pad_embed, config,
                        predictor_graph, talker_graph, max_new_tokens: int = 2048, min_new_tokens: int = 2,
                        temperature: float = 0.9, top_k: int = 50, top_p: float = 1.0, do_sample: bool = True,
                        repetition_penalty: float = 1.05, uniforms: Optional[torch.Tensor] = None,
                        launch_frames: int = 64, return_logprobs: bool = False) -> Tuple[List[Optional[torch.Tensor]], dict]:
    """Batched counterpart of ``fast_generate`` (generate.py:16-215): (list of codes [steps_b,16] or None per row,
    timing with the reference's keys; ``steps`` is the total over rows).  ``return_logprobs``: timing also holds
    "logprobs" (per row float32 [steps_b,16]) and "eos_logprob" (per row, or None)."""
    B = talker_input_embeds.shape[0]
    parts: List[List[torch.Tensor]] = [[] for _ in range(B)]
    lparts: List[List[torch.Tensor]] = [[] for _ in range(B)]
    eos_lp: List[Optional[float]] = [None] * B
    t0 = time.time()
    prefill_ms = 0.0
    for items in fast_generate_streaming_batch(
            talker, talker_input_embeds, attention_mask, trailing_text_hiddens, tts_pad_embed, config, predictor_graph,
            talker_graph, max_new_tokens=max_new_tokens, min_new_tokens=min_new_tokens, temperature=temperature,
            top_k=top_k, top_p=top_p, do_sample=do_sample, repetition_penalty=repetition_penalty,
            chunk_size=launch_frames, uniforms=uniforms, return_logprobs=return_logprobs):
        for b, codes, tm in items:
            parts[b].append(codes)
            if return_logprobs:
                lparts[b].append(tm["logprobs"])
                eos_lp[b] = tm.get("eos_logprob", eos_lp[b])
            prefill_ms = max(prefill_ms, tm["prefill_ms"])
    _sync(talker_input_embeds.device)
    dt = time.time() - t0 - prefill_ms / 1000
    out = [torch.cat(p) if p else None for p in parts]
    n = sum(int(c.shape[0]) for c in out if c is not None)
    timing = {"prefill_ms": prefill_ms, "decode_s": dt, "steps": n, "ms_per_step": (dt / n * 1000) if n else 0,
              "steps_per_s": (n / dt) if dt > 0 else 0}
    if return_logprobs:
        timing["logprobs"] = [torch.cat(p) if p else torch.zeros(0, 16) for p in lparts]
        timing["eos_logprob"] = eos_lp
    return out, timing
