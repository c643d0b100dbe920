"""Incremental text input: a streaming request that is fed its text while it is being spoken.

In the step-by-step text layout (``non_streaming_mode=False``) the prompt holds only the first text token; every later
token is one row of ``trailing_text_hiddens``, and decode frame ``s`` adds row ``s`` to the talker input (``tts_pad``
once the rows run out).  A request therefore needs text row ``k`` only at frame ``k``.  ``TextFeed`` turns text pieces
as they arrive (an LLM's reply, token by token) into committed token ids and talker rows; the engine's open-text gate
(``fq3_set_text_rows``) stops a slot at the frame that would need a row that has not arrived, instead of running ahead
on ``tts_pad``.  The model then sees exactly the inputs of the one-shot request, whatever the split of the text and
however fast it comes.

Commit rule: tokenize the chat template around all text received so far, hold back the last pre-token (Qwen2
pre-tokenization), and commit only ids that are also a prefix of the tokenization of everything received so far.
Committed ids are never retracted; at ``close()`` they must equal the one-shot body ids ``ids[3:-5]``.
"""
from __future__ import annotations

import time
from typing import Iterable, Iterator, List, Optional

import regex
import torch

# transformers.models.qwen2.tokenization_qwen2.PRETOKENIZE_REGEX
PRETOKENIZE_REGEX = (r"""(?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\r\n\p{L}\p{N}]?\p{L}+|\p{N}| ?[^\s\p{L}\p{N}]+[\r\n]*|"""
                     r"""\s*[\r\n]+|\s+(?!\S)|\s+""")
_PRETOKEN = regex.compile(PRETOKENIZE_REGEX)


def stable_prefix(text: str) -> str:
    """``text`` without its last pre-token: the part whose pre-tokenization no later text can change."""
    last = None
    for last in _PRETOKEN.finditer(text):
        pass
    return text[: last.start()] if last is not None else ""


class TextCommitter:
    """Text pieces -> committed body token ids.  ``tokenizer`` is the upstream wrapper (``Qwen3TTSModel`` or the
    synthetic stand-in): only ``_build_assistant_text`` and ``_tokenize_texts`` are called."""

    def __init__(self, tokenizer):
        self.tok = tokenizer
        self.text = ""
        self.ids: List[int] = []
        self.role: Optional[List[int]] = None   # the 3 role ids and 5 closing ids of the assistant turn
        self.tail: Optional[List[int]] = None
        self.closed = False

    def _tokenize(self, text: str) -> List[int]:
        return [int(x) for x in self.tok._tokenize_texts([self.tok._build_assistant_text(text)])[0].reshape(-1).tolist()]

    def push(self, piece: str) -> int:
        """Append text; returns the number of ids committed by this call."""
        if self.closed:
            raise RuntimeError("text stream already closed")
        if not piece:
            return 0
        self.text += piece
        full = self._tokenize(self.text)
        self.role, self.tail = full[:3], full[-5:]
        stable = self._tokenize(stable_prefix(self.text))[3:-5]
        body = full[3:-5]
        n = 0
        while n < min(len(stable), len(body)) and stable[n] == body[n]:
            n += 1
        if n <= len(self.ids):
            return 0
        if stable[: len(self.ids)] != self.ids:
            raise RuntimeError("text commit rule violated: committed ids are no longer a prefix of the text's tokenization")
        new = stable[len(self.ids): n]
        self.ids += new
        return len(new)

    def close(self) -> int:
        """Commit the rest: the committed ids then equal the one-shot body ids."""
        if self.closed:
            return 0
        self.closed = True
        if not self.text:
            return 0
        full = self._tokenize(self.text)
        self.role, self.tail = full[:3], full[-5:]
        body = full[3:-5]
        if body[: len(self.ids)] != self.ids:
            raise RuntimeError("text commit rule violated: committed ids differ from the one-shot tokenization")
        n = len(body) - len(self.ids)
        self.ids = body
        return n


class TextFeed:
    """One text-fed request: committed ids -> talker rows in a preallocated device buffer.

    ``rows`` [max_rows, H] (model dtype) is the buffer the engine latches as trailing text.  Row ``k`` is the text
    embedding of body id ``k + 1``; at ``close()`` the one-shot ``tts_eos`` row follows the last text row.  Rows past
    ``max_rows`` (= max_new_tokens) are never read by the decode loop and are not written.  Each id is embedded in a call
    of its own, so the row numerics do not depend on how the text was split."""

    def __init__(self, model, max_rows: int):
        self.model = model                 # FasterQwen3TTS
        self.committer = TextCommitter(model.model)
        self.talker = model.model.model.talker
        self.max_rows = int(max_rows)
        self.rows: Optional[torch.Tensor] = None
        self.eos_row: Optional[torch.Tensor] = None
        self.n_rows = 0                    # rows valid in ``rows``
        self._embedded = 0                 # body ids already turned into rows (body id 0 lives in the prompt)

    @property
    def closed(self) -> bool:
        return self.committer.closed

    @property
    def n_ids(self) -> int:
        return len(self.committer.ids)

    def push(self, piece: str) -> int:
        return self.committer.push(piece)

    def close(self) -> None:
        self.committer.close()
        if not self.committer.ids:
            raise ValueError("the text stream closed without any text")

    def prompt_ids(self) -> torch.Tensor:
        """role + [body id 0] + closing ids: the prompt of the one-shot request is built from exactly these"""
        c = self.committer
        ids = c.role + c.ids[:1] + c.tail
        return torch.tensor([ids], dtype=torch.long, device=self.talker.device)

    def start(self, eos_row: torch.Tensor, dtype: torch.dtype) -> None:
        """``eos_row``: the trailing row ``build_talker_inputs`` returns for a one-token body (the one-shot eos row)."""
        H = eos_row.shape[-1]
        self.eos_row = eos_row.reshape(1, H).to(dtype)
        self.rows = torch.zeros(max(self.max_rows, 1), H, dtype=dtype, device=eos_row.device)

    @torch.inference_mode()
    def update(self) -> int:
        """Embed the newly committed ids (and the eos row once closed); returns the number of valid rows."""
        ids = self.committer.ids
        emb = self.talker.get_text_embeddings()
        while self._embedded + 1 < len(ids) and self.n_rows < self.max_rows:
            t = torch.tensor([[ids[self._embedded + 1]]], dtype=torch.long, device=self.rows.device)
            self.rows[self.n_rows] = self.talker.text_projection(emb(t))[0, 0].to(self.rows.dtype)
            self._embedded += 1
            self.n_rows += 1
        if self.closed and self._embedded + 1 >= len(ids) and self.n_rows < self.max_rows \
                and self.n_rows == len(ids) - 1:
            self.rows[self.n_rows] = self.eos_row[0]
            self.n_rows += 1
        return self.n_rows


def build_prompt(model, feed: TextFeed, *, language, speaker=None, instruct_ids=None, voice_clone_prompt=None):
    """The prompt of a text-fed request, from the feed's first committed id: ``build_talker_inputs`` on ids
    ``role + [body id 0] + closing ids``, which makes it bit-identical to the one-shot prompt.  Starts the feed's row
    buffer with the one-shot eos row.  -> (tie, tam, tpe)"""
    from .prompt import build_talker_inputs
    m = model.model.model
    tie, tam, tth, tpe = build_talker_inputs(
        m, input_ids=[feed.prompt_ids()], ref_ids=[None], voice_clone_prompt=voice_clone_prompt,
        languages=[language if language is not None else "Auto"], speakers=[speaker], non_streaming_mode=False,
        instruct_ids=[instruct_ids])
    if not model._warmed_up:
        model.warmup(tie.shape[1])
    m.talker.rope_deltas = None
    feed.start(tth[0, 0], model.engine.dtype)
    return tie, tam, tpe


ICL_REFUSAL = ("text streaming is not available for ICL voice cloning: its target text sits under the reference codec "
               "frames inside the prompt, so it must be known before prefill; use x-vector cloning (xvec_only=True)")


def _refuse_unsupported(voice_clone_prompt, non_streaming_mode):
    """``voice_clone_prompt``: None or the resolved dict form (``_resolve_voice_clone_prompt``)"""
    if non_streaming_mode:
        raise ValueError("text streaming needs the step-by-step text layout (non_streaming_mode=False): "
                         "the non-streaming layout puts the whole text into the prompt")
    if voice_clone_prompt is not None and any(voice_clone_prompt.get("icl_mode", [False])):
        raise ValueError(ICL_REFUSAL)


@torch.inference_mode()
def generate_text_streaming(model, text_stream: Iterable[str], *, language: str, speaker=None, instruct_ids=None,
                            voice_clone_prompt=None, chunk_size: int = 12, max_new_tokens: int = 2048,
                            min_new_tokens: int = 2, temperature: float = 0.9, top_k: int = 50, top_p: float = 1.0,
                            do_sample: bool = True, repetition_penalty: float = 1.05, uniforms=None, to_host: bool = True,
                            speed: float = 1.0, sample_rate=None, pitch: float = 0.0,
                            gain_db: float = 0.0) -> Iterator:
    """Yields (pcm, sample_rate, timing) like the ``*_streaming`` methods.  Prefills once the first text id is
    committed, then per launch: pull text until the next chunk's rows exist (window codec policy) or one more row
    exists (stateful codec), or the text closes; announce the rows; decode one chunk.  The request is the one request of
    a ``BatchScheduler`` on the graph's slot: its ``rows_ahead`` rule (``SlotRequest.ready``) says when to launch.

    The window policy gets only full ``chunk_size`` chunks plus the final partial one, exactly the chunking of the
    one-shot request, so its PCM is identical.  The stateful codec decodes whatever frames exist at once: a stream equals
    the one-shot decode whatever the chunking.  ``timing`` has the reference's keys plus ``text_wait_ms``, the time this
    chunk spent blocked on ``text_stream``."""
    from .batching import _chunks, _single
    from .generate import shared_engine
    engine = shared_engine(model.predictor_graph, model.talker_graph)
    if engine is None:
        raise RuntimeError("text streaming needs graph handles backed by one loaded fq3 engine")
    m = model.model.model
    st = m.speech_tokenizer
    feed = TextFeed(model, max_rows=max_new_tokens)
    it = iter(text_stream)
    wait = [0.0]

    def pull(until) -> None:
        while not feed.closed and not until():
            t = time.perf_counter()
            try:
                piece = next(it)
            except StopIteration:
                piece = None
            wait[0] += time.perf_counter() - t
            if piece is None:
                feed.close()
            else:
                feed.push(piece)

    pull(lambda: feed.n_ids >= 1)
    if feed.n_ids == 0:
        feed.close()   # raises: no text at all
    tie, tam, tpe = build_prompt(model, feed, language=language, speaker=speaker, instruct_ids=instruct_ids,
                                 voice_clone_prompt=voice_clone_prompt)
    win = None
    if st is not None:
        from .model import _post_kw
        win = model._make_window(st, None, chunk_size, to_host, **_post_kw(speed, sample_rate, pitch, gain_db))
    # the window policy's PCM depends on the chunking: launch only when a full chunk of rows exists, so that every launch
    # emits a full chunk or ends the request.  A stateful stream (or codes only) is the same in any chunking.
    ahead = 1 if win is None or getattr(win, "any_chunking", False) else chunk_size
    sched, rq, t_prefill = _single(
        engine, m.talker, m.config.talker_config, model.predictor_graph, model.talker_graph,
        dict(tie=tie, tam=tam, tth=feed.rows[None], tpe=tpe, max_new_tokens=max_new_tokens,
             min_new_tokens=min_new_tokens, temperature=temperature, top_k=top_k, top_p=top_p, do_sample=do_sample,
             repetition_penalty=repetition_penalty, uniforms=uniforms, feed=feed, rows_ahead=ahead))
    wait_before = wait[0]   # text wait before the prefill: reported with the first chunk, outside its decode window
    wait[0] = 0.0

    def rows_ready() -> bool:
        feed.update()
        return rq.ready()

    for (_, codes, tm), in _chunks(sched, chunk_size, t_prefill, before_step=lambda: pull(rows_ready)):
        tm.update(decode_ms=tm["decode_ms"] - wait[0] * 1000, is_final=bool(rq.finished),
                  text_wait_ms=(wait[0] + wait_before) * 1000)
        wait[0] = wait_before = 0.0
        if win is None:
            yield (codes.cpu().numpy() if to_host else codes), model.sample_rate, tm
        elif getattr(win, "tempo", None) is None and getattr(win, "resampler", None) is None:
            pcm, sr = win.push(codes)
            yield pcm, sr, tm
        else:   # the last chunk flushes the tempo and the resampler
            pcm, sr = win.push(codes, final=bool(rq.finished))
            yield pcm, sr, tm
    if win is not None:
        from .model import flush_windows
        for _, (pcm, sr) in zip(*flush_windows(st, [win])):   # a request that ended on a step without frames
            yield pcm, sr, {"chunk_steps": 0, "is_final": True}
