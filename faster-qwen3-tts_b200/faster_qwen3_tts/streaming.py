"""Streaming generation: same signature and per-chunk timing keys as the reference's ``fast_generate_streaming``
(faster_qwen3_tts/streaming.py:19-188).  One persistent-kernel launch produces one chunk of ``chunk_size`` frames;
the only host synchronisation is the end-of-chunk result read (the reference synchronises there too,
streaming.py:158)."""
from __future__ import annotations

import time
from typing import Generator, Optional, Tuple

import torch

from .batching import _chunks, _single
from .generate import _sync, shared_engine, special_suppress_mask, stepwise_frames
from .sampling import apply_repetition_penalty, sample_logits


def _timing(idx, n, t_prefill, dt, total, final):
    return {"chunk_index": idx, "chunk_steps": n, "prefill_ms": t_prefill * 1000 if idx == 0 else 0,
            "decode_ms": dt * 1000, "total_steps_so_far": total, "is_final": final}


@torch.inference_mode()
def fast_generate_streaming(
    talker,
    talker_input_embeds: torch.Tensor,
    attention_mask: torch.Tensor,
    trailing_text_hiddens: torch.Tensor,
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
    uniforms: Optional[torch.Tensor] = None,
    return_logprobs: bool = False,
) -> Generator[Tuple[torch.Tensor, dict], None, None]:
    """Yields (codes LongTensor[chunk_steps,16], timing); the last chunk may be short and has is_final=True
    only when it is a partial chunk, exactly like the reference.  ``return_logprobs`` (fused engine path only): every
    timing dict also holds "logprobs" (float32 [chunk_steps,16], the log-probability of every code; see logprobs.py),
    and the last chunk of the request "eos_logprob" (the EOS draw that ends it, or None)."""
    device = talker_input_embeds.device
    skw = dict(max_new_tokens=max_new_tokens, min_new_tokens=min_new_tokens, temperature=temperature, top_k=top_k,
               top_p=top_p, do_sample=do_sample, repetition_penalty=repetition_penalty)
    engine = shared_engine(predictor_graph, talker_graph)
    if return_logprobs and engine is None:
        raise ValueError("return_logprobs needs graph handles backed by one loaded fq3 engine (the fused decode path)")
    if engine is not None:
        sched, _, t_prefill = _single(engine, talker, config, predictor_graph, talker_graph,
                                      dict(tie=talker_input_embeds, tam=attention_mask, tth=trailing_text_hiddens,
                                           tpe=tts_pad_embed, uniforms=uniforms, **skw), return_logprobs)
        for items in _chunks(sched, chunk_size, t_prefill):
            for _, codes, tm in items:
                yield codes, tm
    else:
        yield from _chunked(stepwise_frames(talker, talker_input_embeds, attention_mask, trailing_text_hiddens,
                                            tts_pad_embed, config, predictor_graph, talker_graph, **skw),
                            device, chunk_size, time.time())


def _chunked(frames, device, chunk_size, t0):
    """Shared chunker of the host-driven paths: frames -> (codes [n,16], timing) with the reference's timing keys.  A
    full buffer is flushed (is_final False) when the step after its last frame completes; whatever is left when the
    generator ends -- a partial chunk, or a full one whose last step hit the cache limit -- is flagged is_final
    (streaming.py:158-188)."""
    buf, t_prefill, t1, total, idx = [], 0.0, t0, 0, 0
    for kind, row in frames:
        if kind == "prefill_done":
            _sync(device)
            t_prefill = time.time() - t0
            t1 = time.time()
            continue
        if kind == "frame":
            buf.append(row)
            continue
        if len(buf) >= chunk_size:   # "step_done"
            _sync(device)
            total += len(buf)
            yield torch.stack(buf), _timing(idx, len(buf), t_prefill, time.time() - t1, total, False)
            buf, idx, t1 = [], idx + 1, time.time()
    if buf:
        _sync(device)
        total += len(buf)
        yield torch.stack(buf), _timing(idx, len(buf), t_prefill, time.time() - t1, total, True)


def _dynamic_cache_frames(talker, tie, tam, tth, tpe, config, *, max_new_tokens, min_new_tokens, temperature, top_k,
                          top_p, do_sample, repetition_penalty):
    """The upstream talker driven step by step through its own ``forward`` with a growing (dynamic) KV cache: no
    static cache, no graphs, no engine -- the reference's baseline path (streaming.py:192-359).  Needs the upstream
    decode-step contract: ``forward(input_ids=[1,1], past_key_values=..., generation_step=..., past_hidden=...,
    subtalker_*=...)`` returning ``hidden_states[1]`` = the frame's 16 codes."""
    eos_id = config.codec_eos_token_id
    smask = special_suppress_mask(config.vocab_size, eos_id, tie.device)
    kw = dict(temperature=temperature, top_k=top_k, top_p=top_p, do_sample=do_sample, suppress_mask=smask)
    step_kw = dict(use_cache=True, output_hidden_states=True, return_dict=True, trailing_text_hidden=tth,
                   tts_pad_embed=tpe)
    out = talker.forward(inputs_embeds=tie, attention_mask=tam, generation_step=None, past_hidden=None,
                         past_key_values=None, **step_kw)
    token = sample_logits(out.logits[:, -1, :], suppress_tokens=[eos_id] if min_new_tokens > 0 else None, **kw)
    mask = tam.clone() if tam is not None else None
    yield "prefill_done", None
    history = []
    for _ in range(max_new_tokens):
        if token.item() == eos_id:
            return
        cache_position = None
        if mask is not None:   # one more attended position per step
            mask = torch.cat([mask, mask.new_ones((mask.shape[0], 1))], dim=1)
            cache_position = torch.tensor([mask.shape[1] - 1], device=mask.device)
        out = talker.forward(input_ids=token.view(1, 1), attention_mask=mask, generation_step=out.generation_step,
                             past_hidden=out.past_hidden, past_key_values=out.past_key_values,
                             subtalker_dosample=do_sample, subtalker_top_k=top_k, subtalker_top_p=top_p,
                             subtalker_temperature=temperature, cache_position=cache_position, **step_kw)
        frame = out.hidden_states[1]
        if frame is None:
            return
        history.append(token.detach())
        yield "frame", frame.squeeze(0).detach()
        logits = out.logits[:, -1, :]
        if repetition_penalty != 1.0:
            logits = apply_repetition_penalty(logits, torch.stack(history), repetition_penalty)
        token = sample_logits(logits, suppress_tokens=[eos_id] if len(history) < min_new_tokens else None, **kw)
        yield "step_done", None


@torch.inference_mode()
def parity_generate_streaming(
    talker,
    talker_input_embeds: torch.Tensor,
    attention_mask: torch.Tensor,
    trailing_text_hiddens: torch.Tensor,
    tts_pad_embed: torch.Tensor,
    config,
    max_new_tokens: int = 2048,
    min_new_tokens: int = 2,
    temperature: float = 0.9,
    top_k: int = 50,
    top_p: float = 1.0,
    do_sample: bool = True,
    repetition_penalty: float = 1.05,
    chunk_size: int = 12,
) -> Generator[Tuple[torch.Tensor, dict], None, None]:
    """Same signature, chunking and timing keys as the reference's ``parity_generate_streaming``
    (faster_qwen3_tts/streaming.py:192-359): streaming through the upstream talker's own dynamic-cache step (the
    baseline the fast path is compared with).  Raises NotImplementedError when the talker does not implement the
    upstream decode-step contract (the offline synthetic talker is prefill-only)."""
    if not getattr(talker, "supports_decode_step", hasattr(talker, "generate")):
        raise NotImplementedError("parity_mode needs the upstream qwen-tts talker (dynamic-cache decode step)")
    frames = _dynamic_cache_frames(talker, talker_input_embeds, attention_mask, trailing_text_hiddens, tts_pad_embed,
                                   config, max_new_tokens=max_new_tokens, min_new_tokens=min_new_tokens,
                                   temperature=temperature, top_k=top_k, top_p=top_p, do_sample=do_sample,
                                   repetition_penalty=repetition_penalty)
    yield from _chunked(frames, talker_input_embeds.device, chunk_size, time.time())
