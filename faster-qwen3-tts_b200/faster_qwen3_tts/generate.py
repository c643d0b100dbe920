"""Non-streaming generation: same signature, return value and timing keys as the reference's ``fast_generate``
(faster_qwen3_tts/generate.py:16-215).  When both graph objects are backed by one fq3 engine the whole decode
loop runs on device (one persistent-kernel launch per <=256 frames, issued by the launch loop of the batched drivers
on the graph's slot, batching.py); otherwise a step-wise loop drives any
duck-typed ``PredictorGraph`` / ``TalkerGraph`` (the contract of the reference's tests/test_sampling.py:79-93)."""
from __future__ import annotations

import time
from typing import Optional, Tuple

import torch

from .engine import SamplingParams
from .sampling import apply_repetition_penalty, sample_logits

_MAX_LAUNCH_FRAMES = 256


def shared_engine(predictor_graph, talker_graph):
    e1, e2 = getattr(predictor_graph, "engine", None), getattr(talker_graph, "engine", None)
    if e1 is not None and e1 is e2 and getattr(e1, "loaded", False):
        return e1
    return None


def special_suppress_mask(vocab_size: int, eos_id: int, device) -> torch.Tensor:
    """ids [vocab-1024, vocab) except EOS are never sampled (generate.py:46-50)."""
    mask = torch.zeros(vocab_size, dtype=torch.bool, device=device)
    mask[max(0, vocab_size - 1024):] = True
    if 0 <= eos_id < vocab_size:
        mask[eos_id] = False
    return mask


def _prefill(talker, tie, tam, tth, tpe):
    return talker.forward(inputs_embeds=tie, attention_mask=tam, use_cache=True, output_hidden_states=True,
                          return_dict=True, trailing_text_hidden=tth, tts_pad_embed=tpe, generation_step=None,
                          past_hidden=None, past_key_values=None)


def _native_prefill(engine, talker_graph, tie) -> bool:
    """K3 (the hand-written prefill) serves a [1,P,H] row of a bf16 engine; fp32 engines, graphs that opt out and
    multi-row inputs take the upstream ``talker.forward``."""
    return getattr(engine, "has_prefill", False) and getattr(talker_graph, "use_native_prefill", True) \
        and tie.shape[0] == 1


def _native_out(logits, hidden):
    import types
    return types.SimpleNamespace(logits=logits.view(1, 1, -1), past_hidden=hidden.view(1, 1, -1), generation_step=0,
                                 past_key_values=None)


def _first_token(engine, out, config, uniforms, u0, *, min_new_tokens, temperature, top_k, top_p, do_sample,
                 logprob=False, **_):
    """first cb0 token of a prefilled row (generate.py:119-120), a device tensor [1]; with ``logprob``: (token,
    its log-probability float32 [1])"""
    return engine.sample_logits(out.logits[:, -1, :], SamplingParams(do_sample, top_k, temperature, top_p, 1.0), u=u0,
                                suppress_special=True, eos_id=config.codec_eos_token_id, suppress_eos=min_new_tokens > 0,
                                return_logprob=logprob)


def _uniforms(engine, predictor_graph, uniforms, *, max_new_tokens, do_sample, **_):
    if (do_sample or predictor_graph.do_sample) and uniforms is None:
        uniforms = torch.rand(max_new_tokens + 1, 16, device=engine.device)
    return uniforms


def latch_fused(engine, talker, out, native, pad, tie, tth, tpe, predictor_graph, talker_graph, first, *, slot, uniforms,
                trailing_len, max_new_tokens, min_new_tokens, temperature, top_k, top_p, do_sample, repetition_penalty):
    """Latch half of ``begin_fused``: generation state and request of `slot` from a prefilled row ``out`` whose first
    token ``first`` (int) is sampled (generate.py:120-140)."""
    if native:
        prefill_len = int(tie.shape[1])
        n_left_pad, rope_delta = pad, -pad   # rotary position = cache index - pad count (talker_graph.py:210-211)
    else:
        prefill_len = 0
        for li in range(talker_graph.num_layers):
            k, v = out.past_key_values[li]
            prefill_len = engine.import_kv(li, k, v, slot=slot)
        rd = getattr(talker, "rope_deltas", None)
        n_left_pad = pad
        rope_delta = int(round(float(rd.reshape(-1)[0].item()))) if rd is not None else 0
    engine.set_generation_state(n_left_pad, rope_delta, slot=slot)
    if slot == getattr(talker_graph, "slot", 0):
        talker_graph.prefill_len, talker_graph.n_left_pad, talker_graph.rope_delta = prefill_len, n_left_pad, rope_delta
    gen_step = int(out.generation_step) if out.generation_step is not None else 0
    sp_t = SamplingParams(do_sample=do_sample, top_k=top_k, temperature=temperature, top_p=top_p,
                          repetition_penalty=repetition_penalty)
    engine.begin_request(first_token=int(first), prefill_len=prefill_len, gen_step=gen_step,
                         past_hidden=out.past_hidden, trailing_text=tth, tts_pad=tpe, max_new_tokens=max_new_tokens,
                         min_new_tokens=min_new_tokens, sp_talker=sp_t, sp_predictor=predictor_graph.sampling(),
                         uniforms=uniforms, rope_delta=rope_delta, n_left_pad=n_left_pad, slot=slot,
                         trailing_len=trailing_len)


def begin_fused(engine, talker, tie, tam, tth, tpe, config, predictor_graph, talker_graph, *, max_new_tokens,
                min_new_tokens, temperature, top_k, top_p, do_sample, repetition_penalty, uniforms, slot=None,
                trailing_len=None, logprob=False):
    """Prefill + first token + request latch (generate.py:104-140) for ONE row [1,P,H] into request slot `slot`
    (default: the slot the graph handles drive): the one-row case of ``begin_fused_batch``.  ``trailing_len``: rows of
    ``tth`` valid now (text-fed requests latch a larger buffer and announce rows later, ``Engine.set_text_rows``).
    Returns the first token id; with ``logprob`` (first token id, its log-probability as a float)."""
    row = dict(tie=tie, tam=tam, tth=tth, tpe=tpe, max_new_tokens=max_new_tokens, min_new_tokens=min_new_tokens,
               temperature=temperature, top_k=top_k, top_p=top_p, do_sample=do_sample,
               repetition_penalty=repetition_penalty, uniforms=uniforms, trailing_len=trailing_len)
    slot = int(getattr(talker_graph, "slot", 0) if slot is None else slot)
    got = begin_fused_batch(engine, talker, [row], config, predictor_graph, talker_graph, [slot], logprob=logprob)
    return (got[0][0], got[1][0]) if logprob else got[0]


def _gen(row):
    """the sampling keywords of a ``begin_fused_batch`` row"""
    return {k: v for k, v in row.items() if k not in ("tie", "tam", "tth", "tpe", "uniforms", "trailing_len")}


def _begin_upstream(engine, talker, row, config, predictor_graph, talker_graph, slot, logprob):
    """One row prefilled by the upstream ``talker.forward`` (fp32 engine, a graph that opts out of K3) and latched into
    `slot`, its KV cache imported: -> (first token id, its log-probability as a float or None)."""
    gen = _gen(row)
    pad = int((row["tam"][0] == 0).sum().item()) if row["tam"] is not None else 0
    out = _prefill(talker, row["tie"], row["tam"], row["tth"], row["tpe"])
    uniforms = _uniforms(engine, predictor_graph, row.get("uniforms"), **gen)
    u0 = float(uniforms.reshape(-1)[0]) if (gen["do_sample"] and uniforms is not None) else 0.0
    first = _first_token(engine, out, config, uniforms, u0, logprob=logprob, **gen)
    lp = None
    if logprob:
        first, lp = first
        lp = float(lp.item())
    first = int(first.item())
    latch_fused(engine, talker, out, False, pad, row["tie"], row["tth"], row["tpe"], predictor_graph, talker_graph, first,
                slot=slot, uniforms=uniforms, trailing_len=row.get("trailing_len"), **gen)
    return first, lp


def begin_fused_batch(engine, talker, rows, config, predictor_graph, talker_graph, slots, logprob=False):
    """Prefill + first token + request latch for several rows into distinct slots: ``rows[b]`` holds the arguments of
    one ``begin_fused`` call (tie [1,P,H], tam, tth, tpe, the sampling keywords, uniforms, trailing_len).  On a K3
    engine all prompts go through ONE ``Engine.prefill_batch`` and the first tokens of all rows come back with one host
    synchronisation.  Otherwise (fp32 engine, a graph that opts out of K3) each row is prefilled by the upstream
    ``talker.forward`` in turn.  Returns the first token ids; with ``logprob`` (ids, their log-probabilities as
    floats)."""
    if not all(_native_prefill(engine, talker_graph, r["tie"]) for r in rows):
        got = [_begin_upstream(engine, talker, r, config, predictor_graph, talker_graph, int(s), logprob)
               for r, s in zip(rows, slots)]
        firsts, lps = [f for f, _ in got], [lp for _, lp in got]
        return (firsts, lps) if logprob else firsts
    gens = [_gen(r) for r in rows]
    n = len(rows)
    uniforms = [_uniforms(engine, predictor_graph, r.get("uniforms"), **g) for r, g in zip(rows, gens)]
    # pad counts (host arrays of the C call) and first-token draws of all rows: one transfer (float64 holds both exactly)
    head = [torch.zeros(()) if r["tam"] is None else (r["tam"][0] == 0).sum() for r in rows] + \
        [u.reshape(-1)[0] if (g["do_sample"] and u is not None) else torch.zeros(()) for u, g in zip(uniforms, gens)]
    head = torch.stack([x.to(engine.device, torch.float64) for x in head]).tolist()
    pads, u0 = [int(x) for x in head[:n]], head[n:]
    logits, hidden = engine.prefill_batch([r["tie"][0] for r in rows], pads, slots)
    outs = [_native_out(logits[b], hidden[b]) for b in range(n)]
    got = [_first_token(engine, o, config, u, x, logprob=logprob, **g) for o, u, x, g in zip(outs, uniforms, u0, gens)]
    lps = None
    if logprob:
        got, lps = [t for t, _ in got], torch.cat([lp for _, lp in got]).tolist()
    firsts = torch.cat(got).tolist()   # the one host synchronisation of the first tokens
    for r, s, o, u, g, pad, first in zip(rows, slots, outs, uniforms, gens, pads, firsts):
        latch_fused(engine, talker, o, True, pad, r["tie"], r["tth"], r["tpe"], predictor_graph, talker_graph, first,
                    slot=int(s), uniforms=u, trailing_len=r.get("trailing_len"), **g)
    return (firsts, lps) if logprob else firsts


def stepwise_frames(talker, tie, tam, tth, tpe, config, predictor_graph, talker_graph, *, max_new_tokens,
                    min_new_tokens, temperature, top_k, top_p, do_sample, repetition_penalty):
    """Generator over frames for arbitrary duck-typed graphs (compatibility path; one host round trip per frame).
    Yields ("prefill_done", None) once, then per emitted frame ("frame", LongTensor[16]) and, once the talker step that
    follows it has been taken, ("step_done", None) -- a frame whose step is cut short by the cache limit
    (generate.py:175-177) has no "step_done"."""
    eos_id = config.codec_eos_token_id
    n_groups = config.num_code_groups
    smask = special_suppress_mask(config.vocab_size, eos_id, tie.device)
    embed_cb0 = talker.get_input_embeddings()
    embeds_rest = talker.code_predictor.get_input_embeddings()
    head = talker.codec_head
    kw = dict(temperature=temperature, top_k=top_k, top_p=top_p, do_sample=do_sample, suppress_mask=smask)
    out = _prefill(talker, tie, tam, tth, tpe)
    past_hidden, gen_step = out.past_hidden, out.generation_step
    token = sample_logits(out.logits[:, -1, :], suppress_tokens=[eos_id] if min_new_tokens > 0 else None, **kw)
    prefill_len = talker_graph.prefill_kv(out.past_key_values)
    talker_graph.set_generation_state(tam, getattr(talker, "rope_deltas", None))
    yield "prefill_done", None
    history = []
    for step in range(max_new_tokens):
        if token.item() == eos_id:
            return
        cb0_embed = embed_cb0(token.unsqueeze(1))
        rest = predictor_graph.run(torch.cat((past_hidden, cb0_embed), dim=1))
        history.append(token.detach())
        yield "frame", torch.cat([token.view(1), rest]).detach()
        rows = [cb0_embed] + [embeds_rest[i](rest[i].view(1, 1)) for i in range(n_groups - 1)]
        nxt = torch.cat(rows, dim=1).sum(1, keepdim=True)
        nxt = nxt + (tth[:, gen_step].unsqueeze(1) if gen_step < tth.shape[1] else tpe)
        pos = prefill_len + step
        if pos >= talker_graph.max_seq_len - 1:
            return
        hidden = talker_graph.run(nxt, position=pos)
        logits = head(hidden[:, -1, :]).unsqueeze(0)
        if repetition_penalty != 1.0:
            logits = apply_repetition_penalty(logits, torch.stack(history), repetition_penalty)
        token = sample_logits(logits.squeeze(0), suppress_tokens=[eos_id] if len(history) < min_new_tokens else None, **kw)
        past_hidden = hidden[:, -1:, :].clone()
        gen_step += 1
        yield "step_done", None


def _sync(device):
    if torch.cuda.is_available() and torch.device(device).type == "cuda":
        torch.cuda.synchronize()


@torch.inference_mode()
def fast_generate(
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
    subtalker_dosample: Optional[bool] = None,
    subtalker_top_k: Optional[int] = None,
    subtalker_top_p: Optional[float] = None,
    subtalker_temperature: Optional[float] = None,
    parity_mode: bool = False,
    uniforms: Optional[torch.Tensor] = None,
    return_logprobs: bool = False,
) -> Tuple[Optional[torch.Tensor], dict]:
    """Returns (codes LongTensor[steps,16] or None, timing dict with the reference's keys).  ``return_logprobs`` (fused
    engine path only): the timing dict also holds "logprobs" (float32 [steps,16], the log-probability of every code;
    see logprobs.py) and "eos_logprob" (the EOS draw that ended the request, or None)."""
    device = talker_input_embeds.device
    skw = dict(max_new_tokens=max_new_tokens, min_new_tokens=min_new_tokens, temperature=temperature, top_k=top_k,
               top_p=top_p, do_sample=do_sample, repetition_penalty=repetition_penalty)
    if parity_mode:
        if return_logprobs:
            raise ValueError("return_logprobs needs the fused decode path, not parity_mode")
        return _upstream_generate(talker, talker_input_embeds, attention_mask, trailing_text_hiddens, tts_pad_embed,
                                  config, subtalker_dosample, subtalker_top_k, subtalker_top_p,
                                  subtalker_temperature, **skw)
    engine = shared_engine(predictor_graph, talker_graph)
    if return_logprobs and engine is None:
        raise ValueError("return_logprobs needs graph handles backed by one loaded fq3 engine (the fused decode path)")
    t0 = time.time()
    if engine is not None:
        from .batching import _chunks, _single
        sched, rq, t_prefill = _single(engine, talker, config, predictor_graph, talker_graph,
                                       dict(tie=talker_input_embeds, tam=attention_mask, tth=trailing_text_hiddens,
                                            tpe=tts_pad_embed, uniforms=uniforms, **skw), return_logprobs)
        t1 = time.time()
        parts = [codes for items in _chunks(sched, _MAX_LAUNCH_FRAMES, t_prefill) for _, codes, _ in items]
        t_decode = time.time() - t1
        all_codes = torch.cat(parts) if parts else None
    else:
        frames, t_prefill, t1 = [], 0.0, t0
        for kind, row in stepwise_frames(talker, talker_input_embeds, attention_mask, trailing_text_hiddens,
                                         tts_pad_embed, config, predictor_graph, talker_graph, **skw):
            if kind == "prefill_done":
                _sync(device)
                t_prefill = time.time() - t0
                t1 = time.time()
            elif kind == "frame":
                frames.append(row)
        _sync(device)
        t_decode = time.time() - t1
        all_codes = torch.stack(frames) if frames else None
    n = 0 if all_codes is None else int(all_codes.shape[0])
    timing = {
        "prefill_ms": t_prefill * 1000,
        "decode_s": t_decode,
        "steps": n,
        "ms_per_step": (t_decode / n * 1000) if n > 0 else 0,
        "steps_per_s": (n / t_decode) if t_decode > 0 else 0,
    }
    if return_logprobs:
        timing["logprobs"] = rq.lp.frames()
        timing["eos_logprob"] = rq.eos_logprob
    return all_codes, timing


def _upstream_generate(talker, tie, tam, tth, tpe, config, sub_do, sub_k, sub_p, sub_t, *, max_new_tokens,
                       min_new_tokens, temperature, top_k, top_p, do_sample, repetition_penalty):
    """parity_mode: defer to the upstream dynamic-cache ``talker.generate`` (generate.py:52-97)."""
    if not hasattr(talker, "generate"):
        raise NotImplementedError("parity_mode needs the upstream qwen-tts talker (talker.generate)")
    eos_id, V = config.codec_eos_token_id, config.vocab_size
    t0 = time.time()
    res = talker.generate(
        inputs_embeds=tie, attention_mask=tam, trailing_text_hidden=tth, tts_pad_embed=tpe,
        max_new_tokens=max_new_tokens, min_new_tokens=min_new_tokens, do_sample=do_sample, top_k=top_k, top_p=top_p,
        temperature=temperature, repetition_penalty=repetition_penalty, eos_token_id=eos_id,
        suppress_tokens=[i for i in range(max(0, V - 1024), V) if i != eos_id],
        subtalker_dosample=do_sample if sub_do is None else sub_do,
        subtalker_top_k=top_k if sub_k is None else sub_k,
        subtalker_top_p=top_p if sub_p is None else sub_p,
        subtalker_temperature=temperature if sub_t is None else sub_t,
        output_hidden_states=True, return_dict_in_generate=True)
    codes = torch.stack([h[-1] for h in res.hidden_states if h[-1] is not None], dim=1)[0]
    stop = (codes[:, 0] == eos_id).nonzero()
    if stop.numel():
        codes = codes[: int(stop[0])]
    _sync(tie.device)
    dt = time.time() - t0
    n = int(codes.shape[0])
    return (codes if n else None), {"prefill_ms": 0.0, "decode_s": dt, "steps": n,
                                    "ms_per_step": (dt / n * 1000) if n else 0.0,
                                    "steps_per_s": (n / dt) if dt > 0 else 0.0}
