"""float64 reference of the decode kernels' per-draw log-probabilities (include/fq3_engine.h, fq3_decode_chunk_lp).

``processed_row`` restates, in the model dtype, the row the sampler draws from (the steps of
``qwen3_tts_oracle.filtered_probs`` before its softmax; greedy: the penalised, suppressed logits without temperature),
``logprob64`` is the float64 log-softmax of such a row at one id, and ``teacher_forced_logprobs`` walks the oracle
model along given codes and returns the value of every draw in the kernels' layout."""
from __future__ import annotations

from typing import List, Optional

import numpy as np
import torch
import torch.nn.functional as F

from . import qwen3_tts_oracle as O


def processed_row(logits: torch.Tensor, *, do_sample: bool, temperature: float, top_k: int, top_p: float,
                  suppress_mask: Optional[torch.Tensor] = None, suppress_tokens: Optional[List[int]] = None) -> torch.Tensor:
    """[V] model dtype -> the [V] row (model dtype, -inf where filtered) whose log-softmax the kernels report"""
    lg = logits.detach().cpu().clone()
    if suppress_mask is not None:
        lg[..., suppress_mask] = float("-inf")
    if suppress_tokens:
        lg[..., list(suppress_tokens)] = float("-inf")
    if not do_sample:
        return lg
    lg = lg / temperature
    if top_k > 0:
        tv, _ = torch.topk(lg, min(top_k, lg.size(-1)))
        lg = torch.where(lg < tv[..., -1:], torch.full_like(lg, float("-inf")), lg)
    if top_p < 1.0:   # fp32 nucleus in (value desc, index asc) order, as the kernels and filtered_probs do
        lf = lg.float()
        order = np.lexsort((np.arange(lf.numel()), -lf.numpy()))
        sl = lf[torch.from_numpy(order)]
        pr = F.softmax(sl, dim=-1)
        cum = torch.from_numpy(np.cumsum(pr.numpy(), dtype=np.float32))
        rem = cum > top_p
        rem[0] = False
        sl[rem] = float("-inf")
        out = torch.full_like(lf, float("-inf"))
        out[torch.from_numpy(order)] = sl
        lg = out.to(lg.dtype)
    return lg


def logprob64(row: torch.Tensor, tok: int) -> float:
    """float64 log-softmax of ``row`` at ``tok``"""
    l = row.detach().cpu().double()
    m = l.max()
    return float((l[tok] - m) - torch.log(torch.exp(l - m).sum()))


def teacher_forced_logprobs(om: O.OracleModel, tie: torch.Tensor, tth: torch.Tensor, tpe: torch.Tensor,
                            codes: torch.Tensor, *, sp_talker: O.SamplingParams, sp_pred: O.SamplingParams,
                            min_new_tokens: int, next_token: int, n_left_pad: int = 0):
    """The oracle's generate loop forced along ``codes`` [T,16] (and ``next_token``, the cb0 drawn after the last
    frame).  Returns (first: float, rows float64 [T,16]) where rows[f, k>=1] is codebook k of frame f and rows[f, 0]
    the cb0 drawn after frame f -- the layout of fq3_decode_chunk_lp; first is the first token's value."""
    cfg = om.cfg
    eos = cfg.codec_eos_token_id
    smask = O.suppress_mask_for(cfg)
    pc = cfg.predictor
    T = int(codes.shape[0])

    def talker_lp(logits, tok, n_rows):
        return logprob64(processed_row(logits, do_sample=sp_talker.do_sample, temperature=sp_talker.temperature,
                                       top_k=sp_talker.top_k, top_p=sp_talker.top_p, suppress_mask=smask,
                                       suppress_tokens=[eos] if n_rows < min_new_tokens else None), tok)

    def pred_lp(logits, tok):
        return logprob64(processed_row(logits, do_sample=sp_pred.do_sample, temperature=sp_pred.temperature,
                                       top_k=sp_pred.top_k, top_p=sp_pred.top_p), tok)

    logits, past_hidden, cache = om.talker_prefill(tie, n_left_pad)
    cb0 = [int(c) for c in codes[:, 0]] + [int(next_token)]
    first = talker_lp(logits, cb0[0], 0)
    rows = np.zeros((T, 16), dtype=np.float64)
    rope_delta = -n_left_pad
    for f in range(T):
        token = cb0[f]
        last_id_hidden = om.codec_embed(token)
        pcache = O.KVCache(pc.num_hidden_layers)
        h = om._mtp(torch.stack((past_hidden, last_id_hidden)))
        hid = O.run_stack(om.W, "talker.code_predictor.model", pc, h, torch.arange(2), pcache, om.rope_p, 0, None)
        c15 = [int(c) for c in codes[f, 1:]]
        for i in range(cfg.num_code_groups - 1):
            if i > 0:
                emb = om.W[f"talker.code_predictor.model.codec_embedding.{i - 1}.weight"][c15[i - 1]]
                hid = O.run_stack(om.W, "talker.code_predictor.model", pc, om._mtp(emb[None]), torch.tensor([1 + i]),
                                  pcache, om.rope_p)
            lg = F.linear(hid[-1], om.W[f"talker.code_predictor.lm_head.{i}.weight"])
            rows[f, 1 + i] = pred_lp(lg, c15[i])
        extra = tth[f] if f < tth.shape[0] else tpe
        x = om.next_talker_input(last_id_hidden, c15, extra)
        pos = tie.shape[0] + f
        hid = om.talker_step(x, pos, cache, n_left_pad, rope_delta)
        lg = F.linear(hid, om.W["talker.codec_head.weight"]).cpu()
        if sp_talker.repetition_penalty != 1.0:
            lg = O.apply_repetition_penalty(lg.clone(), torch.tensor(cb0[:f + 1], dtype=torch.long),
                                            sp_talker.repetition_penalty)
        rows[f, 0] = talker_lp(lg, cb0[f + 1], f + 1)
        past_hidden = hid.clone()
    return first, rows
