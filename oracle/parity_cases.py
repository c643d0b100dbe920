"""Deterministic decode-step talker double + case list for the parity (dynamic-cache) streaming path  --  TEST
INFRASTRUCTURE.  Shared by oracle/make_golden.py (which drives the REFERENCE's own ``parity_generate_streaming``,
the reference's faster_qwen3_tts/streaming.py:192-359, with it) and tests/test_parity_stream_cpu.py (which drives the
product's restatement with the same double and compares against the recorded fixture).

The double implements the upstream ``talker.forward`` contract that path relies on: a prefill call
(inputs_embeds, generation_step=None) and one call per frame (input_ids [1,1], past_key_values, generation_step,
past_hidden, subtalker_* kwargs, cache_position) returning logits [1,1,V], hidden_states = (None, codes [1,16] | None),
past_key_values, past_hidden, generation_step.  Its arithmetic is a seeded hash of (step, token): the point is the
CONTROL FLOW around it (EOS / min_new_tokens / suppress range / penalty history / `codes is None` stop / chunking)."""
from __future__ import annotations

import types

import torch

V, EOS = 96 + 1024, 96 + 40      # suppress range = last 1024 ids except EOS (generate.py:46-50)

# name, seed, max_new, min_new, do_sample, penalty, chunk, eos_bias, none_at (frame index whose codes are None, or -1)
CASES = [
    ("greedy", 1, 11, 2, False, 1.05, 4, 0.0, -1),
    ("sampled_eos", 2, 40, 2, True, 1.05, 3, 5.0, -1),
    ("sampled_min6", 3, 40, 6, True, 1.3, 5, 9.0, -1),
    ("none_stop", 4, 20, 2, True, 1.0, 4, 0.0, 6),
    ("min0_chunk1", 5, 5, 0, True, 1.05, 1, 0.0, -1),
    ("exact_multiple", 6, 8, 2, False, 1.05, 4, 0.0, -1),
]


class StepTalker:
    supports_decode_step = True

    def __init__(self, seed: int, eos_bias: float, none_at: int):
        self.seed, self.eos_bias, self.none_at = seed, eos_bias, none_at
        self.calls = []

    def _logits(self, step: int, token: int):
        g = torch.Generator().manual_seed(self.seed * 1_000_003 + step * 7919 + token)
        lg = torch.randn(1, 1, V, generator=g)
        lg[..., EOS] += self.eos_bias
        return lg

    def forward(self, inputs_embeds=None, input_ids=None, attention_mask=None, past_key_values=None,
                generation_step=None, past_hidden=None, cache_position=None, **kw):
        if input_ids is None:   # prefill
            assert generation_step is None and past_key_values is None and past_hidden is None
            self.calls.append(("prefill", int(inputs_embeds.shape[1])))
            return types.SimpleNamespace(logits=self._logits(0, 0), past_key_values=0, past_hidden=torch.zeros(1, 1, 4),
                                         generation_step=0, hidden_states=(None, None))
        step, tok = int(past_key_values) + 1, int(input_ids.view(-1)[0])
        self.calls.append(("step", step, tok, None if attention_mask is None else int(attention_mask.shape[1]),
                           None if cache_position is None else int(cache_position[0]),
                           tuple(sorted(k for k in kw if k.startswith("subtalker_")))))
        g = torch.Generator().manual_seed(self.seed * 31 + step * 17 + tok)
        codes = torch.randint(0, 64, (1, 16), generator=g)
        codes[0, 0] = tok
        if step - 1 == self.none_at:
            codes = None
        return types.SimpleNamespace(logits=self._logits(step, tok), past_key_values=step,
                                     past_hidden=torch.full((1, 1, 4), float(step)), generation_step=generation_step + 1,
                                     hidden_states=(None, codes))


def run_case(fn, case, P: int = 7):
    """Drive `fn` (the reference's or the product's parity_generate_streaming) with one case; -> (chunks, timings, calls)"""
    name, seed, max_new, min_new, do_sample, pen, chunk, eos_bias, none_at = case
    talker = StepTalker(seed, eos_bias, none_at)
    conf = types.SimpleNamespace(codec_eos_token_id=EOS, vocab_size=V, num_code_groups=16)
    torch.manual_seed(1000 + seed)
    chunks, timings = [], []
    for c, t in fn(talker=talker, talker_input_embeds=torch.zeros(1, P, 4), attention_mask=torch.ones(1, P, dtype=torch.long),
                   trailing_text_hiddens=torch.zeros(1, 2, 4), tts_pad_embed=torch.zeros(1, 1, 4), config=conf,
                   max_new_tokens=max_new, min_new_tokens=min_new, temperature=0.9, top_k=50, top_p=1.0,
                   do_sample=do_sample, repetition_penalty=pen, chunk_size=chunk):
        chunks.append(c.clone())
        timings.append(dict(t))
    return chunks, timings, talker.calls
