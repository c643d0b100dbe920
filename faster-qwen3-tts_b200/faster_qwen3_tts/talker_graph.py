"""TalkerGraph -- same public surface as the reference class (faster_qwen3_tts/talker_graph.py:21-214) but backed
by the persistent sm_90a decode kernel instead of StaticCache + torch.cuda.CUDAGraph.

There is nothing to capture: ``capture()`` only validates that the engine is ready, no mask table is built (the
causal / left-pad mask is implicit in ``position`` and ``n_left_pad`` inside the kernel) and no StaticCache exists
(the engine owns a ``[L, n_kv, max_seq_len, 128]`` KV cache)."""
from __future__ import annotations

from typing import Optional

import torch

from .engine import Engine


class TalkerGraph:
    def __init__(self, talker_model=None, talker_config=None, device="cuda", dtype=torch.bfloat16, max_seq_len=512,
                 engine: Optional[Engine] = None):
        self.device = device
        self.dtype = dtype
        self.max_seq_len = max_seq_len
        self.model = talker_model
        self.hidden_size = getattr(talker_config, "hidden_size", None) if talker_config is not None else None
        self.num_layers = getattr(talker_config, "num_hidden_layers", None) if talker_config is not None else None
        self.engine = engine
        if engine is not None:
            self.max_seq_len = engine.max_seq_len
            self.hidden_size = engine.talker_cfg["hidden_size"]
            self.num_layers = engine.talker_cfg["num_hidden_layers"]
        self.captured = False
        self.use_native_prefill = True   # K3 (bf16 engines); False -> talker.forward + prefill_kv like the reference
        self.prefill_len = 0
        self.n_left_pad = 0
        self.rope_delta = 0
        self.slot = 0   # request slot of the engine this handle drives (batch row; the reference is batch-1 here)
        self._out = None

    def _need_engine(self) -> Engine:
        if self.engine is None or not self.engine.loaded:
            raise RuntimeError("TalkerGraph has no loaded fq3 engine: construct it through "
                               "FasterQwen3TTS.from_pretrained(...) or pass engine=Engine(...)")
        return self.engine

    @torch.inference_mode()
    def capture(self, prefill_len=100, num_warmup=3):
        """Kept for API compatibility (model.py:250).  Nothing is captured; a warm-up step is run so that the first
        request does not pay lazy module loading."""
        eng = self._need_engine()
        x = torch.zeros(self.hidden_size, dtype=eng.dtype, device=eng.device)
        pos = min(max(int(prefill_len), 0), self.max_seq_len - 1)
        # a slot of a paged engine (kv_pages > 0) has no cache rows until a request maps them: its first request loads
        # the modules instead
        for _ in range(max(1, min(int(num_warmup), 1)) if not getattr(eng, "paged", False) else 0):
            eng.talker_step(x, pos)
        torch.cuda.synchronize()
        self.captured = True

    def reset(self, prefill_len: int = 0):
        self.prefill_len = 0

    def prefill_kv(self, past_key_values) -> int:
        """Import the prompt KV (indexable [layer] -> (k, v) each [1, n_kv, P, 128]); talker_graph.py:153-170."""
        eng = self._need_engine()
        seq_len = 0
        for li in range(self.num_layers):
            k, v = past_key_values[li]
            seq_len = k.shape[2]
            if seq_len > self.max_seq_len:
                raise RuntimeError(
                    f"Input is too long: prefill has {seq_len} tokens but max_seq_len={self.max_seq_len}. "
                    "Use shorter text or shorter reference audio.")
            eng.import_kv(li, k, v, slot=self.slot)
        self.prefill_len = seq_len
        return seq_len

    def set_generation_state(self, attention_mask: Optional[torch.Tensor], rope_deltas: Optional[torch.Tensor]):
        """Left-pad count + rope delta (talker_graph.py:172-196).  Batch is 1 on this path."""
        pad = 0
        if attention_mask is not None:
            pad = int((attention_mask[0] == 0).sum().item())
        delta = 0
        if rope_deltas is not None:
            delta = int(round(float(rope_deltas.reshape(-1)[0].item())))
        self.n_left_pad, self.rope_delta = pad, delta
        self._need_engine().set_generation_state(pad, delta, slot=self.slot)

    @torch.inference_mode()
    def run(self, input_embeds: torch.Tensor, position: int) -> torch.Tensor:
        """One decode step: [1,1,H] -> [1,1,H] post-norm hidden (aliases an internal buffer like the reference)."""
        eng = self._need_engine()
        if self._out is None:
            self._out = torch.empty(self.hidden_size, dtype=eng.dtype, device=eng.device)
        eng.talker_step(input_embeds, int(position), out=self._out, slot=self.slot)
        return self._out.view(1, 1, -1)
