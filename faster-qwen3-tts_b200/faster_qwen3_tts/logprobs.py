"""Host assembly of per-frame log-probabilities (``return_logprobs=True`` of the generation entry points).

The decode kernels write one float32 row [16] per emitted frame (``Engine.decode_chunk(..., logprobs=True)``): column
k >= 1 is codebook k of that frame, column 0 the cb0 token sampled at the END of the frame, i.e. the next frame's cb0
or the EOS that ends the request.  Callers want column 0 to describe the frame's own cb0, so the rows are shifted here:
frame 0 takes the first-token value (``Engine.sample_logits(..., return_logprob=True)``), frame f > 0 takes column 0
of row f - 1, and the value left over after the last frame is the EOS term when the request ended on EOS.

A log-probability is a statistic of the sampler, not a quality measure of the audio."""
from __future__ import annotations

from typing import Optional

import torch


class FrameLogprobs:
    """Carries column 0 across chunks: ``push`` the kernel's rows of each chunk in order, get the shifted rows back."""

    def __init__(self, first_logprob: float):
        self.carry = float(first_logprob)
        self.rows = []

    def push(self, raw: torch.Tensor) -> torch.Tensor:
        """raw [n,16] as the kernel wrote it -> [n,16] float32 CPU, column 0 = the log-probability of the frame's cb0"""
        raw = raw.detach().to("cpu", torch.float32).reshape(-1, 16)
        out = raw.clone()
        if raw.shape[0]:
            out[0, 0] = self.carry
            out[1:, 0] = raw[:-1, 0]
            self.carry = float(raw[-1, 0])
        self.rows.append(out)
        return out

    def eos_logprob(self, next_token: int, eos_id: int) -> Optional[float]:
        """log-probability of the EOS draw that ends the request -- the cb0 drawn after the last frame pushed is EOS
        (``ChunkResult.next_token``) --, None otherwise"""
        return self.carry if int(next_token) == int(eos_id) else None

    def frames(self) -> torch.Tensor:
        """all rows pushed so far, [T,16]"""
        return torch.cat(self.rows) if self.rows else torch.zeros(0, 16)


def score(per_frame: torch.Tensor, eos_logprob: Optional[float]) -> dict:
    """{"logprobs": [T,16], "eos_logprob", "total_logprob" (EOS term included), "frames"} of one request"""
    total = float(per_frame.double().sum()) + (eos_logprob if eos_logprob is not None else 0.0)
    return {"logprobs": per_frame, "eos_logprob": eos_logprob, "total_logprob": total, "frames": int(per_frame.shape[0])}
