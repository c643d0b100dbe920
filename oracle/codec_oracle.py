"""fp32 oracle of the codec decoder (RVQ codes -> 24 kHz PCM)  --  TEST INFRASTRUCTURE, NOT PRODUCT.

Only ``tests/`` may import this module.  It is the checker for the PCM bar of BASELINE.json's north_star ("output audio
matches the reference on fixed seeds within 1e-3 max-abs PCM"): a purely functional restatement in torch fp32 (no
nn.Module, no product import) that consumes a plain ``{name: tensor}`` weight dict.

What it restates: the decoder behind ``speech_tokenizer.decode`` that the reference calls at
the reference's faster_qwen3_tts/model.py:924,1093,1122.  The real Qwen3-TTS 12 Hz tokenizer decoder ships inside the
un-vendored ``qwen-tts`` package (pyproject.toml:27); the closest readable source in this image is the Qwen3-Omni
``Code2Wav`` of transformers 5.5 (``transformers/models/qwen3_omni_moe/modeling_qwen3_omni_moe.py``):
  code-offset embedding + mean over the 16 quantisers                                   :3766-3772
  sliding-window pre-transformer with RMSNorm, RoPE, layer scale, SwiGLU                :3370-3640
  2 x (ConvTranspose1d k=2,s=2 + ConvNeXt block)                                        :3333-3366, :3750-3760
  causal conv / causal transposed conv (right trim -> exactly `stride` samples per step) :3283-3330
  SnakeBeta                                                                             :3645-3683
  decoder block: SnakeBeta -> ConvTranspose(k=2r, s=r) -> 3 residual units (dil 1,3,9)  :3686-3727
  final SnakeBeta -> conv7 -> clamp(-1, 1)                                               :3774-3790

PARITY STATUS: pinned against that Hugging Face module with shared weights (``tests/test_codec_vs_transformers.py``,
<= 5e-6 PCM; the analogue's two-sided transposed-conv trim patched to the causal right trim that yields exactly 1920
samples per frame, which the reference relies on at model.py:935-937); against upstream ``qwen-tts`` itself: parity
unpinned (no weights, no package).

Weight names are those of the product's torch container (``Code2Wav.state_dict()``), which mirror the analogue's
layout one to one; the dict can also be filled from the Hugging Face module (see the test's name map).
"""
from __future__ import annotations

from typing import Dict, Sequence

import torch
import torch.nn.functional as F


def _rms(x, w, eps):
    return w * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps))


def _snake(x, alpha, beta):   # x [B,C,T]
    a = torch.exp(alpha)[None, :, None]
    b = torch.exp(beta)[None, :, None]
    return x + (1.0 / (b + 1e-9)) * torch.sin(x * a).pow(2)


def _cconv(x, w, b, dilation=1, groups=1):
    k = w.shape[-1]
    return F.conv1d(F.pad(x, ((k - 1) * dilation, 0)), w, b, dilation=dilation, groups=groups)


def _cconvT(x, w, b, stride):
    y = F.conv_transpose1d(x, w, b, stride=stride)
    trim = w.shape[-1] - stride
    return y[..., : y.shape[-1] - trim] if trim else y


def decode(W: Dict[str, torch.Tensor], codes: torch.Tensor, *, codebook_size: int, num_attention_heads: int,
           sliding_window: int = 72, rms_norm_eps: float = 1e-5, rope_theta: float = 10000.0,
           upsampling_ratios: Sequence[int] = (2, 2), upsample_rates: Sequence[int] = (8, 5, 4, 3)) -> torch.Tensor:
    """codes LongTensor [T, Q] -> PCM float32 [prod(rates) * T], every operation in fp32."""
    W = {k: v.detach().to(torch.float32) for k, v in W.items()}
    dev = W["code_embedding.weight"].device
    codes = codes.to(dev)
    T, Q = codes.shape
    off = torch.arange(Q, device=dev) * codebook_size
    x = W["code_embedding.weight"][codes + off[None, :]].mean(1)[None]          # [1,T,H]
    H = x.shape[-1]
    nh = num_attention_heads
    hd = H // nh
    inv = 1.0 / (rope_theta ** (torch.arange(0, hd, 2, dtype=torch.float32, device=dev) / hd))
    fr = torch.arange(T, dtype=torch.float32, device=dev)[:, None] * inv[None]
    emb = torch.cat((fr, fr), dim=-1)
    cos, sin = emb.cos()[None, None], emb.sin()[None, None]
    i = torch.arange(T, device=dev)
    allowed = (i[None, :] <= i[:, None]) & (i[None, :] > i[:, None] - sliding_window)
    bias = torch.zeros(T, T, device=dev).masked_fill_(~allowed, float("-inf"))

    def rot(t):
        return torch.cat((-t[..., hd // 2:], t[..., : hd // 2]), dim=-1)

    li = 0
    while f"layers.{li}.q.weight" in W:
        p = f"layers.{li}."
        h = _rms(x, W[p + "ln1.weight"], rms_norm_eps)
        q = F.linear(h, W[p + "q.weight"]).view(1, T, nh, hd).transpose(1, 2)
        k = F.linear(h, W[p + "k.weight"]).view(1, T, nh, hd).transpose(1, 2)
        v = F.linear(h, W[p + "v.weight"]).view(1, T, nh, hd).transpose(1, 2)
        q = q * cos + rot(q) * sin
        k = k * cos + rot(k) * sin
        att = torch.softmax(torch.matmul(q, k.transpose(2, 3)) * (hd ** -0.5) + bias, dim=-1)
        o = torch.matmul(att, v).transpose(1, 2).reshape(1, T, H)
        x = x + W[p + "s1"] * F.linear(o, W[p + "o.weight"])
        h = _rms(x, W[p + "ln2.weight"], rms_norm_eps)
        x = x + W[p + "s2"] * F.linear(F.silu(F.linear(h, W[p + "gate.weight"])) * F.linear(h, W[p + "up.weight"]),
                                       W[p + "down.weight"])
        li += 1
    x = _rms(x, W["norm.weight"], rms_norm_eps).transpose(1, 2)                  # [1,H,T]
    for ui, r in enumerate(upsampling_ratios):
        p = f"upsample.{ui}."
        x = _cconvT(x, W[p + "0.conv.weight"], W[p + "0.conv.bias"], r)
        h = _cconv(x, W[p + "1.dwconv.conv.weight"], W[p + "1.dwconv.conv.bias"], groups=x.shape[1]).transpose(1, 2)
        h = F.layer_norm(h, (h.shape[-1],), W[p + "1.norm.weight"], W[p + "1.norm.bias"], 1e-6)
        h = F.linear(F.gelu(F.linear(h, W[p + "1.pwconv1.weight"], W[p + "1.pwconv1.bias"])), W[p + "1.pwconv2.weight"],
                     W[p + "1.pwconv2.bias"])
        x = x + (W[p + "1.gamma"] * h).transpose(1, 2)
    x = _cconv(x, W["conv_in.conv.weight"], W["conv_in.conv.bias"])
    for bi, r in enumerate(upsample_rates):
        p = f"blocks.{bi}."
        x = _cconvT(_snake(x, W[p + "act.alpha"], W[p + "act.beta"]), W[p + "up.conv.weight"], W[p + "up.conv.bias"], r)
        for ri, dil in enumerate((1, 3, 9)):
            q = p + f"res.{ri}."
            h = _cconv(_snake(x, W[q + "act1.alpha"], W[q + "act1.beta"]), W[q + "conv1.conv.weight"],
                       W[q + "conv1.conv.bias"], dilation=dil)
            x = x + _cconv(_snake(h, W[q + "act2.alpha"], W[q + "act2.beta"]), W[q + "conv2.conv.weight"],
                           W[q + "conv2.conv.bias"])
    x = _cconv(_snake(x, W["act_out.alpha"], W["act_out.beta"]), W["conv_out.conv.weight"], W["conv_out.conv.bias"])
    return x.clamp(-1, 1).reshape(-1)
