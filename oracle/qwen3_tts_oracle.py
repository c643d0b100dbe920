"""CPU oracle for the Qwen3-TTS decode hot path  --  TEST INFRASTRUCTURE, NOT PRODUCT.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import this module.  The product package
(``faster-qwen3-tts_b200/faster_qwen3_tts``) never imports anything under ``oracle/``.

What it restates (plain torch on CPU, fp32 or bf16, dims taken from a config dict):

* the reference's per-frame orchestration      -- faster_qwen3_tts/generate.py:46-50,124-134,149-199
                                                   faster_qwen3_tts/streaming.py:106-188
* the predictor's 15-step loop                  -- faster_qwen3_tts/predictor_graph.py:115-167
* the talker single-token step + KV/mask state  -- faster_qwen3_tts/talker_graph.py:97-107,153-214
* sampling                                      -- faster_qwen3_tts/sampling.py:10-66

The layer arithmetic itself lives in the un-vendored ``qwen-tts>=0.1.1`` / ``transformers>=4.57,<5``
packages (pyproject.toml:27-28 of the reference), which are absent from this image.  It is restated here
from the published Qwen3 decoder block as readable in the in-image transformers 5.5 analogue
(``transformers/models/qwen3_omni_moe/modeling_qwen3_omni_moe.py``: RMSNorm :2331-2345, attention with
q/k-norm :2352-2423, eager attention :471-493, SwiGLU :2426-2439, block :2442-2481, RoPE :2484-2546,
rotate_half/apply :816-820,1448-1470).

PARITY STATUS
  * sampling + loop control flow: PINNED against the reference's own ``sampling.py`` / ``generate.py`` /
    ``streaming.py`` executed in this container (``oracle/make_golden.py`` -> ``tests/golden/*.npz``).
  * prompt assembly: the product's restatement is PINNED against the reference's own
    ``_build_talker_inputs_local`` executed here (``tests/golden/prompt.npz``, ``tests/test_prompt_cpu.py``).
  * talker / predictor layer arithmetic (``run_stack``): checked at test time against the Hugging Face eager Qwen3
    decoder of the in-image ``transformers`` (same weights; prefill + cached steps): bit-identical in fp32, bf16-ulp
    level in bf16; ``predictor_frame`` against the Hugging Face Qwen3-Omni talker code predictor stepped with the
    same weights: identical greedy codes (``tests/test_oracle_vs_transformers.py``).  That pins the block to an independent implementation
    of the architecture family; against upstream ``qwen-tts`` itself it stays "parity unpinned" -- no weights, no
    ``qwen_tts`` and no golden token/PCM vectors exist in the reference tree (SURVEY.md section 8c).
  * codec decoder (product-side torch module ``codec.py``): checked against the Hugging Face Qwen3-Omni Code2Wav
    analogue with shared weights (``tests/test_codec_vs_transformers.py``); "parity unpinned" against upstream.

Noise contract (replaces ``torch.multinomial`` whose CUDA Philox stream cannot be reproduced):
  one uniform u in [0,1) per draw; token = first index v (ascending) whose inclusive prefix sum of the
  final probabilities exceeds u * total, prefix sums formed in the fixed order documented in
  ``draw_inverse_cdf``.  The engine implements the identical order on device.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

# --------------------------------------------------------------------------------------
# configuration
# --------------------------------------------------------------------------------------


@dataclass
class StackCfg:
    """One transformer stack (talker backbone or code predictor)."""

    hidden_size: int
    intermediate_size: int
    num_hidden_layers: int
    num_attention_heads: int = 16
    num_key_value_heads: int = 8
    head_dim: int = 128
    rms_norm_eps: float = 1e-6
    rope_theta: float = 1_000_000.0
    vocab_size: int = 3072


@dataclass
class ModelCfg:
    talker: StackCfg
    predictor: StackCfg
    num_code_groups: int = 16
    codec_eos_token_id: int = 2150
    has_mtp_projection: bool = True  # small_to_mtp_projection is Linear(+bias) when hidden sizes differ


def cfg_1p7b() -> ModelCfg:
    return ModelCfg(
        talker=StackCfg(2048, 6144, 28, vocab_size=3072),
        predictor=StackCfg(1024, 3072, 5, vocab_size=2048),
        has_mtp_projection=True,
    )


def cfg_0p6b() -> ModelCfg:
    return ModelCfg(
        talker=StackCfg(1024, 3072, 28, vocab_size=3072),
        predictor=StackCfg(1024, 3072, 5, vocab_size=2048),
        has_mtp_projection=False,
    )


def cfg_tiny(layers_t: int = 3, layers_p: int = 2) -> ModelCfg:
    """Small geometry for second-scale CPU tests (same head_dim, GQA ratio 2)."""
    return ModelCfg(
        talker=StackCfg(512, 768, layers_t, num_attention_heads=4, num_key_value_heads=2, vocab_size=1280),
        predictor=StackCfg(256, 512, layers_p, num_attention_heads=4, num_key_value_heads=2, vocab_size=256),
        codec_eos_token_id=300,
        has_mtp_projection=True,
    )


# --------------------------------------------------------------------------------------
# layer arithmetic (restated from the Qwen3 decoder block; see module docstring)
# --------------------------------------------------------------------------------------


def rms_norm(x: torch.Tensor, w: torch.Tensor, eps: float) -> torch.Tensor:
    dt = x.dtype
    xf = x.to(torch.float32)
    var = xf.pow(2).mean(-1, keepdim=True)
    xf = xf * torch.rsqrt(var + eps)
    return w * xf.to(dt)


def rope_tables(head_dim: int, theta: float, max_pos: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """fp32 cos/sin tables [max_pos, head_dim] exactly as the HF rotary module computes them."""
    inv_freq = 1.0 / (theta ** (torch.arange(0, head_dim, 2, dtype=torch.int64).to(torch.float32) / head_dim))
    pos = torch.arange(max_pos, dtype=torch.float32)
    freqs = pos[:, None] * inv_freq[None, :]
    emb = torch.cat((freqs, freqs), dim=-1)
    return emb.cos(), emb.sin()


def _rotate_half(x: torch.Tensor) -> torch.Tensor:
    h = x.shape[-1] // 2
    return torch.cat((-x[..., h:], x[..., :h]), dim=-1)


class KVCache:
    """Dynamic cache: per layer K,V of shape [n_kv, T, d] (the reference's parity path uses HF DynamicCache)."""

    def __init__(self, n_layers: int):
        self.k: List[Optional[torch.Tensor]] = [None] * n_layers
        self.v: List[Optional[torch.Tensor]] = [None] * n_layers

    def append(self, li: int, k: torch.Tensor, v: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        if self.k[li] is None:
            self.k[li], self.v[li] = k, v
        else:
            self.k[li] = torch.cat((self.k[li], k), dim=1)
            self.v[li] = torch.cat((self.v[li], v), dim=1)
        return self.k[li], self.v[li]

    def length(self) -> int:
        return 0 if self.k[0] is None else int(self.k[0].shape[1])


def decoder_layer(
    W: Dict[str, torch.Tensor],
    prefix: str,
    cfg: StackCfg,
    li: int,
    x: torch.Tensor,  # [T, H]
    cos: torch.Tensor,  # [T, d] in x.dtype
    sin: torch.Tensor,
    cache: KVCache,
    n_left_pad: int = 0,
    dbg: Optional[dict] = None,
) -> torch.Tensor:
    p = f"{prefix}.layers.{li}."
    T = x.shape[0]
    nH, nKV, d = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
    res = x
    h = rms_norm(x, W[p + "input_layernorm.weight"], cfg.rms_norm_eps)
    q = F.linear(h, W[p + "self_attn.q_proj.weight"]).view(T, nH, d)
    k = F.linear(h, W[p + "self_attn.k_proj.weight"]).view(T, nKV, d)
    v = F.linear(h, W[p + "self_attn.v_proj.weight"]).view(T, nKV, d)
    if dbg is not None:
        dbg[f"L{li}.qkv"] = torch.cat((q.reshape(T, -1), k.reshape(T, -1), v.reshape(T, -1)), dim=-1).float()
    q = rms_norm(q, W[p + "self_attn.q_norm.weight"], cfg.rms_norm_eps).transpose(0, 1)  # [nH,T,d]
    k = rms_norm(k, W[p + "self_attn.k_norm.weight"], cfg.rms_norm_eps).transpose(0, 1)
    v = v.transpose(0, 1)
    c, s = cos[None], sin[None]
    q = (q * c) + (_rotate_half(q) * s)
    k = (k * c) + (_rotate_half(k) * s)
    past = int(cache.k[li].shape[1]) if cache.k[li] is not None else 0
    kk, vv = cache.append(li, k, v)  # [nKV, S, d]
    S = kk.shape[1]
    rep = nH // nKV
    kk = kk[:, None].expand(nKV, rep, S, d).reshape(nH, S, d)
    vv = vv[:, None].expand(nKV, rep, S, d).reshape(nH, S, d)
    scaling = d ** -0.5
    att = torch.matmul(q, kk.transpose(1, 2)) * scaling  # [nH, T, S]
    # causal + left-pad mask (additive, finfo.min like HF)
    qpos = past + torch.arange(T, device=x.device)
    kpos = torch.arange(S, device=x.device)
    allowed = (kpos[None, :] <= qpos[:, None]) & (kpos[None, :] >= n_left_pad)
    mask = torch.zeros(T, S, dtype=att.dtype, device=x.device)
    mask.masked_fill_(~allowed, torch.finfo(att.dtype).min)
    att = att + mask[None]
    att = F.softmax(att, dim=-1, dtype=torch.float32).to(q.dtype)
    o = torch.matmul(att, vv)  # [nH, T, d]
    o = o.transpose(0, 1).reshape(T, nH * d)
    if dbg is not None:
        dbg[f"L{li}.attn"] = o.float()
    o = F.linear(o, W[p + "self_attn.o_proj.weight"])
    x = res + o
    if dbg is not None:
        dbg[f"L{li}.x1"] = x.float()
    res = x
    h = rms_norm(x, W[p + "post_attention_layernorm.weight"], cfg.rms_norm_eps)
    g = F.linear(h, W[p + "mlp.gate_proj.weight"])
    u = F.linear(h, W[p + "mlp.up_proj.weight"])
    a = F.silu(g) * u
    if dbg is not None:
        dbg[f"L{li}.act"] = a.float()
    x = res + F.linear(a, W[p + "mlp.down_proj.weight"])
    if dbg is not None:
        dbg[f"L{li}.x"] = x.float()
    return x


def run_stack(
    W: Dict[str, torch.Tensor],
    prefix: str,
    cfg: StackCfg,
    x: torch.Tensor,  # [T,H]
    positions: torch.Tensor,  # [T] int64 (already includes rope delta)
    cache: KVCache,
    rope: Tuple[torch.Tensor, torch.Tensor],
    n_left_pad: int = 0,
    dbg: Optional[dict] = None,
) -> torch.Tensor:
    """All layers + final norm.  Returns the post-norm hidden [T,H] (what HF calls last_hidden_state)."""
    cos = rope[0][positions].to(device=x.device, dtype=x.dtype)
    sin = rope[1][positions].to(device=x.device, dtype=x.dtype)
    for li in range(cfg.num_hidden_layers):
        x = decoder_layer(W, prefix, cfg, li, x, cos, sin, cache, n_left_pad, dbg)
    return rms_norm(x, W[prefix + ".norm.weight"], cfg.rms_norm_eps)


# --------------------------------------------------------------------------------------
# sampling  (follows the reference's faster_qwen3_tts/sampling.py:10-66 line by line)
# --------------------------------------------------------------------------------------


def apply_repetition_penalty(logits: torch.Tensor, history: torch.Tensor, penalty: float) -> torch.Tensor:
    """sampling.py:10-29 -- HF-style penalty over unique(all history)."""
    if penalty == 1.0 or history.numel() == 0:
        return logits
    uniq = history.unique()
    t = logits[..., uniq]
    logits[..., uniq] = torch.where(t > 0, t / penalty, t * penalty)
    return logits


def filtered_probs(
    logits: torch.Tensor,  # [V]
    *,
    temperature: float,
    top_k: int,
    top_p: float,
    suppress_mask: Optional[torch.Tensor] = None,
    suppress_tokens: Optional[List[int]] = None,
) -> torch.Tensor:
    """sampling.py:44-66 up to (and including) the final softmax; returns probs in logits.dtype."""
    logits = logits.clone()
    if suppress_mask is not None:
        logits[..., suppress_mask] = float("-inf")
    if suppress_tokens:
        logits[..., list(suppress_tokens)] = float("-inf")
    logits = logits / temperature
    if top_k > 0:
        tv, _ = torch.topk(logits, min(top_k, logits.size(-1)))
        logits = torch.where(logits < tv[..., -1:], torch.full_like(logits, float("-inf")), logits)
    if top_p < 1.0:
        # the engine evaluates nucleus filtering in fp32 with (value desc, index asc) order; in fp32 this is
        # the reference computation; in bf16 the reference's own bf16 cumsum is tolerance-level only.
        lf = logits.float()
        order = np.lexsort((np.arange(lf.numel()), -lf.numpy()))
        sl = lf[torch.from_numpy(order)]
        pr = F.softmax(sl, dim=-1)
        cum = torch.from_numpy(np.cumsum(pr.numpy(), dtype=np.float32))
        rem = cum > top_p
        rem[0] = False
        sl[rem] = float("-inf")
        out = torch.full_like(lf, float("-inf"))
        out[torch.from_numpy(order)] = sl
        logits = out.to(logits.dtype)
    return F.softmax(logits, dim=-1)


_NCHUNK = 256  # the engine's sampling block has 256 threads; each owns a contiguous chunk of the vocabulary


def _ks_scan32(x: np.ndarray) -> np.ndarray:
    """Kogge-Stone inclusive scan over 32 lanes in fp32 (the order __shfl_up_sync produces)."""
    x = x.astype(np.float32).copy()
    d = 1
    while d < 32:
        y = x.copy()
        y[d:] = (x[d:] + x[:-d]).astype(np.float32)
        x = y
        d *= 2
    return x


def draw_inverse_cdf(probs: torch.Tensor, u: float) -> int:
    """Inverse-CDF draw with the engine's summation order.

    chunk c (0..255) owns indices [c*CH, (c+1)*CH), CH = ceil(V/256); chunk sums are sequential fp32;
    the 256 chunk sums are scanned as 8 warps x 32 lanes: Kogge-Stone within a warp, then a sequential
    exclusive scan over the 8 warp totals.  target = u * total (fp32).  Pick the first chunk whose inclusive
    prefix exceeds target, then walk that chunk sequentially from its exclusive prefix.  If rounding leaves
    no index selected, the last index with p > 0 is returned.
    """
    p = probs.detach().to(torch.float32).numpy().astype(np.float32)
    V = p.shape[0]
    CH = (V + _NCHUNK - 1) // _NCHUNK
    pad = np.zeros(_NCHUNK * CH, dtype=np.float32)
    pad[:V] = p
    pc = pad.reshape(_NCHUNK, CH)
    csum = np.zeros(_NCHUNK, dtype=np.float32)
    for j in range(CH):
        csum = (csum + pc[:, j]).astype(np.float32)
    incl = np.zeros(_NCHUNK, dtype=np.float32)
    wtot = np.zeros(8, dtype=np.float32)
    for w in range(8):
        sc = _ks_scan32(csum[w * 32:(w + 1) * 32])
        incl[w * 32:(w + 1) * 32] = sc
        wtot[w] = sc[31]
    woff = np.zeros(8, dtype=np.float32)
    acc = np.float32(0.0)
    for w in range(8):
        woff[w] = acc
        acc = np.float32(acc + wtot[w])
    total = acc
    for w in range(8):
        incl[w * 32:(w + 1) * 32] = (incl[w * 32:(w + 1) * 32] + woff[w]).astype(np.float32)
    target = np.float32(np.float32(u) * total)
    hit = np.nonzero(incl > target)[0]
    if hit.size:
        c = int(hit[0])
        # exclusive prefix of chunk c in the order the engine uses: inclusive(c-1), or the warp offset at lane 0
        lane = c % 32
        w = c // 32
        if lane == 0:
            excl = woff[w]
        else:
            excl = incl[c - 1]
        run = np.float32(excl)
        for j in range(CH):
            idx = c * CH + j
            if idx >= V:
                break
            run = np.float32(run + pad[idx])
            if run > target and pad[idx] > 0:
                return idx
    nz = np.nonzero(p > 0)[0]
    return int(nz[-1]) if nz.size else 0


def sample_token(
    logits: torch.Tensor,  # [V] in model dtype
    *,
    temperature: float,
    top_k: int,
    top_p: float,
    do_sample: bool,
    u: float,
    suppress_mask: Optional[torch.Tensor] = None,
    suppress_tokens: Optional[List[int]] = None,
) -> int:
    """sampling.py:32-66 with torch.multinomial replaced by the inverse-CDF noise contract."""
    logits = logits.detach().cpu()   # the weights (and so the logits) may live on an accelerator when tests host the oracle there
    if not do_sample:
        lg = logits.clone()
        if suppress_mask is not None:
            lg[..., suppress_mask] = float("-inf")
        if suppress_tokens:
            lg[..., list(suppress_tokens)] = float("-inf")
        return int(torch.argmax(lg, dim=-1))
    pr = filtered_probs(
        logits,
        temperature=temperature,
        top_k=top_k,
        top_p=top_p,
        suppress_mask=suppress_mask,
        suppress_tokens=suppress_tokens,
    )
    return draw_inverse_cdf(pr, u)


# --------------------------------------------------------------------------------------
# the model: prefill, talker step, predictor frame
# --------------------------------------------------------------------------------------


@dataclass
class SamplingParams:
    do_sample: bool = True
    temperature: float = 0.9
    top_k: int = 50
    top_p: float = 1.0
    repetition_penalty: float = 1.05


class OracleModel:
    """Holds weights (a flat dict with HF-style names) + rope tables; exposes the three computations."""

    def __init__(self, cfg: ModelCfg, W: Dict[str, torch.Tensor], max_pos: int = 4096):
        self.cfg = cfg
        self.W = W
        self.dtype = W["talker.codec_head.weight"].dtype
        self.rope_t = rope_tables(cfg.talker.head_dim, cfg.talker.rope_theta, max_pos)
        self.rope_p = rope_tables(cfg.predictor.head_dim, cfg.predictor.rope_theta, 64)

    # -- talker ---------------------------------------------------------------------------
    def talker_prefill(self, embeds: torch.Tensor, n_left_pad: int = 0, rope_delta: int = 0, dbg=None):
        """generate.py:107-121 -- full forward over the prompt.  Returns (logits_last[V], past_hidden[H], cache)."""
        P = embeds.shape[0]
        cache = KVCache(self.cfg.talker.num_hidden_layers)
        pos = (torch.arange(P) - n_left_pad).clamp(min=0) + rope_delta
        hid = run_stack(self.W, "talker.model", self.cfg.talker, embeds, pos, cache, self.rope_t, n_left_pad, dbg)
        logits = F.linear(hid[-1], self.W["talker.codec_head.weight"])
        return logits, hid[-1].clone(), cache

    def talker_step(self, x: torch.Tensor, position: int, cache: KVCache, n_left_pad: int = 0, rope_delta: int = 0,
                    dbg=None) -> torch.Tensor:
        """talker_graph.py:198-214 -- one token at cache slot `position`, rotary position = position + rope_delta."""
        assert cache.length() == position, (cache.length(), position)
        pos = torch.tensor([position + rope_delta])
        hid = run_stack(self.W, "talker.model", self.cfg.talker, x[None], pos, cache, self.rope_t, n_left_pad, dbg)
        return hid[0]

    # -- predictor ------------------------------------------------------------------------
    def _mtp(self, x: torch.Tensor) -> torch.Tensor:
        if not self.cfg.has_mtp_projection:
            return x
        return F.linear(x, self.W["talker.code_predictor.small_to_mtp_projection.weight"],
                        self.W.get("talker.code_predictor.small_to_mtp_projection.bias"))

    def predictor_frame(self, past_hidden: torch.Tensor, last_id_hidden: torch.Tensor, sp: SamplingParams,
                        uniforms: Optional[np.ndarray] = None, dbg=None, margins: Optional[list] = None) -> List[int]:
        """predictor_graph.py:115-167 -- 2-token prefill, then 14 single-token decodes; 15 ids."""
        pc = self.cfg.predictor
        nb = self.cfg.num_code_groups - 1
        cache = KVCache(pc.num_hidden_layers)
        h = self._mtp(torch.stack((past_hidden, last_id_hidden)))  # [2, Hp]
        hid = run_stack(self.W, "talker.code_predictor.model", pc, h, torch.arange(2), cache, self.rope_p, 0, dbg)
        out: List[int] = []
        logits = F.linear(hid[-1], self.W["talker.code_predictor.lm_head.0.weight"])
        if dbg is not None:
            dbg["pred.logits0"] = logits.float()
        if margins is not None:   # top-1 minus top-2 logit of every pass (how close a greedy decision is to a tie)
            t2 = torch.topk(logits.float(), 2).values
            margins.append(float(t2[0] - t2[1]))
        tok = sample_token(logits, temperature=sp.temperature, top_k=sp.top_k, top_p=sp.top_p,
                           do_sample=sp.do_sample, u=float(uniforms[0]) if uniforms is not None else 0.0)
        out.append(tok)
        for i in range(1, nb):
            emb = self.W[f"talker.code_predictor.model.codec_embedding.{i - 1}.weight"][tok]
            h = self._mtp(emb[None])
            hid = run_stack(self.W, "talker.code_predictor.model", pc, h, torch.tensor([1 + i]), cache, self.rope_p)
            logits = F.linear(hid[-1], self.W[f"talker.code_predictor.lm_head.{i}.weight"])
            if margins is not None:
                t2 = torch.topk(logits.float(), 2).values
                margins.append(float(t2[0] - t2[1]))
            tok = sample_token(logits, temperature=sp.temperature, top_k=sp.top_k, top_p=sp.top_p,
                               do_sample=sp.do_sample, u=float(uniforms[i]) if uniforms is not None else 0.0)
            out.append(tok)
        return out

    # -- helpers the loop needs -------------------------------------------------------------
    def codec_embed(self, tok: int) -> torch.Tensor:
        return self.W["talker.model.codec_embedding.weight"][tok]

    def next_talker_input(self, last_id_hidden: torch.Tensor, codes15: List[int], extra: torch.Tensor) -> torch.Tensor:
        """generate.py:163-171 -- cat(16 rows).sum(1) then + trailing text row / tts_pad_embed."""
        rows = [last_id_hidden]
        for i, c in enumerate(codes15):
            rows.append(self.W[f"talker.code_predictor.model.codec_embedding.{i}.weight"][c])
        s = torch.stack(rows, dim=0)[None].sum(1)[0]  # [1,16,H].sum(1) like the reference
        return s + extra


def suppress_mask_for(cfg: ModelCfg) -> torch.Tensor:
    """generate.py:46-50."""
    V = cfg.talker.vocab_size
    m = torch.zeros(V, dtype=torch.bool)
    for i in range(max(0, V - 1024), V):
        if i != cfg.codec_eos_token_id:
            m[i] = True
    return m


def generate(
    om: OracleModel,
    talker_input_embeds: torch.Tensor,  # [P, H]
    trailing_text_hiddens: torch.Tensor,  # [Tt, H]
    tts_pad_embed: torch.Tensor,  # [H]
    *,
    max_new_tokens: int = 2048,
    min_new_tokens: int = 2,
    sp_talker: SamplingParams = SamplingParams(),
    sp_pred: SamplingParams = SamplingParams(repetition_penalty=1.0),
    max_seq_len: int = 2048,
    uniforms: Optional[np.ndarray] = None,  # [max_new_tokens+1, 16]; row 0 col 0 = first-token draw
    chunk_size: Optional[int] = None,
    n_left_pad: int = 0,
    gen_step0: int = 0,
    trace: Optional[list] = None,
    rope_delta: Optional[int] = None,
):
    """generate.py:99-215 / streaming.py:57-188 restated.  Returns codes [n,16] (and chunk boundaries).

    uniforms[s+1, 0] is the draw for the cb0 token sampled at the end of frame s; uniforms[s+1, 1:16] are the
    predictor draws of frame s; uniforms[0, 0] is the draw for the first token (from the prefill logits).
    """
    cfg = om.cfg
    eos = cfg.codec_eos_token_id
    smask = suppress_mask_for(cfg)
    # decode positions are cache index + rope_delta on all three mRoPE axes (talker_graph.py:210-211); for a
    # left-padded row upstream's rope_deltas is minus the pad count, so the first generated token continues the
    # prompt's positions (arange - n_left_pad)
    if rope_delta is None:
        rope_delta = -n_left_pad
    if uniforms is None:
        uniforms = np.zeros((max_new_tokens + 1, 16), dtype=np.float32)
    logits, past_hidden, cache = om.talker_prefill(talker_input_embeds, n_left_pad)
    gen_step = gen_step0
    token = sample_token(
        logits, temperature=sp_talker.temperature, top_k=sp_talker.top_k, top_p=sp_talker.top_p,
        do_sample=sp_talker.do_sample, u=float(uniforms[0, 0]), suppress_mask=smask,
        suppress_tokens=[eos] if min_new_tokens > 0 else None)
    prefill_len = talker_input_embeds.shape[0]
    rows: List[List[int]] = []
    chunks: List[int] = []
    buf = 0
    for step_idx in range(max_new_tokens):
        if token == eos:
            break
        last_id_hidden = om.codec_embed(token)
        pm = [] if trace is not None else None
        codes15 = om.predictor_frame(past_hidden, last_id_hidden, sp_pred, uniforms[step_idx + 1, 1:16], margins=pm)
        rows.append([token] + codes15)
        buf += 1
        if gen_step < trailing_text_hiddens.shape[0]:
            extra = trailing_text_hiddens[gen_step]
        else:
            extra = tts_pad_embed
        x = om.next_talker_input(last_id_hidden, codes15, extra)
        pos = prefill_len + step_idx
        if pos >= max_seq_len - 1:
            break
        hid = om.talker_step(x, pos, cache, n_left_pad, rope_delta)
        logits = F.linear(hid, om.W["talker.codec_head.weight"]).cpu()
        if trace is not None:
            trace.append({"x": x.float().cpu(), "hidden": hid.float().cpu(), "logits": logits.float().clone(),
                          "x_raw": x.detach().clone(), "position": pos, "pred_margins": pm})
        if sp_talker.repetition_penalty != 1.0:
            hist = torch.tensor([r[0] for r in rows], dtype=torch.long)
            logits = apply_repetition_penalty(logits.clone(), hist, sp_talker.repetition_penalty)
        token = sample_token(
            logits, temperature=sp_talker.temperature, top_k=sp_talker.top_k, top_p=sp_talker.top_p,
            do_sample=sp_talker.do_sample, u=float(uniforms[step_idx + 1, 0]), suppress_mask=smask,
            suppress_tokens=[eos] if len(rows) < min_new_tokens else None)
        past_hidden = hid.clone()
        gen_step += 1
        if chunk_size is not None and buf >= chunk_size:
            chunks.append(buf)
            buf = 0
    if chunk_size is not None and buf:
        chunks.append(buf)
    codes = torch.tensor(rows, dtype=torch.long).reshape(-1, 16)
    return (codes, chunks) if chunk_size is not None else codes


# --------------------------------------------------------------------------------------
# synthetic weights (seeded).  Shapes/names follow the attribute paths the reference touches:
#   predictor_graph.py:53-57, generate.py:99-102, talker_graph.py:41.
# --------------------------------------------------------------------------------------


def make_weights(cfg: ModelCfg, seed: int = 0, dtype: torch.dtype = torch.float32, std: float = 0.02,
                 norm_jitter: float = 0.1, eos_boost: float = 1.0) -> Dict[str, torch.Tensor]:
    g = torch.Generator().manual_seed(seed)
    W: Dict[str, torch.Tensor] = {}

    def lin(name, out_f, in_f, s=std):
        W[name] = (torch.randn(out_f, in_f, generator=g) * s).to(dtype)

    def norm(name, n):
        W[name] = (1.0 + norm_jitter * torch.randn(n, generator=g)).to(dtype)

    def stack(prefix, c: StackCfg):
        qd, kd = c.num_attention_heads * c.head_dim, c.num_key_value_heads * c.head_dim
        for li in range(c.num_hidden_layers):
            p = f"{prefix}.layers.{li}."
            norm(p + "input_layernorm.weight", c.hidden_size)
            lin(p + "self_attn.q_proj.weight", qd, c.hidden_size)
            lin(p + "self_attn.k_proj.weight", kd, c.hidden_size)
            lin(p + "self_attn.v_proj.weight", kd, c.hidden_size)
            lin(p + "self_attn.o_proj.weight", c.hidden_size, qd)
            norm(p + "self_attn.q_norm.weight", c.head_dim)
            norm(p + "self_attn.k_norm.weight", c.head_dim)
            norm(p + "post_attention_layernorm.weight", c.hidden_size)
            lin(p + "mlp.gate_proj.weight", c.intermediate_size, c.hidden_size)
            lin(p + "mlp.up_proj.weight", c.intermediate_size, c.hidden_size)
            lin(p + "mlp.down_proj.weight", c.hidden_size, c.intermediate_size)
        norm(prefix + ".norm.weight", c.hidden_size)

    Ht, Hp = cfg.talker.hidden_size, cfg.predictor.hidden_size
    stack("talker.model", cfg.talker)
    lin("talker.model.codec_embedding.weight", cfg.talker.vocab_size, Ht, 1.0)
    lin("talker.codec_head.weight", cfg.talker.vocab_size, Ht, std * 4)
    if eos_boost != 1.0:
        W["talker.codec_head.weight"][cfg.codec_eos_token_id] *= eos_boost
    stack("talker.code_predictor.model", cfg.predictor)
    for i in range(cfg.num_code_groups - 1):
        lin(f"talker.code_predictor.model.codec_embedding.{i}.weight", cfg.predictor.vocab_size, Ht, 1.0)
        lin(f"talker.code_predictor.lm_head.{i}.weight", cfg.predictor.vocab_size, Hp, std * 4)
    if cfg.has_mtp_projection:
        lin("talker.code_predictor.small_to_mtp_projection.weight", Hp, Ht)
        W["talker.code_predictor.small_to_mtp_projection.bias"] = (torch.randn(Hp, generator=g) * std).to(dtype)
    return W


def make_inputs(cfg: ModelCfg, P: int, Tt: int, seed: int = 0, dtype: torch.dtype = torch.float32):
    g = torch.Generator().manual_seed(10_000 + seed)
    H = cfg.talker.hidden_size
    tie = torch.randn(P, H, generator=g).to(dtype)
    tth = torch.randn(Tt, H, generator=g).to(dtype)
    tpe = torch.randn(H, generator=g).to(dtype)
    return tie, tth, tpe
