"""Weight ingestion: read tensors out of the loaded upstream ``nn.Module`` tree (the attribute paths the
reference itself touches: predictor_graph.py:53-57, talker_graph.py:41, generate.py:99-102) and hand them to the
engine, which repacks every GEMV matrix into its per-CTA streaming tape."""
from __future__ import annotations

from typing import Dict, Tuple

import torch


def _cfg_get(cfg, name, default=None):
    if isinstance(cfg, dict):
        return cfg.get(name, default)
    return getattr(cfg, name, default)


def rope_theta_of(cfg) -> float:
    th = _cfg_get(cfg, "rope_theta")
    if th is None:
        rp = _cfg_get(cfg, "rope_parameters") or _cfg_get(cfg, "rope_scaling") or {}
        th = rp.get("rope_theta") if isinstance(rp, dict) else None
    return float(th if th is not None else 1_000_000.0)


def stack_config(cfg, vocab_size=None) -> dict:
    """HF config object -> plain dict (talker_graph.py:36-37,63-65 read the same attributes)."""
    nh = int(_cfg_get(cfg, "num_attention_heads"))
    hd = _cfg_get(cfg, "head_dim") or int(_cfg_get(cfg, "hidden_size")) // nh
    if int(hd) != 128:
        raise ValueError(f"engine supports head_dim=128 only (config has {hd})")
    return dict(
        hidden_size=int(_cfg_get(cfg, "hidden_size")),
        intermediate_size=int(_cfg_get(cfg, "intermediate_size")),
        num_hidden_layers=int(_cfg_get(cfg, "num_hidden_layers")),
        num_attention_heads=nh,
        num_key_value_heads=int(_cfg_get(cfg, "num_key_value_heads", nh)),
        vocab_size=int(vocab_size if vocab_size is not None else _cfg_get(cfg, "vocab_size")),
        rms_norm_eps=float(_cfg_get(cfg, "rms_norm_eps", 1e-6)),
        rope_theta=rope_theta_of(cfg),
    )


def rope_tables(theta: float, n_pos: int, head_dim: int = 128) -> Tuple[torch.Tensor, torch.Tensor]:
    """float32 cos/sin [n_pos, head_dim], computed the way the HF rotary module does (default rope type;
    the three mRoPE axes carry identical positions on this path, talker_graph.py:210-211)."""
    inv_freq = 1.0 / (theta ** (torch.arange(0, head_dim, 2, dtype=torch.int64).to(torch.float32) / head_dim))
    freqs = torch.arange(n_pos, dtype=torch.float32)[:, None] * inv_freq[None, :]
    emb = torch.cat((freqs, freqs), dim=-1)
    return emb.cos(), emb.sin()


def _stack_tensors(prefix: str, model, dtype, device) -> Dict[str, torch.Tensor]:
    layers = list(model.layers)

    def cat(fn):
        return torch.stack([fn(l).detach().to(device=device, dtype=dtype) for l in layers]).contiguous()

    return {
        prefix + "q": cat(lambda l: l.self_attn.q_proj.weight),
        prefix + "k": cat(lambda l: l.self_attn.k_proj.weight),
        prefix + "v": cat(lambda l: l.self_attn.v_proj.weight),
        prefix + "o": cat(lambda l: l.self_attn.o_proj.weight),
        prefix + "gate": cat(lambda l: l.mlp.gate_proj.weight),
        prefix + "up": cat(lambda l: l.mlp.up_proj.weight),
        prefix + "down": cat(lambda l: l.mlp.down_proj.weight),
        prefix + "ln_in": cat(lambda l: l.input_layernorm.weight),
        prefix + "ln_post": cat(lambda l: l.post_attention_layernorm.weight),
        prefix + "qnorm": cat(lambda l: l.self_attn.q_norm.weight),
        prefix + "knorm": cat(lambda l: l.self_attn.k_norm.weight),
        prefix + "ln_f": model.norm.weight.detach().to(device=device, dtype=dtype).contiguous(),
    }


def has_mtp_projection(code_predictor) -> bool:
    proj = getattr(code_predictor, "small_to_mtp_projection", None)
    return proj is not None and hasattr(proj, "weight")


def engine_tensors(talker, talker_cfg: dict, pred_cfg: dict, dtype, device, rope_positions: int) -> Dict[str, torch.Tensor]:
    """talker: the upstream talker module (``base_model.model.talker``)."""
    cp = talker.code_predictor
    out = {}
    out.update(_stack_tensors("t.", talker.model, dtype, device))
    out.update(_stack_tensors("p.", cp.model, dtype, device))
    conv = lambda w: w.detach().to(device=device, dtype=dtype).contiguous()  # noqa: E731
    out["t.head"] = conv(talker.codec_head.weight)
    out["t.embed"] = conv(talker.get_input_embeddings().weight)
    out["p.heads"] = torch.stack([conv(h.weight) for h in cp.lm_head]).contiguous()
    out["p.embeds"] = torch.stack([conv(e.weight) for e in cp.get_input_embeddings()]).contiguous()
    if has_mtp_projection(cp):
        out["p.mtp_w"] = conv(cp.small_to_mtp_projection.weight)
        b = getattr(cp.small_to_mtp_projection, "bias", None)
        out["p.mtp_b"] = conv(b) if b is not None else torch.zeros(pred_cfg["hidden_size"], dtype=dtype, device=device)
    c, s = rope_tables(talker_cfg["rope_theta"], rope_positions)
    out["t.cos"], out["t.sin"] = c.to(device), s.to(device)
    c, s = rope_tables(pred_cfg["rope_theta"], 32)
    out["p.cos"], out["p.sin"] = c.to(device), s.to(device)
    return out


def engine_for_talker(talker, dtype=torch.bfloat16, device="cuda", max_seq_len: int = 2048, num_ctas: int = 0,
                      native_prefill: bool = True, max_batch: int = 1, max_slots=None,
                      kv_pages: int = 0):
    """Build and load an fq3 Engine from the upstream talker module (``base_model.model.talker``)."""
    from .engine import Engine

    tcfg_obj = talker.config
    pcfg_obj = talker.code_predictor.model.config
    tcfg = stack_config(tcfg_obj)
    pcfg = stack_config(pcfg_obj)
    eng = Engine(talker=tcfg, predictor=pcfg, dtype=dtype, device=device, max_seq_len=max_seq_len,
                 num_code_groups=int(_cfg_get(tcfg_obj, "num_code_groups", 16)),
                 codec_eos_token_id=int(_cfg_get(tcfg_obj, "codec_eos_token_id")),
                 has_mtp_projection=has_mtp_projection(talker.code_predictor), num_ctas=num_ctas,
                 max_batch=max_batch, max_slots=max_slots, kv_pages=kv_pages)
    tensors = engine_tensors(talker, tcfg, pcfg, dtype, eng.device, eng.rope_positions)
    eng.load_weights(tensors)
    if dtype == torch.bfloat16 and native_prefill:
        L, I, H = tcfg["num_hidden_layers"], tcfg["intermediate_size"], tcfg["hidden_size"]
        eng.set_prefill_weights({
            "t.qkv": torch.cat((tensors["t.q"], tensors["t.k"], tensors["t.v"]), dim=1).contiguous(),
            "t.o": tensors["t.o"],
            "t.gu": torch.stack((tensors["t.gate"], tensors["t.up"]), dim=2).reshape(L, 2 * I, H).contiguous(),
            "t.down": tensors["t.down"],
            "t.head": tensors["t.head"],
        })
    return eng
