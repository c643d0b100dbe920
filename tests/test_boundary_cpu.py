"""CPU-only checks of the drop-in boundary: the C-ABI library loads and exports every symbol include/*.h declares,
the host mirrors keep the reference's signatures, and the step-wise scheduler honours the reference's duck-type
contract (the reference's own tests/test_sampling.py scenario, on CPU)."""
import ctypes
import inspect
import os
import re
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    names = []
    for f in os.listdir(os.path.join(ROOT, "include")):
        src = open(os.path.join(ROOT, "include", f)).read()
        src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
        names += re.findall(r"\b(fq3_[a-z0-9_]+)\s*\(", src)
    return sorted(set(names))


def test_library_exports_every_declared_symbol():
    from faster_qwen3_tts.engine import LIB_PATH, build_extension
    build_extension()
    lib = ctypes.CDLL(LIB_PATH)
    syms = _declared_symbols()
    assert len(syms) >= 18
    for s in syms:
        assert hasattr(lib, s), s
    lib.fq3_version.restype = ctypes.c_char_p
    assert b"sm_90a" in lib.fq3_version()


def test_engine_refuses_to_run_without_cuda():
    from faster_qwen3_tts.engine import Engine
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        Engine(talker=dict(hidden_size=512, intermediate_size=768, num_hidden_layers=1, num_attention_heads=4,
                           num_key_value_heads=2, vocab_size=1280),
               predictor=dict(hidden_size=256, intermediate_size=512, num_hidden_layers=1, num_attention_heads=4,
                              num_key_value_heads=2, vocab_size=256), dtype=torch.float32)


def test_signatures_match_reference():
    from faster_qwen3_tts.generate import fast_generate
    from faster_qwen3_tts.streaming import fast_generate_streaming
    from faster_qwen3_tts.sampling import sample_logits, apply_repetition_penalty
    ref_gen = ["talker", "talker_input_embeds", "attention_mask", "trailing_text_hiddens", "tts_pad_embed", "config",
               "predictor_graph", "talker_graph", "max_new_tokens", "min_new_tokens", "temperature", "top_k", "top_p",
               "do_sample", "repetition_penalty", "subtalker_dosample", "subtalker_top_k", "subtalker_top_p",
               "subtalker_temperature", "parity_mode"]
    got = list(inspect.signature(fast_generate).parameters)
    assert got[:len(ref_gen)] == ref_gen
    ref_stream = ref_gen[:15] + ["chunk_size"]
    got = list(inspect.signature(fast_generate_streaming).parameters)
    assert got[:len(ref_stream)] == ref_stream
    d = {k: v.default for k, v in inspect.signature(fast_generate_streaming).parameters.items()}
    assert (d["max_new_tokens"], d["min_new_tokens"], d["temperature"], d["top_k"], d["top_p"], d["do_sample"],
            d["repetition_penalty"], d["chunk_size"]) == (2048, 2, 0.9, 50, 1.0, True, 1.05, 12)
    assert list(inspect.signature(sample_logits).parameters)[:7] == [
        "logits", "temperature", "top_k", "top_p", "do_sample", "suppress_mask", "suppress_tokens"]
    assert list(inspect.signature(apply_repetition_penalty).parameters) == ["logits", "token_history", "repetition_penalty"]


def test_graph_classes_keep_reference_surface():
    from faster_qwen3_tts.predictor_graph import PredictorGraph
    from faster_qwen3_tts.talker_graph import TalkerGraph
    pg = PredictorGraph(None, types.SimpleNamespace(num_code_groups=16), 1024, device="cpu")
    assert (pg.do_sample, pg.top_k, pg.top_p, pg.temperature, pg.num_codebooks, pg.max_seq) == (True, 50, 1.0, 0.9, 15, 17)
    tg = TalkerGraph(None, types.SimpleNamespace(hidden_size=1024, num_hidden_layers=28), device="cpu", max_seq_len=64)
    assert tg.max_seq_len == 64
    for name in ("capture", "run"):
        assert hasattr(pg, name)
    for name in ("capture", "run", "prefill_kv", "set_generation_state", "reset"):
        assert hasattr(tg, name)
    with pytest.raises(RuntimeError, match="no loaded fq3 engine"):
        tg.run(torch.zeros(1, 1, 1024), 3)


def test_host_sampling_matches_reference_fixtures(golden_dir):
    import numpy as np
    from faster_qwen3_tts.sampling import apply_repetition_penalty, sample_logits
    s = np.load(os.path.join(golden_dir, "sampling.npz"))
    for i in range(int(s["n_cases"])):
        pre = f"c{i}_"
        dt = torch.bfloat16 if int(s[pre + "bf16"]) else torch.float32
        lg = torch.from_numpy(s[pre + "logits"]).to(dt)
        T, k, p, u, eos, sup = s[pre + "params"]
        V = lg.numel()
        mask = torch.zeros(V, dtype=torch.bool)
        mask[(V - 1024 if V > 1024 else V - 32):] = True
        mask[int(eos)] = False
        g = sample_logits(lg[None], temperature=float(T), top_k=int(k), top_p=float(p), do_sample=False,
                          suppress_mask=mask, suppress_tokens=None if sup < 0 else [int(sup)])
        assert int(g[0]) == int(s[pre + "greedy"])
    for j, dt in enumerate((torch.float32, torch.bfloat16)):
        lg = torch.from_numpy(s[f"pen{j}_logits"]).to(dt)
        out = apply_repetition_penalty(lg.clone()[None, None], torch.from_numpy(s[f"pen{j}_hist"]), 1.05)
        assert np.array_equal(out[0, 0].float().numpy(), s[f"pen{j}_out"])


def test_stepwise_scheduler_min_new_tokens_contract():
    """The reference's tests/test_sampling.py:24-118 scenario (dummies that favour EOS), run on CPU."""
    from faster_qwen3_tts.generate import fast_generate

    class Cfg:
        codec_eos_token_id = 1
        num_code_groups = 16
        vocab_size = 5

    emb = [torch.nn.Embedding(5, 4) for _ in range(15)]

    class Talker:
        config = Cfg()
        code_predictor = types.SimpleNamespace(get_input_embeddings=lambda: emb)
        _e = torch.nn.Embedding(5, 4)
        rope_deltas = torch.zeros(1, 1)

        def get_input_embeddings(self):
            return self._e

        @staticmethod
        def codec_head(x):
            lg = torch.full((x.shape[0], 5), -10.0)
            lg[:, 1] = 10.0
            lg[:, 0] = 5.0
            return lg

        def forward(self, inputs_embeds, attention_mask=None, **kw):
            lg = torch.full((1, 1, 5), -10.0)
            lg[..., 1] = 10.0
            lg[..., 0] = 5.0
            return types.SimpleNamespace(past_key_values=[(torch.zeros(1, 1, 1, 1),) * 2],
                                         past_hidden=torch.zeros(1, 1, 4), generation_step=0, logits=lg)

    class PG:
        def run(self, x):
            return torch.zeros(15, dtype=torch.long)

    class TG:
        max_seq_len = 8

        def prefill_kv(self, kv):
            return 1

        def set_generation_state(self, m, d):
            return None

        def run(self, x, position):
            return x

    t = Talker()
    codes, timing = fast_generate(talker=t, talker_input_embeds=torch.zeros(1, 3, 4),
                                  attention_mask=torch.ones(1, 3, dtype=torch.long),
                                  trailing_text_hiddens=torch.zeros(1, 1, 4), tts_pad_embed=torch.zeros(1, 1, 4),
                                  config=t.config, predictor_graph=PG(), talker_graph=TG(), max_new_tokens=3,
                                  min_new_tokens=2, do_sample=False)
    assert codes is not None and codes.shape[0] >= 2
    assert (codes[:2, 0] == 1).sum().item() == 0
    assert set(timing) == {"prefill_ms", "decode_s", "steps", "ms_per_step", "steps_per_s"}
