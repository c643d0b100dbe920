#!/usr/bin/env python3
"""Generate tests/golden/*.npz by EXECUTING THE REFERENCE'S OWN CODE in this container.

TEST INFRASTRUCTURE.  Needs a checkout of the reference (FQ3_REFERENCE_DIR, read-only); never runs on a GPU -- the fixtures it writes
are committed and are what the tests read.

What is executed from the reference (loaded by file path, unmodified):
  * faster_qwen3_tts/sampling.py   apply_repetition_penalty, sample_logits
  * faster_qwen3_tts/generate.py   fast_generate           (non-streaming scheduler)
  * faster_qwen3_tts/streaming.py  fast_generate_streaming (chunk scheduler)

The two graph objects and the talker those schedulers drive are duck-typed doubles (the contract of
the reference's tests/test_sampling.py:26-93) whose arithmetic is the CPU oracle, so the recorded codes pin the
oracle's restatement of the *control flow* (EOS, min_new_tokens, suppress range, penalty history, trailing-text
indexing, max_seq_len stop, chunking).  torch.multinomial inside the reference's sampling module is replaced
by the inverse-CDF noise contract (its Philox stream is not reproducible); the probabilities it was handed are
recorded, which pins suppress/temperature/top-k/top-p/softmax bit for bit.

  * faster_qwen3_tts/model.py      FasterQwen3TTS._build_talker_inputs_local (prompt assembly, model.py:583-805),
                                   driven on the synthetic module tree (oracle/prompt_cases.py); `soundfile`, which
                                   model.py imports at module level and the image lacks, is stubbed (it is not used
                                   by that function)

  * faster_qwen3_tts/model.py      the body of generate_voice_clone_streaming (hybrid Phase-1 / Phase-2 codec window
                                   policy, model.py:1052-1135) with request preparation, token stream and codec
                                   decoder replaced by deterministic doubles (oracle/window_cases.py)

Usage:  python oracle/make_golden.py            (writes tests/golden/{sampling,loop,prompt,window,parity_stream}.npz)
"""
from __future__ import annotations

import importlib.util
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import qwen3_tts_oracle as O  # noqa: E402

REF = os.path.join(os.environ.get("FQ3_REFERENCE_DIR", "reference"), "faster_qwen3_tts")


def load_reference():
    pkg = types.ModuleType("fq3ref")
    pkg.__path__ = [REF]
    sys.modules["fq3ref"] = pkg
    mods = {}
    for name in ("sampling", "predictor_graph", "talker_graph", "generate", "streaming"):
        spec = importlib.util.spec_from_file_location(f"fq3ref.{name}", f"{REF}/{name}.py")
        m = importlib.util.module_from_spec(spec)
        sys.modules[f"fq3ref.{name}"] = m
        spec.loader.exec_module(m)
        mods[name] = m
    return mods


class _TorchProxy:
    """`torch` as seen by the reference's sampling module, with multinomial swapped for the noise contract."""

    def __init__(self):
        self.uniforms = []
        self.captured = []

    def __getattr__(self, k):
        return getattr(torch, k)

    def multinomial(self, probs, n):
        assert n == 1
        self.captured.append(probs.detach().clone())
        u = self.uniforms.pop(0) if self.uniforms else 0.0
        flat = probs.reshape(-1, probs.shape[-1])
        out = [O.draw_inverse_cdf(flat[i], u) for i in range(flat.shape[0])]
        return torch.tensor(out, dtype=torch.long).reshape(*probs.shape[:-1], 1)


# ----------------------------------------------------------------------------------------------
# sampling fixtures
# ----------------------------------------------------------------------------------------------


def gen_sampling(ref, out_path):
    smp = ref["sampling"]
    proxy = _TorchProxy()
    smp.torch = proxy
    rng = np.random.default_rng(1234)
    cases = {}
    idx = 0
    for dtype in (torch.float32, torch.bfloat16):
        for V in (256, 2048, 3072):
            for (T, k, p) in ((0.9, 50, 1.0), (0.7, 5, 1.0), (1.3, 0, 1.0), (0.9, 50, 0.8), (1.0, 0, 0.5)):
                if p < 1.0 and dtype is torch.bfloat16:
                    continue  # nucleus path is fp32-semantics in the engine (see oracle docstring)
                lg = torch.from_numpy((rng.standard_normal(V) * 3.0).astype(np.float32)).to(dtype)
                if idx % 3 == 0:  # force ties at the top-k boundary
                    srt = torch.sort(lg.float(), descending=True).values
                    kk = max(1, min(k if k > 0 else 7, V) - 1)
                    lg[rng.integers(0, V, size=4)] = srt[kk].to(dtype)
                mask = torch.zeros(V, dtype=torch.bool)
                mask[(V - 1024 if V > 1024 else V - 32):] = True
                eos = V - 900 if V > 1024 else V - 10
                mask[eos] = False
                sup = [eos] if idx % 2 == 0 else None
                u = float(rng.random(dtype=np.float32))
                proxy.uniforms = [u]
                proxy.captured = []
                tok = smp.sample_logits(lg[None], temperature=T, top_k=k, top_p=p, do_sample=True,
                                        suppress_mask=mask, suppress_tokens=sup)
                greedy = smp.sample_logits(lg[None], temperature=T, top_k=k, top_p=p, do_sample=False,
                                           suppress_mask=mask, suppress_tokens=sup)
                pre = f"c{idx}_"
                cases[pre + "logits"] = lg.float().numpy()
                cases[pre + "bf16"] = np.array(int(dtype is torch.bfloat16))
                cases[pre + "params"] = np.array([T, k, p, u, eos, -1 if sup is None else sup[0]], dtype=np.float64)
                cases[pre + "probs"] = proxy.captured[0][0].float().numpy()
                cases[pre + "token"] = np.array(int(tok[0]))
                cases[pre + "greedy"] = np.array(int(greedy[0]))
                idx += 1
    # repetition penalty known answers (incl. the reference's own KAT, tests/test_sampling.py:10-21)
    for j, dtype in enumerate((torch.float32, torch.bfloat16)):
        V = 512
        lg = torch.from_numpy((rng.standard_normal(V) * 2.0).astype(np.float32)).to(dtype)
        hist = torch.from_numpy(rng.integers(0, V, size=90)).long()
        out = ref["sampling"].apply_repetition_penalty(lg.clone()[None, None], hist, 1.05)
        cases[f"pen{j}_logits"] = lg.float().numpy()
        cases[f"pen{j}_hist"] = hist.numpy()
        cases[f"pen{j}_out"] = out[0, 0].float().numpy()
    cases["n_cases"] = np.array(idx)
    np.savez_compressed(out_path, **cases)
    smp.torch = torch
    print("sampling fixtures:", idx, "->", out_path)


# ----------------------------------------------------------------------------------------------
# loop fixtures: the reference schedulers driving oracle-backed doubles
# ----------------------------------------------------------------------------------------------


class _Embed:
    def __init__(self, table):
        self.table = table

    def __call__(self, ids):
        return self.table[ids]


class _Talker:
    """Double for qwen_tts's talker as used by generate.py:99-121 / streaming.py:52-78."""

    def __init__(self, om: O.OracleModel):
        self.om = om
        self.rope_deltas = None
        nb = om.cfg.num_code_groups - 1
        self.code_predictor = types.SimpleNamespace(
            get_input_embeddings=lambda: [
                _Embed(om.W[f"talker.code_predictor.model.codec_embedding.{i}.weight"]) for i in range(nb)])
        self.codec_head = lambda h: torch.nn.functional.linear(h, om.W["talker.codec_head.weight"])

    def get_input_embeddings(self):
        return _Embed(self.om.W["talker.model.codec_embedding.weight"])

    def forward(self, inputs_embeds, attention_mask=None, **kw):
        logits, past_hidden, cache = self.om.talker_prefill(inputs_embeds[0])
        return types.SimpleNamespace(past_key_values=cache, past_hidden=past_hidden[None, None],
                                     generation_step=0, logits=logits[None, None])


class _PredGraph:
    def __init__(self, om, sp, uniforms):
        self.om, self.sp, self.uniforms, self.frame = om, sp, uniforms, 0

    def run(self, pred_input):
        u = self.uniforms[self.frame + 1, 1:16]
        self.frame += 1
        return torch.tensor(self.om.predictor_frame(pred_input[0, 0], pred_input[0, 1], self.sp, u), dtype=torch.long)


class _TalkerGraph:
    def __init__(self, om, max_seq_len):
        self.om, self.max_seq_len, self.cache = om, max_seq_len, None

    def prefill_kv(self, cache):
        self.cache = cache
        return cache.length()

    def set_generation_state(self, attention_mask, rope_deltas):
        return None

    def run(self, input_embeds, position):
        return self.om.talker_step(input_embeds[0, 0], position, self.cache)[None, None]


LOOP_CASES = [
    # name, weight seed, P, Tt, max_new, min_new, do_sample, penalty, max_seq_len, chunk, eos_boost, noise seed
    ("greedy_plain", 0, 12, 5, 12, 2, False, 1.0, 2048, 4, 1.0, 0),
    ("greedy_penalty", 1, 9, 0, 14, 2, False, 1.05, 2048, 8, 1.0, 0),
    ("sampled_default", 2, 16, 20, 16, 2, True, 1.05, 2048, 8, 1.0, 7),
    ("sampled_eos", 3, 10, 3, 40, 2, True, 1.05, 2048, 8, 6.0, 11),
    ("sampled_eos_min5", 3, 10, 3, 40, 5, True, 1.05, 2048, 3, 9.0, 12),
    ("maxlen_stop", 4, 10, 2, 30, 2, True, 1.05, 18, 4, 1.0, 13),
    ("min0", 5, 8, 1, 6, 0, True, 1.3, 2048, 12, 1.0, 14),
]


def gen_loop(ref, out_path):
    torch.cuda.synchronize = lambda *a, **k: None  # generate.py:142,201 / streaming.py:96,158,177
    smp = ref["sampling"]
    proxy = _TorchProxy()
    smp.torch = proxy
    out = {}
    for (name, wseed, P, Tt, max_new, min_new, do_sample, pen, max_seq, chunk, boost, nseed) in LOOP_CASES:
        cfg = O.cfg_tiny()
        W = O.make_weights(cfg, seed=wseed, eos_boost=boost)
        om = O.OracleModel(cfg, W)
        tie, tth, tpe = O.make_inputs(cfg, P, Tt, seed=wseed)
        uniforms = np.random.default_rng(nseed).random((max_new + 1, 16), dtype=np.float32)
        sp_pred = O.SamplingParams(do_sample=do_sample, repetition_penalty=1.0)
        conf = types.SimpleNamespace(codec_eos_token_id=cfg.codec_eos_token_id, num_code_groups=cfg.num_code_groups,
                                     vocab_size=cfg.talker.vocab_size)
        kw = dict(talker_input_embeds=tie[None], attention_mask=torch.ones(1, P, dtype=torch.long),
                  trailing_text_hiddens=tth[None], tts_pad_embed=tpe[None, None], config=conf,
                  max_new_tokens=max_new, min_new_tokens=min_new, temperature=0.9, top_k=50, top_p=1.0,
                  do_sample=do_sample, repetition_penalty=pen)
        # non-streaming
        proxy.uniforms = [float(x) for x in uniforms[:, 0]]
        codes, timing = ref["generate"].fast_generate(
            talker=_Talker(om), predictor_graph=_PredGraph(om, sp_pred, uniforms),
            talker_graph=_TalkerGraph(om, max_seq), **kw)
        codes = torch.zeros(0, 16, dtype=torch.long) if codes is None else codes
        # streaming
        proxy.uniforms = [float(x) for x in uniforms[:, 0]]
        chunks, keys, finals = [], None, []
        for c, t in ref["streaming"].fast_generate_streaming(
                talker=_Talker(om), predictor_graph=_PredGraph(om, sp_pred, uniforms),
                talker_graph=_TalkerGraph(om, max_seq), chunk_size=chunk, **kw):
            chunks.append(c)
            finals.append(int(t["is_final"]))
            keys = sorted(t.keys())
        scodes = torch.cat(chunks) if chunks else torch.zeros(0, 16, dtype=torch.long)
        assert torch.equal(scodes, codes), name
        out[name + "_codes"] = codes.numpy()
        out[name + "_chunks"] = np.array([c.shape[0] for c in chunks], dtype=np.int64)
        out[name + "_final"] = np.array(finals, dtype=np.int64)
        out[name + "_params"] = np.array([wseed, P, Tt, max_new, min_new, int(do_sample), pen, max_seq, chunk, boost,
                                          nseed], dtype=np.float64)
        eos_hit = codes.shape[0] < max_new
        print(f"{name}: frames={codes.shape[0]} chunks={[c.shape[0] for c in chunks]} stopped_early={eos_hit} "
              f"timing_keys={keys} nonstream_keys={sorted(timing.keys())}")
    out["names"] = np.array([c[0] for c in LOOP_CASES])
    np.savez_compressed(out_path, **out)
    smp.torch = torch


# ----------------------------------------------------------------------------------------------
# prompt assembly fixtures
# ----------------------------------------------------------------------------------------------


def load_reference_model_class():
    """The reference's FasterQwen3TTS class, loaded by file path with `soundfile` stubbed."""
    if "soundfile" not in sys.modules:
        sys.modules["soundfile"] = types.ModuleType("soundfile")
    for name in ("utils", "model"):
        spec = importlib.util.spec_from_file_location(f"fq3ref.{name}", f"{REF}/{name}.py")
        m = importlib.util.module_from_spec(spec)
        sys.modules[f"fq3ref.{name}"] = m
        spec.loader.exec_module(m)
    return sys.modules["fq3ref.model"].FasterQwen3TTS


def gen_prompt(out_path):
    from oracle import prompt_cases as PC
    ref_cls = load_reference_model_class()
    base = PC.build_base(seed=0)
    out = {}
    names = []
    for name, kw in PC.cases(base).items():
        tie, tam, tth, tpe = ref_cls._build_talker_inputs_local(None, base.model, **kw)
        out[name + "_tie"], out[name + "_tam"] = tie.numpy(), tam.numpy()
        out[name + "_tth"], out[name + "_tpe"] = tth.numpy(), tpe.numpy()
        names.append(name)
        print(f"{name}: embeds {tuple(tie.shape)} mask_sum {tam.sum(1).tolist()} trailing {tuple(tth.shape)}")
    out["names"] = np.array(names)
    np.savez_compressed(out_path, **out)


# ----------------------------------------------------------------------------------------------
# streaming codec-window policy fixtures
# ----------------------------------------------------------------------------------------------


def gen_window(out_path):
    """Runs the body of the reference's generate_voice_clone_streaming (model.py:1019-1137) with a fake `self`:
    request preparation and the token generator are doubles, the Phase-1 / Phase-2 window logic is the reference's."""
    from oracle import window_cases as WC
    ref_cls = load_reference_model_class()
    streaming_mod = sys.modules["fq3ref.streaming"]
    real_stream = streaming_mod.fast_generate_streaming
    out, names = {}, []
    try:
        for name, (chunk_size, sizes, n_ref, tk) in WC.CASES.items():
            tok = WC.FakeTokenizer(**tk)
            ref_codes = WC.ref_codes_for(n_ref)
            chunks = WC.chunk_stream(sizes, seed=len(name))
            streaming_mod.fast_generate_streaming = lambda **kw: iter(chunks)
            fake = types.SimpleNamespace(
                _reject_ggml_cached_reference_args=lambda **kw: None,
                _resolve_non_streaming_mode=lambda v, default: default,
                _prepare_generation=lambda **kw: (types.SimpleNamespace(speech_tokenizer=tok), None, None, None, None,
                                                  None, None, ref_codes),
                predictor_graph=None, talker_graph=None)
            got = list(ref_cls.generate_voice_clone_streaming.__wrapped__(fake, "text", "English", ref_audio="x.wav",
                                                                          chunk_size=chunk_size)
                       if hasattr(ref_cls.generate_voice_clone_streaming, "__wrapped__") else
                       ref_cls.generate_voice_clone_streaming(fake, "text", "English", ref_audio="x.wav",
                                                              chunk_size=chunk_size))
            lens = [len(a) for a, _, _ in got]
            out[name + "_lens"] = np.array(lens, dtype=np.int64)
            out[name + "_audio"] = np.concatenate([np.asarray(a, dtype=np.float32) for a, _, _ in got])
            out[name + "_decoded_T"] = np.array(tok.calls, dtype=np.int64)
            names.append(name)
            print(f"{name}: chunk lens {lens} decode calls (frames) {tok.calls}")
    finally:
        streaming_mod.fast_generate_streaming = real_stream
    # non-streaming: generate_voice_clone's decode + reference trim (model.py:914-938)
    gen_mod = sys.modules["fq3ref.generate"]
    real_gen = gen_mod.fast_generate
    try:
        for name, (n_gen, n_ref, tk) in WC.NONSTREAM_CASES.items():
            tok = WC.FakeTokenizer(**tk)
            ref_codes = WC.ref_codes_for(n_ref)
            gen_mod.fast_generate = lambda **kw: (WC.generated_codes(n_gen), dict(WC.TIMING))
            fake = types.SimpleNamespace(
                _reject_ggml_cached_reference_args=lambda **kw: None,
                _resolve_non_streaming_mode=lambda v, default: default,
                _prepare_generation=lambda **kw: (types.SimpleNamespace(speech_tokenizer=tok), None, None, None, None,
                                                  None, None, ref_codes),
                predictor_graph=None, talker_graph=None, sample_rate=WC.SR)
            fn = ref_cls.generate_voice_clone
            fn = getattr(fn, "__wrapped__", fn)
            audio, sr = fn(fake, "text", "English", ref_audio="x.wav")
            out[name + "_audio"] = np.asarray(audio[0], dtype=np.float32)
            out[name + "_decoded_T"] = np.array(tok.calls, dtype=np.int64)
            names.append(name)
            print(f"{name}: {len(audio[0])} samples, decode calls {tok.calls}, sr {sr}")
    finally:
        gen_mod.fast_generate = real_gen
    out["names"] = np.array(names)
    np.savez_compressed(out_path, **out)


# ----------------------------------------------------------------------------------------------
# parity (dynamic-cache) streaming fixtures: the reference's own parity_generate_streaming, driven with the decode-step
# talker double of oracle/parity_cases.py (torch.multinomial seeded; the probabilities it is handed are pinned bit for
# bit by sampling.npz)
# ----------------------------------------------------------------------------------------------
def gen_parity_stream(ref, out_path):
    from oracle import parity_cases as PC
    torch.cuda.synchronize = lambda *a, **k: None  # streaming.py:262,337,353
    out = {}
    for case in PC.CASES:
        chunks, timings, calls = PC.run_case(ref["streaming"].parity_generate_streaming, case)
        name = case[0]
        codes = torch.cat(chunks) if chunks else torch.zeros(0, 16, dtype=torch.long)
        out[name + "_codes"] = codes.numpy()
        out[name + "_chunks"] = np.array([c.shape[0] for c in chunks], dtype=np.int64)
        out[name + "_final"] = np.array([int(t["is_final"]) for t in timings], dtype=np.int64)
        out[name + "_total"] = np.array([t["total_steps_so_far"] for t in timings], dtype=np.int64)
        out[name + "_ncalls"] = np.array([len(calls)], dtype=np.int64)
        out[name + "_lastcall"] = np.array([str(calls[-1])])
        keys = sorted(timings[0].keys()) if timings else []
        print(f"parity {name}: frames={codes.shape[0]} chunks={[c.shape[0] for c in chunks]} final={[int(t['is_final']) for t in timings]} "
              f"calls={len(calls)} keys={keys}")
    out["names"] = np.array([c[0] for c in PC.CASES])
    out["timing_keys"] = np.array(sorted(timings[0].keys()))
    np.savez_compressed(out_path, **out)


if __name__ == "__main__":
    ref = load_reference()
    gdir = os.path.join(ROOT, "tests", "golden")
    os.makedirs(gdir, exist_ok=True)
    with torch.inference_mode():
        gen_sampling(ref, os.path.join(gdir, "sampling.npz"))
        gen_loop(ref, os.path.join(gdir, "loop.npz"))
        gen_prompt(os.path.join(gdir, "prompt.npz"))
        gen_window(os.path.join(gdir, "window.npz"))
        gen_parity_stream(ref, os.path.join(gdir, "parity_stream.npz"))
