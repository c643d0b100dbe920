"""GPU parity: the sm_90a engine (through the C ABI) against the CPU oracle on the same seeded inputs.

Bars (north_star): codec-token indices bit-exact (fp32, greedy and noise-contract sampling); bf16 within a
stated logit tolerance plus the reference's structural invariants (tests/test_e2e_parity.py:40-101)."""
import dataclasses
import os

import numpy as np
import pytest
import torch

from oracle import qwen3_tts_oracle as O

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from util_models import Pair, report
    from faster_qwen3_tts.engine import SamplingParams
    from faster_qwen3_tts.generate import fast_generate
    from faster_qwen3_tts.streaming import fast_generate_streaming


@pytest.fixture(scope="module")
def tiny32():
    return Pair(O.cfg_tiny(), seed=0, dtype=torch.float32, max_seq_len=128)


@pytest.fixture(scope="module")
def tiny16():
    return Pair(O.cfg_tiny(), seed=0, dtype=torch.bfloat16, max_seq_len=128)


def _prefill_into_engine(p, P=12, seed=0):
    tie, tth, tpe = O.make_inputs(p.cfg, P, 5, seed=seed, dtype=p.dtype)
    with torch.inference_mode():
        logits, ph, cache = p.om.talker_prefill(tie)
    for li in range(p.cfg.talker.num_hidden_layers):
        p.engine.import_kv(li, cache.k[li].cuda(), cache.v[li].cuda())
    p.engine.set_generation_state(0, 0)
    return tie, tth, tpe, logits, ph, cache


@pytest.mark.parametrize("which", ["tiny32", "tiny16"])
def test_talker_step_layerwise(which, request):
    p = request.getfixturevalue(which)
    tol = 2e-4 if p.dtype == torch.float32 else 6e-2
    tie, tth, tpe, logits, ph, cache = _prefill_into_engine(p)
    x = torch.randn(p.cfg.talker.hidden_size, generator=torch.Generator().manual_seed(5)).to(p.dtype)
    dbg = {}
    with torch.inference_mode():
        ref = p.om.talker_step(x, 12, cache, dbg=dbg)
    p.engine.debug_enable(True)
    got = p.engine.talker_step(x.cuda(), 12)
    torch.cuda.synchronize()
    d = p.engine.debug_layers("t", 1)
    p.engine.debug_enable(False)
    worst = 0.0
    for li in range(p.cfg.talker.num_hidden_layers):
        for key in ("qkv", "attn", "x1", "act", "x"):
            worst = max(worst, report(f"L{li}.{key}", d[f"L{li}.{key}"][0], dbg[f"L{li}.{key}"][0]))
    worst = max(worst, report("hidden", got, ref))
    assert worst < tol


@pytest.mark.parametrize("which", ["tiny32", "tiny16"])
def test_predictor_greedy_and_pass0(which, request):
    p = request.getfixturevalue(which)
    g = torch.Generator().manual_seed(3)
    ph = torch.randn(p.cfg.talker.hidden_size, generator=g).to(p.dtype)
    tok = 17
    emb = p.W["talker.model.codec_embedding.weight"][tok]
    dbg = {}
    with torch.inference_mode():
        ref = p.om.predictor_frame(ph, emb, O.SamplingParams(do_sample=False), dbg=dbg)
    p.engine.debug_enable(True)
    got = p.engine.predictor_run(torch.stack((ph, emb)).cuda(), SamplingParams(do_sample=False))
    torch.cuda.synchronize()
    d = p.engine.debug_layers("p", 2)
    p.engine.debug_enable(False)
    worst = 0.0
    for li in range(p.cfg.predictor.num_hidden_layers):
        for key in ("qkv", "attn", "x1", "act", "x"):
            worst = max(worst, report(f"P{li}.{key}", d[f"L{li}.{key}"], dbg[f"L{li}.{key}"]))
    print("codes got", got.tolist(), "ref", ref)
    assert worst < (2e-4 if p.dtype == torch.float32 else 8e-2)
    if p.dtype == torch.float32:
        assert got.tolist() == ref


def test_predictor_sampled_fp32(tiny32):
    p = tiny32
    g = torch.Generator().manual_seed(4)
    ph = torch.randn(p.cfg.talker.hidden_size, generator=g)
    emb = p.W["talker.model.codec_embedding.weight"][33]
    u = np.random.default_rng(9).random(15, dtype=np.float32)
    with torch.inference_mode():
        ref = p.om.predictor_frame(ph, emb, O.SamplingParams(), uniforms=u)
    got = p.engine.predictor_run(torch.stack((ph, emb)).cuda(), SamplingParams(), torch.from_numpy(u).cuda())
    assert got.tolist() == ref


def test_sampler_kernel_vs_reference_fixtures(tiny32, tiny16, golden_dir):
    """fq3_sample_logits on the logits recorded from the reference's sample_logits (oracle/make_golden.py)."""
    s = np.load(os.path.join(golden_dir, "sampling.npz"))
    bad = []
    for i in range(int(s["n_cases"])):
        pre = f"c{i}_"
        bf = bool(int(s[pre + "bf16"]))
        p = tiny16 if bf else tiny32
        T, k, tp, u, eos, sup = s[pre + "params"]
        lg = torch.from_numpy(s[pre + "logits"]).to(p.dtype).cuda()
        V = lg.numel()
        if V <= 1024:
            continue  # the fixture's 32-wide suppress range is not the engine's [V-1024,V) rule
        for do_sample, key in ((True, "token"), (False, "greedy")):
            sp = SamplingParams(do_sample=do_sample, top_k=int(k), temperature=float(T), top_p=float(tp))
            got = p.engine.sample_logits(lg, sp, u=float(u), suppress_special=True, eos_id=int(eos),
                                         suppress_eos=sup >= 0)
            if int(got.item()) != int(s[pre + key]):
                bad.append((i, key, int(got.item()), int(s[pre + key])))
    assert not bad, bad


def test_sampler_penalty_matches_reference(tiny32, golden_dir):
    s = np.load(os.path.join(golden_dir, "sampling.npz"))
    lg = torch.from_numpy(s["pen0_logits"])
    hist = torch.from_numpy(s["pen0_hist"])
    ref = torch.from_numpy(s["pen0_out"])
    want = int(torch.argmax(ref))
    got = tiny32.engine.sample_logits(lg.cuda(), SamplingParams(do_sample=False, repetition_penalty=1.05),
                                      history=hist.cuda())
    assert int(got.item()) == want


def _run_case(p, tie, tth, tpe, uniforms, **kw):
    u = torch.from_numpy(uniforms).cuda() if uniforms is not None else None
    codes, timing = fast_generate(p.talker, tie[None].cuda(), torch.ones(1, tie.shape[0], dtype=torch.long).cuda(),
                                  tth[None].cuda(), tpe[None, None].cuda(), p.config, p.pg, p.tg, uniforms=u, **kw)
    return (torch.zeros(0, 16, dtype=torch.long) if codes is None else codes.cpu()), timing


@pytest.mark.parametrize("idx", range(7))
def test_fused_loop_vs_reference_scheduler_goldens(idx, golden_dir):
    """fp32 engine, whole loop on device, against codes recorded from the REFERENCE's fast_generate /
    fast_generate_streaming driving the oracle (tests/golden/loop.npz)."""
    loop = np.load(os.path.join(golden_dir, "loop.npz"))
    name = str(loop["names"][idx])
    wseed, P, Tt, max_new, min_new, do_sample, pen, max_seq, chunk, boost, nseed = loop[name + "_params"]
    p = Pair(O.cfg_tiny(), seed=int(wseed), dtype=torch.float32, max_seq_len=max(int(max_seq), 8) if max_seq < 2048 else 128,
             eos_boost=float(boost))
    p.pg.do_sample = bool(do_sample)
    tie, tth, tpe = O.make_inputs(p.cfg, int(P), int(Tt), seed=int(wseed))
    uniforms = np.random.default_rng(int(nseed)).random((int(max_new) + 1, 16), dtype=np.float32)
    kw = dict(max_new_tokens=int(max_new), min_new_tokens=int(min_new), do_sample=bool(do_sample),
              repetition_penalty=float(pen))
    codes, timing = _run_case(p, tie, tth, tpe, uniforms, **kw)
    want = loop[name + "_codes"]
    print(name, "got", codes.shape, "want", want.shape)
    assert codes.shape == want.shape and np.array_equal(codes.numpy(), want), name
    assert set(timing) == {"prefill_ms", "decode_s", "steps", "ms_per_step", "steps_per_s"}
    # streaming: same tokens, reference chunk boundaries and timing keys
    chunks, finals = [], []
    u = torch.from_numpy(uniforms).cuda()
    for c, t in fast_generate_streaming(p.talker, tie[None].cuda(), torch.ones(1, int(P), dtype=torch.long).cuda(),
                                        tth[None].cuda(), tpe[None, None].cuda(), p.config, p.pg, p.tg,
                                        chunk_size=int(chunk), uniforms=u, **kw):
        chunks.append(c.cpu())
        finals.append(int(t["is_final"]))
        assert set(t) == {"chunk_index", "chunk_steps", "prefill_ms", "decode_ms", "total_steps_so_far", "is_final"}
    assert [c.shape[0] for c in chunks] == loop[name + "_chunks"].tolist()
    assert finals == loop[name + "_final"].tolist()   # incl. the FULL last chunk the cache limit makes final
    if chunks:
        assert np.array_equal(torch.cat(chunks).numpy(), want)


def test_bf16_generation_structure_and_streaming_equivalence(tiny16):
    """bf16: the reference's own structural gate (tests/test_e2e_parity.py:40-101,729-782)."""
    p = tiny16
    tie, tth, tpe = O.make_inputs(p.cfg, 10, 4, seed=2, dtype=torch.bfloat16)
    uniforms = np.random.default_rng(5).random((41, 16), dtype=np.float32)
    kw = dict(max_new_tokens=40, min_new_tokens=2, do_sample=True)
    codes, _ = _run_case(p, tie, tth, tpe, uniforms, **kw)
    V = p.cfg.talker.vocab_size
    assert codes.ndim == 2 and codes.shape[1] == 16 and codes.shape[0] >= 2
    assert int(codes[:, 0].max()) < V - 1024 and int(codes[:, 0].min()) >= 0
    assert int(codes[:, 1:].max()) < p.cfg.predictor.vocab_size
    assert (codes[:, 0] == p.cfg.codec_eos_token_id).sum() == 0
    chunks = [c.cpu() for c, _ in fast_generate_streaming(
        p.talker, tie[None].cuda(), torch.ones(1, 10, dtype=torch.long).cuda(), tth[None].cuda(),
        tpe[None, None].cuda(), p.config, p.pg, p.tg, chunk_size=8, uniforms=torch.from_numpy(uniforms).cuda(), **kw)]
    assert torch.equal(torch.cat(chunks), codes)


def test_reference_scheduler_drives_engine_duck_types(tiny32):
    """Drop-in proof: the step-wise loop (the reference's algorithm over duck-typed run()/prefill_kv()) with the
    engine-backed graph objects gives the oracle's greedy codes."""
    from faster_qwen3_tts.generate import stepwise_frames
    p = tiny32
    p.pg.do_sample = False
    tie, tth, tpe = O.make_inputs(p.cfg, 9, 3, seed=1)
    with torch.inference_mode():
        rows = [r for k, r in stepwise_frames(
            p.talker, tie[None].cuda(), torch.ones(1, 9, dtype=torch.long).cuda(), tth[None].cuda(),
            tpe[None, None].cuda(), p.config, p.pg, p.tg, max_new_tokens=10, min_new_tokens=2, temperature=0.9,
            top_k=50, top_p=1.0, do_sample=False, repetition_penalty=1.05) if k == "frame"]
    with torch.inference_mode():
        want = O.generate(p.om, tie, tth, tpe, max_new_tokens=10,
                          sp_talker=O.SamplingParams(do_sample=False, repetition_penalty=1.05),
                          sp_pred=O.SamplingParams(do_sample=False), max_seq_len=128)
    p.pg.do_sample = True
    assert torch.equal(torch.stack(rows).cpu(), want)


def test_prompt_too_long_raises(tiny32):
    p = tiny32
    k = torch.zeros(1, 2, 200, 128, device="cuda")
    with pytest.raises(RuntimeError, match="Input is too long"):
        p.tg.prefill_kv([(k, k)] * p.cfg.talker.num_hidden_layers)


@pytest.mark.parametrize("size", ["0.6B"])
def test_full_size_fp32_greedy_tokens_bit_exact(size):
    """BASELINE config 1: 0.6B geometry, P=40, fp32 greedy (the reference's exact-parity protocol,
    tests/test_e2e_parity.py:236-313,431-485); tokens must be identical to the CPU oracle."""
    cfg = O.cfg_0p6b()
    p = Pair(cfg, seed=0, dtype=torch.float32, max_seq_len=256)
    p.pg.do_sample = False
    tie, tth, tpe = O.make_inputs(cfg, 40, 0, seed=0)
    n = 12
    with torch.inference_mode():
        want = O.generate(p.om, tie, tth, tpe, max_new_tokens=n,
                          sp_talker=O.SamplingParams(do_sample=False, repetition_penalty=1.0),
                          sp_pred=O.SamplingParams(do_sample=False), max_seq_len=256)
    codes, _ = _run_case(p, tie, tth, tpe, None, max_new_tokens=n, min_new_tokens=2, do_sample=False,
                         repetition_penalty=1.0)
    print("match rows:", int((codes == want).all(dim=1).sum()), "of", n)
    assert torch.equal(codes, want)


def test_full_size_bf16_step_logits_and_structure():
    """1.7B geometry, bf16: one decode step's hidden within bf16 tolerance of the oracle; 24 sampled frames pass the
    structural gate."""
    cfg = O.cfg_1p7b()
    p = Pair(cfg, seed=1, dtype=torch.bfloat16, max_seq_len=512)
    tie, tth, tpe, logits, ph, cache = _prefill_into_engine(p, P=24, seed=1)
    x = torch.randn(cfg.talker.hidden_size, generator=torch.Generator().manual_seed(6)).to(torch.bfloat16)
    with torch.inference_mode():
        ref = p.om.talker_step(x, 24, cache)
    got = p.engine.talker_step(x.cuda(), 24)
    err = report("hidden1.7B", got, ref)
    assert err < 0.15  # post-norm hidden, |x|~3: a few bf16 ulps after 28 layers
    uniforms = np.random.default_rng(1).random((25, 16), dtype=np.float32)
    codes, _ = _run_case(p, tie, tth, tpe, uniforms, max_new_tokens=24, min_new_tokens=2, do_sample=True)
    assert codes.shape[1] == 16 and codes.shape[0] >= 2
    assert int(codes[:, 0].max()) < 2048 and int(codes[:, 1:].max()) < 2048


def test_codec_stack_kernels_vs_fp32_oracle_reduced_geometry():
    """K4 at a reduced geometry (fast): engine decode against the fp32 oracle decode (oracle/codec_oracle.py) at the
    north_star's PCM bar, plus causality of the window (a prefix decodes to the same samples).  The full-geometry gate
    lives in tests/test_gpu_codec.py."""
    from faster_qwen3_tts.codec import Code2WavConfig, build_codec
    from oracle import codec_oracle
    cfg = Code2WavConfig(hidden_size=256, num_hidden_layers=2, num_attention_heads=4, intermediate_size=512,
                         decoder_dim=512, codebook_size=64)
    st = build_codec(cfg, seed=3, dtype=torch.bfloat16, device="cuda", backend="engine")
    codes = torch.randint(0, 64, (1, 9, 16), device="cuda")
    got, sr = st.decode({"audio_codes": codes})
    assert sr == 24000 and got[0].shape[0] == 9 * 1920
    with torch.inference_mode():
        ref32 = codec_oracle.decode(st.decoder.state_dict(), codes[0], codebook_size=64, num_attention_heads=4,
                                    sliding_window=cfg.sliding_window, rms_norm_eps=cfg.rms_norm_eps)
    e_engine = (got[0] - ref32).abs().max().item()
    print(f"codec max|engine - fp32 oracle| = {e_engine:.4e}  peak {ref32.abs().max().item():.3f} rms {ref32.pow(2).mean().sqrt().item():.3e}")
    assert e_engine < 1e-3
    got2, _ = st.decode({"audio_codes": codes[:, :5]})
    assert (got2[0] - got[0][: 5 * 1920]).abs().max().item() < 1e-6


def test_native_prefill_vs_oracle_bf16(tiny16):
    """K3: hand-written prefill (C ABI) vs the bf16 oracle: logits / past_hidden within bf16 tolerance, and a decode
    step on top of the natively written KV cache equals a step on top of oracle KV."""
    p = tiny16
    tie, tth, tpe = O.make_inputs(p.cfg, 37, 3, seed=4, dtype=torch.bfloat16)
    with torch.inference_mode():
        logits, ph, cache = p.om.talker_prefill(tie)
    lg, hid = p.engine.prefill(tie.cuda())
    e1 = report("prefill.hidden", hid, ph)
    e2 = report("prefill.logits", lg, logits)
    assert e1 < 6e-2 and e2 < 0.25
    x = torch.randn(p.cfg.talker.hidden_size, generator=torch.Generator().manual_seed(8)).to(torch.bfloat16)
    p.engine.set_generation_state(0, 0)
    got = p.engine.talker_step(x.cuda(), 37).clone()
    with torch.inference_mode():
        ref = p.om.talker_step(x, 37, cache)
    assert report("step_after_native_prefill", got, ref) < 6e-2
    # same generation with and without the native prefill (greedy, bf16): identical tokens
    p.pg.do_sample = False
    kw = dict(max_new_tokens=6, min_new_tokens=2, do_sample=False)
    a, _ = _run_case(p, tie, tth, tpe, None, **kw)
    p.tg.use_native_prefill = False
    b, _ = _run_case(p, tie, tth, tpe, None, **kw)
    p.tg.use_native_prefill = True
    p.pg.do_sample = True
    print("native vs module prefill rows equal:", int((a == b).all(dim=1).sum()), "of", a.shape[0])
    assert a.shape == b.shape


@pytest.mark.parametrize("talker_change, reason", [
    ({"num_key_value_heads": 1}, "GQA ratio"),
    ({"vocab_size": 1282}, r"vocab_size 1282 is not a multiple of 8|rows 1282 / K \d+ not tileable")])
def test_native_prefill_refuses_unsupported_talker_geometry(talker_change, reason):
    """K3 takes GQA ratios 1 and 2 and a talker vocabulary that is a multiple of 8 (the head GEMM's N): building a bf16
    engine whose talker has a GQA ratio of 4, or a vocabulary = 2 (mod 8), fails while its weights load.  The bf16 decode
    tape already refuses such a vocabulary (its head rows come in units of 8); fq3_engine_set_prefill_weights refuses it
    again for callers that set the prefill weights first."""
    cfg = O.cfg_tiny()
    cfg = dataclasses.replace(cfg, talker=dataclasses.replace(cfg.talker, **talker_change))
    with pytest.raises(RuntimeError, match=reason):
        Pair(cfg, seed=0, dtype=torch.bfloat16, max_seq_len=128)


def test_public_api_end_to_end_tiny():
    """FasterQwen3TTS public surface on a tiny synthetic model: streaming == non-streaming length bookkeeping, PCM
    chunk sizes follow the reference's window policy (every chunk is frames*1920 samples), x-vector and ICL modes."""
    from faster_qwen3_tts import FasterQwen3TTS
    m = FasterQwen3TTS.from_synthetic("tiny", dtype=torch.bfloat16, max_seq_len=512, seed=3)
    assert m.sample_rate == 24000
    for xvec in (True, False):
        torch.manual_seed(0)
        chunks = list(m.generate_voice_clone_streaming("hello there general kenobi", "English", ref_audio="ref.wav",
                                                       ref_text="ref", max_new_tokens=40, min_new_tokens=40, chunk_size=8,
                                                       xvec_only=xvec))
        assert len(chunks) == 5
        for pcm, sr, t in chunks:
            assert sr == 24000 and pcm.dtype == np.float32 and pcm.shape[0] == t["chunk_steps"] * 1920
            assert np.isfinite(pcm).all() and np.abs(pcm).max() <= 1.0
        torch.manual_seed(0)
        audio, sr = m.generate_voice_clone("hello there general kenobi", "English", ref_audio="ref.wav", ref_text="ref",
                                           max_new_tokens=40, min_new_tokens=40, xvec_only=xvec)
        assert sr == 24000 and audio[0].shape[0] == 40 * 1920
    a, sr = m.generate_custom_voice("good morning", "aiden", "English", max_new_tokens=9, min_new_tokens=9)
    assert a[0].shape[0] == 9 * 1920
    with pytest.raises(ValueError, match="ref_audio is required"):
        m.generate_voice_clone("x", "English")
    # a cached reference in decoded form (SURVEY 8(f) item 4): speaker vector alone = x-vector cloning, with the
    # reference's codec frames = ICL cloning (frames are acoustic context of the codec and trimmed from the output)
    H = m.model.model.config.talker_config.hidden_size
    g = np.random.default_rng(0)
    spk = g.standard_normal(H).astype(np.float32) * 0.1
    a, sr = m.generate_voice_clone("cached voice", "English", ref_spk_emb=spk, max_new_tokens=8, min_new_tokens=8)
    assert a[0].shape[0] == 8 * 1920 and np.isfinite(a[0]).all()
    codes = g.integers(0, 200, size=(20, 16)).astype(np.int32)
    chunks = list(m.generate_voice_clone_streaming("cached voice", "English", ref_text="the reference words", ref_spk_emb=spk,
                                                   ref_codes=codes, max_new_tokens=16, min_new_tokens=16, chunk_size=8))
    assert [c[0].shape[0] for c in chunks] == [8 * 1920, 8 * 1920]
    with pytest.raises(ValueError, match="ref_text is required"):
        m.generate_voice_clone("cached voice", "English", ref_spk_emb=spk, ref_codes=codes, max_new_tokens=4)


@pytest.mark.gpu
def test_split_attention_matches_per_head_attention(monkeypatch):
    """bf16 talker steps: keys split over several CTAs per q-head with TMA-staged K/V slices (default) against one
    CTA per q-head reading the cache directly (FQ3_ATTN_SPLIT=0): same weights, same imported cache, positions that
    exercise empty slices, ragged tiles and multi-tile slices, then two consecutive steps (the second reads the row
    the first one appended through the staged path)."""
    from faster_qwen3_tts.model import FasterQwen3TTS
    import torch.nn.functional as F
    monkeypatch.setenv("FQ3_ATTN_SPLIT", "0")
    a = FasterQwen3TTS.from_synthetic("0.6B", dtype=torch.bfloat16, with_codec=False, max_seq_len=2048, seed=3).engine
    monkeypatch.delenv("FQ3_ATTN_SPLIT")
    b = FasterQwen3TTS.from_synthetic("0.6B", dtype=torch.bfloat16, with_codec=False, max_seq_len=2048, seed=3).engine
    g = torch.Generator().manual_seed(11)
    L, nkv = a.talker_cfg["num_hidden_layers"], a.talker_cfg["num_key_value_heads"]
    H = a.H
    worst = 0.0
    for pos in (3, 40, 333, 1100, 2040):
        for l in range(L):
            k = torch.randn(nkv, pos, 128, generator=g).to(torch.bfloat16).cuda()
            v = torch.randn(nkv, pos, 128, generator=g).to(torch.bfloat16).cuda()
            a.import_kv(l, k, v); b.import_kv(l, k, v)
        for step in range(2):
            x = (torch.randn(H, generator=g) * 0.5).to(torch.bfloat16).cuda()
            ya, yb = a.talker_step(x, pos + step).float(), b.talker_step(x, pos + step).float()
            assert torch.isfinite(yb).all()
            err = (ya - yb).abs().max().item()
            cos = F.cosine_similarity(ya, yb, dim=0).item()
            print(f"pos {pos + step}: max abs {err:.4f} cos {cos:.6f}")
            worst = max(worst, err)
            assert cos > 0.999
    assert worst < 0.25  # post-norm hidden |x|~3 after 28 bf16 layers; the two paths differ only in rounding order


@pytest.mark.gpu
def test_fused_loop_across_split_attention_threshold():
    """Fused on-device loop, bf16, tiny geometry (4 q-heads -> 16 key slices per head): the context grows from below
    the split threshold (192 cached keys) through it and across slice/tile boundaries; the producer warp's K/V tile
    schedule has to stay in lock-step with the consumers for every frame (a mismatch hangs or traps), streaming and
    non-streaming drivers must agree, and the first frames -- generated before the threshold -- must equal those of
    an engine with the split path disabled."""
    cfg = O.cfg_tiny()
    P, n = 170, 72
    tie, tth, tpe = O.make_inputs(cfg, P, 6, seed=4, dtype=torch.bfloat16)
    uniforms = np.random.default_rng(9).random((n + 1, 16), dtype=np.float32)
    kw = dict(max_new_tokens=n, min_new_tokens=n, do_sample=True)
    p = Pair(cfg, seed=0, dtype=torch.bfloat16, max_seq_len=512)
    codes, _ = _run_case(p, tie, tth, tpe, uniforms, **kw)
    assert codes.shape == (n, 16)
    assert int(codes[:, 0].max()) < cfg.talker.vocab_size - 1024 and int(codes[:, 1:].max()) < cfg.predictor.vocab_size
    chunks = [c.cpu() for c, _ in fast_generate_streaming(
        p.talker, tie[None].cuda(), torch.ones(1, P, dtype=torch.long).cuda(), tth[None].cuda(),
        tpe[None, None].cuda(), p.config, p.pg, p.tg, chunk_size=8, uniforms=torch.from_numpy(uniforms).cuda(), **kw)]
    assert torch.equal(torch.cat(chunks), codes)
    os.environ["FQ3_ATTN_SPLIT"] = "0"
    try:
        q = Pair(cfg, seed=0, dtype=torch.bfloat16, max_seq_len=512)
    finally:
        del os.environ["FQ3_ATTN_SPLIT"]
    ref, _ = _run_case(q, tie, tth, tpe, uniforms, **kw)
    assert torch.equal(ref[: 192 - P], codes[: 192 - P])   # identical code path until 192 keys are cached
    same = int((ref == codes).all(dim=1).sum())
    print("frames identical with / without split attention:", same, "of", n)
