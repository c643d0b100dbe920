"""Paged talker KV cache (fq3_config::kv_pages, fq3_map_kv_pages, fq3_kv_pages_to / _from; batching.KvPager).

A request's cache rows live in 64-row pages of one pool, reached through its page table.  Only addresses change, not the
arithmetic or its order, so every result must be bit-identical to the default pool, in which each slot owns one
consecutive run of pages: the single-sequence kernel across the split-key threshold (192 cached keys) with 64-key tiles
straddling pages, up to the max_seq_len rule; the batched kernel with mixed lengths, left padding and rope deltas; the
batched prefill into scattered pages.  Pages here come in a shuffled, non-monotone order and are mapped chunk by chunk.
Parking moves a request's pages to host memory and back into other pages without changing its codes or its PCM.  Every
refusal launches nothing and leaves other slots' caches as they were.  Tiny geometry throughout."""
import numpy as np
import pytest
import torch

from oracle import qwen3_tts_oracle as O

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from util_models import Pair
    import faster_qwen3_tts.batching as B
    import faster_qwen3_tts.weights as Wt
    from faster_qwen3_tts.batching import BatchScheduler
    from faster_qwen3_tts.engine import KV_PAGE, EngineError
    from faster_qwen3_tts.generate import begin_fused, fast_generate
    from faster_qwen3_tts.streaming import fast_generate_streaming
    _ENGINE_FOR_TALKER = Wt.engine_for_talker


def _pair(monkeypatch, kv_pages=0, max_slots=None, **kw):
    """util_models.Pair on an engine with a ``kv_pages`` pool and ``max_slots`` slots"""
    monkeypatch.setattr(Wt, "engine_for_talker",
                        lambda *a, **k: _ENGINE_FOR_TALKER(*a, kv_pages=kv_pages, max_slots=max_slots, **k))
    return Pair(**kw)


def _scrambled(monkeypatch, seed):
    """every KvPager hands out its pages in a shuffled order"""
    real = B.KvPager.__init__

    def init(self, engine):
        real(self, engine)
        np.random.default_rng(seed).shuffle(self.free)
    monkeypatch.setattr(B.KvPager, "__init__", init)


def _request(cfg, P, pad, Tt, n, dtype, seed):
    H = cfg.talker.hidden_size
    e, t, tpe = O.make_inputs(cfg, P, Tt, seed=seed, dtype=dtype)
    tie = torch.cat([torch.zeros(pad, H, dtype=dtype), e])
    tam = torch.cat([torch.zeros(pad, dtype=torch.long), torch.ones(P, dtype=torch.long)])
    u = np.random.default_rng(seed).random((n + 1, 16), dtype=np.float32)
    return dict(tie=tie, tam=tam, tth=t, tpe=tpe, pad=pad, n=n, u=u)


def _args(r, tag=0):
    H = r["tie"].shape[1]
    tth = r["tth"][None].cuda() if r["tth"].shape[0] else torch.zeros(1, 0, H, dtype=r["tie"].dtype).cuda()
    return dict(tie=r["tie"][None].cuda(), tam=r["tam"][None].cuda(), tth=tth, tpe=r["tpe"][None, None].cuda(), tag=tag,
                max_new_tokens=r["n"], min_new_tokens=r["n"], do_sample=True, repetition_penalty=1.05,
                uniforms=torch.from_numpy(r["u"]).cuda())


def _run_sched(p, reqs, chunk):
    """all requests through one BatchScheduler -> ({tag: codes}, {tag: logprobs}, scheduler)"""
    sched = BatchScheduler(p.engine, p.talker, p.config, p.pg, p.tg)
    sched.submit_many([_args(r, i) for i, r in enumerate(reqs)], logprobs=True)
    codes, lps = {i: [] for i in range(len(reqs))}, {i: [] for i in range(len(reqs))}
    while len(sched):
        for rq, c in sched.step(chunk):
            codes[rq.tag].append(c.cpu())
            lps[rq.tag].append(rq.chunk_logprobs.cpu())
    return {i: torch.cat(v) for i, v in codes.items()}, {i: torch.cat(v) for i, v in lps.items()}, sched


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_single_sequence_on_scrambled_pages_grown_chunk_by_chunk(dtype, monkeypatch):
    """one request from a 40-row prompt to the max_seq_len rule: on the default pool in launches of 256 frames, on a
    pool of one request plus 3 pages whose pages arrive shuffled, 24 frames (a page every few launches) at a time.
    bf16 crosses 192 cached keys, from where its split-key attention stages 64-key tiles that straddle pages"""
    cfg = O.cfg_tiny()
    S = 512
    ref = _pair(monkeypatch, cfg=cfg, seed=3, dtype=dtype, max_seq_len=S)
    paged = _pair(monkeypatch, kv_pages=S // KV_PAGE + 3, cfg=cfg, seed=3, dtype=dtype, max_seq_len=S)
    assert paged.engine.paged and not ref.engine.paged and paged.engine.kv_pages == S // KV_PAGE + 3
    if dtype == torch.bfloat16:
        assert ref.engine.lib.fq3_num_ctas(ref.engine.h) >= 2 * cfg.talker.num_attention_heads   # split attention on
    _scrambled(monkeypatch, 1)
    r = _request(cfg, 37, 3, 6, S, dtype, seed=5)
    a = _args(r)
    a.pop("tag")
    ins = [a.pop(k) for k in ("tie", "tam", "tth", "tpe")]
    want, wt = fast_generate(ref.talker, *ins, ref.config, ref.pg, ref.tg, return_logprobs=True, **a)
    parts, lps = [], []
    for codes, tm in fast_generate_streaming(paged.talker, *ins, paged.config, paged.pg, paged.tg, chunk_size=24,
                                             return_logprobs=True, **a):
        parts.append(codes)
        lps.append(tm["logprobs"])
    got = torch.cat(parts)
    assert want.shape[0] + 40 == S, want.shape   # ended by the max_seq_len rule, at row S - 1
    assert torch.equal(got, want)
    assert torch.equal(torch.cat(lps), wt["logprobs"])
    if dtype == torch.float32:
        with torch.inference_mode():
            oracle = O.generate(ref.om, r["tie"], r["tth"], r["tpe"], max_new_tokens=S, min_new_tokens=S,
                                sp_talker=O.SamplingParams(do_sample=True, repetition_penalty=1.05),
                                sp_pred=O.SamplingParams(do_sample=True), max_seq_len=S, uniforms=r["u"], n_left_pad=3)
        assert torch.equal(got.cpu(), oracle)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_batched_rows_on_a_pool_that_parks(dtype, monkeypatch):
    """8 requests of mixed prompt lengths and left pads (rope deltas) in batched launches of 5 frames, from a pool of 8
    pages (each request needs 2): budgets are clamped to the mapped rows and requests are parked and restored.  Codes and log-probabilities
    equal those of the default pool; no page is left over"""
    monkeypatch.setenv("FQ3_ATTN_SPLIT", "0")
    cfg = O.cfg_tiny()
    S = 128
    ref = _pair(monkeypatch, cfg=cfg, seed=4, dtype=dtype, max_seq_len=S, max_batch=8)
    paged = _pair(monkeypatch, kv_pages=8, cfg=cfg, seed=4, dtype=dtype, max_seq_len=S, max_batch=8)
    _scrambled(monkeypatch, 2)
    rng = np.random.default_rng(7)
    reqs = []
    for i in range(8):   # every request ends between rows 70 and 100: all of them reach row 64 and need a second page
        P, pad = int(rng.integers(5, 40)), int(rng.integers(0, 6)) if i % 3 else 0
        reqs.append(_request(cfg, P, pad, int(rng.integers(0, 6)), int(rng.integers(70, 100)) - P - pad, dtype,
                             seed=100 + i))
    want, want_lp, _ = _run_sched(ref, reqs, 5)
    got, got_lp, sched = _run_sched(paged, reqs, 5)
    for i in range(8):
        assert torch.equal(got[i], want[i]), i
        assert torch.equal(got_lp[i], want_lp[i]), i
    assert sched.pager.parks > 0 and sched.pager.peak == 8
    assert sorted(sched.pager.free) == list(range(8)) and not sched.pager.mapped
    assert all(paged.engine.slot_kv_rows(s) == 0 for s in range(8))


def test_prefill_batch_into_scattered_pages(monkeypatch):
    """fq3_prefill_batch into three slots whose tables map permuted pages: K/V of every layer, logits and past_hidden
    equal the default pool's"""
    cfg = O.cfg_tiny()
    S = 256
    ref = _pair(monkeypatch, cfg=cfg, seed=6, dtype=torch.bfloat16, max_seq_len=S, max_batch=4)
    paged = _pair(monkeypatch, kv_pages=13, cfg=cfg, seed=6, dtype=torch.bfloat16, max_seq_len=S, max_batch=4)
    perm = [int(x) for x in np.random.default_rng(3).permutation(13)]
    P, pads, slots = [70, 130, 45], [0, 5, 2], [2, 0, 3]
    taken = 0
    for s, n in zip(slots, P):
        k = -(-n // KV_PAGE)
        paged.engine.map_kv_pages(s, perm[taken:taken + k])
        assert paged.engine.slot_kv_rows(s) == k * KV_PAGE
        taken += k
    rows = [O.make_inputs(cfg, n, 0, seed=20 + i, dtype=torch.bfloat16)[0].cuda() for i, n in enumerate(P)]
    lw, hw = ref.engine.prefill_batch(rows, pads, slots)
    lg, hg = paged.engine.prefill_batch(rows, pads, slots)
    assert torch.equal(lg, lw) and torch.equal(hg, hw)
    for s, n in zip(slots, P):
        for l in range(cfg.talker.num_hidden_layers):
            kw, vw = ref.engine.export_kv(l, n, slot=s)
            kg, vg = paged.engine.export_kv(l, n, slot=s)
            assert torch.equal(kg, kw) and torch.equal(vg, vw), (s, l)


def _kv(eng, slot, P, L):
    return torch.cat([torch.cat([t.flatten() for t in eng.export_kv(l, P, slot=slot)]) for l in range(L)])


def test_refusals_launch_nothing_and_touch_no_other_slot(monkeypatch):
    cfg = O.cfg_tiny()
    S = 256
    npt = S // KV_PAGE
    with pytest.raises(EngineError, match="kv_pages"):
        _pair(monkeypatch, kv_pages=npt - 1, cfg=cfg, seed=1, dtype=torch.bfloat16, max_seq_len=S, max_batch=4)
    p = _pair(monkeypatch, kv_pages=npt + 4, cfg=cfg, seed=1, dtype=torch.bfloat16, max_seq_len=S, max_batch=4)
    eng, L = p.engine, cfg.talker.num_hidden_layers
    assert all(eng.slot_kv_rows(s) == 0 for s in range(4))
    # slot 0: a prefilled request on pages 5, 2
    eng.map_kv_pages(0, [5, 2])
    e0 = O.make_inputs(cfg, 100, 0, seed=2, dtype=torch.bfloat16)[0].cuda()
    eng.prefill_batch([e0], [0], [0])
    before = _kv(eng, 0, 100, L)
    # table refusals: nothing changes
    for pages, msg in (([0, eng.kv_pages], "outside"), ([1, 1], "twice"), ([2], "mapped to slot 0"), ([-1], "outside")):
        with pytest.raises(EngineError, match=msg):
            eng.map_kv_pages(1, pages)
        assert eng.slot_kv_rows(1) == 0 and eng.slot_kv_rows(0) == 128
    with pytest.raises(EngineError, match="pages outside"):
        eng.map_kv_pages(1, list(range(6, 6 + npt + 1)))
    eng.map_kv_pages(1, [7])
    # work on unmapped rows is refused before anything is launched
    n0 = eng.launch_count
    e1 = O.make_inputs(cfg, 65, 0, seed=3, dtype=torch.bfloat16)[0].cuda()
    with pytest.raises(EngineError, match="map 64 rows"):
        eng.prefill_batch([e1, e1[:40]], [0, 0], [1, 3])          # row 0 needs 65 rows; slot 3 maps none either
    with pytest.raises(EngineError, match="map 0 rows"):
        eng.prefill(e1[:10], slot=2)
    k = torch.zeros(cfg.talker.num_key_value_heads, 65, 128, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(EngineError, match="fq3_import_kv"):
        eng.import_kv(0, k, k, slot=1)
    with pytest.raises(EngineError, match="fq3_export_kv"):
        eng.export_kv(0, 65, slot=1)
    with pytest.raises(EngineError, match="fq3_talker_step"):
        eng.talker_step(e1[0], 64, slot=1)
    assert eng.launch_count == n0
    # a request on slot 1 (40-row prompt, one page): a budget whose frames would write row 64 is refused
    r = _request(cfg, 40, 0, 4, 60, torch.bfloat16, seed=9)
    a = _args(r)
    a.pop("tag")
    begin_fused(eng, p.talker, a.pop("tie"), a.pop("tam"), a.pop("tth"), a.pop("tpe"), p.config, p.pg, p.tg, slot=1,
                temperature=0.9, top_k=50, top_p=1.0, **a)
    n0 = eng.launch_count
    with pytest.raises(EngineError, match="frame budget"):
        eng.decode_chunk(25, slot=1)
    with pytest.raises(EngineError, match="frame budget"):
        eng.decode_chunk_batch([1], [30])
    assert eng.launch_count == n0
    codes, res = eng.decode_chunk(24, slot=1)                     # rows 40..63: allowed
    assert int(res.frames_emitted) == 24
    with pytest.raises(EngineError, match="frame budget"):
        eng.decode_chunk(1, slot=1)
    torch.cuda.synchronize()
    assert torch.equal(_kv(eng, 0, 100, L), before)
    # growing the table keeps the rows of the pages it keeps, and the request goes on
    eng.map_kv_pages(1, [7, 0])
    codes2, res = eng.decode_chunk(8, slot=1)
    assert int(res.frames_emitted) == 8 and torch.equal(_kv(eng, 0, 100, L), before)
    # the same request alone on the default pool
    ref = _pair(monkeypatch, cfg=cfg, seed=1, dtype=torch.bfloat16, max_seq_len=S, max_batch=4)
    a = _args(r)
    a.pop("tag")
    ins = [a.pop(k) for k in ("tie", "tam", "tth", "tpe")]
    want, _ = fast_generate(ref.talker, *ins, ref.config, ref.pg, ref.tg, **a)
    assert torch.equal(torch.cat([codes, codes2]), want[:32])


def test_import_export_and_page_copies_through_a_scattered_table(monkeypatch):
    cfg = O.cfg_tiny()
    S = 256
    p = _pair(monkeypatch, kv_pages=10, cfg=cfg, seed=2, dtype=torch.float32, max_seq_len=S, max_batch=2)
    eng, L = p.engine, cfg.talker.num_hidden_layers
    nkv, P = cfg.talker.num_key_value_heads, 150
    eng.map_kv_pages(1, [8, 3, 6])
    g = torch.Generator().manual_seed(0)
    kv = [(torch.randn(nkv, P, 128, generator=g), torch.randn(nkv, P, 128, generator=g)) for _ in range(L)]
    for l, (k, v) in enumerate(kv):
        eng.import_kv(l, k, v, slot=1)
    for l, (k, v) in enumerate(kv):
        ek, ev = eng.export_kv(l, P, slot=1)
        assert torch.equal(ek.cpu(), k) and torch.equal(ev.cpu(), v), l
    # pages to pinned host memory and device memory and back, into other pages
    host = torch.empty(3, eng.kv_page_bytes, dtype=torch.uint8, pin_memory=True)
    dev = torch.empty(3, eng.kv_page_bytes, dtype=torch.uint8, device="cuda")
    eng.kv_pages_to([8, 3, 6], host)
    eng.kv_pages_to([8, 3, 6], dev)
    torch.cuda.synchronize()
    assert torch.equal(host, dev.cpu())
    eng.kv_pages_from([8, 3, 6], torch.zeros_like(dev))
    assert not torch.equal(eng.export_kv(0, P, slot=1)[0].cpu(), kv[0][0])
    eng.map_kv_pages(1, [0, 9, 4])
    eng.kv_pages_from([0, 9, 4], host)
    for l, (k, v) in enumerate(kv):
        ek, ev = eng.export_kv(l, P, slot=1)
        assert torch.equal(ek.cpu(), k) and torch.equal(ev.cpu(), v), l
    with pytest.raises(EngineError, match="twice"):
        eng.kv_pages_to([1, 1], torch.empty(2, eng.kv_page_bytes, dtype=torch.uint8, device="cuda"))
    with pytest.raises(EngineError, match="outside"):
        eng.kv_pages_from([10], dev[:1])
    with pytest.raises(ValueError):
        eng.kv_pages_to([1], torch.empty(eng.kv_page_bytes, dtype=torch.uint8))   # pageable host memory


TEXTS = ["hello there general kenobi", "a much longer sentence that keeps going for a while so that the prompt lengths differ",
         "short one", "the quick brown fox jumps over the lazy dog"]


@pytest.mark.parametrize("codec_mode", ["window", "stateful"])
def test_serving_under_page_pressure(codec_mode, monkeypatch):
    """ContinuousBatcher on a pool of one request plus 2 pages: four requests whose worst case needs more (one of them
    400 frames past its prompt, more than 384 rows) all complete, requests are parked and restored into other pages, and each request's audio equals
    that of the request served alone on the default pool"""
    monkeypatch.setenv("FQ3_ATTN_SPLIT", "0")
    from faster_qwen3_tts import FasterQwen3TTS
    from faster_qwen3_tts.serving import batcher_for_model, voice_clone_request
    S = 512
    models = {}
    for kv_pages in (0, S // KV_PAGE + 2):
        m = FasterQwen3TTS.from_synthetic("tiny", dtype=torch.bfloat16, max_seq_len=S, seed=5, max_batch=4,
                                          kv_pages=kv_pages)
        m.streaming_codec = codec_mode
        m.predictor_graph.do_sample = False
        models[kv_pages] = m
    ref, paged = models[0], models[S // KV_PAGE + 2]
    frames = [150, 400, 150, 200]   # every request outgrows its share of the pool: all of them stall, some park
    want = []
    for i, text in enumerate(TEXTS):
        gen = dict(max_new_tokens=frames[i], min_new_tokens=frames[i], do_sample=False)
        parts = [pcm for pcm, sr, t in ref.generate_voice_clone_streaming(text, "English", ref_audio="ref.wav",
                                                                          ref_text="ref words", chunk_size=8,
                                                                          xvec_only=(i % 2 == 1), **gen)]
        want.append(np.concatenate(parts))
    moved = []
    real_park, real_restore = B.KvPager.park, B.KvPager.restore

    def park(self, slot, rows):
        self._was = getattr(self, "_was", {})
        self._was[slot] = list(self.mapped.get(slot, []))[: self.pages(rows)]
        return real_park(self, slot, rows)

    def restore(self, slot, host, rows):
        ok = real_restore(self, slot, host, rows)
        if ok:
            moved.append(self.mapped[slot][: host.shape[0]] != self._was[slot])
        return ok
    monkeypatch.setattr(B.KvPager, "park", park)
    monkeypatch.setattr(B.KvPager, "restore", restore)
    b = batcher_for_model(paged, chunk_size=8)
    try:
        tickets = [b.submit(voice_clone_request(paged, text, "English", "ref.wav", "ref words", xvec_only=(i % 2 == 1)),
                            max_new_tokens=frames[i], min_new_tokens=frames[i], do_sample=False)
                   for i, text in enumerate(TEXTS)]
        got = [t.audio() for t in tickets]
    finally:
        b.close()
    for i, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape, i
        assert float(np.abs(g - w).max()) == 0.0, i
    pager = b.sched.pager
    assert b.max_concurrent >= 2
    assert pager.parks > 0 and any(moved), (pager.parks, moved)
    assert sorted(pager.free) == list(range(paged.engine.kv_pages)) and not pager.mapped
