"""More resident request slots than launch columns, and a frame budget per slot (fq3_config::max_slots,
fq3_decode_chunk_n): an engine holds ``max_slots`` requests and each launch advances at most ``max_batch`` of them, chosen
by the caller, each by its own number of frames.

A request's codes must not depend on any of that: with slot ids of 32 and above, subsets, column positions and budgets that
change from launch to launch, every request is bit-exact against the oracle (fp32) and bit-identical to the same request
run alone through the single-sequence kernel (bf16); a launch leaves the slots it does not list untouched; a slot that used
up its budget resumes unchanged; rows past a budget are not written.  All through the C ABI, tiny geometry."""
import numpy as np
import pytest
import torch

from oracle import qwen3_tts_oracle as O

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from util_models import Pair
    from faster_qwen3_tts.batching import BatchScheduler
    from faster_qwen3_tts.engine import EngineError
    from faster_qwen3_tts.generate import fast_generate

SENTINEL = -7


def _pair(monkeypatch, max_slots, **kw):
    """util_models.Pair on an engine with ``max_slots`` resident slots"""
    import faster_qwen3_tts.weights as Wt
    real = Wt.engine_for_talker
    monkeypatch.setattr(Wt, "engine_for_talker", lambda *a, **k: real(*a, max_slots=max_slots, **k))
    monkeypatch.setenv("FQ3_ATTN_SPLIT", "0")   # a lone bf16 request must take the attention path a batched row takes
    return Pair(**kw)


def _requests(cfg, n, dtype, seed, n_new=14, sample=True):
    """n requests with mixed prompt lengths, each left-padded by its own amount (zeros in the mask = pad rows, which
    also gives the request a non-zero rope delta), own trailing text and uniforms"""
    rng = np.random.default_rng(seed)
    H = cfg.talker.hidden_size
    out = []
    for i in range(n):
        P, Tt, pad = int(rng.integers(5, 30)), int(rng.integers(0, 6)), int(rng.integers(0, 6)) if i % 3 else 0
        e, t, tpe = O.make_inputs(cfg, P, Tt, seed=seed * 1000 + i, dtype=dtype)
        tie = torch.cat([torch.zeros(pad, H, dtype=dtype), e])
        tam = torch.cat([torch.zeros(pad, dtype=torch.long), torch.ones(P, dtype=torch.long)])
        out.append(dict(tie=tie, tam=tam, tth=t, tpe=tpe, pad=pad, n=n_new,
                        u=rng.random((n_new + 1, 16), dtype=np.float32) if sample else None))
    return out


def _submit_args(r, i, sample=True, **kw):
    H = r["tie"].shape[1]
    tth = r["tth"][None].cuda() if r["tth"].shape[0] else torch.zeros(1, 0, H, dtype=r["tie"].dtype).cuda()
    return dict(tie=r["tie"][None].cuda(), tam=r["tam"][None].cuda(), tth=tth, tpe=r["tpe"][None, None].cuda(), tag=i,
                max_new_tokens=r["n"], min_new_tokens=2, do_sample=sample, repetition_penalty=1.05,
                uniforms=None if r["u"] is None else torch.from_numpy(r["u"]).cuda(), **kw)


def _alone(p, r, sample=True):
    a = _submit_args(r, 0, sample)
    a.pop("tag")
    codes, _ = fast_generate(p.talker, a.pop("tie"), a.pop("tam"), a.pop("tth"), a.pop("tpe"), p.config, p.pg, p.tg, **a)
    return codes.cpu() if codes is not None else torch.zeros(0, 16, dtype=torch.long)


def _oracle(p, r, max_seq_len, sample=True):
    nthr = torch.get_num_threads()
    torch.set_num_threads(1)   # tiny tensors: intra-op threads only add synchronisation
    with torch.inference_mode():
        want = O.generate(p.om, r["tie"], r["tth"], r["tpe"], max_new_tokens=r["n"], min_new_tokens=2,
                          sp_talker=O.SamplingParams(do_sample=sample, repetition_penalty=1.05),
                          sp_pred=O.SamplingParams(do_sample=sample), max_seq_len=max_seq_len, uniforms=r["u"],
                          n_left_pad=r["pad"])
    torch.set_num_threads(nthr)
    return want


def _launch(eng, slots, budgets, logprobs=False):
    """one launch with a budget per slot -> {slot: (codes, logprobs or None, result)}; codes / logprobs are the FULL rows
    of buffers pre-filled with a sentinel"""
    n, F = len(slots), max(budgets)
    if n == 1:
        out = torch.full((F, 16), SENTINEL, dtype=torch.long, device="cuda")
        lp = torch.full((F, 16), float(SENTINEL), device="cuda") if logprobs else None
        got = eng.decode_chunk(budgets[0], out=out, slot=slots[0], logprobs=lp)
        return {slots[0]: (out.cpu(), None if lp is None else lp.cpu(), got[-1])}
    out = torch.full((n, F, 16), SENTINEL, dtype=torch.long, device="cuda")
    lp = torch.full((n, F, 16), float(SENTINEL), device="cuda") if logprobs else None
    got = eng.decode_chunk_batch(slots, budgets, out=out, logprobs=lp)
    return {s: (out[j].cpu(), None if lp is None else lp[j].cpu(), got[-1][j]) for j, s in enumerate(slots)}


def _drive(eng, slots, rng, want_len=None, max_cols=32, budget_hi=6, logprobs=False, done=None):
    """every slot to its end in random subsets (in random column order) with random budgets per launch; ``done``: frames
    the slots emitted before.  -> ({slot: codes}, {slot: logprobs}, column positions seen)"""
    live, parts, lparts, cols = list(slots), {s: [] for s in slots}, {s: [] for s in slots}, set()
    done = {s: (done or {}).get(s, 0) for s in slots}
    launches = 0
    while live:
        launches += 1
        k = min(len(live), max_cols if launches % 2 else int(rng.integers(1, max_cols + 1)))   # full launches too
        subset = [int(s) for s in rng.choice(live, size=k, replace=False)]
        budgets = [int(b) for b in rng.integers(1, budget_hi + 1, size=k)]
        for j, (s, (codes, lp, res)) in enumerate(_launch(eng, subset, budgets, logprobs).items()):
            m = int(res.frames_emitted)
            cols.add(j)
            assert m <= budgets[j]
            if want_len is not None:
                assert m == min(budgets[j], want_len[s] - done[s]), (s, m, budgets[j], want_len[s], done[s])
            assert (codes[m:] == SENTINEL).all(), "rows past frames_emitted were written"
            if lp is not None:
                assert (lp[m:] == SENTINEL).all()
                lparts[s].append(lp[:m])
            parts[s].append(codes[:m])
            done[s] += m
            assert int(res.total_frames) == done[s]
            if res.finished:
                live.remove(s)
    return {s: torch.cat(v) for s, v in parts.items()}, {s: torch.cat(v) for s, v in lparts.items() if v}, cols


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_80_resident_requests_in_rotating_subsets(dtype, monkeypatch):
    cfg = O.cfg_tiny()
    S, N = 96, 80
    p = _pair(monkeypatch, N, cfg=cfg, seed=4, dtype=dtype, max_seq_len=S, eos_boost=3.0, max_batch=32)
    eng = p.engine
    assert eng.max_batch == 32 and eng.max_slots == N == eng.lib.fq3_max_slots(eng.h) and eng.lib.fq3_max_batch(eng.h) == 32
    reqs = _requests(cfg, N, dtype, seed=9)
    # bf16: the yardstick is the single-sequence kernel (whose parity with the oracle has its own tests); fp32: the oracle,
    # and the lone run for a sample
    want = [_oracle(p, r, S) if dtype == torch.float32 else _alone(p, r) for r in reqs]
    sched = BatchScheduler(eng, p.talker, p.config, p.pg, p.tg)
    assert sched.capacity() == N
    for i0 in range(0, N, 32):   # bf16: one batched prefill per 32 prompts, into slot ids up to 79
        sched.submit_many([_submit_args(r, i0 + i) for i, r in enumerate(reqs[i0:i0 + 32])])
    assert not sched.has_capacity()
    slot_of = {rq.tag: s for s, rq in sched.active.items()}
    assert sorted(slot_of.values()) == list(range(N))
    want_len = {slot_of[i]: want[i].shape[0] for i in range(N)}
    got, _, cols = _drive(eng, list(range(N)), np.random.default_rng(1), want_len)
    assert cols == set(range(32)), "not every column position occurred"
    bad = [i for i in range(N) if not torch.equal(got[slot_of[i]], want[i])]
    assert not bad, bad
    assert len({w.shape[0] for w in want}) > 1   # requests ended at different frames
    if dtype == torch.float32:
        for i in range(0, N, 9):
            assert torch.equal(_alone(p, reqs[i]), want[i]), i


def test_a_launch_leaves_unlisted_slots_untouched(monkeypatch):
    cfg = O.cfg_tiny()
    S, N = 64, 40
    p = _pair(monkeypatch, N, cfg=cfg, seed=2, dtype=torch.bfloat16, max_seq_len=S, max_batch=4)
    eng = p.engine
    reqs = _requests(cfg, 8, torch.bfloat16, seed=3, n_new=10)
    want = [_alone(p, r) for r in reqs]
    sched = BatchScheduler(eng, p.talker, p.config, p.pg, p.tg)
    sched.free = [0, 33, 5, 39, 1, 36, 2, 34] + [s for s in sched.free if s not in (0, 33, 5, 39, 1, 36, 2, 34)]
    for i0 in (0, 4):
        sched.submit_many([_submit_args(r, i0 + i) for i, r in enumerate(reqs[i0:i0 + 4])])
    slot_of = {rq.tag: s for s, rq in sched.active.items()}
    listed, unlisted = [slot_of[i] for i in (1, 2, 5)], [slot_of[i] for i in (0, 3, 4, 6, 7)]
    assert any(s >= 32 for s in listed) and any(s >= 32 for s in unlisted)
    L = cfg.talker.num_hidden_layers

    def snap(slots):
        return [torch.cat([torch.cat([t.flatten() for t in eng.export_kv(l, S, slot=s)]) for l in range(L)]
                          + [eng.past_hidden(s).flatten()]) for s in slots]

    idle = [s for s in range(N) if s not in slot_of.values()][:4]   # slots nobody ever used
    before = snap(unlisted + idle)
    got = {s: [] for s in slot_of.values()}
    for budgets in ([3, 1, 2], [2, 4, 1]):
        for s, (codes, _, res) in _launch(eng, listed, budgets).items():
            got[s].append(codes[: res.frames_emitted])
    for scalar in (np.int64(2), torch.tensor(1)):   # any integer scalar is one budget for all
        buf, ress = eng.decode_chunk_batch(listed, scalar)
        assert buf.shape[1] == int(scalar)
        for j, s_ in enumerate(listed):
            got[s_].append(buf[j, : ress[j].frames_emitted].cpu())
    torch.cuda.synchronize()
    after = snap(unlisted + idle)
    assert all(torch.equal(a, b) for a, b in zip(before, after))
    # loop state and penalty bitmap of the unlisted slots: they still produce their own codes from frame 0
    rest, _, _ = _drive(eng, list(slot_of.values()), np.random.default_rng(5), max_cols=4,
                        done={s: sum(c.shape[0] for c in v) for s, v in got.items()})
    for i, s in slot_of.items():
        assert torch.equal(torch.cat(got[s] + [rest[s]]), want[i]), i


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_budgets_per_slot_with_open_text_and_logprobs(dtype, monkeypatch):
    """budgets {1, 3, 8, 8, 2, 5} on slot ids up to 39, one slot fed its text (set_text_rows on a slot id >= 32), log-
    probabilities on: the frames and their log-probabilities equal those of launches with one budget for all"""
    cfg = O.cfg_tiny()
    S, N = 96, 40
    p = _pair(monkeypatch, N, cfg=cfg, seed=6, dtype=dtype, max_seq_len=S, eos_boost=1.5, max_batch=8)
    eng = p.engine
    reqs = _requests(cfg, 6, dtype, seed=12, n_new=20)
    order = [35, 2, 39, 7, 33, 0]
    FED = 0   # request 0 (slot 35): its 5 trailing rows arrive two per launch
    H = cfg.talker.hidden_size
    e, t, tpe = O.make_inputs(cfg, 12, 5, seed=77, dtype=dtype)
    reqs[FED].update(tie=e, tam=torch.ones(12, dtype=torch.long), tth=t, tpe=tpe, pad=0)

    class Feed:   # the part of text_stream.TextFeed a scheduler reads
        def __init__(self):
            self.rows = torch.zeros(20, H, dtype=dtype, device="cuda")
            self.n_rows, self.closed = 0, False

        def update(self):
            return self.n_rows

    def run(budgets_of):
        sched = BatchScheduler(eng, p.talker, p.config, p.pg, p.tg)
        sched.free = order + [s for s in sched.free if s not in order]
        feed = Feed()
        feed.rows[:5] = t.cuda()
        args = [_submit_args(r, i) for i, r in enumerate(reqs)]
        args[FED].update(tth=feed.rows[None], feed=feed)
        sched.submit_many(args)
        fed_slot = order[FED]
        gen0 = eng.gen_step0[fed_slot]
        live, codes, lps, launch = list(order), {s: [] for s in order}, {s: [] for s in order}, 0
        emitted = {s: 0 for s in order}
        while live:
            if not feed.closed:
                feed.n_rows = min(5, feed.n_rows + 2)
                feed.closed = feed.n_rows == 5 and launch >= 4
                eng.set_text_rows(fed_slot, feed.n_rows, not feed.closed)
            budgets = budgets_of(live, launch)
            out = _launch(eng, live, budgets, logprobs=True)
            for s, b in zip(list(live), budgets):
                c, lp, res = out[s]
                m = int(res.frames_emitted)
                if s == fed_slot and not feed.closed and not res.finished:
                    assert m == min(b, feed.n_rows - (gen0 + emitted[s])), (m, b, feed.n_rows, emitted[s])
                assert (c[m:] == SENTINEL).all() and (lp[m:] == SENTINEL).all()
                codes[s].append(c[:m])
                lps[s].append(lp[:m])
                emitted[s] += m
                if res.finished:
                    live.remove(s)
            launch += 1
        return {s: torch.cat(v) for s, v in codes.items()}, {s: torch.cat(v) for s, v in lps.items()}

    mixed = {35: 1, 2: 3, 39: 8, 7: 8, 33: 2, 0: 5}
    c_eq, lp_eq = run(lambda live, k: [4] * len(live))
    c_mx, lp_mx = run(lambda live, k: [mixed[s] if k % 2 == 0 else 1 + (s + k) % 7 for s in live])
    for i, s in enumerate(order):
        assert torch.equal(c_eq[s], c_mx[s]), (i, s)
        # column 0 of a request's last frame is the EOS draw, or unwritten when max_new_tokens ended it
        a, b = lp_eq[s], lp_mx[s]
        assert torch.equal(a[:, 1:], b[:, 1:]) and torch.equal(a[:-1, 0], b[:-1, 0]), (i, s)
        want = _oracle(p, reqs[i], S) if dtype == torch.float32 else _alone(p, reqs[i])
        assert torch.equal(c_mx[s], want), (i, s)


def test_takes_on_slot_ids_of_32_and_above(monkeypatch):
    """the takes of one request, latched into slots 34.. by one batched prefill and decoded with log-probabilities
    (fq3_decode_chunk_lp), are the takes the first slots give"""
    from faster_qwen3_tts import FasterQwen3TTS, batching
    monkeypatch.setenv("FQ3_ATTN_SPLIT", "0")
    m = FasterQwen3TTS.from_synthetic("tiny", dtype=torch.bfloat16, max_seq_len=256, seed=8, max_batch=4, max_slots=40)
    gen = dict(max_new_tokens=24, min_new_tokens=2, n_takes=4, seeds=[3, 4, 5, 6])
    text = "Several takes of the same sentence."
    a0, _, s0 = m.generate_custom_voice_takes(text, "ryan", "English", **gen)
    init, used = batching.BatchScheduler.__init__, []

    def high_slots_first(self, *a, **k):
        init(self, *a, **k)
        self.free = self.free[34:] + self.free[:34]
        used.append(self.free[:4])

    monkeypatch.setattr(batching.BatchScheduler, "__init__", high_slots_first)
    a1, _, s1 = m.generate_custom_voice_takes(text, "ryan", "English", **gen)
    assert used == [[34, 35, 36, 37]]
    for i in range(4):
        assert np.array_equal(a0[i], a1[i]) and torch.equal(s0[i]["logprobs"], s1[i]["logprobs"]), i
        assert s0[i]["total_logprob"] == s1[i]["total_logprob"]


def test_refusals_launch_nothing(monkeypatch):
    cfg = O.cfg_tiny()
    p = _pair(monkeypatch, 6, cfg=cfg, seed=1, dtype=torch.float32, max_seq_len=64, max_batch=4)
    eng = p.engine
    reqs = _requests(cfg, 6, torch.float32, seed=2, n_new=6)
    sched = BatchScheduler(eng, p.talker, p.config, p.pg, p.tg)
    for i, r in enumerate(reqs):
        sched.submit(**_submit_args(r, i))
    torch.cuda.synchronize()
    n0 = eng.launch_count
    with pytest.raises(EngineError, match=r"n_slots 5 outside \[1, max_batch=4\]"):
        eng.decode_chunk_batch([0, 1, 2, 3, 4], 2)
    with pytest.raises(EngineError, match=r"slot 6 outside \[0, max_slots=6\)"):
        eng.decode_chunk_batch([0, 6], 2)
    with pytest.raises(EngineError, match=r"slot 6 outside \[0, max_slots=6\)"):
        eng.past_hidden(6)
    with pytest.raises(EngineError, match=r"slot 7 outside \[0, max_slots=6\)"):
        eng.set_text_rows(7, 0, True)
    with pytest.raises(EngineError, match="n_frames must be positive"):
        eng.decode_chunk_batch([0, 1, 2], [2, 0, 2])
    with pytest.raises(EngineError, match="n_frames must be positive"):
        eng.decode_chunk_batch([0, 1], [2, -1])
    with pytest.raises(EngineError, match="n_frames must be positive"):
        eng.decode_chunk(0, out=torch.empty(1, 16, dtype=torch.long, device="cuda"), slot=5)
    with pytest.raises(ValueError, match="3 slots but 2 frame budgets"):
        eng.decode_chunk_batch([0, 1, 2], [2, 2])
    assert eng.launch_count == n0
    # the requests are where they were: they run to the codes of their lone runs
    got, _, _ = _drive(eng, list(range(6)), np.random.default_rng(0), max_cols=4)
    for i, r in enumerate(reqs):
        assert torch.equal(got[i], _oracle(p, r, 64)), i


def test_engine_create_refusals_and_default():
    cfg = O.cfg_tiny()
    from faster_qwen3_tts.engine import Engine, load_library
    from faster_qwen3_tts.weights import stack_config
    from util_models import syn_cfg_from
    syn = syn_cfg_from(cfg)
    kw = dict(talker=stack_config(syn.talker_config), predictor=stack_config(syn.code_predictor_config),
              dtype=torch.float32, max_seq_len=64, codec_eos_token_id=cfg.codec_eos_token_id,
              has_mtp_projection=cfg.has_mtp_projection)
    free0 = torch.cuda.mem_get_info()[0]
    with pytest.raises(EngineError, match="max_slots 3 is smaller than max_batch 4"):
        Engine(max_batch=4, max_slots=3, **kw)
    with pytest.raises(EngineError, match="max_slots 257 exceeds 256"):
        Engine(max_batch=4, max_slots=257, **kw)
    with pytest.raises(EngineError, match="max_slots -1 is smaller"):
        Engine(max_batch=1, max_slots=-1, **kw)
    assert torch.cuda.mem_get_info()[0] == free0   # refused before any allocation
    e = Engine(max_batch=4, **kw)                  # max_slots = 0 in the C struct
    assert e.max_slots == 4 == load_library().fq3_max_slots(e.h) == load_library().fq3_max_batch(e.h)
    e1 = Engine(max_batch=1, max_slots=3, **kw)    # several resident requests on the single-sequence kernel
    assert (e1.max_batch, e1.max_slots) == (1, 3)


TEXTS = ["hello there general kenobi", "a much longer sentence that keeps going for a while so that the prompt lengths differ",
         "short one", "the quick brown fox jumps over the lazy dog"]


@pytest.mark.parametrize("codec_mode", ["window", "stateful"])
def test_48_paced_listeners_on_32_columns_hear_what_they_would_alone(codec_mode, monkeypatch):
    """serving.ContinuousBatcher on the real engine, 48 real-time listeners on a clock that runs 50 x faster than the wall:
    more requests than a launch carries, launches chosen by lead, listeners held at the watermark -- and every listener's
    PCM is that of its request streamed alone (window policy: same chunk_size; stateful codec: any chunking, so with a
    short first chunk)."""
    import time
    from faster_qwen3_tts import FasterQwen3TTS
    from faster_qwen3_tts.serving import batcher_for_model, voice_clone_request
    monkeypatch.setenv("FQ3_ATTN_SPLIT", "0")
    m = FasterQwen3TTS.from_synthetic("tiny", dtype=torch.bfloat16, max_seq_len=512, seed=5, max_batch=32, max_slots=48)
    m.streaming_codec = codec_mode
    m.predictor_graph.do_sample = False
    gen = dict(max_new_tokens=21, min_new_tokens=21, do_sample=False)
    variants = [(text, xvec) for text in TEXTS for xvec in (True, False)]
    want = {}
    for text, xvec in variants:
        parts = [pcm for pcm, _, _ in m.generate_voice_clone_streaming(text, "English", ref_audio="ref.wav", ref_text="ref words",
                                                                       chunk_size=8, xvec_only=xvec, **gen)]
        want[(text, xvec)] = np.concatenate(parts)
    t0 = time.monotonic()
    b = batcher_for_model(m, chunk_size=8, lead_high_s=0.5, clock=lambda: (time.monotonic() - t0) * 50)
    extra = dict(first_chunk=2) if codec_mode == "stateful" else {}
    try:
        tickets = [b.submit(voice_clone_request(m, *variants[k % 8][:1], "English", "ref.wav", "ref words",
                                                xvec_only=variants[k % 8][1]), pace=1.0, **gen, **extra) for k in range(48)]
        got = [t.audio() for t in tickets]
    finally:
        b.close()
    assert b.max_concurrent > 32, "never more resident requests than columns"
    for k, g in enumerate(got):
        w = want[variants[k % 8]]
        assert g.shape == w.shape and np.array_equal(g, w), k
    assert all(t.frames == 21 for t in tickets)


def test_a_tickets_own_chunk_size_under_the_window_policy(monkeypatch):
    """the window policy's audio depends on the chunk size (it calibrates once max(25, chunk_size) frames exist): a ticket
    with its own chunk_size, served next to tickets with the batcher's, gets the PCM of the streaming call with that size"""
    from faster_qwen3_tts import FasterQwen3TTS
    from faster_qwen3_tts.serving import batcher_for_model, voice_clone_request
    monkeypatch.setenv("FQ3_ATTN_SPLIT", "0")
    m = FasterQwen3TTS.from_synthetic("tiny", dtype=torch.bfloat16, max_seq_len=512, seed=5, max_batch=4, max_slots=8)
    m.streaming_codec = "window"
    m.predictor_graph.do_sample = False
    gen = dict(max_new_tokens=70, min_new_tokens=70, do_sample=False)
    sizes = [8, 28, 30, 8, 28, 12]
    want = []
    for i, cs in enumerate(sizes):
        parts = [pcm for pcm, _, _ in m.generate_voice_clone_streaming(TEXTS[i % 4], "English", ref_audio="ref.wav",
                                                                       ref_text="ref words", chunk_size=cs,
                                                                       xvec_only=(i % 2 == 0), **gen)]
        want.append(np.concatenate(parts))
    b = batcher_for_model(m, chunk_size=8)
    try:
        tickets = [b.submit(voice_clone_request(m, TEXTS[i % 4], "English", "ref.wav", "ref words", xvec_only=(i % 2 == 0)),
                            **gen, **({} if cs == 8 else {"chunk_size": cs})) for i, cs in enumerate(sizes)]
        chunks = [list(t) for t in tickets]
    finally:
        b.close()
    assert b.max_concurrent > 4
    for i, (cs, ch) in enumerate(zip(sizes, chunks)):
        assert [c[2]["chunk_steps"] for c in ch][:2] == [cs, cs], i
        g = np.concatenate([c[0] for c in ch])
        assert g.shape == want[i].shape and np.array_equal(g, want[i]), (i, cs)
