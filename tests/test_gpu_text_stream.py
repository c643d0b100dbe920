"""Incremental text input on the GPU: a request whose trailing text is OPEN (fq3_set_text_rows) is fed its rows between
launches, and the decode kernels stop a slot at the frame that would need a row that has not arrived.  Because the slot
waits instead of running ahead on tts_pad, the model sees exactly the inputs of the one-shot request: its codes are
bit-exact against the oracle on the full rows (fp32) and bit-identical to the same rows latched at once (bf16), for the
single-sequence and the batched kernel, whatever the reveal schedule."""
import numpy as np
import pytest
import torch

from oracle import qwen3_tts_oracle as O

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from util_models import Pair
    from faster_qwen3_tts.batching import BatchScheduler
    from faster_qwen3_tts.engine import EngineError
    from faster_qwen3_tts.generate import begin_fused, fast_generate


def _buffer(tth, max_new, H, dtype):
    buf = torch.zeros(max_new, H, dtype=dtype, device="cuda")
    buf[: tth.shape[0]] = tth.cuda()
    return buf


def _text_fed(p, tie, tth, tpe, n, rng, uniforms, do_sample, n_frames=3, slot=0, check_bound=True):
    """One request through the C ABI: rows revealed 0..3 at a time between launches (some launches starve), then the
    text is closed.  Returns (codes, starved launches)."""
    H = tie.shape[-1]
    buf = _buffer(tth, n, H, p.dtype)
    P = tie.shape[0]
    begin_fused(p.engine, p.talker, tie[None].cuda(), torch.ones(1, P, dtype=torch.long).cuda(), buf[None],
                tpe[None, None].cuda(), p.config, p.pg, p.tg, max_new_tokens=n, min_new_tokens=2, temperature=0.9,
                top_k=50, top_p=1.0, do_sample=do_sample, repetition_penalty=1.05,
                uniforms=None if uniforms is None else torch.from_numpy(uniforms).cuda(), slot=slot, trailing_len=0)
    eng = p.engine
    gen0 = eng.gen_step0[slot]
    Tt, rows, closed, total, starved, parts = tth.shape[0], 0, False, 0, 0, []
    eng.set_text_rows(slot, 0, True)
    while True:
        if not closed:
            rows = min(Tt, rows + int(rng.choice([0, 0, 1, 1, 2, 3])))
            closed = rows == Tt and rng.random() < 0.5
            eng.set_text_rows(slot, rows, not closed)
        codes, res = eng.decode_chunk(n_frames, slot=slot)
        k = int(res.frames_emitted)
        if check_bound and not closed:
            bound = min(n_frames, rows - (gen0 + total))
            if res.finished == 0:
                assert k == bound, (k, bound, rows, total)
            else:
                assert k <= bound
        if res.finished == 0 and k < n_frames:
            starved += 1
        total += k
        if k:
            parts.append(codes.clone().cpu())
        if res.finished:
            break
    return (torch.cat(parts) if parts else torch.zeros(0, 16, dtype=torch.long)), starved


@pytest.mark.parametrize("do_sample", [False, True])
def test_text_fed_fp32_bit_exact_against_oracle(do_sample):
    cfg = O.cfg_tiny()
    p = Pair(cfg, seed=11, dtype=torch.float32, max_seq_len=96, eos_boost=2.0 if do_sample else 1.0)
    p.pg.do_sample = do_sample
    sp_t = O.SamplingParams(do_sample=do_sample, repetition_penalty=1.05)
    sp_p = O.SamplingParams(do_sample=do_sample)
    rng = np.random.default_rng(7)
    starved = 0
    for case, (P, Tt, n) in enumerate([(10, 12, 18), (6, 5, 14), (20, 1, 9), (14, 16, 16)]):
        tie, tth, tpe = O.make_inputs(cfg, P, Tt, seed=30 + case)
        uniforms = rng.random((n + 1, 16), dtype=np.float32) if do_sample else None
        with torch.inference_mode():
            want = O.generate(p.om, tie, tth, tpe, max_new_tokens=n, min_new_tokens=2, sp_talker=sp_t, sp_pred=sp_p,
                              max_seq_len=96, uniforms=uniforms)
        got, s = _text_fed(p, tie, tth, tpe, n, rng, uniforms, do_sample)
        starved += s
        print(f"case {case}: {got.shape[0]} frames (oracle {want.shape[0]}), {s} starved launches")
        assert torch.equal(got, want), case
    assert starved > 0


def test_set_text_rows_refusals():
    cfg = O.cfg_tiny()
    p = Pair(cfg, seed=1, dtype=torch.float32, max_seq_len=64, max_batch=2)
    tie, tth, tpe = O.make_inputs(cfg, 8, 4, seed=1)
    with pytest.raises(EngineError, match="fq3_begin_request"):
        p.engine.set_text_rows(1, 0, True)                   # inactive slot
    buf = _buffer(tth, 8, cfg.talker.hidden_size, torch.float32)
    begin_fused(p.engine, p.talker, tie[None].cuda(), torch.ones(1, 8, dtype=torch.long).cuda(), buf[None],
                tpe[None, None].cuda(), p.config, p.pg, p.tg, max_new_tokens=8, min_new_tokens=2, temperature=0.9,
                top_k=50, top_p=1.0, do_sample=False, repetition_penalty=1.05, uniforms=None, slot=0, trailing_len=2)
    p.engine.set_text_rows(0, 3, True)
    with pytest.raises(EngineError, match="withdrawn"):
        p.engine.set_text_rows(0, 2, True)                   # shrinking
    p.engine.set_text_rows(0, 4, False)
    with pytest.raises(EngineError, match="reopened"):
        p.engine.set_text_rows(0, 4, True)                   # reopening a closed text
    with pytest.raises(EngineError, match="cannot grow"):
        p.engine.set_text_rows(0, 5, False)                  # rows after the end of the text
    p.engine.set_text_rows(0, 4, False)                      # the closing call may be repeated
    with pytest.raises(ValueError, match="exceeds"):
        p.engine.set_text_rows(0, 9, False)                  # beyond the latched buffer
    # no buffer latched: any row is refused by the engine itself
    begin_fused(p.engine, p.talker, tie[None].cuda(), torch.ones(1, 8, dtype=torch.long).cuda(),
                torch.zeros(1, 0, cfg.talker.hidden_size).cuda(), tpe[None, None].cuda(), p.config, p.pg, p.tg,
                max_new_tokens=8, min_new_tokens=2, temperature=0.9, top_k=50, top_p=1.0, do_sample=False,
                repetition_penalty=1.05, uniforms=None, slot=1)
    rc = p.engine.lib.fq3_set_text_rows(p.engine.h, 1, 1, 1)
    assert rc == -1 and b"no trailing text" in p.engine.lib.fq3_last_error()


@pytest.mark.parametrize("size", ["tiny", "1.7B"])
def test_text_fed_bf16_bit_identical_to_rows_latched_at_once(size):
    cfg = O.cfg_tiny() if size == "tiny" else O.cfg_1p7b()
    p = Pair(cfg, seed=4, dtype=torch.bfloat16, max_seq_len=256, eos_boost=1.5,
             oracle_device="cpu" if size == "tiny" else "cuda")
    rng = np.random.default_rng(3)
    cases = [(24, 14, 20), (9, 3, 12)] if size == "tiny" else [(40, 12, 16)]
    for case, (P, Tt, n) in enumerate(cases):
        tie, tth, tpe = O.make_inputs(cfg, P, Tt, seed=50 + case, dtype=torch.bfloat16)
        uniforms = rng.random((n + 1, 16), dtype=np.float32)
        want, _ = fast_generate(p.talker, tie[None].cuda(), torch.ones(1, P, dtype=torch.long).cuda(), tth[None].cuda(),
                                tpe[None, None].cuda(), p.config, p.pg, p.tg, max_new_tokens=n, min_new_tokens=2,
                                do_sample=True, repetition_penalty=1.05, uniforms=torch.from_numpy(uniforms).cuda())
        got, s = _text_fed(p, tie, tth, tpe, n, rng, uniforms, True, n_frames=4)
        print(f"{size} case {case}: {got.shape[0]} frames, {s} starved launches")
        assert torch.equal(got, want.cpu()), case


class _Reveal:
    """A feed whose rows all exist already and are revealed on a schedule (the scheduler's view of a TextFeed)."""

    def __init__(self, rows, schedule):
        self.rows, self.schedule, self.n_rows, self.closed, self.t = rows, schedule, 0, False, 0

    def advance(self):
        k = self.schedule(self.t)
        self.t += 1
        self.n_rows = min(self.rows.shape[0], self.n_rows + k)
        if self.n_rows == self.rows.shape[0] and self.t > 3:
            self.closed = True

    def update(self):
        return self.n_rows


def test_batched_text_fed_rows_bit_identical_to_single_slot_runs():
    cfg = O.cfg_tiny()
    B = 8
    p = Pair(cfg, seed=9, dtype=torch.bfloat16, max_seq_len=160, eos_boost=1.5, max_batch=B)
    rng = np.random.default_rng(12)
    n = 22
    reqs = []
    for b in range(B):
        P, Tt = int(rng.integers(8, 40)), int(rng.integers(2, 16))
        tie, tth, tpe = O.make_inputs(cfg, P, Tt, seed=70 + b, dtype=torch.bfloat16)
        reqs.append((tie, tth, tpe, rng.random((n + 1, 16), dtype=np.float32)))
    kw = dict(max_new_tokens=n, min_new_tokens=2, do_sample=True, repetition_penalty=1.05)
    want = []
    for tie, tth, tpe, u in reqs:
        codes, _ = fast_generate(p.talker, tie[None].cuda(), torch.ones(1, tie.shape[0], dtype=torch.long).cuda(),
                                 tth[None].cuda(), tpe[None, None].cuda(), p.config, p.pg, p.tg,
                                 uniforms=torch.from_numpy(u).cuda(), **kw)
        want.append(codes.cpu())
    schedules = [lambda t: 1, lambda t: 2, lambda t: 0 if t < 12 else 5,    # slot 2 starves for 12 launches
                 lambda t: t % 2, lambda t: 3 if t % 4 == 0 else 0, lambda t: 100, lambda t: 1 if t % 3 else 0,
                 lambda t: int(rng.integers(0, 3))]
    sched = BatchScheduler(p.engine, p.talker, p.config, p.pg, p.tg)
    feeds = []
    for b, (tie, tth, tpe, u) in enumerate(reqs):
        buf = _buffer(tth, n, cfg.talker.hidden_size, torch.bfloat16)
        f = _Reveal(buf[: tth.shape[0]], schedules[b])
        feeds.append(f)
        sched.submit(tie[None].cuda(), torch.ones(1, tie.shape[0], dtype=torch.long).cuda(), buf[None],
                     tpe[None, None].cuda(), tag=b, uniforms=torch.from_numpy(u).cuda(), feed=f, **kw)
    got = {b: [] for b in range(B)}
    launches = starved_launches = 0
    while len(sched):
        for f in feeds:
            f.advance()
        out = sched.step(4)
        launches += 1
        for rq, codes in out:
            got[rq.tag].append(codes.cpu())
            if not rq.finished and codes.shape[0] < 4:
                starved_launches += 1
        assert launches < 500
    print("launches", launches, "slot-launches that stopped for text", starved_launches)
    for b in range(B):
        assert torch.equal(torch.cat(got[b]), want[b]), b


def _model(codec_mode, max_batch=1):
    from faster_qwen3_tts import FasterQwen3TTS
    m = FasterQwen3TTS.from_synthetic("tiny", dtype=torch.bfloat16, max_seq_len=256, seed=8, max_batch=max_batch)
    m.streaming_codec = codec_mode
    m.predictor_graph.do_sample = False
    return m


TEXT = "Hello there, general Kenobi! It's 3 pm; we're streaming text into speech, word by word."


def _splits(text):
    rng = np.random.default_rng(5)
    cuts = sorted(set(int(x) for x in rng.integers(1, len(text), size=15)))
    return {"whole": [text], "chars": list(text),
            "random": [text[a:b] for a, b in zip([0] + cuts, cuts + [len(text)])]}


@pytest.mark.parametrize("codec_mode", ["window", "stateful"])
def test_public_text_streaming_is_split_independent(codec_mode):
    from faster_qwen3_tts.model import _StreamWindow
    from faster_qwen3_tts.text_stream import TextFeed, build_prompt
    m = _model(codec_mode)
    gen = dict(max_new_tokens=40, min_new_tokens=40, do_sample=False, chunk_size=8)
    pushed = []
    make = m._make_window

    def recording(*a, **k):
        w = make(*a, **k)
        push = w.push

        def rec(c):
            pushed[-1].append(c.clone())
            return push(c)
        w.push = rec
        return w
    m._make_window = recording
    pcm = {}
    for name, pieces in _splits(TEXT).items():
        pushed.append([])
        chunks = list(m.generate_custom_voice_text_streaming(iter(pieces), "aiden", "English", **gen))
        for _, sr, tm in chunks:
            assert {"chunk_index", "chunk_steps", "prefill_ms", "decode_ms", "total_steps_so_far", "is_final",
                    "text_wait_ms"} <= set(tm)
        if codec_mode == "window":
            assert [c.shape[0] for c in pushed[-1]] == [8] * 5
        pcm[name] = np.concatenate([c[0] for c in chunks])
        assert pcm[name].shape[0] == 40 * 1920
    for name in pcm:
        assert np.array_equal(pcm[name], pcm["whole"]), name
    m._make_window = make
    if codec_mode == "window":   # the window policy on the same codes in the one-shot chunking
        codes = torch.cat(pushed[0])
        w = _StreamWindow(m, m.speech_tokenizer, None, 8)
        ref = np.concatenate([w.push(codes[i:i + 8])[0] for i in range(0, codes.shape[0], 8)])
        assert np.array_equal(ref, pcm["whole"])
    # the prompt is the one-shot prompt bit for bit; the rows are within one bf16 rounding step of the one-shot rows
    _, _, _, tie1, tam1, tth1, tpe1 = m._prepare_generation_custom(TEXT, "English", "aiden", non_streaming_mode=False)
    feed = TextFeed(m, max_rows=64)
    for piece in _splits(TEXT)["random"]:
        feed.push(piece)
    feed.close()
    tie, tam, tpe = build_prompt(m, feed, language="English", speaker="aiden")
    n = feed.update()
    assert torch.equal(tie, tie1) and torch.equal(tam, tam1) and torch.equal(tpe, tpe1)
    assert n == tth1.shape[1]
    rows, ref = feed.rows[:n].float(), tth1[0].float()
    d = (rows - ref).abs()
    ulp = ref.abs().clamp_min(1e-30) * 2.0 ** -7
    print(f"trailing rows: max|text-fed - one-shot| = {d.max().item():.3e}")
    assert bool((d <= ulp).all())
    assert torch.equal(feed.rows[n - 1], tth1[0, -1])        # the eos row
    # an independent run: the one-shot stream with the text-fed rows latched at once gives the text-fed PCM (so rows
    # written after the latch do reach the kernel)
    ref = np.concatenate([c[0] for c in m.stream_from_embeds(tie, tam, feed.rows[:n][None], tpe, chunk_size=8,
                                                             max_new_tokens=40, min_new_tokens=40, do_sample=False)])
    assert np.array_equal(ref, pcm["whole"])


FED = ("a text that arrives slowly from another thread, piece by piece, so that the request waits for its words "
       "again and again while the others run")


@pytest.mark.parametrize("codec_mode", ["window", "stateful"])
def test_serving_text_fed_ticket_and_cancel(codec_mode, monkeypatch):
    import threading
    import time
    from faster_qwen3_tts.serving import batcher_for_model, custom_voice_text_request
    monkeypatch.setenv("FQ3_ATTN_SPLIT", "0")
    m = _model(codec_mode, max_batch=4)
    gen = dict(max_new_tokens=21, min_new_tokens=21, do_sample=False)
    texts = ["hello there general kenobi", "short one", "the quick brown fox jumps over the lazy dog"]
    want = []
    for t in texts:
        want.append(np.concatenate([c[0] for c in m.generate_custom_voice_streaming(
            t, "aiden", "English", non_streaming_mode=False, chunk_size=8, **gen)]))
    want_fed = np.concatenate([c[0] for c in m.generate_custom_voice_text_streaming(
        iter([FED]), "ryan", "English", chunk_size=8, **gen)])
    b = batcher_for_model(m, chunk_size=8)
    try:
        tt = b.submit_text(custom_voice_text_request(m, "ryan", "English"), **gen)

        def writer():
            words = FED.split(" ")
            for i, w in enumerate(words):
                tt.write(w + (" " if i + 1 < len(words) else ""))
                time.sleep(0.05)
            tt.close()
        th = threading.Thread(target=writer)
        th.start()

        def plain(text):
            def prepare():
                _, _, _, tie, tam, tth, tpe = m._prepare_generation_custom(text, "English", "aiden",
                                                                           non_streaming_mode=False)
                return tie, tam, tth, tpe, None
            return prepare
        tickets = [b.submit(plain(t), **gen) for t in texts]
        got = [t.audio() for t in tickets]
        fed = tt.audio()
        th.join()
        for i, (g, w) in enumerate(zip(got, want)):
            d = float(np.abs(g - w).max())
            print(f"request {i}: max|served - alone| = {d:.3e}")
            assert g.shape == w.shape and d == 0.0, i
        d = float(np.abs(fed - want_fed).max())
        print(f"text-fed ticket: max|served - text-streamed alone| = {d:.3e}")
        assert fed.shape == want_fed.shape == (21 * 1920,) and d == 0.0
        # a client that never closes its text: cancel frees the slot, and a queued fifth request is admitted into it
        hang = [b.submit_text(custom_voice_text_request(m, "ryan", "English"), **gen) for _ in range(4)]
        for h in hang:
            h.write("never closed ")
        deadline = time.time() + 60
        while len(b.sched) < 4 and time.time() < deadline:
            time.sleep(0.01)
        assert len(b.sched) == 4 and not b.sched.has_capacity()
        fifth = b.submit(plain(texts[1]), **gen)
        time.sleep(0.2)
        assert fifth.first_chunk_at is None
        hang[0].cancel()
        out = fifth.audio()
        assert np.array_equal(out, want[1])
        for h in hang[1:]:
            h.cancel()
        for h in hang:
            h.audio()
    finally:
        b.close()
