"""Batched prefill (fq3_prefill_batch / Engine.prefill_batch): several prompts of mixed lengths and left pads into
non-consecutive request slots with one chain of launches.  For every listed slot the K/V cache of every layer, the logits
and past_hidden are bit-identical to fq3_prefill of the same prompt into the same slot on the same engine (the attention
aligns query blocks and key tiles to each prompt's own row 0); slots not listed keep their caches; a call whose rows
fit max_seq_len costs the launches of one fq3_prefill, a longer one runs in groups; refused calls change no slot.
End to end: the batched streaming driver and the continuous batcher admit a burst with one batched prefill and produce
what the same requests produce admitted one at a time."""
import ctypes as C
import threading

import numpy as np
import pytest
import torch

from oracle import qwen3_tts_oracle as O

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from util_models import Pair
    from faster_qwen3_tts.engine import EngineError

MAXS = 320
NSLOT = 8


def _cfg(ratio):
    cfg = O.cfg_tiny()
    if ratio == 1:
        cfg.talker.num_key_value_heads = cfg.talker.num_attention_heads
    return cfg


@pytest.fixture(scope="module", params=[2, 1], ids=["gqa2", "gqa1"])
def tiny(request):
    return Pair(_cfg(request.param), seed=13, dtype=torch.bfloat16, max_seq_len=MAXS, max_batch=NSLOT)


def _prompt(cfg, P, pad, seed):
    tie = O.make_inputs(cfg, P, 1, seed=seed, dtype=torch.bfloat16)[0]
    tie[:pad] = 0
    return tie.cuda()


def _snapshot(p, slots=range(NSLOT)):
    L = p.cfg.talker.num_hidden_layers
    return {s: [tuple(t.clone() for t in p.engine.export_kv(l, p.engine.max_seq_len, slot=s)) for l in range(L)] for s in slots}


def _same(a, b):
    return a.keys() == b.keys() and all(torch.equal(x[0], y[0]) and torch.equal(x[1], y[1])
                                        for s in a for x, y in zip(a[s], b[s]))


def _check_bit_exact(p, specs, seed0=0):
    """specs: (P, pad, slot); single prefills first, the slots clobbered, then one batched call"""
    L = p.cfg.talker.num_hidden_layers
    prompts = [_prompt(p.cfg, P, pad, seed=seed0 + i) for i, (P, pad, _) in enumerate(specs)]
    want = []
    for x, (P, pad, s) in zip(prompts, specs):
        lg, ph = p.engine.prefill(x, pad, slot=s)
        kv = [tuple(t.clone() for t in p.engine.export_kv(l, P, slot=s)) for l in range(L)]
        want.append((lg.clone(), ph.clone(), kv))
    for i, (_, _, s) in enumerate(specs):   # other contents, so that the batched call has to write every row again
        p.engine.prefill(_prompt(p.cfg, p.engine.max_seq_len, 0, seed=999 + i), 0, slot=s)
    listed = {s for _, _, s in specs}
    others = _snapshot(p, [s for s in range(p.engine.max_batch) if s not in listed])
    lg, ph = p.engine.prefill_batch(prompts, [pad for _, pad, _ in specs], [s for _, _, s in specs])
    for b, ((P, pad, s), (wl, wh, wkv)) in enumerate(zip(specs, want)):
        assert torch.equal(lg[b], wl) and torch.equal(ph[b], wh), (b, P, pad, s)
        for l, (k, v) in enumerate(wkv):
            gk, gv = p.engine.export_kv(l, P, slot=s)
            assert torch.equal(gk[:, pad:], k[:, pad:]) and torch.equal(gv[:, pad:], v[:, pad:]), (b, P, pad, s, l)
    assert _same(others, _snapshot(p, others.keys())), "a slot that was not listed changed"


# (P, pad, slot): lengths at and around the 32-row tiles, pads inside a tile, on a boundary and past whole query blocks,
# slots non-consecutive and out of order
FITS = [(33, 32, 5), (1, 0, 0), (100, 70, 3), (31, 9, 6)]                  # 165 rows: one group
GROUPS = [(300, 9, 2), (32, 0, 7), (1, 0, 0), (100, 70, 5), (31, 9, 3), (33, 32, 1), (200, 70, 4)]   # groups of 300,
# 197 and 200 rows (max_seq_len 320)


def test_batch_is_bit_exact_to_single_prefills(tiny):
    _check_bit_exact(tiny, FITS, seed0=10)


def test_batch_over_max_seq_len_runs_in_groups_bit_exact(tiny):
    _check_bit_exact(tiny, GROUPS, seed0=20)


def test_left_padded_batch_tensor_is_packed_by_reshape(tiny):
    """a [B,P,H] left-padded batch (the reference's prompt layout) equals the same rows passed as a list"""
    cfg = tiny.cfg
    x = torch.stack([_prompt(cfg, 40, pad, seed=40 + pad) for pad in (0, 7, 33)])
    a = tiny.engine.prefill_batch(x, [0, 7, 33], [4, 1, 6])
    b = tiny.engine.prefill_batch(list(x), [0, 7, 33], [4, 1, 6])
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_one_group_costs_the_launches_of_one_prefill(tiny):
    e = tiny.engine
    x = _prompt(tiny.cfg, 50, 0, seed=1)
    n0 = e.launch_count
    e.prefill(x, 0, slot=0)
    single = e.launch_count - n0
    prompts = [_prompt(tiny.cfg, P, pad, seed=i) for i, (P, pad, _) in enumerate(FITS)]
    n0 = e.launch_count
    e.prefill_batch(prompts, [pad for _, pad, _ in FITS], [s for _, _, s in FITS])
    assert e.launch_count - n0 == single
    prompts = [_prompt(tiny.cfg, P, pad, seed=i) for i, (P, pad, _) in enumerate(GROUPS)]
    n0 = e.launch_count
    e.prefill_batch(prompts, [pad for _, pad, _ in GROUPS], [s for _, _, s in GROUPS])
    assert e.launch_count - n0 == 3 * single


def test_refusals_change_no_slot(tiny):
    e, cfg = tiny.engine, tiny.cfg
    H = cfg.talker.hidden_size
    for s in range(NSLOT):
        e.prefill(_prompt(cfg, 60, 0, seed=70 + s), 0, slot=s)
    before = _snapshot(tiny)
    a, b = _prompt(cfg, 20, 0, seed=1), _prompt(cfg, 30, 3, seed=2)
    cases = [
        (EngineError, "slot 2 listed twice", lambda: e.prefill_batch([a, b], [0, 3], [2, 2])),
        (EngineError, r"slot 8 outside \[0, max_batch=8\) \(row 1\)", lambda: e.prefill_batch([a, b], [0, 3], [1, 8])),
        (EngineError, r"empty prompt \(row 1\)", lambda: e.prefill_batch([a, a[:0]], [0, 0], [1, 2])),
        (RuntimeError, "Input is too long: prefill has 321 tokens but max_seq_len=320",
         lambda: e.prefill_batch([a, _prompt(cfg, MAXS + 1, 0, seed=3)], [0, 0], [1, 2])),
        (EngineError, "n 0 outside", lambda: e.prefill_batch([], [], [])),
        (EngineError, "n 9 outside", lambda: e.prefill_batch([a] * 9, [0] * 9, list(range(9)))),
    ]
    for exc, msg, call in cases:
        with pytest.raises(exc, match=msg):
            call()
        torch.cuda.synchronize()
        assert _same(before, _snapshot(tiny)), msg
    # misaligned logits, through the C ABI
    x = torch.cat([a, b])
    logits = torch.empty(2 * cfg.talker.vocab_size + 8, dtype=torch.bfloat16, device="cuda")
    hidden = torch.empty(2, H, dtype=torch.bfloat16, device="cuda")
    arr = C.c_int32 * 2
    rc = e.lib.fq3_prefill_batch(e.h, 2, arr(1, 2), x.data_ptr(), arr(20, 30), arr(0, 3), logits.data_ptr() + 2,
                                 hidden.data_ptr(), e._stream())
    assert rc == -1 and b"16-byte aligned" in e.lib.fq3_last_error()
    torch.cuda.synchronize()
    assert _same(before, _snapshot(tiny))


def test_batch_is_bit_exact_1p7b():
    p = Pair(O.cfg_1p7b(), seed=3, dtype=torch.bfloat16, max_seq_len=256, max_batch=4)
    _check_bit_exact(p, [(100, 40, 2), (17, 0, 0), (64, 5, 3)], seed0=30)


# ---- end to end --------------------------------------------------------------------------------------------------
def test_streaming_batch_equals_rows_admitted_one_submit_at_a_time():
    from faster_qwen3_tts.batching import BatchScheduler, fast_generate_streaming_batch
    cfg = O.cfg_tiny()
    p = Pair(cfg, seed=4, dtype=torch.bfloat16, max_seq_len=160, max_batch=4)
    p.pg.do_sample = False
    lens, Tts = [40, 12, 33, 27], [3, 1, 5, 2]
    H = cfg.talker.hidden_size
    tie, tam, tth = torch.zeros(4, 40, H, dtype=torch.bfloat16), torch.zeros(4, 40, dtype=torch.long), None
    tths = []
    for b, (P, Tt) in enumerate(zip(lens, Tts)):   # left-padded like the reference's batch builder (model.py:774-787)
        e, t, tpe = O.make_inputs(cfg, P, Tt, seed=8 + b, dtype=torch.bfloat16)
        tie[b, 40 - P:], tam[b, 40 - P:] = e, 1
        tths.append(torch.cat([t, tpe[None].expand(5 - Tt, H)]))
    tie, tam, tth, tpe = tie.cuda(), tam.cuda(), torch.stack(tths).cuda(), tpe[None, None].cuda()
    kw = dict(max_new_tokens=16, min_new_tokens=2, do_sample=False, repetition_penalty=1.05)
    calls = []
    orig = p.engine.prefill_batch
    p.engine.prefill_batch = lambda rows, pads, slots: (calls.append(list(slots)), orig(rows, pads, slots))[1]
    got = [[] for _ in range(4)]
    for items in fast_generate_streaming_batch(p.talker, tie, tam, tth, tpe, p.config, p.pg, p.tg, chunk_size=8, **kw):
        for b, codes, _ in items:
            got[b].append(codes.cpu())
    assert calls == [[0, 1, 2, 3]]
    sched = BatchScheduler(p.engine, p.talker, p.config, p.pg, p.tg)
    for b in range(4):
        sched.submit(tie[b:b + 1], tam[b:b + 1], tth[b:b + 1], tpe, tag=b, **kw)
    want = [[] for _ in range(4)]
    while len(sched):
        for rq, codes in sched.step(8):
            want[rq.tag].append(codes.cpu())
    for b in range(4):
        assert torch.equal(torch.cat(got[b]), torch.cat(want[b])), b


TEXTS = ["hello there general kenobi", "a much longer sentence that keeps going for a while so that the prompt lengths differ",
         "short one", "the quick brown fox jumps over the lazy dog"]


def test_continuous_batcher_admits_a_burst_with_one_batched_prefill(monkeypatch):
    monkeypatch.setenv("FQ3_ATTN_SPLIT", "0")   # as in test_gpu_serving.py: both sides stay on the per-head attention
    from faster_qwen3_tts import FasterQwen3TTS
    from faster_qwen3_tts.serving import ContinuousBatcher, batcher_for_model, voice_clone_request
    m = FasterQwen3TTS.from_synthetic("tiny", dtype=torch.bfloat16, max_seq_len=512, seed=5, max_batch=4)
    assert m.engine.has_prefill
    m.predictor_graph.do_sample = False
    gen = dict(max_new_tokens=21, min_new_tokens=21, do_sample=False)
    want = []
    for i, text in enumerate(TEXTS):
        parts = [pcm for pcm, sr, t in m.generate_voice_clone_streaming(text, "English", ref_audio="ref.wav", ref_text="ref words",
                                                                        chunk_size=8, xvec_only=(i % 2 == 0), **gen)]
        want.append(np.concatenate(parts))
    calls = []
    orig = m.engine.prefill_batch
    monkeypatch.setattr(m.engine, "prefill_batch", lambda rows, pads, slots: (calls.append(list(slots)), orig(rows, pads, slots))[1])
    gate = threading.Event()
    admit = ContinuousBatcher._admit
    monkeypatch.setattr(ContinuousBatcher, "_admit", lambda self: (gate.wait(), admit(self))[1])
    b = batcher_for_model(m, chunk_size=8)
    try:
        tickets = [b.submit(voice_clone_request(m, text, "English", "ref.wav", "ref words", xvec_only=(i % 2 == 0)), **gen)
                   for i, text in enumerate(TEXTS)]
        gate.set()
        got = [t.audio() for t in tickets]
    finally:
        gate.set()
        b.close()
    assert calls == [[0, 1, 2, 3]], calls
    for i, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape and float(np.abs(g - w).max()) == 0.0, i
