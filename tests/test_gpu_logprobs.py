"""GPU tests of the per-draw log-probabilities of the decode kernels (fq3_decode_chunk_lp / fq3_sample_logits_lp).

  * nothing changes when they are off: codes of fq3_decode_chunk_lp equal fq3_decode_chunk's bit for bit, single-sequence
    and batched kernel, fp32 and bf16, sampled and greedy;
  * fp32 (logits bit-exact against the oracle): every value within 2e-5 of the float64 log-softmax of the oracle's
    processed row, teacher-forced along the engine's own codes (oracle/logprob_oracle.py), for sampling, greedy,
    top-k = 1 (exactly 0), top-p < 1, the repetition penalty, min_new_tokens suppression and the EOS draw;
  * bf16: batched rows bit-identical to single-sequence runs; the first-token value against its own input row;
  * edges: a text-gated slot writes no row past frames_emitted; rows of slots not in a launch are untouched."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import logprob_oracle as LO
from oracle import qwen3_tts_oracle as O

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from util_models import Pair
    from faster_qwen3_tts.engine import ChunkResult, SamplingParams
    from faster_qwen3_tts.generate import begin_fused, fast_generate

BAR = 2e-5


def _inputs(cfg, P, Tt, seed, dtype):
    e, t, pad = O.make_inputs(cfg, P, Tt, seed=seed, dtype=dtype)
    return e, t, pad, (e[None].cuda(), torch.ones(1, P, dtype=torch.long).cuda(), t[None].cuda(), pad[None, None].cuda())


def _begin(p, args, slot, n, uniforms, **kw):
    skw = dict(max_new_tokens=n, min_new_tokens=2, temperature=0.9, top_k=50, top_p=1.0, do_sample=True,
               repetition_penalty=1.05)
    skw.update(kw)
    with torch.inference_mode():
        begin_fused(p.engine, p.talker, *args, p.config, p.pg, p.tg, uniforms=uniforms, slot=slot, **skw)


def _plain_chunk(engine, slots, n_frames):
    """the existing entry point, called as it is"""
    out = torch.zeros(len(slots), n_frames, 16, dtype=torch.long, device=engine.device)
    res = (ChunkResult * len(slots))()
    rc = engine.lib.fq3_decode_chunk(engine.h, (C.c_int32 * len(slots))(*slots), len(slots), n_frames, out.data_ptr(),
                                     res, engine._stream())
    assert rc == 0
    return out, list(res)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("do_sample", [True, False])
@pytest.mark.parametrize("B", [1, 3])
def test_codes_unchanged_by_logprobs(dtype, do_sample, B):
    cfg = O.cfg_tiny()
    p = Pair(cfg, seed=5, dtype=dtype, max_seq_len=128, eos_boost=2.0, max_batch=4)
    p.pg.do_sample = do_sample
    n = 20
    rng = np.random.default_rng(B)
    reqs = [_inputs(cfg, 8 + 5 * b, 3, 40 + b, dtype)[3] for b in range(B)]
    U = [torch.from_numpy(rng.random((n + 1, 16), dtype=np.float32)).cuda() for _ in range(B)]
    slots = list(range(B))
    got = []
    for with_lp in (False, True):
        for b in range(B):
            _begin(p, reqs[b], b, n, U[b], do_sample=do_sample)
        if with_lp:
            codes, lp, res = p.engine.decode_chunk_batch(slots, n, logprobs=True) if B > 1 else \
                (lambda c, l, r: (c[None], l[None], [r]))(*p.engine.decode_chunk(n, slot=0, logprobs=True))
        else:
            codes, res = _plain_chunk(p.engine, slots, n)
        got.append([codes[j, :res[j].frames_emitted].cpu() for j in range(B)])
        if with_lp:
            for j in range(B):
                assert torch.isfinite(lp[j, :res[j].frames_emitted, 1:]).all()
    for a, b in zip(*got):
        assert torch.equal(a, b)


def _check_against_oracle(p, e, t, pad, args, n, sp_t, min_new, uniforms=None, top_k1=False):
    codes, timing = fast_generate(p.talker, *args, p.config, p.pg, p.tg, max_new_tokens=n, min_new_tokens=min_new,
                                  temperature=sp_t.temperature, top_k=sp_t.top_k, top_p=sp_t.top_p,
                                  do_sample=sp_t.do_sample, repetition_penalty=sp_t.repetition_penalty,
                                  uniforms=None if uniforms is None else torch.from_numpy(uniforms).cuda(),
                                  return_logprobs=True)
    codes = codes.cpu()
    got = timing["logprobs"]
    assert got.shape == codes.shape
    ended_eos = timing["eos_logprob"] is not None
    sp_p = O.SamplingParams(do_sample=p.pg.do_sample, temperature=p.pg.temperature, top_k=p.pg.top_k, top_p=p.pg.top_p)
    nxt = p.config.codec_eos_token_id if ended_eos else int(codes[-1, 0])   # not EOS: column 0 of the last row unused
    with torch.inference_mode():
        first, rows = LO.teacher_forced_logprobs(p.om, e, t, pad, codes, sp_talker=sp_t, sp_pred=sp_p,
                                                 min_new_tokens=min_new, next_token=nxt)
    want = rows.copy()
    want[0, 0] = first
    want[1:, 0] = rows[:-1, 0]
    d = np.abs(got.double().numpy() - want)
    assert d.max() <= BAR, (d.max(), np.unravel_index(d.argmax(), d.shape))
    if ended_eos:
        assert abs(timing["eos_logprob"] - rows[-1, 0]) <= BAR
    if top_k1:
        assert (got == 0).all()
    return codes, timing


@pytest.mark.parametrize("case", ["sample", "greedy", "top_k_1", "top_p", "no_penalty"])
def test_fp32_logprobs_match_float64_oracle(case):
    cfg = O.cfg_tiny()
    p = Pair(cfg, seed=11, dtype=torch.float32, max_seq_len=128, eos_boost=3.0)
    sp_t = O.SamplingParams(do_sample=case != "greedy", repetition_penalty=1.0 if case == "no_penalty" else 1.3)
    if case == "top_k_1":
        sp_t.top_k = 1
        p.pg.top_k = 1
    if case == "top_p":
        sp_t.top_p = 0.8
        p.pg.top_p = 0.7
    p.pg.do_sample = case != "greedy"
    e, t, pad, args = _inputs(cfg, 14, 4, 3, torch.float32)
    n = 24
    u = np.random.default_rng(7).random((n + 1, 16), dtype=np.float32)
    _check_against_oracle(p, e, t, pad, args, n, sp_t, min_new=2, uniforms=u, top_k1=case == "top_k_1")


def test_fp32_min_new_suppression_and_eos_row():
    """EOS is likely (eos_boost) but suppressed for the first 6 frames; the request ends on EOS, whose value is reported
    separately"""
    cfg = O.cfg_tiny()
    p = Pair(cfg, seed=2, dtype=torch.float32, max_seq_len=128, eos_boost=6.0)
    sp_t = O.SamplingParams(do_sample=True, repetition_penalty=1.05)
    e, t, pad, args = _inputs(cfg, 10, 2, 9, torch.float32)
    n = 60
    u = np.random.default_rng(1).random((n + 1, 16), dtype=np.float32)
    codes, timing = _check_against_oracle(p, e, t, pad, args, n, sp_t, min_new=6, uniforms=u)
    assert codes.shape[0] >= 6 and codes.shape[0] < n
    assert timing["eos_logprob"] is not None and timing["eos_logprob"] <= 0.0


def test_fp32_greedy_eos_row():
    cfg = O.cfg_tiny()
    p = Pair(cfg, seed=4, dtype=torch.float32, max_seq_len=128, eos_boost=8.0)
    p.pg.do_sample = False
    sp_t = O.SamplingParams(do_sample=False, repetition_penalty=1.05)
    e, t, pad, args = _inputs(cfg, 12, 2, 5, torch.float32)
    codes, timing = _check_against_oracle(p, e, t, pad, args, 40, sp_t, min_new=3)
    assert timing["eos_logprob"] is not None


def _single_rows(p, reqs, U, n, chunk):
    """each request alone through the single-sequence kernel, raw kernel rows"""
    out = []
    for b, args in enumerate(reqs):
        _begin(p, args, 0, n, U[b])
        rows, codes = [], []
        while True:
            c, lp, res = p.engine.decode_chunk(chunk, slot=0, logprobs=True)
            rows.append(lp.cpu())
            codes.append(c.cpu())
            if res.finished or res.frames_emitted == 0:
                break
        out.append((torch.cat(codes), torch.cat(rows)))
    return out


@pytest.mark.parametrize("B", [2, 8, 32])
def test_bf16_batched_rows_bit_identical_to_single(B):
    cfg = O.cfg_tiny()
    p = Pair(cfg, seed=B, dtype=torch.bfloat16, max_seq_len=128, eos_boost=2.0, max_batch=B)
    n, chunk = 24, 7
    rng = np.random.default_rng(B)
    lens = [int(x) for x in rng.integers(5, 40, size=B)]
    reqs = []
    for b in range(B):
        e, t, pad, _ = _inputs(cfg, lens[b], 3, 100 + b, torch.bfloat16)
        Pm = max(lens)
        tie = torch.zeros(1, Pm, e.shape[1], dtype=torch.bfloat16)
        tam = torch.zeros(1, Pm, dtype=torch.long)
        tie[0, Pm - lens[b]:] = e
        tam[0, Pm - lens[b]:] = 1       # left padding, as the batch builder lays rows out
        reqs.append((tie.cuda(), tam.cuda(), t[None].cuda(), pad[None, None].cuda()))
    U = [torch.from_numpy(rng.random((n + 1, 16), dtype=np.float32)).cuda() for _ in range(B)]
    want = _single_rows(p, reqs, U, n, chunk)
    for b in range(B):
        _begin(p, reqs[b], b, n, U[b])
    got = [([], []) for _ in range(B)]
    live = list(range(B))
    while live:
        codes, lp, res = p.engine.decode_chunk_batch(live, chunk, logprobs=True)
        nxt = []
        for j, s in enumerate(live):
            k = res[j].frames_emitted
            got[s][0].append(codes[j, :k].cpu())
            got[s][1].append(lp[j, :k].cpu())
            if not res[j].finished and k:
                nxt.append(s)
        live = nxt
    for b in range(B):
        gc, gl = torch.cat(got[b][0]), torch.cat(got[b][1])
        wc, wl = want[b]
        assert torch.equal(gc, wc), b
        # every frame below the cache limit has its talker step, so every column is written
        assert torch.equal(gl.view(torch.int32), wl.view(torch.int32)), b


@pytest.mark.parametrize("do_sample", [True, False])
def test_bf16_first_token_value_against_its_input_row(do_sample):
    cfg = O.cfg_tiny()
    p = Pair(cfg, seed=8, dtype=torch.bfloat16, max_seq_len=64)
    V = cfg.talker.vocab_size
    g = torch.Generator().manual_seed(3)
    for trial in range(6):
        lg = (torch.randn(V, generator=g) * 3).to(torch.bfloat16)
        hist = torch.randint(0, 64, (5,), generator=g)
        sp = SamplingParams(do_sample, 50 if trial % 2 else 0, 0.9, 1.0 if trial < 3 else 0.85, 1.2)
        u = float(torch.rand(1, generator=g))
        tok, lp = p.engine.sample_logits(lg.cuda(), sp, u=u, history=hist.cuda(), suppress_special=True,
                                         eos_id=cfg.codec_eos_token_id, suppress_eos=trial % 3 == 0, return_logprob=True)
        tok2 = p.engine.sample_logits(lg.cuda(), sp, u=u, history=hist.cuda(), suppress_special=True,
                                      eos_id=cfg.codec_eos_token_id, suppress_eos=trial % 3 == 0)
        assert int(tok) == int(tok2)
        pen = O.apply_repetition_penalty(lg.clone(), hist, 1.2)
        smask = O.suppress_mask_for(cfg)
        row = LO.processed_row(pen, do_sample=do_sample, temperature=0.9, top_k=sp.top_k, top_p=sp.top_p,
                               suppress_mask=smask, suppress_tokens=[cfg.codec_eos_token_id] if trial % 3 == 0 else None)
        assert abs(float(lp) - LO.logprob64(row, int(tok))) <= BAR, trial


def test_text_gated_slot_writes_nothing_past_frames_emitted():
    cfg = O.cfg_tiny()
    p = Pair(cfg, seed=6, dtype=torch.bfloat16, max_seq_len=128, max_batch=2)
    n = 30
    e, t, pad, args = _inputs(cfg, 10, 12, 21, torch.bfloat16)
    _, _, _, args2 = _inputs(cfg, 14, 3, 22, torch.bfloat16)
    U = torch.rand(n + 1, 16, device="cuda")
    _begin(p, args, 0, n, U, min_new_tokens=n, trailing_len=0)
    _begin(p, args2, 1, n, U)
    p.engine.set_text_rows(0, 4, open=True)      # slot 0 may run 4 frames, then waits for text
    sentinel = -12345.0
    buf = torch.full((2, 10, 16), sentinel, device="cuda")
    codes, lp, res = p.engine.decode_chunk_batch([0, 1], 10, logprobs=buf)
    assert res[0].finished == 0 and res[0].frames_emitted == 4
    assert (buf[0, 4:] == sentinel).all()
    assert (buf[0, :4] != sentinel).all()
    # single-sequence kernel
    p.engine.set_text_rows(0, 6, open=True)
    one = torch.full((10, 16), sentinel, device="cuda")
    c, l, r = p.engine.decode_chunk(10, slot=0, logprobs=one)
    assert r.frames_emitted == 2 and (one[2:] == sentinel).all() and (one[:2] != sentinel).all()


def _lp_chunk(engine, slots, n_frames, lp_ptr):
    """fq3_decode_chunk_lp called as it is, log-probabilities into caller memory at lp_ptr"""
    out = torch.zeros(len(slots), n_frames, 16, dtype=torch.long, device=engine.device)
    res = (ChunkResult * len(slots))()
    rc = engine.lib.fq3_decode_chunk_lp(engine.h, (C.c_int32 * len(slots))(*slots), len(slots), n_frames, out.data_ptr(),
                                        lp_ptr, res, engine._stream())
    assert rc == 0
    return out, list(res)


def test_slots_not_listed_are_untouched():
    """A launch of slots [1, 2] into rows 1..2 of a [4][n][16] buffer leaves rows 0 and 3 (the unlisted slots 0 and 3)
    as they were, and leaves slots 0 and 3 themselves untouched: their next launch writes exactly the rows it writes
    when no other launch came first."""
    cfg = O.cfg_tiny()
    p = Pair(cfg, seed=6, dtype=torch.bfloat16, max_seq_len=128, max_batch=4)
    n = 6
    reqs = [_inputs(cfg, 9 + s, 2, 30 + s, torch.bfloat16)[3] for s in range(4)]
    U = [torch.rand(2 * n + 1, 16, device="cuda") for _ in range(4)]

    def begin_all():
        for s in range(4):
            _begin(p, reqs[s], s, 2 * n, U[s], min_new_tokens=2 * n)

    begin_all()
    want = torch.empty(2, n, 16, device="cuda")
    want_codes, _ = _lp_chunk(p.engine, [0, 3], n, want.data_ptr())
    begin_all()
    sentinel = -777.0
    big = torch.full((4, n, 16), sentinel, device="cuda")
    before = [p.engine.past_hidden(s).clone() for s in (0, 3)]
    _, res = _lp_chunk(p.engine, [1, 2], n, big[1].data_ptr())
    torch.cuda.synchronize()
    assert all(r.frames_emitted == n for r in res)
    assert (big[1:3] != sentinel).all()
    assert (big[0] == sentinel).all() and (big[3] == sentinel).all()
    for s, b in zip((0, 3), before):
        assert torch.equal(p.engine.past_hidden(s), b)
    got = torch.empty(2, n, 16, device="cuda")
    got_codes, _ = _lp_chunk(p.engine, [0, 3], n, got.data_ptr())
    assert torch.equal(got_codes, want_codes)
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))
