"""The hand-written prefill (K3: fq3_prefill) at its edges, through the C ABI: prompt lengths at and around the 32-key
tiles of the tensor-core attention (1 row up to max_seq_len), left pads that end inside a tile, on a tile boundary and
past whole query blocks (kt_first > 0), GQA ratios 2 and 1 (attn_prefill_mma_kernel<2> and <1>), request slots other
than 0, a slot reused for a shorter prompt, and decode steps on top of a padded native prefill that cross from the
per-head attention to the split attention.

Against the oracle (hosted on the GPU), every tensor is held to the bar of test_split_attention_step_vs_oracle_layerwise:
|engine - bf16 oracle| <= 3 x |bf16 oracle - fp32 oracle on the same bf16 weights| + 1 % of the tensor's range + 1e-3,
i.e. the engine is as close to the bf16 oracle as one valid bf16 evaluation is to another.  K and V are compared at
every layer (rows >= pad), so an error is localised to the layer where it starts.  The invariants are bit for bit."""
import pytest
import torch

from oracle import qwen3_tts_oracle as O

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from util_models import Pair
    from faster_qwen3_tts.weights import engine_for_talker

MAXS = 320
WORST = {}


def _cfg(ratio):
    cfg = O.cfg_tiny()
    if ratio == 1:
        cfg.talker.num_key_value_heads = cfg.talker.num_attention_heads
    return cfg


@pytest.fixture(scope="module", params=[2, 1], ids=["gqa2", "gqa1"])
def tiny(request):
    p = Pair(_cfg(request.param), seed=11, dtype=torch.bfloat16, max_seq_len=MAXS, oracle_device="cuda", max_batch=3)
    p.om32 = O.OracleModel(p.cfg, {k: v.float().cuda() for k, v in p.W.items()})
    p.ratio = request.param
    return p


def _env_check(tag, name, got, ref, ref32):
    got, ref, ref32 = got.float().cpu(), ref.float().cpu(), ref32.float().cpu()
    err = (got - ref).abs().max().item()
    env = (ref - ref32).abs().max().item()
    mag = ref.abs().max().item()
    bar = 3.0 * env + 0.01 * mag + 1e-3
    WORST[tag] = max(WORST.get(tag, 0.0), err / bar)
    assert err <= bar, (tag, name, err, env, mag)


def _prompt(cfg, P, pad, seed):
    tie = O.make_inputs(cfg, P, 1, seed=seed, dtype=torch.bfloat16)[0]
    tie[:pad] = 0
    return tie


def _prefill_vs_oracle(p, P, pad, tag, slot=0):
    cfg = p.cfg
    tie = _prompt(cfg, P, pad, seed=P * 131 + pad)
    with torch.inference_mode():
        lg, ph, cache = p.om.talker_prefill(tie.cuda(), n_left_pad=pad)
        lg32, ph32, cache32 = p.om32.talker_prefill(tie.float().cuda(), n_left_pad=pad)
    elg, eph = p.engine.prefill(tie.cuda(), pad, slot=slot)
    for l in range(cfg.talker.num_hidden_layers):
        k, v = p.engine.export_kv(l, P, slot=slot)
        _env_check(tag, f"K layer {l}", k[:, pad:], cache.k[l][:, pad:], cache32.k[l][:, pad:])
        _env_check(tag, f"V layer {l}", v[:, pad:], cache.v[l][:, pad:], cache32.v[l][:, pad:])
    _env_check(tag, "past_hidden", eph, ph, ph32)
    _env_check(tag, "logits", elg, lg, lg32)
    return tie, cache, cache32


PAD0 = [(P, 0) for P in (1, 2, 31, 32, 33, 65, 300, MAXS)]
PADDED = [(100, pad) for pad in (1, 31, 32, 33, 70, 99)]   # 70: query blocks 0 and 1 lie wholly inside the pad


@pytest.mark.parametrize("P,pad", PAD0 + PADDED, ids=[f"P{P}-pad{pad}" for P, pad in PAD0 + PADDED])
def test_prefill_vs_oracle_tiny(tiny, P, pad):
    _prefill_vs_oracle(tiny, P, pad, f"gqa{tiny.ratio} P{P} pad{pad}")


def test_prefill_vs_oracle_1p7b_padded():
    """the 1.7B geometry with a pad of 40: the first query block lies inside the pad and tile 1 starts masked"""
    p = Pair(O.cfg_1p7b(), seed=3, dtype=torch.bfloat16, max_seq_len=128, oracle_device="cuda")
    p.om32 = O.OracleModel(p.cfg, {k: v.float().cuda() for k, v in p.W.items()})
    _prefill_vs_oracle(p, 100, 40, "1.7B P100 pad40")


def _export(p, slot, P=MAXS):
    return [p.engine.export_kv(l, P, slot=slot) for l in range(p.cfg.talker.num_hidden_layers)]


@pytest.mark.parametrize("k", [1, 2])
def test_pad_by_whole_tiles_is_bit_exact(tiny, k):
    """[32 k zero rows ; prompt] with n_left_pad = 32 k equals the unpadded prompt bit for bit: the attention sees the
    same key tiles in the same order, and every GEMM, norm and RoPE row is computed on its own"""
    cfg = tiny.cfg
    P0, pad = 45, 32 * k
    tie = _prompt(cfg, P0, 0, seed=5)
    padded = torch.cat((torch.zeros(pad, cfg.talker.hidden_size, dtype=tie.dtype), tie))
    lg0, ph0 = tiny.engine.prefill(tie.cuda(), 0, slot=0)
    lg1, ph1 = tiny.engine.prefill(padded.cuda(), pad, slot=1)
    assert torch.equal(lg0, lg1) and torch.equal(ph0, ph1)
    for l, ((k0, v0), (k1, v1)) in enumerate(zip(_export(tiny, 0, P0), _export(tiny, 1, P0 + pad))):
        assert torch.equal(k0, k1[:, pad:]) and torch.equal(v0, v1[:, pad:]), l


def test_prefill_into_other_slots(tiny):
    """a prefill into slot 2 equals the same prefill into slot 0, and leaves the caches of slots 0 and 1 untouched"""
    cfg = tiny.cfg
    a, b = _prompt(cfg, 77, 9, seed=1), _prompt(cfg, 140, 0, seed=2)
    lg0, ph0 = tiny.engine.prefill(a.cuda(), 9, slot=0)
    tiny.engine.prefill(b.cuda(), 0, slot=1)
    before = [_export(tiny, 0), _export(tiny, 1)]
    lg2, ph2 = tiny.engine.prefill(a.cuda(), 9, slot=2)
    assert torch.equal(lg0, lg2) and torch.equal(ph0, ph2)
    for (k0, v0), (k2, v2) in zip(_export(tiny, 0, 77), _export(tiny, 2, 77)):
        assert torch.equal(k0[:, 9:], k2[:, 9:]) and torch.equal(v0[:, 9:], v2[:, 9:])
    for s, want in enumerate(before):
        for l, ((kw, vw), (kg, vg)) in enumerate(zip(want, _export(tiny, s))):
            assert torch.equal(kw, kg) and torch.equal(vw, vg), (s, l)


def test_slot_reused_for_a_shorter_prompt(tiny):
    """a shorter prompt prefilled into a slot that held a longer one gives the logits and the following decode steps of
    a fresh engine: nothing of the longer prompt's cache rows leaks into them"""
    cfg = tiny.cfg
    long_, short = _prompt(cfg, 300, 0, seed=3), _prompt(cfg, 50, 20, seed=4)
    tiny.engine.prefill(long_.cuda(), 0, slot=0)
    fresh = engine_for_talker(tiny.talker, dtype=torch.bfloat16, device="cuda", max_seq_len=MAXS, max_batch=3)
    outs = []
    for eng in (tiny.engine, fresh):
        lg, ph = eng.prefill(short.cuda(), 20, slot=0)
        eng.set_generation_state(20, -20, slot=0)
        g = torch.Generator().manual_seed(6)
        steps = [eng.talker_step((torch.randn(cfg.talker.hidden_size, generator=g) * 0.5).to(torch.bfloat16).cuda(),
                                 50 + s, slot=0).clone() for s in range(4)]
        outs.append((lg.clone(), ph.clone(), steps))
    tiny.engine.set_generation_state(0, 0, slot=0)
    (lg_a, ph_a, st_a), (lg_b, ph_b, st_b) = outs
    assert torch.equal(lg_a, lg_b) and torch.equal(ph_a, ph_b)
    for s, (x, y) in enumerate(zip(st_a, st_b)):
        assert torch.equal(x, y), s


def test_decode_crosses_split_threshold_after_padded_prefill(tiny):
    """P = 280 with pad = 100 leaves 180 keys; 20 teacher-forced talker steps take that to 200.  The split decision
    counts keys from kv_start = pad, so steps 0-11 run the per-head attention and steps 12-19 the split attention"""
    cfg = tiny.cfg
    P, pad = 280, 100
    tag = f"gqa{tiny.ratio} decode P{P} pad{pad}"
    tie, cache, cache32 = _prefill_vs_oracle(tiny, P, pad, tag)
    tiny.engine.set_generation_state(pad, -pad)
    g = torch.Generator().manual_seed(12)
    for s in range(20):
        x = (torch.randn(cfg.talker.hidden_size, generator=g) * 0.5).to(torch.bfloat16)
        with torch.inference_mode():
            ref = tiny.om.talker_step(x.cuda(), P + s, cache, n_left_pad=pad, rope_delta=-pad)
            ref32 = tiny.om32.talker_step(x.float().cuda(), P + s, cache32, n_left_pad=pad, rope_delta=-pad)
        got = tiny.engine.talker_step(x.cuda(), P + s)
        _env_check(tag, f"hidden step {s}", got, ref, ref32)
    tiny.engine.set_generation_state(0, 0)


def test_prefill_report_worst():
    """worst error / bar per prefill case of the oracle comparisons above"""
    print({k: round(v, 3) for k, v in sorted(WORST.items())})
