"""GPU tests of the code predictor's per-pass chain in the decode kernels: the predictor attention at every cache
position, the block sampler under every filter combination, and the per-pass input rows.

  * fp32 (bit-exact against the oracle): all 15 predictor passes of a frame (cache slots 0..16, i.e. every position a
    predictor attention runs at) for greedy decoding and for sampling with top-k off (0), top-k = V, top-k < V, top-p < 1
    alone and together with top-k, and a temperature above 1;
  * the sampler on its own (fq3_sample_logits_lp, the `sample_block` both decode kernels run) at the predictor's and the
    talker's vocabulary sizes: the drawn id equals the oracle's draw, and the log-probability is within 2e-5 of the
    float64 log-softmax of the oracle's processed row, greedy included;
  * bf16: rows of the batched kernel bit-identical to the single-sequence kernel (codes and log-probabilities) under the
    same sampler settings."""
import numpy as np
import pytest
import torch

from oracle import logprob_oracle as LO
from oracle import qwen3_tts_oracle as O

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from util_models import Pair
    from faster_qwen3_tts.batching import fast_generate_batch
    from faster_qwen3_tts.engine import SamplingParams
    from faster_qwen3_tts.generate import fast_generate

# (do_sample, temperature, top_k, top_p); the tiny predictor's vocabulary is 256
SAMPLERS = {
    "greedy": (False, 1.0, 0, 1.0),
    "topk50": (True, 0.9, 50, 1.0),
    "topk0": (True, 0.9, 0, 1.0),
    "topkV": (True, 0.9, 256, 1.0),
    "topp": (True, 0.9, 0, 0.8),
    "topk_topp": (True, 0.7, 20, 0.6),
    "hot": (True, 1.3, 5, 1.0),
}


@pytest.fixture(scope="module")
def tiny32():
    return Pair(O.cfg_tiny(), seed=11, dtype=torch.float32, max_seq_len=64)


@pytest.mark.parametrize("name", list(SAMPLERS))
def test_predictor_every_position_fp32_vs_oracle(tiny32, name):
    p = tiny32
    do_sample, T, k, tp = SAMPLERS[name]
    bad = []
    for case in range(4):
        g = torch.Generator().manual_seed(100 + case)
        ph = torch.randn(p.cfg.talker.hidden_size, generator=g)
        tok = [3, 41, 200, 299][case]
        emb = p.W["talker.model.codec_embedding.weight"][tok]
        u = np.random.default_rng(case).random(15, dtype=np.float32)
        with torch.inference_mode():
            ref = p.om.predictor_frame(ph, emb, O.SamplingParams(do_sample=do_sample, temperature=T, top_k=k, top_p=tp),
                                       uniforms=u if do_sample else None)
        got = p.engine.predictor_run(torch.stack((ph, emb)).cuda(),
                                     SamplingParams(do_sample=do_sample, temperature=T, top_k=k, top_p=tp),
                                     torch.from_numpy(u).cuda() if do_sample else None).tolist()
        if got != ref:
            bad.append((case, got, ref))
    assert not bad, bad


@pytest.mark.parametrize("V", [2048, 3072])
@pytest.mark.parametrize("name", list(SAMPLERS))
def test_sampler_draw_and_logprob_fp32_vs_oracle(tiny32, V, name):
    p = tiny32
    do_sample, T, k, tp = SAMPLERS[name]
    if k == 256:
        k = V
    g = torch.Generator().manual_seed(V + len(name))
    rng = np.random.default_rng(V)
    bad = []
    for r in range(12):
        lg = torch.randn(V, generator=g) * (1.0 + r % 4)
        if r % 3 == 0:
            lg[torch.randint(0, V, (7,), generator=g)] = lg.max()   # ties at the top
        u = float(rng.random(dtype=np.float32))
        want = O.sample_token(lg, temperature=T, top_k=k, top_p=tp, do_sample=do_sample, u=u)
        tok, lp = p.engine.sample_logits(lg.cuda(), SamplingParams(do_sample=do_sample, temperature=T, top_k=k, top_p=tp),
                                         u=u, return_logprob=True)
        row = LO.processed_row(lg, do_sample=do_sample, temperature=T, top_k=k, top_p=tp)
        ref_lp = LO.logprob64(row, want)
        # top-p: the kernel accumulates the sorted probabilities one by one in fp32, the oracle's processed row with
        # torch.cumsum; a probability at the nucleus edge can land on either side, which moves the normaliser by that
        # probability (the draw itself follows the engine's rule and is compared exactly)
        bar = 2e-5 if tp >= 1.0 else 2e-3
        if int(tok.item()) != want or abs(float(lp.item()) - ref_lp) > bar:
            bad.append((r, int(tok.item()), want, float(lp.item()), ref_lp))
    assert not bad, bad


@pytest.mark.parametrize("name", ["greedy", "topk0", "topkV", "topp", "topk_topp"])
def test_bf16_batched_rows_match_single_sequence_across_samplers(name):
    do_sample, T, k, tp = SAMPLERS[name]
    cfg = O.cfg_tiny()
    B = 4
    p = Pair(cfg, seed=3, dtype=torch.bfloat16, max_seq_len=96, eos_boost=2.0, max_batch=B)
    # the predictor draws with the same settings as the talker (its vocabulary is 256: topkV is top-k = V there)
    p.pg.do_sample, p.pg.temperature, p.pg.top_k, p.pg.top_p = do_sample, T, k, tp
    rng = np.random.default_rng(7)
    n = 12
    uniforms = rng.random((B, n + 1, 16), dtype=np.float32)
    kw = dict(max_new_tokens=n, min_new_tokens=2, do_sample=do_sample, temperature=T, top_k=k, top_p=tp,
              repetition_penalty=1.05, return_logprobs=True)
    P = 14
    reqs = [O.make_inputs(cfg, P, 3, seed=20 + b, dtype=torch.bfloat16) for b in range(B)]
    tie = torch.stack([e for e, _, _ in reqs])
    tth = torch.stack([t for _, t, _ in reqs])
    tpe = reqs[0][2]
    tam = torch.ones(B, P, dtype=torch.long)
    want = []
    for b in range(B):
        codes, tm = fast_generate(p.talker, tie[b:b + 1].cuda(), tam[b:b + 1].cuda(), tth[b:b + 1].cuda(),
                                  tpe[None, None].cuda(), p.config, p.pg, p.tg,
                                  uniforms=torch.from_numpy(uniforms[b]).cuda(), **kw)
        want.append((codes.cpu(), tm["logprobs"].cpu()))
    got, tm = fast_generate_batch(p.talker, tie.cuda(), tam.cuda(), tth.cuda(), tpe[None, None].cuda(), p.config, p.pg,
                                  p.tg, uniforms=torch.from_numpy(uniforms).cuda(), launch_frames=5, **kw)
    for b in range(B):
        assert torch.equal(got[b].cpu(), want[b][0]), b
        assert torch.equal(tm["logprobs"][b].cpu(), want[b][1]), b
