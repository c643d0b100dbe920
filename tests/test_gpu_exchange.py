"""The bf16 single-sequence kernel's tagged activation exchange (fq3_decode.cuh xput / xload, DESIGN §4): a launch long
enough to wrap the 16-bit exchange tag decodes exactly what the same request decodes in short launches, whose tags
never come near the wrap."""
import numpy as np
import pytest
import torch

from oracle import qwen3_tts_oracle as O

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from util_models import Pair
    from faster_qwen3_tts.generate import begin_fused


def _exchanges_per_frame(cfg):
    """tagged exchanges of one frame: QKV, O and down of every layer of both stacks, the 15 predictor heads and the
    predictor's input projection (the talker's head keeps its grid barrier)"""
    ncb = cfg.num_code_groups - 1
    return 3 * cfg.talker.num_hidden_layers + ncb * (3 * cfg.predictor.num_hidden_layers + 1) + int(cfg.has_mtp_projection)


def test_bf16_tag_wrap_matches_short_launches():
    cfg = O.cfg_tiny()
    n = 640
    assert n * _exchanges_per_frame(cfg) > 65535 + 1000   # the long launch wraps the tag
    p = Pair(cfg, seed=9, dtype=torch.bfloat16, max_seq_len=1024)
    e, t, pad = O.make_inputs(cfg, 8, 3, seed=21, dtype=torch.bfloat16)
    args = (e[None].cuda(), torch.ones(1, 8, dtype=torch.long).cuda(), t[None].cuda(), pad[None, None].cuda())
    U = torch.from_numpy(np.random.default_rng(3).random((n + 1, 16), dtype=np.float32)).cuda()

    def run(chunk):
        with torch.inference_mode():
            # min_new_tokens = n holds eos back: every launch runs its full budget
            begin_fused(p.engine, p.talker, *args, p.config, p.pg, p.tg, uniforms=U, slot=0, max_new_tokens=n,
                        min_new_tokens=n, temperature=0.9, top_k=50, top_p=1.0, do_sample=True, repetition_penalty=1.05)
        codes, lps = [], []
        while True:
            c, lp, res = p.engine.decode_chunk(chunk, slot=0, logprobs=True)
            codes.append(c.cpu())
            lps.append(lp.cpu())
            if res.finished or res.frames_emitted == 0:
                break
        return torch.cat(codes), torch.cat(lps)

    long_codes, long_lp = run(n)
    short_codes, short_lp = run(8)
    assert long_codes.shape[0] == n
    assert torch.equal(long_codes, short_codes)
    assert torch.equal(long_lp.view(torch.int32), short_lp.view(torch.int32))
