import os, sys, json, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "faster-qwen3-tts_b200")]
from faster_qwen3_tts.model import FasterQwen3TTS
from faster_qwen3_tts.engine import SamplingParams
def timeit(fn, n=20, warm=3):
    for _ in range(warm): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); e1.synchronize()
    return e0.elapsed_time(e1) / n
m = FasterQwen3TTS.from_synthetic("1.7B", dtype=torch.bfloat16, with_codec=False)
eng = m.engine; H = eng.H
x = torch.randn(H, device="cuda").bfloat16()
out = {"env": {k: v for k, v in os.environ.items() if k.startswith("FQ3_")}}
for pos in (300, 400, 500, 700):
    out[f"talker@{pos}"] = round(timeit(lambda: eng.talker_step(x, pos)), 4)
sp = SamplingParams(do_sample=True, top_k=50, temperature=0.9, top_p=1.0, repetition_penalty=1.05)
spp = SamplingParams(do_sample=True, top_k=50, temperature=0.9, top_p=1.0, repetition_penalty=1.0)
def fused(n_chunks, chunk=8, prefill=232):
    eng.begin_request(first_token=5, prefill_len=prefill, gen_step=0, past_hidden=torch.randn(H, device="cuda").bfloat16(),
                      trailing_text=torch.randn(25, H, device="cuda").bfloat16() * 0.02,
                      tts_pad=torch.randn(H, device="cuda").bfloat16() * 0.02, max_new_tokens=4096, min_new_tokens=4096,
                      sp_talker=sp, sp_predictor=spp, uniforms=torch.rand(4097, 16, device="cuda"))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); n = 0
    for _ in range(n_chunks):
        o, res = eng.decode_chunk(chunk); n += o.shape[0]
    e1.record(); e1.synchronize()
    return e0.elapsed_time(e1) / max(n, 1)
fused(2)
out["fused_ms_per_frame"] = round(min(fused(16), fused(16)), 4)
print(json.dumps(out))
