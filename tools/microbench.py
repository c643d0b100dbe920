#!/usr/bin/env python3
"""GPU micro-benchmarks of the persistent kernel's pieces (needs one GPU; prints one line per measurement)."""
import os, sys, time, json
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "faster-qwen3-tts_b200")]
import torch
from faster_qwen3_tts import synthetic
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

size = sys.argv[1] if len(sys.argv) > 1 else "1.7B"
ctas = int(sys.argv[2]) if len(sys.argv) > 2 else 0
m = FasterQwen3TTS.from_synthetic(size, dtype=torch.bfloat16, with_codec=False, num_ctas=ctas)
eng = m.engine
H = eng.H
x = torch.randn(H, device="cuda").bfloat16()
tb, pb = eng.tape_bytes()
for pos in (16, 256, 1024, 2000):
    ms = timeit(lambda: eng.talker_step(x, pos))
    print(json.dumps({"what": "talker_step", "size": size, "ctas": eng.num_ctas, "pos": pos, "ms": ms, "GBps": tb / ms / 1e6}))
pi = torch.randn(2, H, device="cuda").bfloat16()
u = torch.rand(15, device="cuda")
for ds in (False, True):
    ms = timeit(lambda: eng.predictor_run(pi, SamplingParams(do_sample=ds), u))
    print(json.dumps({"what": "predictor_run", "do_sample": ds, "ms": ms, "GBps": pb / ms / 1e6}))

# ---- phase timeline of CTA 0 (clock64 probes)
names = ["norm_in", "gemv_qkv", "B1", "attn", "B2", "gemv_o(+load)", "B3", "norm+gemv_gu", "B4", "gemv_dn(+load)", "B5"]
def timeline(label, fn, L):
    eng.debug_enable(2)
    fn(); torch.cuda.synchronize()
    ts = eng.probe_timestamps(12 * L).double()
    eng.debug_enable(0)
    ts = ts.view(L, 12)
    d = (ts[:, 1:] - ts[:, :-1]) / 1.965e3  # us at 1965 MHz
    segs = ["norm_in", "gemv_qkv", "B1", "attn", "B2", "load+gemv_o", "B3", "norm+gemv_gu", "B4", "load+gemv_dn", "B5"]
    avg = d[1:].mean(0) if L > 1 else d.mean(0)
    print(json.dumps({"what": "timeline_us", "label": label, **{k: round(float(v), 2) for k, v in zip(segs, avg)},
                      "layer_total": round(float(avg.sum()), 2)}))
timeline("talker pos256", lambda: eng.talker_step(x, 256), eng.talker_cfg["num_hidden_layers"])
timeline("talker pos2000", lambda: eng.talker_step(x, 2000), eng.talker_cfg["num_hidden_layers"])
timeline("predictor pass1", lambda: eng.predictor_run(pi, SamplingParams(do_sample=False), u), eng.pred_cfg["num_hidden_layers"])

# ---- frame-level phases of one predictor frame (slots 1024 + 8*pass + k)
for samp in (False, True):
    eng.debug_enable(2)
    eng.predictor_run(pi, SamplingParams(do_sample=samp), u)
    torch.cuda.synchronize()
    ts = eng.probe_timestamps(1024 + 8 * 16).double()[1024:].view(16, 8)[:15, :5]
    d = (ts[:, 1:] - ts[:, :-1]) / 1.965e3
    avg = d[1:].mean(0)
    print(json.dumps({"what": "pred_pass_us", "do_sample": samp, "embed+mtp": round(float(avg[0]), 2), "layers": round(float(avg[1]), 2),
                      "head": round(float(avg[2]), 2), "sample": round(float(avg[3]), 2), "pass0_layers": round(float(d[0, 1]), 2)}))
    eng.debug_enable(0)

# ---- fused on-device loop: chunks of 8 frames at a bench-like context (prompt 232), sampled
sp = SamplingParams(do_sample=True, top_k=50, temperature=0.9, top_p=1.0, repetition_penalty=1.05)
spp = SamplingParams(do_sample=True, top_k=50, temperature=0.9, top_p=1.0, repetition_penalty=1.0)
def fused(n_chunks, chunk=8, prefill=232, dbg=0):
    eng.begin_request(first_token=5, prefill_len=prefill, gen_step=0, past_hidden=torch.randn(H, device="cuda").bfloat16(),
                      trailing_text=torch.randn(25, H, device="cuda").bfloat16() * 0.02,
                      tts_pad=torch.randn(H, device="cuda").bfloat16() * 0.02, max_new_tokens=4096, min_new_tokens=4096,
                      sp_talker=sp, sp_predictor=spp, uniforms=torch.rand(4097, 16, device="cuda"))
    eng.debug_enable(dbg)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    n = 0
    for _ in range(n_chunks):
        out, res = eng.decode_chunk(chunk)
        n += out.shape[0]
    e1.record(); e1.synchronize()
    eng.debug_enable(0)
    return e0.elapsed_time(e1) / max(n, 1), n
fused(2)
for chunk in (8, 64):
    msf, n = fused(128 // chunk, chunk)
    print(json.dumps({"what": "fused_ms_per_frame", "chunk": chunk, "frames": n, "ms": round(msf, 4)}))
msf, n = fused(1, 8, dbg=2)
tl = eng.probe_timestamps(12 * 28).double().view(28, 12)[8:]
dl = ((tl[:, 1:] - tl[:, :-1]) / 1.965e3).mean(0)
print(json.dumps({"what": "fused_talker_layer_us", **{k: round(float(v), 2) for k, v in zip(
    ["norm_in", "gemv_qkv", "B1", "attn", "B2", "load+gemv_o", "B3", "norm+gemv_gu", "B4", "load+gemv_dn", "B5"], dl)},
    "layer_total": round(float(dl.sum()), 2)}))
ts = eng.probe_timestamps(2048 + 8 * 8).double()[2048:].view(8, 8)[:, :6]
d = (ts[:, 1:] - ts[:, :-1]) / 1.965e3
nxt = (ts[1:, 0] - ts[:-1, 5]) / 1.965e3
avg = d[1:].mean(0)
print(json.dumps({"what": "fused_frame_us", "predictor": round(float(avg[0]), 1), "embed_sum": round(float(avg[1]), 1),
                  "talker_layers": round(float(avg[2]), 1), "head": round(float(avg[3]), 1), "sample": round(float(avg[4]), 1),
                  "loop_top": round(float(nxt.mean()), 1), "frame0_predictor": round(float(d[0, 0]), 1),
                  "frame0_talker": round(float(d[0, 2]), 1), "chunk_ms_per_frame": round(msf, 4)}))
