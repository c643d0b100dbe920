#!/usr/bin/env python3
"""Batched prefill against serial prefills (1.7B geometry, bf16, synthetic weights, max_seq_len 2048, 32 slots).

For n prompts of P rows: n serial ``Engine.prefill`` calls against one ``Engine.prefill_batch`` call, CUDA events
around each, after warm-up, the two alternated ``--reps`` times (median and spread reported).  Then a burst of 32
requests through ``stream_batch_from_embeds`` (left-padded batch, codec on): host time from the call to the first chunk
of the last request, with the scheduler admitting the rows by one ``submit_many`` (batched prefill) and, alternated
with it, by one ``submit`` per row (the serial prefills).  One JSON line per measurement, GPU name and power limit in
each.   python tools/prefill_batch_bench.py [--ns 1,8,32] [--ps 12,40,232] [--reps 7] [--out file.jsonl]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "faster-qwen3-tts_b200"))
import torch  # noqa: E402

from faster_qwen3_tts import batching, synthetic  # noqa: E402
from faster_qwen3_tts.model import FasterQwen3TTS  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--ns", default="1,8,32")
ap.add_argument("--ps", default="12,40,232")
ap.add_argument("--reps", type=int, default=7)
ap.add_argument("--burst", type=int, default=32)
ap.add_argument("--burst-prompt", type=int, default=40)
ap.add_argument("--out", default=None)
a = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("prefill_batch_bench needs a CUDA device")


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception:   # noqa: BLE001 -- the name torch reports is still recorded
        return torch.cuda.get_device_name(), "unknown"


GPU, POWER = gpu_info()
out = open(a.out, "a") if a.out else None


def emit(rec):
    rec = dict(rec, gpu=GPU, power_limit=POWER, model="1.7B synthetic bf16", max_seq_len=2048)
    line = json.dumps(rec)
    print(line, flush=True)
    if out:
        out.write(line + "\n")
        out.flush()


ns, ps = [int(x) for x in a.ns.split(",")], [int(x) for x in a.ps.split(",")]
model = FasterQwen3TTS.from_synthetic("1.7B", dtype=torch.bfloat16, max_seq_len=2048, max_batch=max(ns + [a.burst]))
eng = model.engine
cfg = synthetic.make_config("1.7B")
H = cfg.talker_config.hidden_size


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


for P in ps:
    for n in ns:
        g = torch.Generator().manual_seed(P * 100 + n)
        x = (torch.randn(n, P, H, generator=g) * 0.5).to(torch.bfloat16).cuda()
        pads, slots = [0] * n, list(range(n))

        def serial():
            for b in range(n):
                eng.prefill(x[b], 0, slot=b)

        def batched():
            eng.prefill_batch(x, pads, slots)
        for f in (serial, batched, serial, batched):   # warm-up
            f()
        torch.cuda.synchronize()
        ts, tb = [], []
        for _ in range(a.reps):
            ts.append(timed(serial))
            tb.append(timed(batched))
        ms_s, ms_b = statistics.median(ts), statistics.median(tb)
        emit({"what": "prefill", "P": P, "n": n, "serial_ms": round(ms_s, 3), "batched_ms": round(ms_b, 3),
              "serial_ms_range": [round(min(ts), 3), round(max(ts), 3)],
              "batched_ms_range": [round(min(tb), 3), round(max(tb), 3)], "speedup": round(ms_s / ms_b, 2),
              "groups": -(-n * P // 2048), "reps": a.reps})

# ---- burst of requests through the batched streaming API: submit -> first chunk of the last request --------------
B, P = a.burst, a.burst_prompt
prompts = [synthetic.make_prompt(cfg, P - (b % 8), 4, seed=b, dtype=torch.bfloat16, device="cuda") for b in range(B)]
tie = torch.zeros(B, P, H, dtype=torch.bfloat16, device="cuda")
tam = torch.zeros(B, P, dtype=torch.long, device="cuda")
tth = torch.cat([p[2] for p in prompts])
for b, (t, m_, _, _) in enumerate(prompts):
    tie[b, P - t.shape[1]:], tam[b, P - t.shape[1]:] = t[0], 1
tpe = prompts[0][3]
many = batching.BatchScheduler.submit_many


def one_by_one(self, requests, logprobs=False):
    return [many(self, [r], logprobs=logprobs)[0] for r in requests]


def burst(mode):
    batching.BatchScheduler.submit_many = many if mode == "batched" else one_by_one
    try:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        seen, t_last = set(), None
        for items in model.stream_batch_from_embeds(tie, tam, tth, tpe, chunk_size=8, max_new_tokens=16,
                                                    min_new_tokens=16, do_sample=False):
            seen.update(b for b, *_ in items)
            if len(seen) == B:
                t_last = time.perf_counter() - t0
                break
        torch.cuda.synchronize()
        return t_last * 1000
    finally:
        batching.BatchScheduler.submit_many = many


for mode in ("serial", "batched", "serial", "batched"):   # warm-up
    burst(mode)
res = {"serial": [], "batched": []}
for _ in range(a.reps):
    for mode in ("serial", "batched"):
        res[mode].append(burst(mode))
emit({"what": "burst_first_chunk", "requests": B, "P": P, "chunk": 8,
      "serial_ms": round(statistics.median(res["serial"]), 2), "batched_ms": round(statistics.median(res["batched"]), 2),
      "serial_ms_range": [round(min(res["serial"]), 2), round(max(res["serial"]), 2)],
      "batched_ms_range": [round(min(res["batched"]), 2), round(max(res["batched"]), 2)], "reps": a.reps})
