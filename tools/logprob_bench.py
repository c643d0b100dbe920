#!/usr/bin/env python3
"""Cost of the per-draw log-probabilities and of several takes in one batched launch (1.7B geometry, bf16, synthetic
weights, max_seq_len 2048).

  decode: the fused loop through BatchScheduler, ms per frame-step (chunk 8, fixed length), with and without
          log-probabilities, single-sequence (B = 1) and batched (B = 32), CUDA events, the settings alternated --reps
          times after a warm-up of each;
  takes:  wall time of generate_custom_voice_takes(n_takes = n) against n serial generate_custom_voice calls of the same
          text and length (codec included), alternated --reps times.
One JSON line per measurement (median and spread), GPU name and power limit in each.
    python tools/logprob_bench.py [--frames 64] [--reps 5] [--takes 1,2,4,8] [--out file.jsonl]"""
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

from faster_qwen3_tts import synthetic  # noqa: E402
from faster_qwen3_tts.batching import BatchScheduler  # noqa: E402
from faster_qwen3_tts.model import FasterQwen3TTS  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--frames", type=int, default=64)
ap.add_argument("--chunk", type=int, default=8)
ap.add_argument("--prompt", type=int, default=40)
ap.add_argument("--batches", default="1,32")
ap.add_argument("--takes", default="1,2,4,8")
ap.add_argument("--take-frames", type=int, default=96)
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--out", default=None)
a = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("logprob_bench needs a CUDA device")


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


def stats(xs):
    return {"median": round(statistics.median(xs), 4), "min": round(min(xs), 4), "max": round(max(xs), 4), "n": len(xs)}


Bs = [int(x) for x in a.batches.split(",")]
Ns = [int(x) for x in a.takes.split(",")]
dt = torch.bfloat16
cfg = synthetic.make_config("1.7B")
model = FasterQwen3TTS.from_synthetic("1.7B", dtype=dt, max_seq_len=2048, max_batch=max(Bs + Ns))
eng, m = model.engine, model.model.model
prompts = [synthetic.make_prompt(cfg, a.prompt, 4, seed=b, dtype=dt, device="cuda") for b in range(max(Bs))]


def decode_ms_per_step(B, lp):
    sched = BatchScheduler(eng, m.talker, m.config.talker_config, model.predictor_graph, model.talker_graph)
    sched.submit_many([dict(tie=tie, tam=tam, tth=tth, tpe=tpe, tag=b, max_new_tokens=a.frames, min_new_tokens=a.frames)
                       for b, (tie, tam, tth, tpe) in enumerate(prompts[:B])], logprobs=lp)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    n = 0
    while len(sched):
        for rq, codes in sched.step(a.chunk):
            n += codes.shape[0]
    e1.record()
    e1.synchronize()
    assert n == B * a.frames
    return e0.elapsed_time(e1) / a.frames


settings = [(B, lp) for B in Bs for lp in (False, True)]
for s in settings:
    decode_ms_per_step(*s)
res = {s: [] for s in settings}
for _ in range(a.reps):
    for s in settings:
        res[s].append(decode_ms_per_step(*s))
for (B, lp), xs in res.items():
    emit({"what": "decode_ms_per_frame_step", "B": B, "logprobs": lp, "chunk": a.chunk, "frames": a.frames,
          "prompt": a.prompt, **stats(xs)})

TEXT = "The quick brown fox jumps over the lazy dog, and then it runs far away into the forest."
gen = dict(max_new_tokens=a.take_frames, min_new_tokens=a.take_frames)


def takes_s(n):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    model.generate_custom_voice_takes(TEXT, "ryan", "English", n_takes=n, seeds=list(range(n)), **gen)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def serial_s(n):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        model.generate_custom_voice(TEXT, "ryan", "English", **gen)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


for n in Ns:
    takes_s(n)
    serial_s(n)
tk = {n: [] for n in Ns}
se = {n: [] for n in Ns}
for _ in range(a.reps):
    for n in Ns:
        tk[n].append(takes_s(n))
        se[n].append(serial_s(n))
for n in Ns:
    emit({"what": "takes_wall_s", "n_takes": n, "frames_per_take": a.take_frames, "takes": stats(tk[n]),
          "serial": stats(se[n]), "serial_over_takes": round(statistics.median(se[n]) / statistics.median(tk[n]), 3)})
