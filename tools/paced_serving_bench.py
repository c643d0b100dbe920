#!/usr/bin/env python3
"""How many real-time listeners one engine serves: N paced clients (serving.ContinuousBatcher, pace = 1.0) on a
1.7B synthetic bf16 engine with max_batch = 32 columns and max_slots resident requests, chunk 8.

Every listener is a thread that submits a voice-clone request of 10-20 s at a time staggered over the first seconds and
drains its ticket.  Per run: underruns per listener (deliveries that found the listener dry; the first chunk cannot be
one), time to first audio p50 / p95, the launches (scheduler steps that launched something: their number, mean time and
mean number of slots; a step that finds every listener held launches nothing and is not counted), the GPU busy fraction
(wall time of the launches, prefills and codec decodes over the run's wall time) and where the worker's time went.  One
JSON record per run, each with the card's name, power limit and SM clock read in this process.  Besides the paced runs,
N = 32 unpaced requests (pace = None: the engine calls of a build without paced listeners) give the reference point.
``--kv-pages N`` serves the listeners from a pool of N 64-row talker KV pages instead of max_seq_len rows per slot: the
records then also hold the parks and the most pages in use at once.

    python tools/paced_serving_bench.py --listeners 32,64,96,128,160,192 --codec window,stateful --repeats 2 \\
        --out profiles/h100_paced_serving.jsonl
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "faster-qwen3-tts_b200")]
import numpy as np  # noqa: E402
import torch  # noqa: E402

TEXTS = ["The weather report for the coming week, read slowly and clearly.",
         "A short reply.",
         "Thank you for calling, your request has been noted and somebody will be in touch with you tomorrow morning.",
         "Turn left at the next junction, then keep right for two hundred metres."]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().split("\n")[0]
    name, power, sm, sm_max = [x.strip() for x in q.split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


class Timed:
    """adds up the wall time of the calls of a callable that did something (returned a non-empty result), and the sizes
    of their results; a call ends in a device synchronise"""

    def __init__(self, fn):
        self.fn, self.s, self.n, self.items = fn, 0.0, 0, 0

    def __call__(self, *a, **k):
        t0 = time.perf_counter()
        out = self.fn(*a, **k)
        if out:
            torch.cuda.synchronize()
            self.s += time.perf_counter() - t0
            self.n += 1
            self.items += len(out)
        return out


def run(model, n, codec, first_chunk, seed, stagger_s, chunk, pace=1.0):
    from faster_qwen3_tts.serving import batcher_for_model, voice_clone_request
    model.streaming_codec = codec
    rng = np.random.default_rng(seed)
    b = batcher_for_model(model, chunk_size=chunk)
    step, admit = Timed(b.sched.step), Timed(b.sched.submit_many)
    b.sched.step, b.sched.submit_many = step, admit
    decode = Timed(b.batch_decode)
    b.batch_decode = decode
    frames = [int(f) for f in rng.integers(125, 251, size=n)]          # 10-20 s at 12.5 frames per second
    offsets = np.sort(rng.random(n) * stagger_s)
    extra = {"first_chunk": first_chunk} if first_chunk else {}
    tickets, ttfa, t_start = [None] * n, [None] * n, time.monotonic()

    def listener(i):
        time.sleep(max(0.0, t_start + offsets[i] - time.monotonic()))
        t = b.submit(voice_clone_request(model, TEXTS[i % len(TEXTS)], "English", "ref.wav", "ref words", xvec_only=True),
                     pace=pace, max_new_tokens=frames[i], min_new_tokens=frames[i], **extra)
        tickets[i] = t
        for _ in t:
            if ttfa[i] is None:
                ttfa[i] = t.first_chunk_at - t.submitted_at

    threads = [threading.Thread(target=listener, args=(i,)) for i in range(n)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    wall = time.monotonic() - t_start
    b.close()
    under = [t.underruns for t in tickets]
    assert all(t.frames == f for t, f in zip(tickets, frames)), "a listener did not get all its audio"
    return {"listeners": n, "pace": pace, "codec": codec, "first_chunk": first_chunk, "chunk": chunk, "seed": seed,
            "audio_s": round(sum(frames) * 0.08, 1), "wall_s": round(wall, 2),
            "underruns_total": int(sum(under)), "listeners_with_underruns": int(sum(u > 0 for u in under)),
            "underruns_per_listener": round(float(np.mean(under)), 3), "underruns_max": int(max(under)),
            "ttfa_p50_ms": round(float(np.percentile(ttfa, 50)) * 1e3, 1),
            "ttfa_p95_ms": round(float(np.percentile(ttfa, 95)) * 1e3, 1),
            "launches": step.n, "launch_ms_mean": round(step.s / max(step.n, 1) * 1e3, 2),
            "slots_per_launch_mean": round(step.items / max(step.n, 1), 2),
            "slot_chunks_per_launch_s": round(step.items / max(step.s, 1e-9), 1),
            "decode_step_s": round(step.s, 2), "prefill_s": round(admit.s, 2), "codec_s": round(decode.s, 2),
            "gpu_busy": round((step.s + admit.s + decode.s) / wall, 3), "max_concurrent": b.max_concurrent,
            **({"parks": b.sched.pager.parks, "peak_pages": b.sched.pager.peak} if b.sched.pager else {})}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--listeners", default="32,64,96,128,160,192")
    ap.add_argument("--codec", default="window,stateful")
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--max-seq-len", type=int, default=384, help="prompt of about 30 rows + 250 frames fit")
    ap.add_argument("--stagger-s", type=float, default=3.0)
    ap.add_argument("--chunk", type=int, default=8)
    ap.add_argument("--size", default="1.7B")
    ap.add_argument("--kv-pages", type=int, default=0, help="talker KV page pool (0: max_seq_len rows per slot)")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_paced_serving.jsonl"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("paced_serving_bench needs the GPU: a CPU run would measure nothing")
    from faster_qwen3_tts import FasterQwen3TTS
    from faster_qwen3_tts.batching import KvPager
    from faster_qwen3_tts.engine import slot_bytes
    ns = [int(x) for x in args.listeners.split(",")]
    model = FasterQwen3TTS.from_synthetic(args.size, dtype=torch.bfloat16, max_seq_len=args.max_seq_len, max_batch=32,
                                          max_slots=max(max(ns), 32), kv_pages=args.kv_pages)
    eng = model.engine
    base = {"model": f"synthetic:{args.size} bf16", "max_batch": eng.max_batch, "max_slots": eng.max_slots,
            "max_seq_len": args.max_seq_len,
            "kv_gb": round(eng.max_slots * slot_bytes(eng.talker_cfg, eng.pred_cfg, torch.bfloat16, args.max_seq_len) / 2 ** 30, 2)}
    if args.kv_pages:   # the talker pool replaces the slots' talker caches
        talker_kv = KvPager.pages(args.max_seq_len) * eng.kv_page_bytes
        base.update(kv_pages=eng.kv_pages, kv_gb=round((eng.max_slots * (
            slot_bytes(eng.talker_cfg, eng.pred_cfg, torch.bfloat16, args.max_seq_len) - talker_kv) +
            eng.kv_pages * eng.kv_page_bytes) / 2 ** 30, 2))
    run(model, 8, "stateful", None, 0, 0.5, args.chunk)   # warm-up: modules, codec shapes, the prefill path
    run(model, 8, "window", None, 0, 0.5, args.chunk)
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "a") as f:
        def record(*a, **k):
            rec = dict(base, **card(), **run(model, *a, **k))
            print(json.dumps(rec), flush=True)
            f.write(json.dumps(rec) + "\n")
            f.flush()

        for codec in args.codec.split(","):
            for rep in range(args.repeats):   # 32 requests that want their audio as fast as possible
                record(32, codec, None, 100 + rep, args.stagger_s, args.chunk, pace=None)
            for n in ns:
                for rep in range(args.repeats):
                    # window policy: two seeds show the spread.  Stateful codec: the same seed (arrivals and lengths)
                    # with and without the short first chunk, which the window policy does not take
                    if codec == "stateful":
                        record(n, codec, 2 if rep % 2 else None, 100 + rep // 2, args.stagger_s, args.chunk)
                    else:
                        record(n, codec, None, 100 + rep, args.stagger_s, args.chunk)


if __name__ == "__main__":
    main()
