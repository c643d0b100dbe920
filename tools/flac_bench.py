#!/usr/bin/env python3
"""Cost of the FLAC stage (csrc/fq3_flac.cu) for n streams that each push one 8-frame chunk (0.64 s: 15 360 samples at
24 kHz, that many at the stream's rate) of s16, all in one call.  ``call_ms_*``: CUDA events around one whole
``flac.process`` call after warm-up -- the packing of the pushes, the job-table upload, the encoding and packing
launches and the read-back of the byte counts, the stage's one host synchronisation.  ``kernel_us_mean``: the device
time of ``encode_kernel`` and of ``pack_kernel`` per call, from ``torch.profiler`` (CUDA activities) over a separate
run of the same calls, so that tracing does not disturb the event timing.  The chunks are cut from the speech fixture
(tests/golden/speech.npz, resampled to the stream's rate on the device), so the frames are real speech.  One more
record gives the compressed / s16 byte ratio of each fixture file encoded at 24 kHz in 8-frame pushes.  Every record
carries the card's name and power limit, read in this process.

    python tools/flac_bench.py --out profiles/h100_flac.jsonl
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "faster-qwen3-tts_b200")]
import numpy as np  # noqa: E402
import torch  # noqa: E402

CHUNK_S = 0.64


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().split("\n")[0]
    name, power = [x.strip() for x in q.split(",")]
    return name, power


def kernel_times_us(call, iters):
    """mean device time per call of encode_kernel and of pack_kernel, from the profiler's kernel records"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            call()
        torch.cuda.synchronize()
    out = {}
    for name in ("encode_kernel", "pack_kernel"):
        evs = [e for e in prof.key_averages() if name in e.key]
        assert evs, f"the profiler recorded no {name} launch"
        out[name] = sum(e.device_time_total for e in evs) / iters
    return out


def speech():
    return [v.astype(np.int16) for _, v in sorted(np.load(os.path.join(ROOT, "tests", "golden", "speech.npz")).items())]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", default="1,8,32,192")
    ap.add_argument("--rates", default="8000,16000,24000,48000")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the FLAC bench times the kernels on a CUDA device"
    from faster_qwen3_tts import flac as F
    from faster_qwen3_tts import resample as R
    name, power = card()
    files = speech()
    pcm24 = torch.as_tensor(np.concatenate(files).astype(np.float32) / 32768, device="cuda")
    recs = []
    for rate in [int(s) for s in args.rates.split(",")]:
        s16 = R.convert(pcm24, rate, "s16")
        m = int(round(CHUNK_S * rate))
        for n in [int(s) for s in args.streams.split(",")]:
            starts = [(i * 7919 * m // 13) % (s16.numel() - 4 * m) for i in range(n)]
            encs = [F.Encoder(rate, "cuda") for _ in range(n)]
            pos = [0]

            def push():
                # each stream moves on through its own stretch of speech
                k = pos[0] % 4
                pos[0] += 1
                return F.process(encs, [s16[a + k * m:a + (k + 1) * m] for a in starts], False)

            for _ in range(3):
                push()
            torch.cuda.synchronize()
            ms, nbytes = [], 0
            for _ in range(args.iters):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                out = push()
                e1.record()
                e1.synchronize()
                ms.append(e0.elapsed_time(e1))
                nbytes += sum(int(o.numel()) for o in out)
            kern = kernel_times_us(push, args.iters)
            for e in encs:
                e.close()
            rec = dict(bench="flac", gpu=name, power_limit=power, streams=n, rate=rate, push_samples=m,
                       blocks_per_stream=-(-m // F.BLOCK), call_ms_median=float(np.median(ms)),
                       call_ms_min=float(min(ms)), encode_kernel_us_mean=kern["encode_kernel"],
                       pack_kernel_us_mean=kern["pack_kernel"],
                       bytes_over_s16=nbytes / (args.iters * n * 2 * m))
            print(json.dumps(rec), flush=True)
            recs.append(rec)
    ratios = []
    for x in files:
        e = F.Encoder(24000, "cuda")
        t = torch.as_tensor(x, device="cuda")
        m = int(CHUNK_S * 24000)
        parts = [F.process([e], [t[i:i + m]], i + m >= t.numel())[0] for i in range(0, t.numel(), m)]
        e.close()
        ratios.append(sum(int(p.numel()) for p in parts) / (2 * t.numel()))
    rec = dict(bench="flac_ratio", gpu=name, power_limit=power, rate=24000, push_samples=int(CHUNK_S * 24000),
               files=len(files), samples=int(sum(len(x) for x in files)), bytes_over_s16_per_file=ratios,
               bytes_over_s16_all=float(np.average(ratios, weights=[len(x) for x in files])))
    print(json.dumps(rec), flush=True)
    recs.append(rec)
    if args.out:
        with open(args.out, "w") as f:
            for r in recs:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
