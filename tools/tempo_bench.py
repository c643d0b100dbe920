#!/usr/bin/env python3
"""Cost of the speaking-rate stage (csrc/fq3_tempo.cu): kernel time per call, CUDA events after warm-up, for n streams
that each push one 8-frame chunk (15 360 samples at 24 kHz) at one speed, all in one launch; the same work in the
float64 oracle on the host for comparison (one stream, times n).  One JSON record per (n, speed), with the card's name
and power limit read in this process.

    python tools/tempo_bench.py --out profiles/h100_tempo.jsonl
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "faster-qwen3-tts_b200")]
import numpy as np  # noqa: E402
import torch  # noqa: E402

CHUNK = 8 * 1920


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().split("\n")[0]
    name, power = [x.strip() for x in q.split(",")]
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", default="1,8,32,192")
    ap.add_argument("--speeds", default="0.5,1.25,2.0")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the tempo bench times the kernel on a CUDA device"
    from faster_qwen3_tts import tempo as T
    from oracle import tempo_oracle as O
    name, power = card()
    rng = np.random.default_rng(0)
    recs = []
    for speed in [float(s) for s in args.speeds.split(",")]:
        q = T.quantize(speed)
        for n in [int(s) for s in args.streams.split(",")]:
            x = torch.as_tensor(rng.standard_normal((n, CHUNK)).astype(np.float32) * 0.1, device="cuda")
            pcms = list(x)
            tempos = [T.Tempo(speed, "cuda") for _ in range(n)]
            for _ in range(3):    # warm-up: steady-state pushes (the first chunk of a stream runs fewer frames)
                T.process(tempos, pcms, False)
            torch.cuda.synchronize()
            ms = []
            for _ in range(args.iters):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                frames = T.frames_run(tempos[0].total_in, CHUNK, q, False)
                e0.record()
                T.process(tempos, pcms, False)
                e1.record()
                e1.synchronize()
                ms.append(e0.elapsed_time(e1))
            for t in tempos:
                t.close()
            x64 = rng.standard_normal(4 * CHUNK) * 0.1
            s = O.Wsola(speed)
            s.push(x64[:3 * CHUNK])
            t0 = time.perf_counter()
            s.push(x64[3 * CHUNK:])
            host_ms = (time.perf_counter() - t0) * 1000 * n
            rec = dict(bench="tempo", gpu=name, power_limit=power, streams=n, speed=speed, push_samples=CHUNK,
                       frames_per_stream=frames, kernel_ms_median=float(np.median(ms)), kernel_ms_min=float(min(ms)),
                       host_float64_oracle_ms=host_ms,
                       audio_ms_out_per_stream=T.released(3 * CHUNK, CHUNK, q, False) / 24.0)
            print(json.dumps(rec), flush=True)
            recs.append(rec)
    if args.out:
        with open(args.out, "w") as f:
            for r in recs:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
