#!/usr/bin/env python3
"""Cost of the output-rate and encoding stage (csrc/fq3_resample.cu) for n streams that each push one 8-frame chunk
(15 360 samples at 24 kHz) at one rate and encoding, all in one launch.  ``call_ms_*``: CUDA events around one whole
``resample.process`` call after warm-up -- the packing of the pushes, the job-table upload and the kernel.
``kernel_us_mean``: the device time of ``resample_kernel`` alone, from ``torch.profiler`` (CUDA activities) over a
separate run of the same calls, so that tracing does not disturb the event timing.  ``host_float64_oracle_ms``: the same
work in the float64 oracle on the host (one stream, times n; at pitch 0 only).  One JSON record per (n, rate, encoding,
pitch), with the card's name and power limit read in this process.  ``--pitch 7,-7`` times those pitches (every stream
at that pitch, its rho, table size and taps per output in the record) and adds one ``resample_design`` record per
pitched (rate, rho): the host design of its table alone (``fq3_resample_taps_pitch``) and the first create, design plus
upload, timed to a device synchronise.

    python tools/resample_bench.py --out profiles/h100_resample.jsonl
    python tools/resample_bench.py --pitch 7,-7 --rates 8000,24000,48000 --out profiles/h100_pitch.jsonl
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


def kernel_time_us(call, iters):
    """mean device time of one resample_kernel launch over ``iters`` calls, from the profiler's kernel records"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            call()
        torch.cuda.synchronize()
    evs = [e for e in prof.key_averages() if "resample_kernel" in e.key]
    assert evs, "the profiler recorded no resample_kernel launch"
    total = sum(e.device_time_total for e in evs)
    return total / sum(e.count for e in evs)


def design_record(rate, pitch, name, power):
    """host design time of a (rate, rho) table, and its first create (design + upload) timed to a device synchronise"""
    import ctypes as C
    from faster_qwen3_tts import resample as R
    from faster_qwen3_tts.engine import load_library
    lib = load_library()
    rho = R.pitch_rho(pitch)
    n = lib.fq3_resample_taps_pitch(rate, rho, None, 0)
    buf = (C.c_double * n)()
    t0 = time.perf_counter()
    lib.fq3_resample_taps_pitch(rate, rho, buf, n)
    design_ms = (time.perf_counter() - t0) * 1000
    dev = torch.cuda.current_device()
    before = lib.fq3_resample_table_bytes(dev)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = R.Resampler(rate, "f32", "cuda", pitch)
    torch.cuda.synchronize()
    create_ms = (time.perf_counter() - t0) * 1000
    uploaded = lib.fq3_resample_table_bytes(dev) - before
    r.close()
    rec = dict(bench="resample_design", gpu=name, power_limit=power, rate=rate, pitch=pitch, rho=rho, taps=n,
               table_bytes_uploaded=uploaded, host_design_ms=design_ms, first_create_ms=create_ms)
    print(json.dumps(rec), flush=True)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", default="1,8,32,192")
    ap.add_argument("--rates", default="8000,16000,22050,24000,32000,44100,48000")
    ap.add_argument("--encodings", default="f32,ulaw")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--pitch", default="0", help="semitones, comma-separated (default 0: the plain rates)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the resample bench times the kernel on a CUDA device"
    from faster_qwen3_tts import resample as R
    from oracle import resample_oracle as O
    name, power = card()
    rng = np.random.default_rng(0)
    recs = []
    pitches = [float(p) for p in args.pitch.split(",")]
    for rate in [int(s) for s in args.rates.split(",")]:
        for pitch in pitches:
            if pitch != 0:
                recs.append(design_record(rate, pitch, name, power))
        for enc, pitch in [(e, p) for e in args.encodings.split(",") for p in pitches]:
            if (rate, enc, pitch) == (R.IN_RATE, "f32", 0):
                continue   # the identity: nothing is launched
            rho = R.pitch_rho(pitch)
            L, M, half = R.ratio(rate, rho)
            for n in [int(s) for s in args.streams.split(",")]:
                x = torch.as_tensor(rng.standard_normal((n, CHUNK)).astype(np.float32) * 0.1, device="cuda")
                pcms = list(x)
                rs = [R.Resampler(rate, enc, "cuda", pitch) for _ in range(n)]
                for _ in range(3):    # warm-up: steady-state pushes (the first push of a stream holds back the look-ahead)
                    R.process(rs, pcms, False)
                torch.cuda.synchronize()
                ms = []
                for _ in range(args.iters):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    out = rs[0].released(CHUNK, False)
                    e0.record()
                    R.process(rs, pcms, False)
                    e1.record()
                    e1.synchronize()
                    ms.append(e0.elapsed_time(e1))
                kernel_us = kernel_time_us(lambda: R.process(rs, pcms, False), args.iters)
                for r in rs:
                    r.close()
                host_ms = None
                if pitch == 0:
                    x64 = rng.standard_normal(4 * CHUNK) * 0.1
                    s = O.Stream(rate)
                    s.push(x64[:3 * CHUNK])
                    t0 = time.perf_counter()
                    s.push(x64[3 * CHUNK:])
                    host_ms = (time.perf_counter() - t0) * 1000 * n
                rec = dict(bench="resample", gpu=name, power_limit=power, streams=n, rate=rate, encoding=enc,
                           **({} if pitch == 0 else dict(pitch=pitch, rho=rho, table_bytes=L * (2 * half // L + 1) * 4,
                                                         taps_per_output=2 * half // L + 1)),
                           push_samples=CHUNK, out_samples_per_stream=out,
                           out_bytes_per_stream=out * R.SAMPLE_BYTES[enc],
                           call_ms_median=float(np.median(ms)), call_ms_min=float(min(ms)), kernel_us_mean=kernel_us,
                           host_float64_oracle_ms=host_ms)
                print(json.dumps(rec), flush=True)
                recs.append(rec)
    if args.out:
        with open(args.out, "w") as f:
            for r in recs:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
