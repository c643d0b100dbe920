#!/usr/bin/env python3
"""Codec decode (codes -> PCM through fq3_codec_decode_codes) timed with CUDA events; reports ms and TFLOP/s of the
dense layers per BxT case.  python tools/codec_bench3.py [--cases 1x33,1x182,8x33,32x33]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "faster-qwen3-tts_b200")]
import torch  # noqa: E402

from faster_qwen3_tts.codec import build_codec  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--cases", default="1x33,1x182,32x33,8x33")
a = ap.parse_args()
st = build_codec(dtype=torch.bfloat16, device="cuda", seed=1)
for case in a.cases.split(","):
    B, T = (int(x) for x in case.split("x"))
    codes = torch.randint(0, 2048, (B, T, 16), generator=torch.Generator().manual_seed(T)).cuda()
    flops = B * (st.flops(T) + st.frontend_flops(T))
    for _ in range(3):
        st.decode({"audio_codes": codes})
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 10
    e0.record()
    for _ in range(n):
        st.decode({"audio_codes": codes})
    e1.record()
    e1.synchronize()
    ms = e0.elapsed_time(e1) / n
    print(json.dumps({"case": case, "ms": round(ms, 4), "tflops": round(flops / ms / 1e9, 1),
                      "gflop": round(flops / 1e9, 1)}), flush=True)
