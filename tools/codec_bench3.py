#!/usr/bin/env python3
"""Codec decode (codes -> PCM through fq3_codec_decode_codes) timed with CUDA events for the GEMM variants:
one-tile-per-CTA wgmma (default), persistent wgmma, mma.sync; reports ms, TFLOP/s of the dense layers and
the max PCM difference between variants.  python tools/codec_bench3.py [--variants wgmma,wgmma_persistent,mma]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "faster-qwen3-tts_b200")]
import torch  # noqa: E402

from faster_qwen3_tts.codec import build_codec  # noqa: E402
from faster_qwen3_tts.engine import set_gemm_backend  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--variants", default="wgmma,wgmma_persistent")
ap.add_argument("--cases", default="1x33,1x182,32x33,8x33")
a = ap.parse_args()
st = build_codec(dtype=torch.bfloat16, device="cuda", seed=1)
ref = {}
for case in a.cases.split(","):
    B, T = (int(x) for x in case.split("x"))
    codes = torch.randint(0, 2048, (B, T, 16), generator=torch.Generator().manual_seed(T)).cuda()
    flops = B * (st.flops(T) + st.frontend_flops(T))
    for v in a.variants.split(","):
        set_gemm_backend(v)
        for _ in range(3):
            pcm, _ = st.decode({"audio_codes": codes})
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n = 10
        e0.record()
        for _ in range(n):
            pcm, _ = st.decode({"audio_codes": codes})
        e1.record()
        e1.synchronize()
        ms = e0.elapsed_time(e1) / n
        out = torch.stack(pcm)
        key = case
        d = None if key not in ref else (out - ref[key]).abs().max().item()
        ref.setdefault(key, out.clone())
        print(json.dumps({"case": case, "variant": v, "ms": round(ms, 4), "tflops": round(flops / ms / 1e9, 1),
                          "gflop": round(flops / 1e9, 1), "max_abs_diff_vs_first_variant": d}), flush=True)
set_gemm_backend("wgmma")
