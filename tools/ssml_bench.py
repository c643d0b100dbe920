#!/usr/bin/env python3
"""SSML against plain split: a 40-turn two-voice dialogue with prosody spans, on a synthetic 1.7B bf16 engine with the
example server's default of 16 launch columns (serving.ContinuousBatcher, chunk 8, unpaced).

``ssml``: the dialogue as one SSML document -- two custom voices taking turns, every third turn inside
``<prosody rate='1.25' pitch='-2st' volume='-3dB'>``, a 300 ms ``<break>`` between turns.  ``plain``: the same words,
unmarked, in one voice, with ``split=True`` and ``pause_ms=300``.  Both are one request with the same segments.  Random
weights give no meaningful EOS, so every row makes a fixed number of frames (``min_new_tokens = max_new_tokens``, the
longest segment's at ``--chars-per-s``).  Per mode the record holds the wall time from submission to the first audio
and to the last sample, the scheduler steps, and per step the decode launches, the codec launches and the post-codec
stage launches (tempo, resampler and join calls, each one launch).  Every record carries the card's name and power
limit, read in this process.

    python tools/ssml_bench.py --out profiles/h100_ssml.jsonl
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "faster-qwen3-tts_b200")]
import torch  # noqa: E402

LINES = ["Did you see the message from the harbour office this morning?",
         "I did, and they want the boats moved before the storm arrives.",
         "Then we should start with the small ones near the north wall.",
         "Agreed, but the crane will not be free until after lunch.",
         "We can use the ramp for the dinghies and wait for the crane."]
VOICES = {"A": {"speaker": "ryan", "language": "English"}, "B": {"speaker": "serena", "language": "English"}}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().split("\n")[0]
    name, power = [x.strip() for x in q.split(",")]
    return {"gpu": name, "power_limit": power}


def dialogue(turns):
    """(SSML document, the same words unmarked)"""
    parts, plain = [], []
    for i in range(turns):
        line = LINES[i % len(LINES)]
        plain.append(line)
        body = f"<prosody rate='1.25' pitch='-2st' volume='-3dB'>{line}</prosody>" if i % 3 == 2 else line
        parts.append(f"<voice name='{'AB'[i % 2]}'>{body}</voice>")
    return "<speak>" + "<break time='300ms'/>".join(parts) + "</speak>", " ".join(plain)


class Launches:
    """host-side count of post-codec stage calls; each is one launch"""

    def __init__(self):
        from faster_qwen3_tts import join, resample, tempo
        self.n = 0
        for mod in (join, resample, tempo):
            fn = mod.process

            def counted(*a, _fn=fn, **k):
                self.n += 1
                return _fn(*a, **k)
            mod.process = counted


def one(model, b, mode, doc, plain, args, launches):
    from faster_qwen3_tts.serving import custom_voice_request, ssml_request
    if mode == "ssml":
        prep = ssml_request(model, doc, VOICES, "A")
    else:
        prep = custom_voice_request(model, plain, "ryan", "English", split=True)
    n = max(min(args.max_new_tokens, max(2, math.ceil(len(s) / args.chars_per_s * 12.5))) for s in prep.texts)
    eng0, codec0, st0, steps0 = model.engine.launch_count, model.codec_launches(), launches.n, b.steps
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    t = b.submit(prep, split=True, pause_ms=300, seed=1, max_new_tokens=n, min_new_tokens=n)
    first, samples = None, 0
    for audio, sr, timing in t:
        if first is None and len(audio):
            first = time.perf_counter() - t0
        samples += len(audio)
    wall = time.perf_counter() - t0
    steps = b.steps - steps0
    return {"mode": mode, "segments": len(prep), "frames_per_row": n, "audio_s": samples / 24000, "ttfa_s": first,
            "wall_s": wall, "steps": steps,
            "decode_launches_per_step": (model.engine.launch_count - eng0) / steps,
            "codec_launches_per_step": (model.codec_launches() - codec0) / steps,
            "stage_launches_per_step": (launches.n - st0) / steps}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--turns", type=int, default=40)
    ap.add_argument("--max-new-tokens", type=int, default=2048)
    ap.add_argument("--chars-per-s", type=float, default=14.0, help="speech rate that sets each row's frames")
    ap.add_argument("--max-batch", type=int, default=16, help="launch columns (the example server's default)")
    ap.add_argument("--size", default="1.7B")
    ap.add_argument("--codec", default="stateful", choices=["window", "stateful"])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_ssml.jsonl"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("ssml_bench measures the GPU: no CUDA device")
    from faster_qwen3_tts import FasterQwen3TTS
    from faster_qwen3_tts.serving import batcher_for_model
    model = FasterQwen3TTS.from_synthetic(args.size, dtype=torch.bfloat16, max_batch=args.max_batch)
    model.streaming_codec = args.codec
    base = dict(card(), size=args.size, dtype="bf16", max_batch=args.max_batch, codec=args.codec, chunk=8,
                turns=args.turns)
    doc, plain = dialogue(args.turns)
    launches = Launches()
    b = batcher_for_model(model, chunk_size=8)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    try:
        warm_doc, warm_plain = dialogue(4)
        for mode in ("plain", "ssml"):   # warm-up: module loads, codec streams, the pitch's table
            one(model, b, mode, warm_doc, warm_plain, args, launches)
        with open(args.out, "a") as f:
            for r in range(args.repeats):   # alternate the two modes
                for mode in ("plain", "ssml"):
                    rec = dict(base, **one(model, b, mode, doc, plain, args, launches), repeat=r)
                    print(json.dumps(rec), flush=True)
                    f.write(json.dumps(rec) + "\n")
    finally:
        b.close()


if __name__ == "__main__":
    main()
