#!/usr/bin/env python3
"""Long inputs, split against unsplit: one 4096-character request on a synthetic 1.7B bf16 engine with the example
server's default of 16 launch columns (serving.ContinuousBatcher, chunk 8, x-vector voice clone, unpaced).

Per mode (``split`` = the text spoken sentence by sentence as rows, ``unsplit`` = one request) the record holds the wall
time from submission to the first audio and to the last sample, the audio seconds delivered and the segments.  Random
weights give no meaningful EOS, so every row makes a fixed number of frames, set by its text at ``--chars-per-s``
(``min_new_tokens = max_new_tokens``): ``frames = ceil(chars / chars_per_s * 12.5)``, capped at ``--max-new-tokens``.
The unsplit request therefore stops at its cap, which is the truncation split removes, and the split one makes every
segment's frames; compare the wall times together with the audio each mode delivered.

The paced row mixes ``--listeners`` paced short requests (pace 1) with ``--long-listeners`` paced split requests of
``--paced-chars`` characters, and records underruns and time to first audio of both kinds, as ``paced_serving_bench``
does.  Every record carries the card's name and power limit, read in this process.

    python tools/longform_bench.py --out profiles/h100_longform.jsonl
"""
import argparse
import json
import math
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "faster-qwen3-tts_b200")]
import numpy as np  # noqa: E402
import torch  # noqa: E402

SENTENCES = ["The committee met on Tuesday to review the budget for the coming year.",
             "Several members asked whether the new library could open before the winter.",
             "After a long discussion, they agreed to publish the plan next month!",
             "Is there still time to change the route of the northern bus line?",
             "Residents will be invited to comment at three public meetings; the first is in May."]
SHORT = ["Turn left at the next junction, then keep right for two hundred metres.",
         "Thank you for calling, your request has been noted.",
         "The weather report for the coming week, read slowly and clearly."]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().split("\n")[0]
    name, power = [x.strip() for x in q.split(",")]
    return {"gpu": name, "power_limit": power}


def long_text(chars):
    out, i = "", 0
    while len(out) < chars:
        out += SENTENCES[i % len(SENTENCES)] + " "
        i += 1
    return out[:chars].rstrip()


def frames_for(text, chars_per_s, cap):
    return min(cap, max(2, math.ceil(len(text) / chars_per_s * 12.5)))


def one(model, b, text, split, args):
    """-> record of one unpaced request (split or not)"""
    from faster_qwen3_tts.segment import split_text
    from faster_qwen3_tts.serving import voice_clone_request
    segs = split_text(text, args.max_segment_chars) if split else [text]
    # one budget for every row: the longest segment's; the unsplit request gets the whole text's, capped
    n = max(frames_for(s, args.chars_per_s, args.max_new_tokens) for s in segs)
    prep = voice_clone_request(model, text, "English", "ref.wav", "", xvec_only=True, split=split,
                               max_segment_chars=args.max_segment_chars)
    kw = dict(split=True, seed=1) if split else {}
    t0 = time.perf_counter()
    t = b.submit(prep, max_new_tokens=n, min_new_tokens=n, **kw)
    first, samples, frames = None, 0, 0
    for audio, sr, timing in t:
        if first is None and len(audio):
            first = time.perf_counter() - t0
        samples += len(audio)
        frames = timing["total_steps_so_far"]
    wall = time.perf_counter() - t0
    return {"mode": "split" if split else "unsplit", "chars": len(text), "segments": len(segs),
            "frames_per_row": n, "frames": frames, "audio_s": samples / 24000, "ttfa_s": first, "wall_s": wall}


def paced(model, b, args):
    """short paced listeners with long-input paced listeners mixed in"""
    text = long_text(args.paced_chars)
    res, lock = [], threading.Lock()

    def listener(i, long):
        from faster_qwen3_tts.segment import split_text
        from faster_qwen3_tts.serving import voice_clone_request
        time.sleep(i * args.stagger_s / max(1, args.listeners + args.long_listeners))
        s = text if long else SHORT[i % len(SHORT)]
        n = max(frames_for(x, args.chars_per_s, args.max_new_tokens)
                for x in (split_text(s, args.max_segment_chars) if long else [s]))
        prep = voice_clone_request(model, s, "English", "ref.wav", "", xvec_only=True, split=long)
        kw = dict(split=True, seed=i) if long else {}
        t0 = time.perf_counter()
        t = b.submit(prep, pace=1.0, max_new_tokens=n, min_new_tokens=n, **kw)
        first = None
        for audio, _, _ in t:
            if first is None and len(audio):
                first = time.perf_counter() - t0
        with lock:
            res.append((long, first, t.underruns, time.perf_counter() - t0))

    total = args.listeners + args.long_listeners
    longs = {k * total // max(1, args.long_listeners) for k in range(args.long_listeners)}   # spread over arrivals
    th = [threading.Thread(target=listener, args=(i, i in longs)) for i in range(total)]
    t0 = time.perf_counter()
    for x in th:
        x.start()
    for x in th:
        x.join()
    rec = {"mode": "paced", "listeners": args.listeners, "long_listeners": args.long_listeners,
           "paced_chars": args.paced_chars, "wall_s": time.perf_counter() - t0}
    for long in (False, True):
        r = [x for x in res if x[0] == long]
        k = "long" if long else "short"
        ttfa = np.array([x[1] for x in r if x[1] is not None])
        rec[k] = {"n": len(r), "underruns": int(sum(x[2] for x in r)),
                  "ttfa_s_p50": float(np.percentile(ttfa, 50)) if len(ttfa) else None,
                  "ttfa_s_p95": float(np.percentile(ttfa, 95)) if len(ttfa) else None}
    return rec


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--chars", type=int, default=4096)
    ap.add_argument("--max-segment-chars", type=int, default=400)
    ap.add_argument("--max-new-tokens", type=int, default=2048)
    ap.add_argument("--chars-per-s", type=float, default=14.0, help="speech rate that sets each row's frames")
    ap.add_argument("--max-batch", type=int, default=16, help="launch columns (the example server's default)")
    ap.add_argument("--max-seq-len", type=int, default=3072)
    ap.add_argument("--size", default="1.7B")
    ap.add_argument("--codec", default="stateful", choices=["window", "stateful"])
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--listeners", type=int, default=24, help="paced short requests of the paced row (0: no paced row)")
    ap.add_argument("--long-listeners", type=int, default=4, help="paced split requests of the paced row")
    ap.add_argument("--paced-chars", type=int, default=1200)
    ap.add_argument("--stagger-s", type=float, default=2.0)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_longform.jsonl"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("longform_bench measures the GPU: no CUDA device")
    from faster_qwen3_tts import FasterQwen3TTS
    from faster_qwen3_tts.serving import batcher_for_model
    model = FasterQwen3TTS.from_synthetic(args.size, dtype=torch.bfloat16, max_seq_len=args.max_seq_len,
                                          max_batch=args.max_batch)
    model.streaming_codec = args.codec
    base = dict(card(), size=args.size, dtype="bf16", max_batch=args.max_batch, codec=args.codec, chunk=8)
    text = long_text(args.chars)
    b = batcher_for_model(model, chunk_size=8)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    try:
        one(model, b, long_text(300), True, args)   # warm-up: module loads, codec streams, the voice prompt
        with open(args.out, "a") as f:
            def write(rec):
                rec = dict(base, **rec)
                print(json.dumps(rec), flush=True)
                f.write(json.dumps(rec) + "\n")
            for r in range(args.repeats):   # alternate the two modes
                for split in (False, True):
                    write(dict(one(model, b, text, split, args), repeat=r))
            if args.listeners or args.long_listeners:
                write(paced(model, b, args))
    finally:
        b.close()


if __name__ == "__main__":
    main()
