"""Incremental text input under a fixed text rate: the 1.7B custom-voice request (synthetic weights, bf16, chunk 8) fed
its text at 10 / 25 / 50 / 200 tokens per second through ``generate_custom_voice_text_streaming``, for both streaming
codec modes, plus the same request with all of its text known up front.  Per run (JSON lines):

* ``first_text_to_pcm_ms``: from the first text piece handed over to the first PCM chunk;
* ``starved_launches``: launches that stopped unfinished for want of text (the generator pulls text before launching,
  so a launch only starves when a piece commits fewer ids than it carried text);
* ``underruns``: chunks that arrived after the playback of everything before them had ended (real-time playback
  starting at the first chunk).

The model consumes 12.5 text rows per second of audio, so rates below that must stall."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "faster-qwen3-tts_b200")]

TEXT = ("Streaming speech from a language model means the words arrive one at a time, and the voice has to keep up "
        "without waiting for the whole reply. This paragraph is long enough to give the decoder several seconds of "
        "audio to produce, so that the rate at which text arrives decides whether playback ever runs dry.")


def _pieces(text):
    import regex
    from faster_qwen3_tts.text_stream import PRETOKENIZE_REGEX
    return [m.group(0) for m in regex.finditer(PRETOKENIZE_REGEX, text)]


def _run(m, rate, mode, frames, chunk):
    m.streaming_codec = mode
    pieces = _pieces(TEXT)
    t_first = [None]

    def stream():
        for i, p in enumerate(pieces):
            if rate:
                now = time.perf_counter()
                if t_first[0] is None:
                    t_first[0] = now
                target = t_first[0] + i / rate
                if target > now:
                    time.sleep(target - now)
            elif t_first[0] is None:
                t_first[0] = time.perf_counter()
            yield p
    arrivals, samples, starved, waits = [], [], 0, 0.0
    eng = m.engine
    for pcm, sr, tm in m.generate_custom_voice_text_streaming(stream(), "aiden", "English", max_new_tokens=frames,
                                                             min_new_tokens=frames, chunk_size=chunk):
        arrivals.append(time.perf_counter())
        samples.append(len(pcm))
        waits += tm["text_wait_ms"]
    starved = getattr(eng, "starved_launches", 0)
    underruns, play_end = 0, None
    for t, n in zip(arrivals, samples):
        if play_end is not None and t > play_end:
            underruns += 1
            play_end = t
        play_end = (play_end or t) + n / sr
    return {"rate_tok_s": rate or "all_up_front", "codec": mode, "first_text_to_pcm_ms": (arrivals[0] - t_first[0]) * 1000,
            "chunks": len(arrivals), "audio_s": sum(samples) / sr, "underruns": underruns, "starved_launches": starved,
            "text_wait_ms": waits}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", default="1.7B")
    ap.add_argument("--frames", type=int, default=160)
    ap.add_argument("--chunk", type=int, default=8)
    ap.add_argument("--rates", default="10,25,50,200")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from faster_qwen3_tts import FasterQwen3TTS
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    m = FasterQwen3TTS.from_synthetic(a.size, dtype=torch.bfloat16, max_seq_len=2048, seed=0)
    m.predictor_graph.do_sample = False
    eng = m.engine
    decode = eng.decode_chunk

    def counting(n_frames, out=None, slot=0):
        codes, res = decode(n_frames, out=out, slot=slot)
        if res.finished == 0 and res.frames_emitted < n_frames:
            eng.starved_launches += 1
        return codes, res
    eng.decode_chunk = counting
    rows = []
    for mode in ("window", "stateful"):
        eng.starved_launches = 0
        _run(m, 0, mode, 16, a.chunk)   # warm-up
        for rate in [0] + [int(r) for r in a.rates.split(",")]:
            eng.starved_launches = 0
            r = _run(m, rate, mode, a.frames, a.chunk)
            r.update(size=a.size, frames=a.frames, chunk=a.chunk, gpu=gpu)
            print(json.dumps(r), flush=True)
            rows.append(r)
    if a.out:
        with open(a.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
