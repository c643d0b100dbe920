#!/usr/bin/env python3
"""Where does a streaming request spend its time before the first audio, window policy vs stateful codec?
Synchronised wall-clock split of one request of the bench workload (config 3): window / stream set-up (incl. the
reference warm-up), prefill + first chunk, first codec decode, then the steady-state chunks."""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "faster-qwen3-tts_b200")]
import torch  # noqa: E402

import bench  # noqa: E402
from faster_qwen3_tts.model import FasterQwen3TTS  # noqa: E402
from faster_qwen3_tts.streaming import fast_generate_streaming  # noqa: E402

model = FasterQwen3TTS.from_synthetic("1.7B", device="cuda", dtype=torch.bfloat16, max_seq_len=2048, seed=1234)
text, ref_text, ref_audio, prep, P = bench.craft_request(model, 232, 174)
_, _, _, tie, tam, tth, tpe, ref_codes = prep
m = model.model.model
st = m.speech_tokenizer
sync = torch.cuda.synchronize


def one(mode):
    model.streaming_codec = mode
    m.talker.rope_deltas = None
    sync()
    t = [time.perf_counter()]
    win = model._make_window(st, ref_codes, 8, to_host=False)
    sync(); t.append(time.perf_counter())
    chunks = fast_generate_streaming(talker=m.talker, talker_input_embeds=tie, attention_mask=tam, trailing_text_hiddens=tth,
                                     tts_pad_embed=tpe, config=m.config.talker_config, chunk_size=8,
                                     predictor_graph=model.predictor_graph, talker_graph=model.talker_graph,
                                     **model._gen_kwargs(64, 64, 0.9, 50, 1.0, True, 1.05))
    codes, tm = next(chunks)
    sync(); t.append(time.perf_counter())
    win.push(codes)
    sync(); t.append(time.perf_counter())
    rest_dec, rest_codec = 0.0, 0.0
    n = 0
    while True:
        a = time.perf_counter()
        try:
            codes, tm = next(chunks)
        except StopIteration:
            break
        sync(); b = time.perf_counter()
        win.push(codes)
        sync(); c = time.perf_counter()
        rest_dec += b - a; rest_codec += c - b; n += 1
    d = [(t[i + 1] - t[i]) * 1e3 for i in range(3)]
    return {"mode": mode, "window_setup_ms": round(d[0], 3), "prefill_plus_first_chunk_ms": round(d[1], 3),
            "first_codec_ms": round(d[2], 3), "later_chunk_decode_ms": round(rest_dec / max(n, 1) * 1e3, 3),
            "later_chunk_codec_ms": round(rest_codec / max(n, 1) * 1e3, 3), "ref_codes_device": str(ref_codes.device)}


for mode in ("window", "stateful", "window", "stateful"):
    print(json.dumps(one(mode)), flush=True)
