#!/usr/bin/env python3
"""OpenAI-compatible TTS server over the H100 engine with CONTINUOUS BATCHING.

Same endpoint and wire format as the reference's example server (POST /v1/audio/speech, response_format wav | pcm,
streaming WAV with an unknown-length header; the reference's examples/openai_server.py:91-118,215-263), but requests are
not serialised behind a lock (:71,181): up to --max-batch requests share every pass over the model weights and new
requests join between chunks (faster_qwen3_tts/serving.py).  A streamed response is a listener: it is paced at real time
by default, so the engine, which makes audio several times faster than it is played, serves the clients closest to running
dry first and holds up to --max-slots requests (each costs its KV cache) on --max-batch launch columns.  The request field
"pace" overrides that: a number = playback speed relative to real time, null = as fast as possible.

    python examples/openai_server.py --model synthetic:1.7B --max-batch 16 --port 8000
    curl -s localhost:8000/v1/audio/speech -H 'Content-Type: application/json' \\
         -d '{"model": "tts-1", "input": "Hello!", "voice": "default", "response_format": "wav"}' -o out.wav
"""
import argparse
import asyncio
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "faster-qwen3-tts_b200"))


def build_app(model, batcher, voices, default_voice):
    from fastapi import FastAPI, HTTPException
    from fastapi.responses import StreamingResponse
    from typing import Optional
    from pydantic import BaseModel
    from faster_qwen3_tts.serving import to_pcm16, voice_clone_request, wav_header

    app = FastAPI(title="faster-qwen3-tts (H100 engine) OpenAI-compatible API")

    class SpeechRequest(BaseModel):
        model: str = "tts-1"
        input: str
        voice: str = "alloy"
        response_format: str = "wav"   # wav | pcm
        speed: float = 1.0             # accepted, not applied (as in the reference)
        pace: Optional[float] = 1.0    # the client plays at pace x real time; null: everything as fast as possible

    @app.get("/health")
    async def health():
        return {"status": "ok", "active": len(batcher.sched), "max_concurrent_seen": batcher.max_concurrent}

    @app.post("/v1/audio/speech")
    async def create_speech(req: SpeechRequest):
        if not req.input.strip():
            raise HTTPException(status_code=400, detail="'input' text is empty")
        v = voices.get(req.voice) or (voices.get(default_voice) if default_voice else None)
        if v is None:
            raise HTTPException(status_code=400, detail=f"Voice {req.voice!r} is not configured. Available voices: {list(voices)}")
        fmt = req.response_format.lower()
        if fmt not in ("wav", "pcm"):
            raise HTTPException(status_code=400, detail=f"response_format {fmt!r} not supported. Use: wav, pcm")
        if req.pace is not None and not req.pace > 0:
            raise HTTPException(status_code=400, detail=f"'pace' must be a positive number or null, got {req.pace}")
        ticket = batcher.submit(voice_clone_request(model, req.input, v.get("language", "Auto"), v["ref_audio"],
                                                    v.get("ref_text", "")), pace=req.pace,
                                max_new_tokens=v.get("max_new_tokens", 2048))
        loop = asyncio.get_event_loop()
        it = iter(ticket)

        async def audio_stream():
            if fmt == "wav":
                yield wav_header(model.sample_rate)
            while True:
                item = await loop.run_in_executor(None, lambda: next(it, None))
                if item is None:
                    return
                yield to_pcm16(item[0])

        return StreamingResponse(audio_stream(), media_type="audio/wav" if fmt == "wav" else "audio/pcm")

    return app


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--model", default=os.environ.get("QWEN_TTS_MODEL", "synthetic:1.7B"))
    ap.add_argument("--voices", default=os.environ.get("QWEN_TTS_VOICES"), metavar="FILE")
    ap.add_argument("--ref-audio", default=os.environ.get("QWEN_TTS_REF_AUDIO", "ref_audio.wav"))
    ap.add_argument("--ref-text", default=os.environ.get("QWEN_TTS_REF_TEXT", ""))
    ap.add_argument("--language", default=os.environ.get("QWEN_TTS_LANGUAGE", "Auto"))
    ap.add_argument("--max-batch", type=int, default=16, help="requests one launch advances together (<= 32)")
    ap.add_argument("--max-slots", type=int, default=None,
                    help="resident requests (default: --max-batch); more serves more paced listeners, each costs its KV cache")
    ap.add_argument("--chunk-size", type=int, default=8)
    ap.add_argument("--streaming-codec", default="window", choices=["window", "stateful"],
                    help="window: the reference's two-phase window policy (sample-exact); stateful: one decoder stream per "
                         "request, a third of the codec work under load, audio = the non-streaming decode")
    ap.add_argument("--host", default="0.0.0.0")
    ap.add_argument("--port", type=int, default=8000)
    ap.add_argument("--device", default="cuda")
    args = ap.parse_args()
    import torch
    import uvicorn
    from faster_qwen3_tts import FasterQwen3TTS
    from faster_qwen3_tts.serving import batcher_for_model
    if args.model.startswith("synthetic:"):
        model = FasterQwen3TTS.from_synthetic(args.model.split(":", 1)[1], device=args.device, dtype=torch.bfloat16,
                                              max_batch=args.max_batch, max_slots=args.max_slots)
    else:
        model = FasterQwen3TTS.from_pretrained(args.model, device=args.device, max_batch=args.max_batch,
                                               max_slots=args.max_slots)
    model.streaming_codec = args.streaming_codec
    if args.voices:
        voices = json.load(open(args.voices))
        default = next(iter(voices))
    else:
        voices = {"default": {"ref_audio": args.ref_audio, "ref_text": args.ref_text, "language": args.language}}
        default = "default"
    batcher = batcher_for_model(model, chunk_size=args.chunk_size)
    uvicorn.run(build_app(model, batcher, voices, default), host=args.host, port=args.port)


if __name__ == "__main__":
    main()
