#!/usr/bin/env python3
"""OpenAI-compatible TTS server over the H100 engine with CONTINUOUS BATCHING.

Same endpoint and wire format as the reference's example server (POST /v1/audio/speech, response_format wav | pcm, plus
ulaw | alaw: raw 8-bit G.711, and flac: lossless FLAC; streaming WAV with an unknown-length header; the reference's
examples/openai_server.py:91-118,215-263), but requests are not serialised behind a lock (:71,181): up to --max-batch
requests share every pass over the model weights and new requests join between chunks (faster_qwen3_tts/serving.py).  A
streamed response is a listener: it is paced at real time by default, so the engine, which makes audio several times
faster than it is played, serves the clients closest to running dry first and holds up to --max-slots requests (each
costs its KV cache) on --max-batch launch columns.  The request field "pace" overrides that: a number = playback speed
relative to real time, null = as fast as possible.  "speed" (0.25 - 4.0) is the speaking rate: the audio is
time-stretched on the GPU after the codec, at the same pitch.  "sample_rate" (8000, 16000, 22050, 24000, 32000, 44100 or
48000; default 24000) is the rate of the response: the audio is resampled and encoded (s16 for wav / pcm, G.711 for ulaw
/ alaw, s16 compressed to a FLAC stream for flac) on the GPU, so only the encoded bytes leave it.  "pitch" (semitones,
-12 - 12) shifts the voice up or down (formants move with it) and "gain_db" (-96 - 16) scales the level before the
encoding clips; both are applied on the GPU by the same time-stretch and resampler.  "split" (default false, true for every
request with --split) speaks a long input sentence by sentence: the segments are decoded side by side and joined on the
GPU, "pause_ms" (0 - 2000) of silence between them.  "input_format": "ssml" reads the input as an SSML document
(faster_qwen3_tts/ssml.py: <voice>, <prosody>, <break>, <p>, <s>, <sub>): "voice" is then the voice spoken outside every
<voice>, "pause_ms" the pause at a boundary without a <break>, and "split" must be null or true.  A --voices file maps
names to voice specs: {"ref_audio": ..., "ref_text": ..., "xvec_only": ...} (a clone), {"speaker": ..., "instruct": ...}
(a custom voice) or {"design": ...} (a voice design), each with an optional "language" and "max_new_tokens".

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


def build_app(model, batcher, voices, default_voice, split_default=False):
    from fastapi import FastAPI, HTTPException
    from fastapi.responses import StreamingResponse
    from typing import Optional
    from pydantic import BaseModel
    from faster_qwen3_tts.join import check_pause
    from faster_qwen3_tts.resample import RATES, check_prosody
    from faster_qwen3_tts.serving import ssml_request, wav_header
    from faster_qwen3_tts.ssml import voice_request

    app = FastAPI(title="faster-qwen3-tts (H100 engine) OpenAI-compatible API")

    class SpeechRequest(BaseModel):
        model: str = "tts-1"
        input: str
        voice: str = "alloy"
        response_format: str = "wav"   # wav | pcm (16-bit) | ulaw | alaw (8-bit G.711) | flac (lossless, 16-bit)
        sample_rate: int = 24000        # one of 8000, 16000, 22050, 24000, 32000, 44100, 48000
        speed: float = 1.0             # speaking rate in [0.25, 4.0], same pitch
        pitch: float = 0.0             # semitones in [-12, 12]
        gain_db: float = 0.0           # level in [-96, 16] dB
        pace: Optional[float] = 1.0    # the client plays at pace x real time; null: everything as fast as possible
        split: Optional[bool] = None   # speak the input segment by segment (null: the server's --split)
        pause_ms: int = 0              # silence between segments, 0 - 2000 ms
        input_format: str = "text"     # text | ssml

    @app.get("/health")
    async def health():
        return {"status": "ok", "active": len(batcher.sched), "max_concurrent_seen": batcher.max_concurrent}

    @app.post("/v1/audio/speech")
    async def create_speech(req: SpeechRequest):
        if not req.input.strip():
            raise HTTPException(status_code=400, detail="'input' text is empty")
        name = req.voice if req.voice in voices else default_voice
        v = voices.get(name) if name else None
        if v is None:
            raise HTTPException(status_code=400, detail=f"Voice {req.voice!r} is not configured. Available voices: {list(voices)}")
        if req.input_format not in ("text", "ssml"):
            raise HTTPException(status_code=400, detail=f"'input_format' must be text or ssml, got {req.input_format!r}")
        ssml = req.input_format == "ssml"
        if ssml and req.split is False:
            raise HTTPException(status_code=400, detail="an SSML input is spoken segment by segment: 'split' must be "
                                                        "null or true")
        fmt = req.response_format.lower()
        encoding = {"wav": "s16", "pcm": "s16", "ulaw": "ulaw", "alaw": "alaw", "flac": "flac"}.get(fmt)
        if encoding is None:
            raise HTTPException(status_code=400,
                                detail=f"response_format {fmt!r} not supported. Use: wav, pcm, ulaw, alaw, flac")
        if req.sample_rate not in RATES:
            raise HTTPException(status_code=400, detail=f"'sample_rate' must be one of {list(RATES)}, got {req.sample_rate}")
        if req.pace is not None and not req.pace > 0:
            raise HTTPException(status_code=400, detail=f"'pace' must be a positive number or null, got {req.pace}")
        if not 0.25 <= req.speed <= 4.0:
            raise HTTPException(status_code=400, detail=f"'speed' must be in [0.25, 4.0], got {req.speed}")
        split = ssml or (split_default if req.split is None else req.split)
        try:
            check_prosody(req.speed, req.pitch, req.gain_db)
            check_pause(req.pause_ms)
            if ssml:
                prepare = ssml_request(model, req.input, voices, voice=name)
            else:
                prepare = voice_request(model, v, req.input, split=split)
        except ValueError as ex:
            raise HTTPException(status_code=400, detail=str(ex))
        ticket = batcher.submit(prepare, pace=req.pace, speed=req.speed, sample_rate=req.sample_rate, encoding=encoding,
                                pitch=req.pitch, gain_db=req.gain_db, split=split, pause_ms=req.pause_ms,
                                max_new_tokens=v.get("max_new_tokens", 2048))
        loop = asyncio.get_event_loop()
        it = iter(ticket)

        async def audio_stream():
            if fmt == "wav":
                yield wav_header(req.sample_rate)
            while True:
                item = await loop.run_in_executor(None, lambda: next(it, None))
                if item is None:
                    return
                yield item[0].tobytes()   # encoded on the device

        media = {"wav": "audio/wav", "pcm": "audio/pcm", "ulaw": "audio/basic", "alaw": "audio/x-alaw-basic",
                 "flac": "audio/flac"}[fmt]
        return StreamingResponse(audio_stream(), media_type=media)

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
    ap.add_argument("--split", action="store_true",
                    help="speak every request's input segment by segment unless the request sets \"split\"")
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
    uvicorn.run(build_app(model, batcher, voices, default, split_default=args.split), host=args.host, port=args.port)


if __name__ == "__main__":
    main()
