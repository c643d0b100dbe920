"""FasterQwen3TTS -- the reference's public wrapper (faster_qwen3_tts/model.py:21-1505) over the H100 engine.

Kept verbatim from the reference: constructor signature, ``from_pretrained`` / ``warmup`` / ``_warmup`` /
``generate`` / ``generate_voice_clone[_streaming]`` / ``generate_custom_voice[_streaming]`` /
``generate_voice_design[_streaming]`` names, positional order, keyword defaults, return shapes, error types, the
``speech_tokenizer`` / ``sample_rate`` surface, and the streaming codec-window policy (model.py:1052-1135).

Replaced: the two graph objects are thin handles on one fq3 engine (persistent sm_90a kernel); per-chunk work
is one kernel launch + one codec decode.

Prompt assembly (model.py:278-805) is restated here and in ``prompt.py`` (embedding layout pinned against the
reference's own function, tests/test_prompt_cpu.py).  Tokeniser, speaker encoder, codec encoder and the ICL prompt
are upstream ``qwen-tts`` methods of the wrapped model -- called through exactly the attributes the reference calls;
the synthetic model (``from_synthetic``) answers them with deterministic stand-ins (``synthetic_frontend.py``).
"""
from __future__ import annotations

import logging
import os
import time
from pathlib import Path
from typing import Any, Dict, Generator, List, Optional, Tuple, Union

import numpy as np
import torch

logger = logging.getLogger(__name__)

CONTEXT_FRAMES = 25  # model.py:1056


def take_uniforms(seed: int, max_new_tokens: int, device="cuda") -> torch.Tensor:
    """The draws of one take (``*_takes``): [max_new_tokens + 1, 16] uniforms from a CPU generator seeded with ``seed``,
    so a take can be re-rendered alone (``fast_generate(..., uniforms=take_uniforms(seed, n))``) on any device."""
    g = torch.Generator(device="cpu").manual_seed(int(seed))
    return torch.rand(int(max_new_tokens) + 1, 16, generator=g).to(device)


def _check_speed(speed, pitch=0.0, gain_db=0.0):
    """a speaking rate outside [0.25, 4.0], a pitch outside [-12, 12] semitones, a gain outside [-96, 16] dB or a speed
    and pitch whose tempo falls outside [0.25, 4.0] are refused (ValueError) before anything is tokenized"""
    from .resample import check_prosody
    check_prosody(speed, pitch, gain_db)


def _check_rate(sample_rate):
    """an output rate outside ``resample.RATES`` is refused (ValueError) before anything is tokenized"""
    from .resample import check_rate
    check_rate(sample_rate)


def _refuse_split(split):
    """takes and text fed while it is spoken are not split (ValueError before anything is tokenized)"""
    if split:
        raise ValueError("split=True is supported by the one-shot and streaming calls only, not by takes or text fed "
                         "while it is spoken")


def _post_kw(speed, sample_rate=None, pitch=0.0, gain_db=0.0):
    """``speed=`` / ``sample_rate=`` / ``pitch=`` / ``gain_db=`` for the delivery calls, only where they are not the
    identity (speed 1, 24 kHz, pitch 0, 0 dB): at the defaults every call is made exactly as without them"""
    kw = {} if speed == 1.0 else {"speed": speed}
    if sample_rate is not None and int(sample_rate) != 24000:
        kw["sample_rate"] = sample_rate
    if pitch != 0:
        kw["pitch"] = pitch
    if gain_db != 0:
        kw["gain_db"] = gain_db
    return kw


def _rate_of(sr, sample_rate):
    """the rate a delivery returns: the requested one, else what the codec gave"""
    return sr if sample_rate is None else int(sample_rate)


def _pcm_device(speech_tokenizer):
    """the device the codec leaves its PCM on"""
    dev = getattr(speech_tokenizer, "_dev", None)
    return dev if dev is not None else next(speech_tokenizer.decoder.parameters()).device


class _StreamWindow:
    """Per-request state of the streaming codec-window policy (model.py:1052-1135), push-style so that several
    requests of a batch can each keep their own window while their code chunks arrive interleaved.

    Phase 1 with an ICL reference is where the reference spends most of its codec time: every chunk re-decodes the
    reference frames plus everything generated so far and keeps only the new tail.  The decoder is causal, so that tail
    is exactly what a decoder STREAM that has already seen the reference produces for the new frames alone (bit for bit,
    tests/test_gpu_codec.py).  When the tokenizer offers streams (engine codec) Phase 1 therefore runs on a copy of the
    reference's warmed template stream (``SpeechTokenizer.reference_stream``): same samples, one chunk's worth of work,
    and the reference itself is decoded once per voice instead of four times per request.  Phase 2 (25-frame context
    windows without the reference) is the reference's approximation and is decoded exactly as the reference does.
    ``FQ3_PHASE1_STREAM=0`` keeps the literal re-decode.  ``tempo``: the request's speaking rate (``tempo.Tempo``),
    ``resampler``: its output rate and encoding (``resample.Resampler``), and ``flac``: its FLAC encoder
    (``flac.Encoder``, after an s16 resampler), applied in that order to the new samples on the device before they are
    converted (``decode_windows_batched``)."""

    def __init__(self, owner, speech_tokenizer, ref_codes, chunk_size, to_host=True, tempo=None, resampler=None,
                 flac=None):
        self.st, self.ref_codes, self.tempo, self.resampler, self.flac = (speech_tokenizer, ref_codes, tempo, resampler,
                                                                          flac)
        self.min_cal = max(CONTEXT_FRAMES, chunk_size)
        self.all_codes, self.prev_len, self.spf = [], 0, None
        self.conv = owner._to_numpy if to_host else (lambda a: a.flatten())
        self.p1, self._p1_pending = None, False
        if (ref_codes is not None and ref_codes.shape[0] > 0 and getattr(speech_tokenizer, "supports_streams", False)
                and os.environ.get("FQ3_PHASE1_STREAM", "1") != "0"):
            # known voice: a copy of its warmed template, ready before the first chunk.  New voice: the FIRST chunk takes the
            # literal re-decode (one decode of reference + 8 frames -- nothing cheaper exists for the first audio), the
            # template is warmed when the second chunk arrives, i.e. off the time-to-first-audio path.
            self.p1 = speech_tokenizer.reference_stream(ref_codes, create=False)
            self._p1_pending = self.p1 is None

    def window(self, codec_chunk):
        """-> (codes [T,16] to decode, meta): the decode call the policy makes for this chunk"""
        self.all_codes.append(codec_chunk)
        n_new = codec_chunk.shape[0]
        if self._p1_pending and self.spf is None and len(self.all_codes) > 1:
            self._p1_pending = False
            self.p1 = self.st.reference_stream(self.ref_codes)            # warms and caches the voice's template
            self.p1.warm(torch.cat(self.all_codes[:-1], dim=0))           # catch up on the frames already played
        if self.spf is None and self.p1 is not None:
            return codec_chunk, ("phase1_stream", sum(int(c.shape[0]) for c in self.all_codes), 0)
        flat = torch.cat(self.all_codes, dim=0)
        n_total = flat.shape[0]
        if self.spf is None:
            ref_codes = self.ref_codes
            inp = torch.cat([ref_codes.to(flat.device), flat], dim=0) if ref_codes is not None else flat
            return inp, ("phase1", n_total, int(inp.shape[0]))
        start = max(0, n_total - n_new - CONTEXT_FRAMES)
        window = flat[start:]
        return window, ("phase2", window.shape[0] - n_new, 0)

    def finish(self, audio, meta):
        """decoded window -> the new samples of this chunk (trim of the reference / of the 25-frame context), still where
        the codec left them"""
        audio = audio.flatten()
        kind, a, b = meta
        if kind == "phase1_stream":   # the stream produced exactly gen_audio[prev_len:] of the reference's Phase 1
            self.prev_len += len(audio)
            if a >= self.min_cal:
                self.spf = self.prev_len / a
                self.p1.close()
                self.p1 = None
            return audio
        if kind == "phase1":
            n_total, n_inp = a, b
            if self.ref_codes is not None:
                cut = int(self.ref_codes.shape[0] / max(n_inp, 1) * len(audio))
                gen_audio = audio[cut:]
            else:
                gen_audio = audio
            new_audio = gen_audio[self.prev_len:]
            self.prev_len = len(gen_audio)
            if n_total >= self.min_cal:
                self.spf = len(gen_audio) / n_total
            return new_audio
        n_ctx = a
        return audio[int(round(n_ctx * self.spf)):] if n_ctx > 0 else audio

    def push(self, codec_chunk, final=False):
        return decode_windows_batched(self.st, [self], [codec_chunk], [final])[0]


class _StatefulWindow:
    """Streaming decode on a stateful codec stream (SURVEY 8(f) item 2, ``streaming_codec="stateful"``): every chunk costs
    only its own frames -- no Phase-1 re-decode of everything so far, no 25-frame Phase-2 context (model.py:1085-1135).
    The audio of a request equals the non-streaming decode of the same codes (``generate_voice_clone``), i.e. the
    reference's Phase-1 output continued for the whole utterance; Phase-2 chunks of the reference differ slightly because
    they see only 25 frames of context.  ICL reference frames warm the stream's state up front; no audio is made for them."""

    any_chunking = True   # the PCM of a stream does not depend on how its frames are split into chunks

    def __init__(self, owner, speech_tokenizer, ref_codes, chunk_size, to_host=True, tempo=None, resampler=None,
                 flac=None):
        self.st, self.tempo, self.resampler, self.flac = speech_tokenizer, tempo, resampler, flac
        self.stream = speech_tokenizer.open_stream()
        self.conv = owner._to_numpy if to_host else (lambda a: a.flatten())
        if ref_codes is not None and ref_codes.shape[0] > 0:
            self.stream.warm(ref_codes)   # 174 reference frames: ~3 ms once, instead of re-decoding them for four chunks

    def push(self, codec_chunk, final=False):
        return decode_windows_batched(self.st, [self], [codec_chunk], [final])[0]


def decode_windows_batched(speech_tokenizer, wins, chunks, finals=None):
    """One chunk of several requests: windows of equal length are decoded as ONE batch (every codec launch covers all of
    them), then the new samples of every window with a tempo are time-stretched in ONE launch, and those of every window
    with a resampler are resampled and encoded in ONE more launch, and those of every window with a FLAC encoder are
    compressed in one more encoding launch (and its packing launch), still on the device; returns [(new_audio,
    sample_rate)] in the order of `wins`.  ``finals[i]`` ends request i: its tempo, resampler and FLAC encoder flush.  A
    chunk of no frames decodes nothing (a flush after the last frames)."""
    raw = [None] * len(wins)
    sr = speech_tokenizer.sample_rate if hasattr(speech_tokenizer, "sample_rate") else 24000
    live = [i for i, c in enumerate(chunks) if int(c.shape[0])]
    if live and isinstance(wins[0], _StatefulWindow):
        # stateful streams: rows with the same number of new frames advance together in one set of launches
        groups = {}
        for i in live:
            groups.setdefault(int(chunks[i].shape[0]), []).append(i)
        for n, idxs in groups.items():
            pcm = speech_tokenizer.push_streams([wins[i].stream for i in idxs], torch.stack([chunks[i] for i in idxs]))
            for i, a in zip(idxs, pcm):
                raw[i] = a
    elif live:
        prepared = {i: wins[i].window(chunks[i]) for i in live}
        groups, sgroups = {}, {}
        for i, (codes, meta) in prepared.items():
            (sgroups if meta[0] == "phase1_stream" else groups).setdefault(int(codes.shape[0]), []).append(i)
        for T, idxs in groups.items():
            audio_list, sr = speech_tokenizer.decode({"audio_codes": torch.stack([prepared[i][0] for i in idxs])})
            for i, a in zip(idxs, audio_list):
                raw[i] = wins[i].finish(a, prepared[i][1])
        for n, idxs in sgroups.items():   # Phase-1 rows riding on reference-warmed streams: one call for all of them
            pcm = speech_tokenizer.push_streams([wins[i].p1 for i in idxs], torch.stack([prepared[i][0] for i in idxs]))
            for i, a in zip(idxs, pcm):
                raw[i] = wins[i].finish(a, prepared[i][1])
    return run_stages(wins, raw, finals, sr)


def run_stages(wins, raw, finals, sr):
    """The device stages of several windows (or ``_Chain``s) on their new 24 kHz PCM ``raw`` (None: no samples): every
    tempo in one launch, every resampler in one more, every FLAC encoder in one more; ``finals[i]`` flushes window i's
    stages.  Returns [(audio, sample_rate)] converted by each window's ``conv``."""
    stretched = [i for i, w in enumerate(wins) if getattr(w, "tempo", None) is not None]
    if stretched:
        from . import tempo
        finals = finals or [False] * len(wins)
        for i in stretched:
            if raw[i] is None:
                raw[i] = torch.zeros(0, dtype=torch.float32, device=wins[i].tempo.device)
        pcm = tempo.process([wins[i].tempo for i in stretched], [raw[i] for i in stretched], [finals[i] for i in stretched])
        for i, a in zip(stretched, pcm):
            raw[i] = a
    resampled = [i for i, w in enumerate(wins) if getattr(w, "resampler", None) is not None]
    if resampled:
        from . import resample
        finals = finals or [False] * len(wins)
        for i in resampled:
            if raw[i] is None:
                raw[i] = torch.zeros(0, dtype=torch.float32, device=wins[i].resampler.device)
        out = resample.process([wins[i].resampler for i in resampled], [raw[i] for i in resampled],
                               [finals[i] for i in resampled])
        for i, a in zip(resampled, out):
            raw[i] = a
    compressed = [i for i, w in enumerate(wins) if getattr(w, "flac", None) is not None]
    if compressed:
        from . import flac
        finals = finals or [False] * len(wins)
        out = flac.process([wins[i].flac for i in compressed], [raw[i] for i in compressed],
                           [finals[i] for i in compressed])
        for i, a in zip(compressed, out):
            raw[i] = a
    return [(w.conv(a if a is not None else torch.zeros(0)), _window_rate(w, sr)) for w, a in zip(wins, raw)]


def _stages(speech_tokenizer, speed=1.0, sample_rate=None, encoding="f32", pitch=0.0, gain_db=0.0):
    """a request's post-codec stages: at a speed or pitch other than 1 / 0 its ``tempo.Tempo`` (at
    ``resample.tempo_speed``), at an output rate or encoding other than 24 kHz f32, a pitch or a gain its
    ``resample.Resampler``; ``encoding="flac"`` is an s16 resampler followed by a ``flac.Encoder``"""
    from .resample import resampler_for, tempo_speed
    from .tempo import tempo_for
    tempo = (tempo_for(tempo_speed(speed, pitch), _pcm_device(speech_tokenizer))
             if speed != 1.0 or pitch != 0 else None)
    rs = enc = None
    if encoding == "flac":
        from .flac import Encoder
        rs = resampler_for(sample_rate, "s16", _pcm_device(speech_tokenizer), pitch, gain_db)
        enc = Encoder(rs.rate, _pcm_device(speech_tokenizer))
    elif sample_rate is not None or encoding != "f32" or pitch != 0 or gain_db != 0:
        rs = resampler_for(sample_rate, encoding, _pcm_device(speech_tokenizer), pitch, gain_db)
    return dict(tempo=tempo, resampler=rs, flac=enc)


class _Chain:
    """The post-codec stages of a segmented request, run once on its joined stream (``run_stages``)"""

    def __init__(self, owner, speech_tokenizer, to_host=True, **out):
        for k, v in _stages(speech_tokenizer, **out).items():
            setattr(self, k, v)
        self.conv = owner._to_numpy if to_host else (lambda a: a.flatten())


def _window_rate(win, sr):
    r = getattr(win, "resampler", None)
    return sr if r is None else r.rate


def _open_stages(win):
    """whether a window still holds device stages that have not flushed (a tempo, a resampler or a FLAC encoder)"""
    return any(s is not None and not s.final
               for s in (getattr(win, "tempo", None), getattr(win, "resampler", None), getattr(win, "flac", None)))


def flush_windows(speech_tokenizer, wins):
    """The end of several requests: every window with device stages flushes, in one launch per stage ->
    [(last samples, sample_rate)] of those windows, in order (their look-ahead; other windows have nothing left)"""
    wins = [w for w in wins if _open_stages(w)]
    empty = torch.zeros(0, 16, dtype=torch.long)
    return wins, decode_windows_batched(speech_tokenizer, wins, [empty] * len(wins), [True] * len(wins))


class FasterQwen3TTS:
    def __init__(self, base_model, predictor_graph, talker_graph, device: str = "cuda",
                 dtype: torch.dtype = torch.bfloat16, max_seq_len: int = 2048):
        self.model = base_model
        self.predictor_graph = predictor_graph
        self.talker_graph = talker_graph
        self.device = device
        self.dtype = dtype
        self.max_seq_len = max_seq_len
        self.sample_rate = self._infer_sample_rate(base_model)
        self._warmed_up = False
        self._voice_prompt_cache = {}
        # "window": the reference's two-phase re-decode policy (sample-exact, default); "stateful": one stateful decoder
        # stream per request (engine codec only) -- each chunk costs its own frames, audio = the non-streaming decode
        self.streaming_codec = os.environ.get("FQ3_STREAMING_CODEC", "window")

    # ------------------------------------------------------------------ small surface kept from the reference
    @staticmethod
    def _get_speech_tokenizer(base_model):
        return getattr(getattr(base_model, "model", None), "speech_tokenizer", None)

    @property
    def speech_tokenizer(self):
        st = self._get_speech_tokenizer(self.model)
        if st is None:
            raise AttributeError("Underlying model does not expose a speech_tokenizer")
        return st

    @property
    def engine(self):
        return getattr(self.talker_graph, "engine", None)

    @staticmethod
    def _infer_sample_rate(base_model) -> int:
        sr = None
        st = FasterQwen3TTS._get_speech_tokenizer(base_model)
        if st is not None:
            sr = getattr(st, "sample_rate", None)
        if sr is None:
            sr = getattr(base_model, "sample_rate", None)
        if sr is None:
            logger.warning("Could not infer sample rate from base model; defaulting to 24000 Hz.")
            return 24000
        return int(sr)

    @staticmethod
    def _resolve_non_streaming_mode(non_streaming_mode: Optional[bool], *, default: bool) -> bool:
        return default if non_streaming_mode is None else non_streaming_mode

    def _cached_reference_prompt(self, ref_spk_emb, ref_codes, voice_clone_prompt):
        """SURVEY 8(f) item 4, in-memory half: a cached reference in decoded form -> the voice_clone_prompt dict the prompt
        builder consumes (what ggml_backend.py:476-509 hands to qwentts.cpp).  ref_spk_emb: [H_talker] floats; ref_codes:
        None (x-vector cloning) or int array [T,16] of reference codec frames (ICL cloning, needs ref_text)."""
        if ref_spk_emb is None and ref_codes is None:
            return voice_clone_prompt
        if voice_clone_prompt is not None:
            raise ValueError("pass either voice_clone_prompt or ref_spk_emb/ref_codes, not both")
        if ref_spk_emb is None:
            raise ValueError("ref_spk/ref_spk_emb is required for cached voice cloning.")
        emb = torch.as_tensor(np.ascontiguousarray(np.asarray(ref_spk_emb, dtype=np.float32)).reshape(-1))
        if emb.numel() == 0:
            raise ValueError("ref_spk_emb must not be empty.")
        H = self.model.model.config.talker_config.hidden_size
        if emb.numel() != H:
            raise ValueError(f"ref_spk_emb has {emb.numel()} values, the talker expects {H}")
        codes = None
        if ref_codes is not None:
            codes = torch.as_tensor(np.ascontiguousarray(np.asarray(ref_codes, dtype=np.int64)))
            ng = self.model.model.config.talker_config.num_code_groups
            if codes.dim() != 2 or codes.shape[1] != ng or codes.shape[0] == 0:
                raise ValueError(f"ref_codes must be a non-empty [T, {ng}] array of codec frames")
        return dict(ref_spk_embedding=[emb], ref_code=[codes], x_vector_only_mode=[codes is None], icl_mode=[codes is not None])

    # ------------------------------------------------------------------ construction
    @classmethod
    def from_pretrained(cls, model_name: str, device: str = "cuda", dtype: Union[str, torch.dtype] = torch.bfloat16,
                        attn_implementation: str = "sdpa", max_seq_len: int = 2048, backend: str = "torch",
                        quant: str = "BF16", gguf_talker_path=None, gguf_codec_path=None, qwentts_library_path=None,
                        qwentts_use_fa: bool = True, qwentts_clamp_fp16: bool = False, qwentts_ref_cache_dir=None,
                        cache_dir=None, local_files_only: bool = False, max_batch: int = 1,
                        max_slots: Optional[int] = None, kv_pages: int = 0):
        """Same arguments as the reference (model.py:106-124); trailing and engine-specific: ``max_batch`` = requests one
        launch advances together (> 1 enables the batched persistent kernel / continuous batching, serving.py; <= 32),
        ``max_slots`` = request slots that exist (default ``max_batch``; more serves more paced listeners than a launch
        has columns, each slot costing its KV cache), ``kv_pages`` = a pool of that many 64-row talker KV pages that
        requests map as they grow, instead of max_seq_len rows reserved per slot (0: the reservation)."""
        if backend not in ("torch", "ggml", "qwentts"):
            raise ValueError(f"Unsupported backend {backend!r}. Expected 'torch', 'ggml', or 'qwentts'.")
        if backend in ("ggml", "qwentts"):
            raise NotImplementedError("the qwentts.cpp / GGML adapter is out of scope of the H100 engine "
                                      "(SURVEY.md section 2 row 9); use backend='torch'")
        if isinstance(dtype, str):
            dtype = getattr(torch, dtype)
        if not device.startswith("cuda") or not torch.cuda.is_available():
            raise ValueError("CUDA graphs require CUDA device")
        if str(model_name).startswith("synthetic:"):
            return cls.from_synthetic(str(model_name).split(":", 1)[1], device=device, dtype=dtype, max_seq_len=max_seq_len,
                                      max_batch=max_batch, max_slots=max_slots, kv_pages=kv_pages)
        try:
            from qwen_tts import Qwen3TTSModel
        except ImportError as ex:
            raise ImportError("qwen-tts is required to load real checkpoints; use model_name='synthetic:1.7B' "
                              "for random-init weights of the real geometry") from ex
        base = Qwen3TTSModel.from_pretrained(model_name, device_map=device, torch_dtype=dtype,
                                             attn_implementation=attn_implementation)
        return cls._wrap(base, device, dtype, max_seq_len, max_batch=max_batch, max_slots=max_slots, kv_pages=kv_pages)

    @classmethod
    def _wrap(cls, base_model, device, dtype, max_seq_len, num_ctas: int = 0, max_batch: int = 1, max_slots=None,
              kv_pages: int = 0):
        from .predictor_graph import PredictorGraph
        from .talker_graph import TalkerGraph
        from .weights import engine_for_talker
        talker = base_model.model.talker
        tcfg = base_model.model.config.talker_config
        engine = engine_for_talker(talker, dtype=dtype, device=device, max_seq_len=max_seq_len, num_ctas=num_ctas,
                                   max_batch=max_batch, max_slots=max_slots, kv_pages=kv_pages)
        pg = PredictorGraph(talker.code_predictor, talker.code_predictor.model.config, tcfg.hidden_size, device=device,
                            dtype=dtype, do_sample=True, top_k=50, temperature=0.9, engine=engine)
        tg = TalkerGraph(talker.model, tcfg, device=device, dtype=dtype, max_seq_len=max_seq_len, engine=engine)
        return cls(base_model, pg, tg, device=device, dtype=dtype, max_seq_len=max_seq_len)

    @classmethod
    def from_synthetic(cls, size: str = "1.7B", device: str = "cuda", dtype: torch.dtype = torch.bfloat16,
                       max_seq_len: int = 2048, seed: int = 0, num_ctas: int = 0, with_codec: bool = True,
                       codec_config=None, max_batch: int = 1, max_slots: Optional[int] = None,
                       kv_pages: int = 0):
        """Random-init weights at the real geometry (no checkpoint exists offline)."""
        from . import synthetic
        from .codec import build_codec
        cfg = synthetic.make_config(size)
        if codec_config is None and size == "tiny":
            from .codec import Code2WavConfig
            codec_config = Code2WavConfig(codebook_size=256, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                                          intermediate_size=512, decoder_dim=512)
        st = build_codec(codec_config, seed=seed + 1, dtype=dtype, device=device) if with_codec else None
        base = synthetic.build_base_model(cfg, None, seed=seed, dtype=dtype, device=device, speech_tokenizer=st)
        base.syn_cfg = cfg
        m = cls._wrap(base, device, dtype, max_seq_len, num_ctas=num_ctas, max_batch=max_batch, max_slots=max_slots, kv_pages=kv_pages)
        return m

    def warmup(self, prefill_len: int = 100) -> None:
        if self._warmed_up:
            return
        self.predictor_graph.capture(num_warmup=3)
        self.talker_graph.capture(prefill_len=prefill_len, num_warmup=3)
        self._warmed_up = True

    def _warmup(self, prefill_len: int) -> None:
        self.warmup(prefill_len=prefill_len)

    def generate(self, text: str, language: str = "English", max_new_tokens: int = 2048, temperature: float = 0.9,
                 top_k: int = 50, do_sample: bool = True, repetition_penalty: float = 1.05) -> Tuple[list, int]:
        raise NotImplementedError("Default voice generation not yet implemented. "
                                  "Use generate_voice_clone() with reference audio.")

    def codec_launches(self) -> int:
        """kernels launched by the hand-written codec stack (bench.py gpu_launches)"""
        st = self._get_speech_tokenizer(self.model)
        if st is None or getattr(st, "backend", "torch") != "engine":
            return 0
        return int(st._lib.fq3_codec_launch_count(st._h))

    # ------------------------------------------------------------------ prompt assembly (model.py:278-581)
    def _is_synthetic(self) -> bool:
        return bool(getattr(self.model, "synthetic", False))

    @staticmethod
    def _read_audio(path) -> Tuple[np.ndarray, int]:
        """float32 samples + rate.  soundfile when installed (the reference's reader), else 16-bit PCM WAV via stdlib."""
        try:
            import soundfile as sf
            return sf.read(str(path), dtype="float32", always_2d=False)
        except ImportError:
            import wave
            with wave.open(str(path), "rb") as w:
                if w.getsampwidth() != 2:
                    raise ValueError("without soundfile only 16-bit PCM WAV reference audio can be read")
                raw = np.frombuffer(w.readframes(w.getnframes()), dtype="<i2").astype(np.float32) / 32768.0
                if w.getnchannels() > 1:
                    raw = raw.reshape(-1, w.getnchannels())
                return raw, w.getframerate()

    def _load_ref_audio_with_silence(self, ref_audio, silence_secs: float = 0.5) -> Tuple[np.ndarray, int]:
        """model.py:278-293: mono, optionally followed by silence so the ICL prompt does not end mid-phoneme."""
        audio, sr = self._read_audio(ref_audio)
        if audio.ndim > 1:
            audio = audio.mean(axis=1)
        if silence_secs > 0:
            audio = np.concatenate([audio, np.zeros(int(silence_secs * sr), dtype=np.float32)])
        return audio, sr

    def _resolve_voice_clone_prompt(self, input_ids, ref_audio, ref_text: str, xvec_only: bool, append_silence: bool,
                                    voice_clone_prompt):
        """-> (prompt dict, ref_ids, using_icl_mode)   (model.py:295-320)"""
        if voice_clone_prompt is not None:
            return self._resolve_precomputed_voice_clone_prompt(input_ids=input_ids, ref_text=ref_text,
                                                                voice_clone_prompt=voice_clone_prompt)
        if ref_audio is None:
            raise ValueError("ref_audio is required when voice_clone_prompt is not provided")
        return self._resolve_voice_clone_prompt_from_reference(input_ids=input_ids, ref_audio=ref_audio,
                                                               ref_text=ref_text, xvec_only=xvec_only,
                                                               append_silence=append_silence)

    def _ref_ids_for(self, ref_text: str):
        return self.model._tokenize_texts([self.model._build_ref_text(ref_text)])[0]

    def _resolve_precomputed_voice_clone_prompt(self, input_ids, ref_text: str, voice_clone_prompt):
        """model.py:322-413: a list of prompt items or a dict of per-request lists; validates the mode flags."""
        n = len(input_ids)
        if isinstance(voice_clone_prompt, list):
            if len(voice_clone_prompt) != n:
                raise ValueError(f"voice_clone_prompt must have length {n}, got {len(voice_clone_prompt)}")
            vcp = self.model._prompt_items_to_voice_clone_prompt(voice_clone_prompt)
            ref_ids = []
            for item in voice_clone_prompt:
                if not bool(item.icl_mode):
                    ref_ids.append(None)
                    continue
                item_text = item.ref_text if item.ref_text else ref_text
                if not item_text:
                    raise ValueError("ref_text is required when voice_clone_prompt uses ICL mode.")
                ref_ids.append(self._ref_ids_for(item_text))
            return vcp, ref_ids, any(vcp["icl_mode"])

        required = ("ref_spk_embedding",)
        missing = [k for k in required if k not in voice_clone_prompt]
        if missing:
            raise ValueError(f"voice_clone_prompt missing required keys: {missing}. Expected keys: {list(required)}")
        for key in ("ref_spk_embedding", "x_vector_only_mode", "icl_mode", "ref_code"):
            if key in voice_clone_prompt:
                value = voice_clone_prompt[key]
                if not isinstance(value, list) or len(value) != n:
                    raise ValueError(f"voice_clone_prompt[{key!r}] must be a list with length {n}")
        xvec = voice_clone_prompt.get("x_vector_only_mode", [True] * n)
        if "icl_mode" in voice_clone_prompt:
            icl = [bool(v) for v in voice_clone_prompt["icl_mode"]]
            for i, (x, c) in enumerate(zip(xvec, icl)):
                if bool(x) == bool(c):
                    raise ValueError(f"voice_clone_prompt has inconsistent mode flags at index {i}: "
                                     "x_vector_only_mode and icl_mode must be opposites")
        else:
            icl = [not bool(v) for v in xvec]
        codes = voice_clone_prompt.get("ref_code", [None] * n)
        for i, (x, c, code) in enumerate(zip(xvec, icl, codes)):
            if bool(x) and code is not None:
                raise ValueError(f"voice_clone_prompt index {i}: ref_code must be None in x_vector_only mode")
            if bool(c) and code is None:
                raise ValueError(f"voice_clone_prompt index {i}: ref_code is required in ICL mode")
        vcp = dict(ref_code=codes, ref_spk_embedding=voice_clone_prompt["ref_spk_embedding"],
                   x_vector_only_mode=[bool(v) for v in xvec], icl_mode=[bool(v) for v in icl])
        if not any(vcp["icl_mode"]):
            return vcp, [None] * n, False
        if not ref_text:
            raise ValueError("ref_text is required when voice_clone_prompt uses ICL mode.")
        shared = self._ref_ids_for(ref_text)        # one ref_text is shared by every ICL item of the batch
        return vcp, [shared if c else None for c in vcp["icl_mode"]], True

    def _resolve_voice_clone_prompt_from_reference(self, input_ids, ref_audio, ref_text: str, xvec_only: bool,
                                                   append_silence: bool):
        """model.py:415-463: speaker vector (+ codec frames and reference-text ids for ICL), cached per reference."""
        using_icl = not xvec_only
        key = (str(ref_audio), ref_text, xvec_only, append_silence)
        if key in self._voice_prompt_cache:
            vcp, ref_ids = self._voice_prompt_cache[key]
            return vcp, ref_ids, using_icl
        if xvec_only:
            items = self.model.create_voice_clone_prompt(ref_audio=str(ref_audio), ref_text="", x_vector_only_mode=True)
            vcp = dict(ref_code=[None], ref_spk_embedding=[items[0].ref_spk_embedding], x_vector_only_mode=[True],
                       icl_mode=[False])
            ref_ids = [None] * len(input_ids)
        else:
            try:
                audio_in = self._load_ref_audio_with_silence(ref_audio, silence_secs=0.5 if append_silence else 0.0)
            except (OSError, EOFError, ValueError):
                if not self._is_synthetic():
                    raise
                audio_in = str(ref_audio)   # synthetic voices are derived from the name; nothing has to be readable
            items = self.model.create_voice_clone_prompt(ref_audio=audio_in, ref_text=ref_text)
            vcp = self.model._prompt_items_to_voice_clone_prompt(items)
            rt = items[0].ref_text
            ref_ids = [self._ref_ids_for(rt) if rt else None]
        self._voice_prompt_cache[key] = (vcp, ref_ids)
        return vcp, ref_ids, using_icl

    def _prepare_generation(self, text, ref_audio=None, ref_text="", language="English", xvec_only=False,
                            non_streaming_mode=False, append_silence=True, voice_clone_prompt=None, instruct=None):
        """Inputs of the decode path for voice cloning (model.py:465-543); `xvec_only` is ignored when a precomputed
        `voice_clone_prompt` is given."""
        from .prompt import build_talker_inputs
        input_ids = self.model._tokenize_texts([self.model._build_assistant_text(text)])
        instruct_ids = [None]
        if instruct:
            instruct_ids = [self.model._tokenize_texts([self.model._build_instruct_text(instruct)])[0]]
        vcp, ref_ids, using_icl = self._resolve_voice_clone_prompt(
            input_ids=input_ids, ref_audio=ref_audio, ref_text=ref_text, xvec_only=xvec_only,
            append_silence=append_silence, voice_clone_prompt=voice_clone_prompt)
        if instruct and not using_icl:
            logger.warning("Base-model instruct with x-vector-only voice cloning is experimental; prefer xvec_only=False "
                           "(ICL mode) when using instruct for voice cloning.")
        m = self.model.model
        tie, tam, tth, tpe = build_talker_inputs(
            m, input_ids=input_ids, ref_ids=ref_ids, voice_clone_prompt=vcp,
            languages=[language] if language is not None else ["Auto"], speakers=None,
            non_streaming_mode=non_streaming_mode, instruct_ids=instruct_ids)
        if not self._warmed_up:
            self.warmup(tie.shape[1])
        talker = m.talker
        talker.rope_deltas = None
        ref_codes = None   # ICL: the decoder gets the reference frames as acoustic context (model.py:536-539)
        if using_icl and vcp.get("ref_code") and vcp["ref_code"][0] is not None:
            ref_codes = vcp["ref_code"][0]
        return m, talker, m.config.talker_config, tie, tam, tth, tpe, ref_codes

    def _prepare_generation_custom(self, text, language, speaker, instruct=None, non_streaming_mode=True):
        """Inputs for one custom-voice / voice-design request (model.py:545-581): the one-row call of
        ``_prepare_generation_custom_batch``; voice design has speaker None."""
        return self._prepare_generation_custom_batch([text], [language], [speaker], [instruct], non_streaming_mode)

    def _prepare_generation_custom_batch(self, texts, languages, speakers, instructs, non_streaming_mode):
        """Inputs for custom-voice / voice-design requests, one row per text, left-padded like the reference's builder
        pads a list of requests (model.py:583-805)."""
        from .prompt import build_talker_inputs
        input_ids = self.model._tokenize_texts([self.model._build_assistant_text(t) for t in texts])
        instruct_ids = [self.model._tokenize_texts([self.model._build_instruct_text(i)])[0] if i else None
                        for i in instructs]
        m = self.model.model
        tie, tam, tth, tpe = build_talker_inputs(
            m, input_ids=input_ids, ref_ids=[None] * len(texts), voice_clone_prompt=None,
            languages=[l if l is not None else "Auto" for l in languages], speakers=list(speakers),
            non_streaming_mode=non_streaming_mode, instruct_ids=instruct_ids)
        if not self._warmed_up:
            self.warmup(tie.shape[1])
        m.talker.rope_deltas = None
        return m, m.talker, m.config.talker_config, tie, tam, tth, tpe

    # ------------------------------------------------------------------ codec helpers
    @staticmethod
    def _to_numpy(a):
        if hasattr(a, "cpu"):   # encoded output (int16 / uint8) leaves the device as it is
            return (a.flatten().float() if a.is_floating_point() else a.flatten()).cpu().numpy()
        return a.flatten() if hasattr(a, "flatten") else a

    def _decode_all(self, speech_tokenizer, codec_ids, ref_codes, speed=1.0, sample_rate=None, pitch=0.0, gain_db=0.0):
        """Non-streaming decode + proportional reference trim (model.py:918-938)."""
        return self._decode_takes(speech_tokenizer, [codec_ids], ref_codes, **_post_kw(speed, sample_rate, pitch, gain_db))

    def _stream_audio(self, chunks, speech_tokenizer, ref_codes, chunk_size, to_host=True, speed=1.0,
                      sample_rate=None, pitch=0.0, gain_db=0.0):
        """The reference's hybrid streaming decode (model.py:1052-1135): Phase 1 re-decodes everything so far
        (reference codes prepended in ICL mode) until max(25, chunk_size) frames exist and calibrates
        samples_per_frame; Phase 2 decodes a 25-frame left-context window and trims the context.  At a speed other than
        1, or an output rate other than 24 kHz, the stream ends with one more item: the last samples of the tempo and
        the resampler (``chunk_steps`` 0)."""
        win = self._make_window(speech_tokenizer, ref_codes, chunk_size, to_host, **_post_kw(speed, sample_rate, pitch, gain_db))
        timing = {}
        for codec_chunk, timing in chunks:
            new_audio, sr = win.push(codec_chunk)
            yield new_audio, sr, timing
        for _, (tail, sr) in zip(*flush_windows(speech_tokenizer, [win])):
            yield tail, sr, dict(timing, chunk_steps=0, is_final=True)

    def _make_window(self, speech_tokenizer, ref_codes, chunk_size, to_host=True, speed=1.0, sample_rate=None,
                     encoding="f32", pitch=0.0, gain_db=0.0):
        """the codec window of one request; at a speed or pitch other than 1 / 0 it carries the request's
        ``tempo.Tempo`` (at ``resample.tempo_speed``), at an output rate or encoding other than 24 kHz f32, a pitch or a
        gain its ``resample.Resampler``; ``encoding="flac"`` is an s16 resampler followed by a ``flac.Encoder``"""
        if self.streaming_codec not in ("window", "stateful"):
            raise ValueError("streaming_codec must be 'window' or 'stateful'")
        kw = _stages(speech_tokenizer, speed, sample_rate, encoding, pitch, gain_db)
        if self.streaming_codec == "stateful" and getattr(speech_tokenizer, "supports_streams", False):
            return _StatefulWindow(self, speech_tokenizer, ref_codes, chunk_size, to_host, **kw)
        return _StreamWindow(self, speech_tokenizer, ref_codes, chunk_size, to_host, **kw)

    @staticmethod
    def _gen_kwargs(max_new_tokens, min_new_tokens, temperature, top_k, top_p, do_sample, repetition_penalty):
        return dict(max_new_tokens=max_new_tokens, min_new_tokens=min_new_tokens, temperature=temperature, top_k=top_k,
                    top_p=top_p, do_sample=do_sample, repetition_penalty=repetition_penalty)

    # ------------------------------------------------------------------ the embeddings-in entry (bench / servers)
    @torch.inference_mode()
    def stream_from_embeds(self, tie, tam, tth, tpe, ref_codes=None, chunk_size: int = 8, to_host: bool = True,
                           max_new_tokens: int = 2048, min_new_tokens: int = 2, temperature: float = 0.9,
                           top_k: int = 50, top_p: float = 1.0, do_sample: bool = True,
                           repetition_penalty: float = 1.05, uniforms=None, speed: float = 1.0,
                           sample_rate: Optional[int] = None, pitch: float = 0.0, gain_db: float = 0.0):
        """generate_voice_clone_streaming from the point where the prompt embeddings exist (model.py:1079-1137).
        ``speed``: speaking rate in [0.25, 4.0]; ``sample_rate``: output rate (None: 24000), one of
        ``resample.RATES`` (see ``_stream_audio``)."""
        from .streaming import fast_generate_streaming
        _check_speed(speed, pitch, gain_db)
        _check_rate(sample_rate)
        m = self.model.model
        m.talker.rope_deltas = None
        chunks = fast_generate_streaming(
            talker=m.talker, talker_input_embeds=tie, attention_mask=tam, trailing_text_hiddens=tth, tts_pad_embed=tpe,
            config=m.config.talker_config, chunk_size=chunk_size, uniforms=uniforms,
            predictor_graph=self.predictor_graph, talker_graph=self.talker_graph,
            **self._gen_kwargs(max_new_tokens, min_new_tokens, temperature, top_k, top_p, do_sample, repetition_penalty))
        st = m.speech_tokenizer
        if st is None:
            for codes, timing in chunks:
                yield (codes.cpu().numpy() if to_host else codes), self.sample_rate, timing
            return
        yield from self._stream_audio(chunks, st, ref_codes, chunk_size, to_host=to_host,
                                      **_post_kw(speed, sample_rate, pitch, gain_db))

    @torch.inference_mode()
    def stream_batch_from_embeds(self, tie, tam, tth, tpe, ref_codes=None, chunk_size: int = 8, to_host: bool = True,
                                 max_new_tokens: int = 2048, min_new_tokens: int = 2, temperature: float = 0.9,
                                 top_k: int = 50, top_p: float = 1.0, do_sample: bool = True,
                                 repetition_penalty: float = 1.05, uniforms=None, decode_audio: bool = True,
                                 speed: float = 1.0, sample_rate: Optional[int] = None, pitch: float = 0.0, gain_db: float = 0.0):
        """Batched streaming from the point where the (left-padded) prompt batch exists (the tuple
        ``_build_talker_inputs_local`` returns for a list of requests, model.py:774-805): all rows advance together, one
        persistent-kernel launch per chunk; yields [(row, pcm_or_codes, sr, timing)] per chunk.  ``ref_codes``: None or
        a list with one entry per row (ICL reference frames / None).  ``speed``: speaking rate of every row, in [0.25,
        4.0]; ``sample_rate``: output rate of every row (None: 24000); other than the identity, a last item holds every
        row's final samples (``chunk_steps`` 0)."""
        from .batching import fast_generate_streaming_batch
        _check_speed(speed, pitch, gain_db)
        _check_rate(sample_rate)
        m = self.model.model
        m.talker.rope_deltas = None
        B = tie.shape[0]
        st = m.speech_tokenizer if decode_audio else None
        wins = None
        if st is not None:
            wins = [self._make_window(st, None if ref_codes is None else ref_codes[b], chunk_size, to_host,
                                      **_post_kw(speed, sample_rate, pitch, gain_db)) for b in range(B)]
        kw = self._gen_kwargs(max_new_tokens, min_new_tokens, temperature, top_k, top_p, do_sample, repetition_penalty)
        for items in fast_generate_streaming_batch(
                talker=m.talker, talker_input_embeds=tie, attention_mask=tam, trailing_text_hiddens=tth,
                tts_pad_embed=tpe, config=m.config.talker_config, chunk_size=chunk_size, uniforms=uniforms,
                predictor_graph=self.predictor_graph, talker_graph=self.talker_graph, **kw):
            if wins is None:
                yield [(b, codes.cpu().numpy() if to_host else codes, self.sample_rate, timing) for b, codes, timing in items]
                continue
            dec = decode_windows_batched(st, [wins[b] for b, _, _ in items], [codes for _, codes, _ in items])
            yield [(b, audio, sr, timing) for (b, _, timing), (audio, sr) in zip(items, dec)]
        if wins is not None:
            ended, tails = flush_windows(st, wins)
            if ended:
                yield [(wins.index(w), audio, sr, {"chunk_steps": 0, "is_final": True}) for w, (audio, sr) in zip(ended, tails)]

    @torch.inference_mode()
    def generate_custom_voice_batch(self, texts: List[str], speakers: List[str], languages: List[str],
                                    instructs: Optional[List[Optional[str]]] = None, max_new_tokens: int = 2048,
                                    min_new_tokens: int = 2, temperature: float = 0.9, top_k: int = 50,
                                    top_p: float = 1.0, do_sample: bool = True, repetition_penalty: float = 1.05,
                                    non_streaming_mode: Optional[bool] = None, chunk_size: int = 8,
                                    speed: float = 1.0, sample_rate: Optional[int] = None, pitch: float = 0.0, gain_db: float = 0.0):
        """Concurrent custom-voice requests (BASELINE config 4) sharing every pass over the weights: the prompts are
        batched and left-padded exactly like the reference's builder does for a list of requests (model.py:583-805),
        then decoded together.  ``speed`` (one for all requests): speaking rate in [0.25, 4.0], and ``sample_rate``: output
        rate (None: 24000), both applied on the device.  Returns ([audio per request], sample_rate)."""
        _check_speed(speed, pitch, gain_db)
        _check_rate(sample_rate)
        instructs, nsm = self._custom_voice_rules(texts, languages, speakers, instructs or [None] * len(texts),
                                                  non_streaming_mode)
        _, _, _, tie, tam, tth, tpe = self._prepare_generation_custom_batch(texts, languages, speakers, instructs, nsm)
        parts = [[] for _ in texts]
        sr = _rate_of(self.sample_rate, sample_rate)
        for items in self.stream_batch_from_embeds(tie, tam, tth, tpe, chunk_size=chunk_size, **_post_kw(speed, sample_rate, pitch, gain_db), **self._gen_kwargs(
                max_new_tokens, min_new_tokens, temperature, top_k, top_p, do_sample, repetition_penalty)):
            for b, audio, sr, _ in items:
                parts[b].append(audio)
        return [np.concatenate(p) if p else np.zeros(0, dtype=np.float32) for p in parts], sr

    # ------------------------------------------------------------------ voice clone
    @torch.inference_mode()
    def generate_voice_clone(self, text: str, language: str, ref_audio=None, ref_text: str = "",
                             max_new_tokens: int = 2048, min_new_tokens: int = 2, temperature: float = 0.9,
                             top_k: int = 50, top_p: float = 1.0, do_sample: bool = True,
                             repetition_penalty: float = 1.05, xvec_only: bool = False,
                             non_streaming_mode: Optional[bool] = None, append_silence: bool = True,
                             instruct: Optional[str] = None, ref_spk=None, ref_rvq=None, ref_spk_emb=None,
                             ref_codes=None, voice_clone_prompt=None, speed: float = 1.0,
                             sample_rate: Optional[int] = None, pitch: float = 0.0, gain_db: float = 0.0, split: bool = False,
                              max_segment_chars: int = 400, pause_ms: int = 0, seed: Optional[int] = None) -> Tuple[list, int]:
        _check_speed(speed, pitch, gain_db)
        _check_rate(sample_rate)
        voice_clone_prompt, nsm = self._voice_clone_rules(voice_clone_prompt, non_streaming_mode, ref_spk, ref_rvq,
                                                          ref_spk_emb, ref_codes)
        if self._check_split(split, max_segment_chars, pause_ms, seed):
            return self._split_one_shot(
                self._clone_make(language, ref_audio, ref_text, xvec_only, nsm, append_silence, voice_clone_prompt,
                                 instruct), text, max_segment_chars, pause_ms, seed, 12,
                self._gen_kwargs(max_new_tokens, min_new_tokens, temperature, top_k, top_p, do_sample,
                                 repetition_penalty), **_post_kw(speed, sample_rate, pitch, gain_db))
        *prep, ref_codes = self._prepare_generation(
            text=text, language=language, ref_audio=ref_audio, ref_text=ref_text, xvec_only=xvec_only,
            non_streaming_mode=nsm, append_silence=append_silence, voice_clone_prompt=voice_clone_prompt,
            instruct=instruct)
        return self._one_shot(prep, ref_codes, self._gen_kwargs(max_new_tokens, min_new_tokens, temperature, top_k,
                                                                top_p, do_sample, repetition_penalty), speed, sample_rate, pitch, gain_db)

    @torch.inference_mode()
    def generate_voice_clone_streaming(self, text: str, language: str, ref_audio=None, ref_text: str = "",
                                       max_new_tokens: int = 2048, min_new_tokens: int = 2, temperature: float = 0.9,
                                       top_k: int = 50, top_p: float = 1.0, do_sample: bool = True,
                                       repetition_penalty: float = 1.05, chunk_size: int = 12,
                                       xvec_only: bool = False, non_streaming_mode: Optional[bool] = None,
                                       append_silence: bool = True, parity_mode: bool = False,
                                       instruct: Optional[str] = None, ref_spk=None, ref_rvq=None, ref_spk_emb=None,
                                       ref_codes=None, voice_clone_prompt=None, speed: float = 1.0,
                                       sample_rate: Optional[int] = None, pitch: float = 0.0, gain_db: float = 0.0, split: bool = False,
                              max_segment_chars: int = 400, pause_ms: int = 0, seed: Optional[int] = None
                                       ) -> Generator[Tuple[np.ndarray, int, dict], None, None]:
        _check_speed(speed, pitch, gain_db)
        _check_rate(sample_rate)
        voice_clone_prompt, nsm = self._voice_clone_rules(voice_clone_prompt, non_streaming_mode, ref_spk, ref_rvq,
                                                          ref_spk_emb, ref_codes)
        if self._check_split(split, max_segment_chars, pause_ms, seed):
            if parity_mode:
                raise ValueError("split=True runs on the engine's batched decode, not the parity_mode baseline")
            yield from self._split_stream(
                self._clone_make(language, ref_audio, ref_text, xvec_only, nsm, append_silence, voice_clone_prompt,
                                 instruct), text, max_segment_chars, pause_ms, seed, chunk_size,
                self._gen_kwargs(max_new_tokens, min_new_tokens, temperature, top_k, top_p, do_sample,
                                 repetition_penalty), **_post_kw(speed, sample_rate, pitch, gain_db))
            return
        m, talker, config, tie, tam, tth, tpe, ref_codes = self._prepare_generation(
            text=text, language=language, ref_audio=ref_audio, ref_text=ref_text, xvec_only=xvec_only,
            non_streaming_mode=nsm, append_silence=append_silence, voice_clone_prompt=voice_clone_prompt,
            instruct=instruct)
        gen = self._gen_kwargs(max_new_tokens, min_new_tokens, temperature, top_k, top_p, do_sample, repetition_penalty)
        if parity_mode:   # the reference's dynamic-cache baseline (model.py:1064-1077 -> streaming.py:192-359)
            from .streaming import parity_generate_streaming
            chunks = parity_generate_streaming(
                talker=talker, talker_input_embeds=tie, attention_mask=tam, trailing_text_hiddens=tth, tts_pad_embed=tpe,
                config=config, chunk_size=chunk_size, **gen)
            yield from self._stream_audio(chunks, m.speech_tokenizer, ref_codes, chunk_size, **_post_kw(speed, sample_rate, pitch, gain_db))
            return
        yield from self.stream_from_embeds(tie, tam, tth, tpe, ref_codes=ref_codes, chunk_size=chunk_size,
                                           **_post_kw(speed, sample_rate, pitch, gain_db), **gen)

    def _voice_clone_rules(self, voice_clone_prompt, non_streaming_mode, ref_spk=None, ref_rvq=None, ref_spk_emb=None,
                           ref_codes=None):
        """What every voice-clone request checks before anything is tokenized -> (voice_clone_prompt, non_streaming_mode
        with the voice-clone default False).

        ``.spk`` / ``.rvq`` FILES are qwentts.cpp's own on-disk formats (read by qwentts-cpp-python,
        ggml_backend.py:476-509): like the reference's torch backend they are refused here with the reference's message
        (tests/test_voice_clone_prompt_api.py:116-134).  The DECODED form of such a cached reference -- ``ref_spk_emb`` (the
        speaker vector) and ``ref_codes`` (the reference's codec frames) as arrays -- is accepted and becomes the
        ``voice_clone_prompt``, see ``_cached_reference_prompt``."""
        if any(v is not None for v in (ref_spk, ref_rvq)):
            raise NotImplementedError(
                "ref_spk/ref_rvq cached qwentts.cpp references require backend='ggml'. "
                "Use voice_clone_prompt for precomputed prompts with the torch backend.")
        return (self._cached_reference_prompt(ref_spk_emb, ref_codes, voice_clone_prompt),
                self._resolve_non_streaming_mode(non_streaming_mode, default=False))

    # ------------------------------------------------------------------ custom voice / voice design
    def _require_type(self, kind: str, msg: str):
        t = getattr(self.model.model, "tts_model_type", None)
        if t is not None and t != kind:
            raise ValueError(msg)
        if t is None and not self._is_synthetic():
            raise ValueError(msg)

    def _validate(self, language, speaker=None, check_speaker=False):
        """upstream's own validators, called exactly where the reference calls them (model.py:1158-1159,1243-1244,
        1346,1426); a wrapped model without them (duck-typed test doubles) is not validated."""
        v = getattr(self.model, "_validate_languages", None)
        if v is not None:
            v([language])
        if check_speaker:
            v = getattr(self.model, "_validate_speakers", None)
            if v is not None:
                v([speaker])

    def _custom_voice_rules(self, texts, languages, speakers, instructs, non_streaming_mode):
        """What every custom-voice request checks before anything is tokenized: the model type, one speaker and language
        per text and upstream's validators.  -> (instructs, non_streaming_mode with the custom-voice default True); the
        0.6B custom-voice checkpoint ignores instructions, so they are dropped (model.py:1166-1167,1251-1252)."""
        self._require_type("custom_voice", "Loaded model does not support custom voice generation")
        if not (len(speakers) == len(texts) and len(languages) == len(texts)):
            raise ValueError("texts, speakers and languages must have the same length")
        for language, speaker in zip(languages, speakers):
            self._validate(language, speaker, check_speaker=True)
        size = getattr(self.model.model, "tts_model_size", None)
        if size is not None and size in "0b6":
            instructs = [None] * len(instructs)
        return instructs, self._resolve_non_streaming_mode(non_streaming_mode, default=True)

    def _voice_design_rules(self, language, non_streaming_mode):
        """What every voice-design request checks before anything is tokenized -> non_streaming_mode with the
        voice-design default True."""
        self._require_type("voice_design", "Loaded model does not support voice design generation")
        self._validate(language)
        return self._resolve_non_streaming_mode(non_streaming_mode, default=True)

    def _split_stream(self, make, text, max_segment_chars, pause_ms, seed, chunk_size, gen, speed=1.0,
                      sample_rate=None, pitch=0.0, gain_db=0.0):
        """A ``split=True`` request (DESIGN.md "Long inputs"): ``text`` cut by ``segment.split_text``, one row per
        segment with the prompt ``make(segment_text)()`` builds, all decoded side by side through a
        ``serving.ContinuousBatcher`` on this model and joined on the device; yields (audio, sample_rate, timing)."""
        from .serving import segment_requests
        yield from self._segments_stream(segment_requests(make, text, max_segment_chars), pause_ms, seed, chunk_size,
                                         gen, speed, sample_rate, pitch, gain_db)

    def _segments_stream(self, segs, pause_ms, seed, chunk_size, gen, speed=1.0, sample_rate=None, pitch=0.0,
                         gain_db=0.0):
        """``serving.Segments`` spoken side by side through a ``serving.ContinuousBatcher`` on this model and joined on
        the device; yields (audio, sample_rate, timing)."""
        from .serving import batcher_for_model
        b = batcher_for_model(self, chunk_size=chunk_size)
        try:
            ticket = b.submit(segs, split=True, pause_ms=pause_ms, seed=seed, **_post_kw(speed, sample_rate, pitch, gain_db),
                              **gen)
            yield from ticket
        finally:
            b.close()

    def _clone_make(self, language, ref_audio, ref_text, xvec_only, nsm, append_silence, voice_clone_prompt, instruct):
        """segment text -> ``prepare`` of its voice-clone prompt (same voice for every segment)"""
        def make(text):
            return lambda: self._prepare_generation(
                text=text, language=language, ref_audio=ref_audio, ref_text=ref_text, xvec_only=xvec_only,
                non_streaming_mode=nsm, append_silence=append_silence, voice_clone_prompt=voice_clone_prompt,
                instruct=instruct)[3:]
        return make

    def _custom_make(self, language, speaker, instruct, nsm):
        """segment text -> ``prepare`` of its custom-voice (voice-design: speaker None) prompt"""
        def make(text):
            return lambda: self._prepare_generation_custom(text, language, speaker, instruct, nsm)[3:] + (None,)
        return make

    def _split_one_shot(self, *args, **kw):
        return self._collect(self._split_stream(*args, **kw), kw.get("sample_rate"))

    def _collect(self, chunks, sample_rate):
        sr, parts = None, []
        for audio, sr, _ in chunks:
            parts.append(audio)
        if sr is None:
            sr = _rate_of(self.sample_rate, sample_rate)
        return [np.concatenate(parts) if parts else np.zeros(1, dtype=np.float32)], sr

    # ------------------------------------------------------------------ SSML
    _SAMPLING = dict(max_new_tokens=2048, min_new_tokens=2, temperature=0.9, top_k=50, top_p=1.0, do_sample=True,
                     repetition_penalty=1.05)

    @torch.inference_mode()
    def speak_ssml(self, ssml: str, voices: Dict[str, dict], voice: Optional[str] = None, language: str = "Auto",
                      max_segment_chars: int = 400, pause_ms: int = 0, seed: Optional[int] = None, speed: float = 1.0,
                      pitch: float = 0.0, gain_db: float = 0.0, sample_rate: Optional[int] = None,
                      **sampling) -> Tuple[list, int]:
        """An SSML document (``ssml.py``; DESIGN.md "SSML") spoken as segment rows and joined on the device.  ``voices``:
        name -> voice spec (``ssml.voice_request``); ``voice``: the name spoken outside every ``<voice>``;
        ``pause_ms``: the pause at an inner boundary without a ``<break>``; ``speed`` / ``pitch`` / ``gain_db`` /
        ``sample_rate`` apply once to the joined stream, on top of the document's prosody; ``sampling``: the keywords
        of ``generate_custom_voice`` from ``max_new_tokens`` to ``repetition_penalty`` (``max_new_tokens`` is per
        segment).  Returns ([audio], sample_rate).  (Not a ``generate_*`` method: those share one argument layout, with
        ``text`` first and ``pitch`` / ``gain_db`` right after ``sample_rate``.)"""
        return self._collect(self.speak_ssml_streaming(
            ssml, voices, voice, language, max_segment_chars, pause_ms, seed, speed, pitch, gain_db, sample_rate,
            **sampling), sample_rate)

    @torch.inference_mode()
    def speak_ssml_streaming(self, ssml: str, voices: Dict[str, dict], voice: Optional[str] = None,
                                language: str = "Auto", max_segment_chars: int = 400, pause_ms: int = 0,
                                seed: Optional[int] = None, speed: float = 1.0, pitch: float = 0.0, gain_db: float = 0.0,
                                sample_rate: Optional[int] = None, chunk_size: int = 12, **sampling
                                ) -> Generator[Tuple[np.ndarray, int, dict], None, None]:
        """``speak_ssml`` as a stream of (audio, sample_rate, timing); the timing carries ``segment`` and
        ``n_segments``."""
        from .serving import ssml_request
        _check_speed(speed, pitch, gain_db)
        _check_rate(sample_rate)
        self._check_split(True, max_segment_chars, pause_ms, seed)
        unknown = set(sampling) - set(self._SAMPLING)
        if unknown:
            raise TypeError(f"speak_ssml got unexpected keyword arguments {sorted(unknown)}")
        segs = ssml_request(self, ssml, voices, voice, language, max_segment_chars)
        yield from self._segments_stream(segs, pause_ms, seed, chunk_size, dict(self._SAMPLING, **sampling),
                                         **_post_kw(speed, sample_rate, pitch, gain_db))

    @staticmethod
    def _check_split(split, max_segment_chars, pause_ms, seed=None):
        """the long-input arguments, refused (ValueError) before anything is tokenized; ``seed`` is the seed of a split
        request (``segment.segment_seed``) and is refused without ``split``"""
        from .join import check_pause
        from .segment import check_max_chars
        check_max_chars(max_segment_chars)
        check_pause(pause_ms)
        if seed is not None and not split:
            raise ValueError("seed= is the seed of a split request: it needs split=True")
        return bool(split)

    def _one_shot(self, prep, ref_codes, gen, speed=1.0, sample_rate=None, pitch=0.0, gain_db=0.0):
        """The delivery of the three one-shot methods: generate, then decode every frame at once (model.py:893-947),
        time-stretched on the device at a speed other than 1, resampled at an output rate other than 24 kHz."""
        from .generate import fast_generate
        m, talker, config, tie, tam, tth, tpe = prep
        codec_ids, timing = fast_generate(
            talker=talker, talker_input_embeds=tie, attention_mask=tam, trailing_text_hiddens=tth, tts_pad_embed=tpe,
            config=config, predictor_graph=self.predictor_graph, talker_graph=self.talker_graph, **gen)
        if codec_ids is None:
            logger.warning("Generation returned no tokens")
            return [np.zeros(1, dtype=np.float32)], _rate_of(self.sample_rate, sample_rate)
        audio, sr = self._decode_all(m.speech_tokenizer, codec_ids, ref_codes, **_post_kw(speed, sample_rate, pitch, gain_db))
        self._log_rtf(timing)
        return audio, sr

    @torch.inference_mode()
    def generate_custom_voice(self, text: str, speaker: str, language: str, instruct: Optional[str] = None,
                              non_streaming_mode: Optional[bool] = None, max_new_tokens: int = 2048,
                              min_new_tokens: int = 2, temperature: float = 0.9, top_k: int = 50, top_p: float = 1.0,
                              do_sample: bool = True, repetition_penalty: float = 1.05, speed: float = 1.0,
                              sample_rate: Optional[int] = None, pitch: float = 0.0, gain_db: float = 0.0, split: bool = False,
                              max_segment_chars: int = 400, pause_ms: int = 0, seed: Optional[int] = None
                              ) -> Tuple[list, int]:
        _check_speed(speed, pitch, gain_db)
        _check_rate(sample_rate)
        (instruct,), nsm = self._custom_voice_rules([text], [language], [speaker], [instruct], non_streaming_mode)
        if self._check_split(split, max_segment_chars, pause_ms, seed):
            return self._split_one_shot(
                self._custom_make(language, speaker, instruct, nsm), text, max_segment_chars, pause_ms, seed, 12,
                self._gen_kwargs(max_new_tokens, min_new_tokens, temperature, top_k, top_p, do_sample,
                                 repetition_penalty), **_post_kw(speed, sample_rate, pitch, gain_db))
        prep = self._prepare_generation_custom(text, language, speaker, instruct, nsm)
        return self._one_shot(prep, None, self._gen_kwargs(max_new_tokens, min_new_tokens, temperature, top_k, top_p,
                                                           do_sample, repetition_penalty), speed, sample_rate, pitch, gain_db)

    @torch.inference_mode()
    def generate_custom_voice_streaming(self, text: str, speaker: str, language: str, instruct: Optional[str] = None,
                                        non_streaming_mode: Optional[bool] = None, max_new_tokens: int = 2048,
                                        min_new_tokens: int = 2, temperature: float = 0.9, top_k: int = 50,
                                        top_p: float = 1.0, do_sample: bool = True, repetition_penalty: float = 1.05,
                                        chunk_size: int = 12, speed: float = 1.0,
                                        sample_rate: Optional[int] = None, pitch: float = 0.0, gain_db: float = 0.0, split: bool = False,
                              max_segment_chars: int = 400, pause_ms: int = 0, seed: Optional[int] = None
                                        ) -> Generator[Tuple[np.ndarray, int, dict], None, None]:
        _check_speed(speed, pitch, gain_db)
        _check_rate(sample_rate)
        (instruct,), nsm = self._custom_voice_rules([text], [language], [speaker], [instruct], non_streaming_mode)
        if self._check_split(split, max_segment_chars, pause_ms, seed):
            yield from self._split_stream(
                self._custom_make(language, speaker, instruct, nsm), text, max_segment_chars, pause_ms, seed,
                chunk_size, self._gen_kwargs(max_new_tokens, min_new_tokens, temperature, top_k, top_p, do_sample,
                                             repetition_penalty), **_post_kw(speed, sample_rate, pitch, gain_db))
            return
        _, _, _, tie, tam, tth, tpe = self._prepare_generation_custom(text, language, speaker, instruct, nsm)
        yield from self.stream_from_embeds(tie, tam, tth, tpe, chunk_size=chunk_size, **_post_kw(speed, sample_rate, pitch, gain_db), **self._gen_kwargs(
            max_new_tokens, min_new_tokens, temperature, top_k, top_p, do_sample, repetition_penalty))

    @torch.inference_mode()
    def generate_voice_design(self, text: str, instruct: str, language: str,
                              non_streaming_mode: Optional[bool] = None, max_new_tokens: int = 2048,
                              min_new_tokens: int = 2, temperature: float = 0.9, top_k: int = 50, top_p: float = 1.0,
                              do_sample: bool = True, repetition_penalty: float = 1.05, speed: float = 1.0,
                              sample_rate: Optional[int] = None, pitch: float = 0.0, gain_db: float = 0.0, split: bool = False,
                              max_segment_chars: int = 400, pause_ms: int = 0, seed: Optional[int] = None
                              ) -> Tuple[list, int]:
        _check_speed(speed, pitch, gain_db)
        _check_rate(sample_rate)
        nsm = self._voice_design_rules(language, non_streaming_mode)
        if self._check_split(split, max_segment_chars, pause_ms, seed):
            return self._split_one_shot(
                self._custom_make(language, None, instruct, nsm), text, max_segment_chars, pause_ms, seed, 12,
                self._gen_kwargs(max_new_tokens, min_new_tokens, temperature, top_k, top_p, do_sample,
                                 repetition_penalty), **_post_kw(speed, sample_rate, pitch, gain_db))
        prep = self._prepare_generation_custom(text, language, None, instruct, nsm)
        return self._one_shot(prep, None, self._gen_kwargs(max_new_tokens, min_new_tokens, temperature, top_k, top_p,
                                                           do_sample, repetition_penalty), speed, sample_rate, pitch, gain_db)

    @torch.inference_mode()
    def generate_voice_design_streaming(self, text: str, instruct: str, language: str,
                                        non_streaming_mode: Optional[bool] = None, max_new_tokens: int = 2048,
                                        min_new_tokens: int = 2, temperature: float = 0.9, top_k: int = 50,
                                        top_p: float = 1.0, do_sample: bool = True, repetition_penalty: float = 1.05,
                                        chunk_size: int = 12, speed: float = 1.0,
                                        sample_rate: Optional[int] = None, pitch: float = 0.0, gain_db: float = 0.0, split: bool = False,
                              max_segment_chars: int = 400, pause_ms: int = 0, seed: Optional[int] = None
                                        ) -> Generator[Tuple[np.ndarray, int, dict], None, None]:
        _check_speed(speed, pitch, gain_db)
        _check_rate(sample_rate)
        nsm = self._voice_design_rules(language, non_streaming_mode)
        if self._check_split(split, max_segment_chars, pause_ms, seed):
            yield from self._split_stream(
                self._custom_make(language, None, instruct, nsm), text, max_segment_chars, pause_ms, seed,
                chunk_size, self._gen_kwargs(max_new_tokens, min_new_tokens, temperature, top_k, top_p, do_sample,
                                             repetition_penalty), **_post_kw(speed, sample_rate, pitch, gain_db))
            return
        _, _, _, tie, tam, tth, tpe = self._prepare_generation_custom(text, language, None, instruct, nsm)
        yield from self.stream_from_embeds(tie, tam, tth, tpe, chunk_size=chunk_size, **_post_kw(speed, sample_rate, pitch, gain_db), **self._gen_kwargs(
            max_new_tokens, min_new_tokens, temperature, top_k, top_p, do_sample, repetition_penalty))

    # ------------------------------------------------------------------ several takes of one request
    def _check_takes(self, n_takes, seeds):
        """refusals of the ``*_takes`` calls, before anything is launched; returns the seeds"""
        mb = getattr(self.engine, "max_batch", 1)
        if mb < 2:
            raise ValueError("takes need an engine built with max_batch >= 2 (they decode in one batched launch)")
        if not 1 <= int(n_takes) <= mb:
            raise ValueError(f"n_takes={n_takes} must be in [1, max_batch={mb}]")
        if seeds is None:
            seeds = torch.randint(0, 2 ** 62, (int(n_takes),)).tolist()
        seeds = [int(s) for s in seeds]
        if len(seeds) != int(n_takes):
            raise ValueError(f"{len(seeds)} seeds for {n_takes} takes")
        return seeds

    def _takes(self, prep, ref_codes, seeds, gen, chunk_size=64, speed=1.0, sample_rate=None, pitch=0.0, gain_db=0.0):
        """The one implementation behind the three ``*_takes`` methods: the prompt ``prep`` latched into one slot per take
        with ONE batched prefill (``BatchScheduler.submit_many``), all takes decoded together (one launch per chunk),
        their PCM decoded with one codec call per length.  Take i draws its uniforms from ``take_uniforms(seeds[i])``."""
        from .batching import BatchScheduler
        from .logprobs import score
        m, talker, config, tie, tam, tth, tpe = prep
        talker.rope_deltas = None
        n = len(seeds)
        sched = BatchScheduler(self.engine, talker, config, self.predictor_graph, self.talker_graph)
        reqs = [dict(tie=tie, tam=tam, tth=tth, tpe=tpe, tag=i,
                     uniforms=take_uniforms(seeds[i], gen["max_new_tokens"], self.engine.device), **gen) for i in range(n)]
        sched.submit_many(reqs, logprobs=True)
        parts, done = [[] for _ in range(n)], [None] * n
        while len(sched):
            for rq, codes in sched.step(chunk_size):
                parts[rq.tag].append(codes)
                if rq.finished:
                    done[rq.tag] = rq
        codes = [torch.cat(p) if p else None for p in parts]
        scores = []
        for i, rq in enumerate(done):
            sc = score(rq.lp.frames(), rq.eos_logprob)
            sc["seed"] = seeds[i]
            scores.append(sc)
        audio, _ = self._decode_takes(m.speech_tokenizer, codes, ref_codes, **_post_kw(speed, sample_rate, pitch, gain_db))
        return audio, _rate_of(self.sample_rate, sample_rate), scores

    def _decode_takes(self, st, codes, ref_codes, speed=1.0, sample_rate=None, pitch=0.0, gain_db=0.0):
        """Non-streaming decode + proportional reference trim of every take, takes of equal length in ONE codec call (the
        decoder's rows are independent); at a speed other than 1 every take is time-stretched on the device, all in ONE
        launch, and at an output rate other than 24 kHz resampled, all in ONE more launch, each as one push with flush.
        Returns (audio per take, the sample rate the codec returned, or the requested one)."""
        from . import resample, tempo
        out = [np.zeros(1, dtype=np.float32)] * len(codes)
        pcms, at = [], []
        sr = self.sample_rate
        groups = {}
        for i, c in enumerate(codes):
            if c is not None:
                groups.setdefault(int(c.shape[0]), []).append(i)
        ref_len = ref_codes.shape[0] if ref_codes is not None else 0
        for T, idxs in groups.items():
            batch = torch.stack([codes[i] if ref_codes is None else torch.cat([ref_codes.to(codes[i].device), codes[i]])
                                 for i in idxs])
            audio_list, sr = st.decode({"audio_codes": batch})
            for i, a in zip(idxs, audio_list):
                a = a.flatten()
                if ref_len > 0:
                    a = a[int(ref_len / max(batch.shape[1], 1) * len(a)):]
                if speed == 1.0 and sample_rate is None and pitch == 0 and gain_db == 0:
                    out[i] = self._to_numpy(a)
                else:
                    pcms.append(a)
                    at.append(i)
        if at:
            tempos = [tempo.tempo_for(resample.tempo_speed(speed, pitch), a.device) for a in pcms]   # None at q 1024
            if tempos[0] is not None:
                pcms = tempo.process(tempos, pcms, True)
                for t in tempos:
                    t.close()
            rss = [resample.resampler_for(sample_rate, "f32", a.device, pitch, gain_db) for a in pcms]
            if rss and rss[0] is not None:
                pcms = resample.process(rss, pcms, True)
                for r in rss:
                    r.close()
            for i, a in zip(at, pcms):
                out[i] = self._to_numpy(a)
        return out, _rate_of(sr, sample_rate)

    @torch.inference_mode()
    def generate_voice_clone_takes(self, text: str, language: str, ref_audio=None, ref_text: str = "",
                                   max_new_tokens: int = 2048, min_new_tokens: int = 2, temperature: float = 0.9,
                                   top_k: int = 50, top_p: float = 1.0, do_sample: bool = True,
                                   repetition_penalty: float = 1.05, xvec_only: bool = False,
                                   non_streaming_mode: Optional[bool] = None, append_silence: bool = True,
                                   instruct: Optional[str] = None, voice_clone_prompt=None, speed: float = 1.0,
                                   sample_rate: Optional[int] = None, pitch: float = 0.0,
                                   gain_db: float = 0.0, split: bool = False, max_segment_chars: int = 400,
                                    pause_ms: int = 0, n_takes: int = 4, seeds: Optional[List[int]] = None):
        """``n_takes`` renderings of one ``generate_voice_clone`` request for the price of one batched decode: one prompt,
        one batched prefill, one launch per chunk for all takes.  Take i is the request run alone with the uniforms of
        ``take_uniforms(seeds[i], max_new_tokens)`` -- bit for bit while both run the per-head talker attention (a lone
        request past 192 cached keys switches to the split-key path unless ``FQ3_ATTN_SPLIT=0``).  Returns (audios, sample_rate, scores): ``scores[i]``
        holds "logprobs" (float32 [T,16], the log-probability of every code), "eos_logprob", "total_logprob" (their sum,
        EOS term included), "frames" and "seed".  A log-probability says how likely the sampler found its draws, not
        how good the audio is: the calls rank nothing and pick nothing."""
        _refuse_split(split)
        _check_speed(speed, pitch, gain_db)
        _check_rate(sample_rate)
        voice_clone_prompt, nsm = self._voice_clone_rules(voice_clone_prompt, non_streaming_mode)
        seeds = self._check_takes(n_takes, seeds)
        *prep, ref_codes = self._prepare_generation(
            text=text, language=language, ref_audio=ref_audio, ref_text=ref_text, xvec_only=xvec_only,
            non_streaming_mode=nsm, append_silence=append_silence, voice_clone_prompt=voice_clone_prompt,
            instruct=instruct)
        return self._takes(prep, ref_codes, seeds, self._gen_kwargs(max_new_tokens, min_new_tokens, temperature, top_k,
                                                                    top_p, do_sample, repetition_penalty), speed=speed,
                           sample_rate=sample_rate, pitch=pitch, gain_db=gain_db)

    @torch.inference_mode()
    def generate_custom_voice_takes(self, text: str, speaker: str, language: str, instruct: Optional[str] = None,
                                    non_streaming_mode: Optional[bool] = None, max_new_tokens: int = 2048,
                                    min_new_tokens: int = 2, temperature: float = 0.9, top_k: int = 50,
                                    top_p: float = 1.0, do_sample: bool = True, repetition_penalty: float = 1.05,
                                    speed: float = 1.0, sample_rate: Optional[int] = None, pitch: float = 0.0,
                                    gain_db: float = 0.0, split: bool = False, max_segment_chars: int = 400,
                                    pause_ms: int = 0, n_takes: int = 4,
                                    seeds: Optional[List[int]] = None):
        """``n_takes`` renderings of one ``generate_custom_voice`` request (see ``generate_voice_clone_takes``)."""
        _refuse_split(split)
        _check_speed(speed, pitch, gain_db)
        _check_rate(sample_rate)
        (instruct,), nsm = self._custom_voice_rules([text], [language], [speaker], [instruct], non_streaming_mode)
        seeds = self._check_takes(n_takes, seeds)
        prep = self._prepare_generation_custom(text, language, speaker, instruct, nsm)
        return self._takes(prep, None, seeds, self._gen_kwargs(max_new_tokens, min_new_tokens, temperature, top_k,
                                                               top_p, do_sample, repetition_penalty), speed=speed,
                           sample_rate=sample_rate, pitch=pitch, gain_db=gain_db)

    @torch.inference_mode()
    def generate_voice_design_takes(self, text: str, instruct: str, language: str,
                                    non_streaming_mode: Optional[bool] = None, max_new_tokens: int = 2048,
                                    min_new_tokens: int = 2, temperature: float = 0.9, top_k: int = 50,
                                    top_p: float = 1.0, do_sample: bool = True, repetition_penalty: float = 1.05,
                                    speed: float = 1.0, sample_rate: Optional[int] = None, pitch: float = 0.0,
                                    gain_db: float = 0.0, split: bool = False, max_segment_chars: int = 400,
                                    pause_ms: int = 0, n_takes: int = 4,
                                    seeds: Optional[List[int]] = None):
        """``n_takes`` renderings of one ``generate_voice_design`` request (see ``generate_voice_clone_takes``)."""
        _refuse_split(split)
        _check_speed(speed, pitch, gain_db)
        _check_rate(sample_rate)
        nsm = self._voice_design_rules(language, non_streaming_mode)
        seeds = self._check_takes(n_takes, seeds)
        prep = self._prepare_generation_custom(text, language, None, instruct, nsm)
        return self._takes(prep, None, seeds, self._gen_kwargs(max_new_tokens, min_new_tokens, temperature, top_k,
                                                               top_p, do_sample, repetition_penalty), speed=speed,
                           sample_rate=sample_rate, pitch=pitch, gain_db=gain_db)

    # ------------------------------------------------------------------ incremental text input (text_stream.py)
    def _text_streaming(self, text_stream, language, speaker, instruct, voice_clone_prompt, non_streaming_mode,
                        chunk_size, gen, speed=1.0, sample_rate=None, pitch=0.0, gain_db=0.0):
        """The one implementation behind the three ``*_text_streaming`` methods.  Text streaming has one text layout,
        so the raw ``non_streaming_mode`` is checked here, not the voice kind's default."""
        from .text_stream import _refuse_unsupported, generate_text_streaming
        _refuse_unsupported(voice_clone_prompt, non_streaming_mode)
        instruct_ids = None
        if instruct:
            instruct_ids = self.model._tokenize_texts([self.model._build_instruct_text(instruct)])[0]
        yield from generate_text_streaming(self, text_stream, language=language, speaker=speaker,
                                           instruct_ids=instruct_ids, voice_clone_prompt=voice_clone_prompt,
                                           chunk_size=chunk_size, **_post_kw(speed, sample_rate, pitch, gain_db), **gen)

    @torch.inference_mode()
    def generate_custom_voice_text_streaming(self, text_stream, speaker: str, language: str,
                                             instruct: Optional[str] = None, non_streaming_mode: Optional[bool] = None,
                                             max_new_tokens: int = 2048, min_new_tokens: int = 2,
                                             temperature: float = 0.9, top_k: int = 50, top_p: float = 1.0,
                                             do_sample: bool = True, repetition_penalty: float = 1.05,
                                             chunk_size: int = 12, speed: float = 1.0,
                                             sample_rate: Optional[int] = None, pitch: float = 0.0, gain_db: float = 0.0, split: bool = False,
                                             max_segment_chars: int = 400, pause_ms: int = 0
                                             ) -> Generator[Tuple[np.ndarray, int, dict], None, None]:
        """``generate_custom_voice_streaming`` with the text fed while it is spoken: ``text_stream`` is any iterable of
        ``str`` pieces (an LLM's reply token by token).  The audio equals that of the one-shot streaming request for the
        same text, whatever the split and however fast the pieces come; generation waits where the text has not arrived
        yet.  Timing dicts add ``text_wait_ms``, the time spent blocked on ``text_stream``."""
        _refuse_split(split)
        _check_speed(speed, pitch, gain_db)
        _check_rate(sample_rate)
        (instruct,), _ = self._custom_voice_rules([text_stream], [language], [speaker], [instruct], non_streaming_mode)
        yield from self._text_streaming(text_stream, language, speaker, instruct, None, non_streaming_mode, chunk_size,
                                        self._gen_kwargs(max_new_tokens, min_new_tokens, temperature, top_k, top_p,
                                                         do_sample, repetition_penalty), speed, sample_rate, pitch, gain_db)

    @torch.inference_mode()
    def generate_voice_design_text_streaming(self, text_stream, instruct: str, language: str,
                                             non_streaming_mode: Optional[bool] = None, max_new_tokens: int = 2048,
                                             min_new_tokens: int = 2, temperature: float = 0.9, top_k: int = 50,
                                             top_p: float = 1.0, do_sample: bool = True,
                                             repetition_penalty: float = 1.05, chunk_size: int = 12, speed: float = 1.0,
                                             sample_rate: Optional[int] = None, pitch: float = 0.0, gain_db: float = 0.0, split: bool = False,
                                             max_segment_chars: int = 400, pause_ms: int = 0
                                             ) -> Generator[Tuple[np.ndarray, int, dict], None, None]:
        """``generate_voice_design_streaming`` with the text fed while it is spoken (see
        ``generate_custom_voice_text_streaming``)."""
        _refuse_split(split)
        _check_speed(speed, pitch, gain_db)
        _check_rate(sample_rate)
        self._voice_design_rules(language, non_streaming_mode)
        yield from self._text_streaming(text_stream, language, None, instruct, None, non_streaming_mode, chunk_size,
                                        self._gen_kwargs(max_new_tokens, min_new_tokens, temperature, top_k, top_p,
                                                         do_sample, repetition_penalty), speed, sample_rate, pitch, gain_db)

    @torch.inference_mode()
    def generate_voice_clone_text_streaming(self, text_stream, language: str, ref_audio=None, ref_text: str = "",
                                            max_new_tokens: int = 2048, min_new_tokens: int = 2,
                                            temperature: float = 0.9, top_k: int = 50, top_p: float = 1.0,
                                            do_sample: bool = True, repetition_penalty: float = 1.05,
                                            chunk_size: int = 12, xvec_only: bool = True,
                                            non_streaming_mode: Optional[bool] = None, append_silence: bool = True,
                                            ref_spk=None, ref_rvq=None, ref_spk_emb=None, ref_codes=None,
                                            voice_clone_prompt=None, speed: float = 1.0,
                                            sample_rate: Optional[int] = None, pitch: float = 0.0, gain_db: float = 0.0, split: bool = False,
                                             max_segment_chars: int = 400, pause_ms: int = 0
                                            ) -> Generator[Tuple[np.ndarray, int, dict], None, None]:
        """``generate_voice_clone_streaming`` with the text fed while it is spoken, x-vector cloning only: ICL cloning
        puts the target text under the reference codec frames inside the prompt, so it must be known before prefill
        (ValueError)."""
        _refuse_split(split)
        _check_speed(speed, pitch, gain_db)
        _check_rate(sample_rate)
        voice_clone_prompt, _ = self._voice_clone_rules(voice_clone_prompt, non_streaming_mode, ref_spk, ref_rvq,
                                                        ref_spk_emb, ref_codes)
        from .text_stream import ICL_REFUSAL, _refuse_unsupported
        _refuse_unsupported(None, non_streaming_mode)
        if voice_clone_prompt is None and not xvec_only:
            raise ValueError(ICL_REFUSAL)
        # one request: only the length of input_ids is read while a prompt is resolved
        vcp, _, _ = self._resolve_voice_clone_prompt(
            input_ids=[None], ref_audio=ref_audio, ref_text=ref_text, xvec_only=True, append_silence=append_silence,
            voice_clone_prompt=voice_clone_prompt)
        yield from self._text_streaming(text_stream, language, None, None, vcp, non_streaming_mode, chunk_size,
                                        self._gen_kwargs(max_new_tokens, min_new_tokens, temperature, top_k, top_p,
                                                         do_sample, repetition_penalty), speed, sample_rate, pitch, gain_db)

    def _log_rtf(self, timing):
        n = timing["steps"]
        total = timing["prefill_ms"] / 1000 + timing["decode_s"]
        if total > 0:
            logger.info(f"Generated {n / 12.0:.2f}s audio in {total:.2f}s ({timing['ms_per_step']:.1f}ms/step, "
                        f"RTF: {n / 12.0 / total:.2f})")
