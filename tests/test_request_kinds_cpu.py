"""Every public request method of ``FasterQwen3TTS`` (three voice kinds times one-shot, streaming, takes, text
streaming, plus the custom-voice batch) and both ``serving`` request helpers on the CPU synthetic model, with the
delivery layer replaced by recorders:

- each delivery receives the prompt ``_prepare_generation`` / ``build_talker_inputs`` build for the same request, bit
  for bit, with the caller's sampling keywords;
- bad arguments raise the same exception with the same message, the voice kind's refusals before the delivery's, and
  neither after anything was tokenized;
- an empty generation returns one zero sample and says so in the log."""
import logging
import types

import numpy as np
import pytest
import torch

from oracle import prompt_cases as PC

from faster_qwen3_tts import batching, generate, serving, streaming, text_stream  # noqa: E402
from faster_qwen3_tts.model import FasterQwen3TTS, take_uniforms  # noqa: E402
from faster_qwen3_tts.prompt import build_talker_inputs  # noqa: E402

TEXT = "Good morning, how are you today?"
REF = dict(ref_audio="voice_a.wav", ref_text="the reference words")
GEN = dict(max_new_tokens=77, min_new_tokens=3, temperature=0.7, top_k=20, top_p=0.9, do_sample=False,
           repetition_penalty=1.1)
TIMING = dict(steps=24, prefill_ms=5.0, decode_s=0.2, ms_per_step=8.0)


class _Stop(Exception):
    """the takes scheduler double stops the request once it has recorded it"""


@pytest.fixture(scope="module")
def base():
    return PC.build_base(seed=1)


@pytest.fixture
def tts(base):
    engine = types.SimpleNamespace(max_batch=4, device=torch.device("cpu"), dtype=torch.float32)
    m = FasterQwen3TTS(base, types.SimpleNamespace(engine=engine), types.SimpleNamespace(engine=engine), device="cpu",
                       dtype=torch.float32, max_seq_len=512)
    m._warmed_up = True     # no graphs to capture on CPU
    return m


@pytest.fixture
def seen(tts, monkeypatch):
    """The delivery layer as recorders: each stores what it was handed under its delivery's name."""
    rec = {}

    def fast_generate(**kw):
        rec["one_shot"] = kw
        return torch.zeros(TIMING["steps"], 16, dtype=torch.long), dict(TIMING)

    def decode_all(st, codes, ref_codes):
        rec["one_shot_ref_codes"] = ref_codes
        return [np.ones(3, dtype=np.float32)], 24000

    def parity(**kw):
        rec["parity"] = kw
        return iter(())

    def stream_audio(chunks, st, ref_codes, chunk_size, to_host=True):
        rec["parity_ref_codes"] = ref_codes
        return iter(())

    def stream_from_embeds(tie, tam, tth, tpe, **kw):
        rec["streaming"] = dict(kw, prompt=(tie, tam, tth, tpe))
        return iter(())

    def stream_batch_from_embeds(tie, tam, tth, tpe, **kw):
        rec["batch"] = dict(kw, prompt=(tie, tam, tth, tpe))
        return iter(())

    class Scheduler:
        def __init__(self, engine, talker, config, predictor_graph, talker_graph):
            assert engine is tts.engine and predictor_graph is tts.predictor_graph and talker_graph is tts.talker_graph

        def submit_many(self, reqs, logprobs=False):
            rec["takes"] = reqs
            raise _Stop

    def text_streaming(model, pieces, *, language, speaker=None, instruct_ids=None, voice_clone_prompt=None,
                       chunk_size=12, **gen):
        # the prompt a text-fed request gets once its whole text has arrived
        feed = text_stream.TextFeed(model, max_rows=gen["max_new_tokens"])
        for p in pieces:
            feed.push(p)
        feed.close()
        tie, tam, tpe = text_stream.build_prompt(model, feed, language=language, speaker=speaker,
                                                 instruct_ids=instruct_ids, voice_clone_prompt=voice_clone_prompt)
        rec["text"] = dict(gen, chunk_size=chunk_size, prompt=(tie, tam, tpe), ids=feed.prompt_ids(),
                           voice_clone_prompt=voice_clone_prompt)
        return iter(())

    monkeypatch.setattr(generate, "fast_generate", fast_generate)
    monkeypatch.setattr(streaming, "parity_generate_streaming", parity)
    monkeypatch.setattr(batching, "BatchScheduler", Scheduler)
    monkeypatch.setattr(text_stream, "generate_text_streaming", text_streaming)
    monkeypatch.setattr(tts, "_decode_all", decode_all)
    monkeypatch.setattr(tts, "_stream_audio", stream_audio)
    monkeypatch.setattr(tts, "stream_from_embeds", stream_from_embeds)
    monkeypatch.setattr(tts, "stream_batch_from_embeds", stream_batch_from_embeds)
    return rec


def _run(out):
    """a generator method's refusals and deliveries happen when it is iterated"""
    return list(out) if isinstance(out, types.GeneratorType) else out


def _equal(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert (g is None and w is None) or (g.dtype == w.dtype and g.shape == w.shape and torch.equal(g, w))


def _sampling(kw):
    return {k: kw[k] for k in GEN}


def _prompt(kw):
    return kw["talker_input_embeds"], kw["attention_mask"], kw["trailing_text_hiddens"], kw["tts_pad_embed"]


def _speaker_prompt(tts, text, language, speaker, instruct, non_streaming_mode):
    """``build_talker_inputs`` on the ids of one custom-voice / voice-design request"""
    up = tts.model
    ins = up._tokenize_texts([up._build_instruct_text(instruct)])[0] if instruct else None
    with torch.inference_mode():
        return build_talker_inputs(tts.model.model, input_ids=up._tokenize_texts([up._build_assistant_text(text)]),
                                   ref_ids=[None], voice_clone_prompt=None, languages=[language], speakers=[speaker],
                                   non_streaming_mode=non_streaming_mode, instruct_ids=[ins])


def _text_fed_prompt(tts, ids, language, speaker, instruct, vcp):
    up = tts.model
    ins = up._tokenize_texts([up._build_instruct_text(instruct)])[0] if instruct else None
    with torch.inference_mode():
        tie, tam, tth, tpe = build_talker_inputs(tts.model.model, input_ids=[ids], ref_ids=[None], voice_clone_prompt=vcp,
                                                 languages=[language], speakers=[speaker], non_streaming_mode=False,
                                                 instruct_ids=[ins])
    return tie, tam, tpe


def _check_deliveries(rec, want, ref_codes, seeds, chunk_size):
    """one-shot, streaming and takes records against the prompt ``want`` (tie, tam, tth, tpe) and ``ref_codes``"""
    kw = rec["one_shot"]
    _equal(_prompt(kw), want)
    assert _sampling(kw) == GEN
    _equal([rec["one_shot_ref_codes"]], [ref_codes])
    _equal(rec["streaming"]["prompt"], want)
    _equal([rec["streaming"].get("ref_codes")], [ref_codes])
    assert _sampling(rec["streaming"]) == GEN and rec["streaming"]["chunk_size"] == chunk_size
    reqs = rec["takes"]
    assert [r["tag"] for r in reqs] == list(range(len(seeds)))
    for r, s in zip(reqs, seeds):
        _equal((r["tie"], r["tam"], r["tth"], r["tpe"]), want)
        assert _sampling(r) == GEN
        assert torch.equal(r["uniforms"], take_uniforms(s, GEN["max_new_tokens"], "cpu"))


SEEDS = [5, 6]


@pytest.mark.parametrize("mode", ["xvec", "icl", "icl_nsm", "cached_icl", "cached_xvec"])
def test_voice_clone_deliveries_get_the_prepared_prompt(tts, seen, mode):
    emb = torch.randn(tts.model.model.config.talker_config.hidden_size, generator=torch.Generator().manual_seed(3))
    codes = torch.randint(0, 64, (9, 16), generator=torch.Generator().manual_seed(4))
    if mode.startswith("cached"):
        args = dict(ref_spk_emb=emb.numpy(), ref_codes=codes.numpy() if mode == "cached_icl" else None,
                    ref_text=REF["ref_text"])
        vcp = tts._cached_reference_prompt(args["ref_spk_emb"], args["ref_codes"], None)
        prep = dict(voice_clone_prompt=vcp, ref_text=REF["ref_text"])
        takes_args = dict(voice_clone_prompt=vcp, ref_text=REF["ref_text"])
    else:
        args = dict(REF, xvec_only=mode == "xvec", non_streaming_mode=True if mode == "icl_nsm" else None,
                    instruct="slowly" if mode == "icl" else None)
        prep = dict(REF, xvec_only=args["xvec_only"], non_streaming_mode=mode == "icl_nsm", instruct=args["instruct"])
        takes_args = args
    with torch.inference_mode():
        *want, ref_codes = tts._prepare_generation(TEXT, language="English", **prep)[3:]
    assert (ref_codes is None) == (mode in ("xvec", "cached_xvec"))

    tts.generate_voice_clone(TEXT, "English", **args, **GEN)
    _run(tts.generate_voice_clone_streaming(TEXT, "English", chunk_size=7, **args, **GEN))
    with pytest.raises(_Stop):
        tts.generate_voice_clone_takes(TEXT, "English", n_takes=2, seeds=SEEDS, **takes_args, **GEN)
    _check_deliveries(seen, want, ref_codes, SEEDS, 7)

    _run(tts.generate_voice_clone_streaming(TEXT, "English", chunk_size=5, parity_mode=True, **args, **GEN))
    _equal(_prompt(seen["parity"]), want)
    assert _sampling(seen["parity"]) == GEN and seen["parity"]["chunk_size"] == 5
    _equal([seen["parity_ref_codes"]], [ref_codes])


def test_voice_clone_text_streaming_gets_the_resolved_x_vector(tts, seen):
    _run(tts.generate_voice_clone_text_streaming(iter(["Good morning, ", "how are you today?"]), "English",
                                                 chunk_size=9, **REF, **GEN))
    rec = seen["text"]
    vcp, _, _ = tts._resolve_voice_clone_prompt(input_ids=[None], ref_audio=REF["ref_audio"], ref_text=REF["ref_text"],
                                                xvec_only=True, append_silence=True, voice_clone_prompt=None)
    assert rec["voice_clone_prompt"]["x_vector_only_mode"] == [True]
    _equal(rec["prompt"], _text_fed_prompt(tts, rec["ids"], "English", None, None, vcp))
    assert _sampling(rec) == GEN and rec["chunk_size"] == 9


@pytest.mark.parametrize("kind", ["custom_voice", "voice_design"])
@pytest.mark.parametrize("size", [None, "0b6"])
@pytest.mark.parametrize("nsm", [None, False])
def test_custom_voice_and_voice_design_deliveries_get_the_built_prompt(tts, seen, monkeypatch, kind, size, nsm):
    if size is not None:
        monkeypatch.setattr(tts.model.model, "tts_model_size", size, raising=False)
    instruct = "a calm, warm voice"
    if kind == "custom_voice":
        who, speaker = dict(speaker="Aiden"), "Aiden"
        dropped = size is not None     # the 0.6B custom-voice checkpoint ignores instructions
    else:
        who, speaker, dropped = {}, None, False
    f = {k: getattr(tts, f"generate_{kind}{k}") for k in ("", "_streaming", "_takes", "_text_streaming")}
    req = dict(who, instruct=instruct, language="English", non_streaming_mode=nsm)
    want = _speaker_prompt(tts, TEXT, "English", speaker, None if dropped else instruct, nsm is not False)

    f[""](TEXT, **req, **GEN)
    _run(f["_streaming"](TEXT, chunk_size=7, **req, **GEN))
    with pytest.raises(_Stop):
        f["_takes"](TEXT, n_takes=2, seeds=SEEDS, **req, **GEN)
    _check_deliveries(seen, want, None, SEEDS, 7)

    _run(f["_text_streaming"](iter(["Good morning, ", "how are you today?"]), chunk_size=9, **req, **GEN))
    rec = seen["text"]
    _equal(rec["prompt"], _text_fed_prompt(tts, rec["ids"], "English", speaker, None if dropped else instruct, None))
    assert _sampling(rec) == GEN and rec["chunk_size"] == 9

    if kind == "custom_voice":     # a request alone and as the one row of a batch: the same prompt
        tts.generate_custom_voice_batch([TEXT], ["Aiden"], ["English"], [instruct], non_streaming_mode=nsm,
                                        chunk_size=11, **GEN)
        _equal(seen["batch"]["prompt"], want)
        assert _sampling(seen["batch"]) == GEN and seen["batch"]["chunk_size"] == 11


def test_serving_request_helpers_build_the_public_prompt(tts, seen):
    prepare = serving.custom_voice_text_request(tts, "Aiden", "English", instruct="cheerful")
    feed = text_stream.TextFeed(tts, max_rows=16)
    feed.push(TEXT)
    feed.close()
    with torch.inference_mode():
        tie, tam, tpe, ref_codes = prepare(feed)
    assert ref_codes is None
    _equal((tie, tam, tpe), _text_fed_prompt(tts, feed.prompt_ids(), "English", "Aiden", "cheerful", None))

    prepare = serving.voice_clone_request(tts, TEXT, "English", xvec_only=False, **REF)
    with torch.inference_mode():
        got = prepare()
        want = tts._prepare_generation(TEXT, language="English", **REF)[3:]
    _equal(got, want)
    assert seen == {}


# ---------------------------------------------------------------------------------------------------- refusals
BAD_LANG, BAD_SPK = "Klingon", "zorg"
CACHED = dict(ref_spk_emb=np.zeros(512, dtype=np.float32), voice_clone_prompt={"ref_spk_embedding": [torch.zeros(512)]})
ICL_VCP = dict(ref_spk_embedding=[torch.zeros(512)], ref_code=[torch.zeros(3, 16, dtype=torch.long)],
               x_vector_only_mode=[False], icl_mode=[True])
TS = ["Good morning."]

# (id, model type to set, call, exception, message, raised before anything is tokenized)
REFUSALS = [
    # custom voice: model type, then language, then speaker, then the delivery's own refusals
    ("cv_type_lang", "voice_design", lambda m: m.generate_custom_voice(TEXT, BAD_SPK, BAD_LANG),
     ValueError, "does not support custom voice", True),
    ("cv_stream_type", "base", lambda m: m.generate_custom_voice_streaming(TEXT, BAD_SPK, BAD_LANG),
     ValueError, "does not support custom voice", True),
    ("cv_takes_type", "voice_design", lambda m: m.generate_custom_voice_takes(TEXT, "Aiden", "English", n_takes=99),
     ValueError, "does not support custom voice", True),
    ("cv_text_type", "voice_design",
     lambda m: m.generate_custom_voice_text_streaming(iter(TS), "Aiden", "English", non_streaming_mode=True),
     ValueError, "does not support custom voice", True),
    ("cv_batch_type_len", "voice_design", lambda m: m.generate_custom_voice_batch([TEXT], ["Aiden", "ryan"], ["English"]),
     ValueError, "does not support custom voice", True),
    ("cv_serving_type", "voice_design", lambda m: serving.custom_voice_text_request(m, BAD_SPK, BAD_LANG),
     ValueError, "does not support custom voice", True),
    ("cv_lang_spk", None, lambda m: m.generate_custom_voice(TEXT, BAD_SPK, BAD_LANG),
     ValueError, "Unsupported language", True),
    ("cv_stream_lang_spk", None, lambda m: m.generate_custom_voice_streaming(TEXT, BAD_SPK, BAD_LANG),
     ValueError, "Unsupported language", True),
    ("cv_spk", None, lambda m: m.generate_custom_voice(TEXT, BAD_SPK, "English"),
     ValueError, "Unsupported speaker", True),
    ("cv_takes_spk_n", None, lambda m: m.generate_custom_voice_takes(TEXT, BAD_SPK, "English", n_takes=99),
     ValueError, "Unsupported speaker", True),
    ("cv_takes_n_seeds", None, lambda m: m.generate_custom_voice_takes(TEXT, "Aiden", "English", n_takes=99, seeds=[1]),
     ValueError, r"n_takes=99 must be in \[1, max_batch=4\]", True),
    ("cv_takes_seeds", None, lambda m: m.generate_custom_voice_takes(TEXT, "Aiden", "English", n_takes=2, seeds=[1]),
     ValueError, "1 seeds for 2 takes", True),
    ("cv_text_spk_nsm", None,
     lambda m: m.generate_custom_voice_text_streaming(iter(TS), BAD_SPK, "English", non_streaming_mode=True),
     ValueError, "Unsupported speaker", True),
    ("cv_text_nsm", None,
     lambda m: m.generate_custom_voice_text_streaming(iter(TS), "Aiden", "English", non_streaming_mode=True),
     ValueError, "step-by-step text layout", True),
    ("cv_batch_len_lang", None, lambda m: m.generate_custom_voice_batch([TEXT], ["Aiden", "ryan"], [BAD_LANG]),
     ValueError, "texts, speakers and languages must have the same length", True),
    ("cv_batch_lang_spk", None, lambda m: m.generate_custom_voice_batch([TEXT, TEXT], ["Aiden", BAD_SPK],
                                                                        ["English", BAD_LANG]),
     ValueError, "Unsupported language", True),
    ("cv_serving_spk", None, lambda m: serving.custom_voice_text_request(m, BAD_SPK, "English"),
     ValueError, "Unsupported speaker", True),
    # voice design: model type, then language, then the delivery's own refusals
    ("vd_type_lang", "custom_voice", lambda m: m.generate_voice_design(TEXT, "calm", BAD_LANG),
     ValueError, "does not support voice design", True),
    ("vd_stream_type", "custom_voice", lambda m: m.generate_voice_design_streaming(TEXT, "calm", BAD_LANG),
     ValueError, "does not support voice design", True),
    ("vd_takes_type", "custom_voice", lambda m: m.generate_voice_design_takes(TEXT, "calm", "English", n_takes=0),
     ValueError, "does not support voice design", True),
    ("vd_text_type", "custom_voice",
     lambda m: m.generate_voice_design_text_streaming(iter(TS), "calm", BAD_LANG, non_streaming_mode=True),
     ValueError, "does not support voice design", True),
    ("vd_lang", None, lambda m: m.generate_voice_design(TEXT, "calm", BAD_LANG),
     ValueError, "Unsupported language", True),
    ("vd_takes_lang_n", None, lambda m: m.generate_voice_design_takes(TEXT, "calm", BAD_LANG, n_takes=0),
     ValueError, "Unsupported language", True),
    ("vd_takes_n", None, lambda m: m.generate_voice_design_takes(TEXT, "calm", "English", n_takes=0),
     ValueError, "n_takes=0", True),
    ("vd_text_lang_nsm", None,
     lambda m: m.generate_voice_design_text_streaming(iter(TS), "calm", BAD_LANG, non_streaming_mode=True),
     ValueError, "Unsupported language", True),
    ("vd_text_nsm", None,
     lambda m: m.generate_voice_design_text_streaming(iter(TS), "calm", "English", non_streaming_mode=True),
     ValueError, "step-by-step text layout", True),
    # voice clone: .spk/.rvq files, then the cached reference, then the delivery's refusals, then prompt resolution
    ("vc_ggml_cached", None, lambda m: m.generate_voice_clone(TEXT, "English", ref_spk="a.spk", **CACHED),
     NotImplementedError, "backend='ggml'", True),
    ("vc_stream_ggml", None, lambda m: m.generate_voice_clone_streaming(TEXT, "English", ref_rvq="a.rvq", **CACHED),
     NotImplementedError, "backend='ggml'", True),
    ("vc_text_ggml_nsm", None,
     lambda m: m.generate_voice_clone_text_streaming(iter(TS), "English", ref_spk="a.spk", non_streaming_mode=True,
                                                     **CACHED),
     NotImplementedError, "backend='ggml'", True),
    ("vc_cached_both", None, lambda m: m.generate_voice_clone(TEXT, "English", **CACHED),
     ValueError, "either voice_clone_prompt or ref_spk_emb/ref_codes, not both", True),
    ("vc_stream_cached_both", None, lambda m: m.generate_voice_clone_streaming(TEXT, "English", **CACHED),
     ValueError, "not both", True),
    ("vc_text_cached_both_nsm", None,
     lambda m: m.generate_voice_clone_text_streaming(iter(TS), "English", non_streaming_mode=True, **CACHED),
     ValueError, "not both", True),
    ("vc_codes_without_emb", None,
     lambda m: m.generate_voice_clone(TEXT, "English", ref_codes=np.zeros((3, 16), dtype=np.int64)),
     ValueError, "ref_spk/ref_spk_emb is required", True),
    ("vc_takes_n_no_ref", None, lambda m: m.generate_voice_clone_takes(TEXT, "English", n_takes=99),
     ValueError, "n_takes=99", True),
    ("vc_takes_seeds", None, lambda m: m.generate_voice_clone_takes(TEXT, "English", n_takes=2, seeds=[1, 2, 3], **REF),
     ValueError, "3 seeds for 2 takes", True),
    ("vc_text_nsm_icl", None,
     lambda m: m.generate_voice_clone_text_streaming(iter(TS), "English", xvec_only=False, non_streaming_mode=True,
                                                     **REF),
     ValueError, "step-by-step text layout", True),
    ("vc_text_icl", None,
     lambda m: m.generate_voice_clone_text_streaming(iter(TS), "English", xvec_only=False, **REF),
     ValueError, "text streaming is not available for ICL voice cloning", True),
    ("vc_text_icl_prompt", None,
     lambda m: m.generate_voice_clone_text_streaming(iter(TS), "English", voice_clone_prompt=ICL_VCP,
                                                     ref_text="words"),
     ValueError, "text streaming is not available for ICL voice cloning", False),
    ("vc_text_icl_cached_no_ref_text", None,
     lambda m: m.generate_voice_clone_text_streaming(iter(TS), "English", ref_spk_emb=np.zeros(512, dtype=np.float32),
                                                     ref_codes=np.zeros((3, 16), dtype=np.int64)),
     ValueError, "ref_text is required when voice_clone_prompt uses ICL mode", True),
    ("vc_no_ref_audio", None, lambda m: m.generate_voice_clone(TEXT, "English"),
     ValueError, "ref_audio is required", False),
    ("vc_takes_no_ref_audio", None, lambda m: m.generate_voice_clone_takes(TEXT, "English", n_takes=2),
     ValueError, "ref_audio is required", False),
    ("takes_one_column_engine", None,
     lambda m: (setattr(m.engine, "max_batch", 1), m.generate_voice_design_takes(TEXT, "calm", "English", n_takes=1)),
     ValueError, "max_batch >= 2", True),
]


@pytest.mark.parametrize("mtype,call,exc,match,untokenized", [r[1:] for r in REFUSALS], ids=[r[0] for r in REFUSALS])
def test_refusals_keep_their_exception_and_order(tts, seen, monkeypatch, mtype, call, exc, match, untokenized):
    if mtype is not None:
        monkeypatch.setattr(tts.model.model, "tts_model_type", mtype, raising=False)
    tokenized = []
    tok = tts.model._tokenize_texts
    monkeypatch.setattr(tts.model, "_tokenize_texts", lambda texts: tokenized.append(texts) or tok(texts))
    with pytest.raises(exc, match=match):
        _run(call(tts))
    assert seen == {}
    if untokenized:
        assert tokenized == []


# ---------------------------------------------------------------------------------------------------- one-shot log
ONE_SHOT = {
    "voice_clone": lambda m: m.generate_voice_clone(TEXT, "English", **REF),
    "custom_voice": lambda m: m.generate_custom_voice(TEXT, "Aiden", "English"),
    "voice_design": lambda m: m.generate_voice_design(TEXT, "calm", "English"),
}


@pytest.mark.parametrize("kind", list(ONE_SHOT))
def test_one_shot_logs_an_empty_generation(tts, seen, monkeypatch, caplog, kind):
    monkeypatch.setattr(generate, "fast_generate", lambda **kw: (None, {}))
    with caplog.at_level(logging.WARNING, logger="faster_qwen3_tts.model"):
        audio, sr = ONE_SHOT[kind](tts)
    assert sr == tts.sample_rate and len(audio) == 1
    assert audio[0].dtype == np.float32 and np.array_equal(audio[0], np.zeros(1, dtype=np.float32))
    assert any(r.levelno == logging.WARNING and r.getMessage() == "Generation returned no tokens" for r in caplog.records)


@pytest.mark.parametrize("kind", list(ONE_SHOT))
def test_one_shot_logs_its_real_time_factor(tts, seen, caplog, kind):
    with caplog.at_level(logging.INFO, logger="faster_qwen3_tts.model"):
        audio, sr = ONE_SHOT[kind](tts)
    assert sr == 24000 and np.array_equal(audio[0], np.ones(3, dtype=np.float32))
    logged = [r.getMessage() for r in caplog.records if r.getMessage().startswith("Generated")]
    assert len(logged) == 1 and logged[0].startswith("Generated 2.00s audio in") and "(8.0ms/step, RTF:" in logged[0]
