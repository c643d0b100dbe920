"""SSML input without a GPU: the parser's subset and refusals (faster_qwen3_tts/ssml.py), the join oracle's pause plan,
the constants, a document through ``ContinuousBatcher`` on a fake scheduler (voices, seeds, row prosody, pause plan,
due), and the example server's ``input_format``."""
import os
import re

import numpy as np
import pytest
import torch

from oracle import prompt_cases  # noqa: F401  (puts the package on sys.path)
from faster_qwen3_tts import join as J
from faster_qwen3_tts import ssml as X
from faster_qwen3_tts.segment import segment_seed, split_text
from faster_qwen3_tts.serving import ContinuousBatcher, Segments

import join_oracle as O
from join_pauses_oracle import join_pauses

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
V = {"a": {"ref_audio": "a.wav"}, "b": {"speaker": "ryan", "language": "German"}, "d": {"design": "calm"}}


def _doc(body, voice="a", **kw):
    return X.parse(f"<speak>{body}</speak>", V, voice, **kw)


def _one(body, **kw):
    d = _doc(body, **kw)
    assert len(d.spans) == 1, d
    return d.spans[0]


# ---- parser: accepted forms -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("attrs,ms", [("time='250ms'", 250), ("time='2s'", 2000), ("time='1.5s'", 1500),
                                      ("time='0.0004s'", 0), ("time='0.0005s'", 1), ("time='12.5ms'", 13),
                                      ("time=' 3 ms '", 3), ("time='.5s'", 500), ("time='300ms' strength='x-strong'", 300)]
                         + [(f"strength='{k}'", v) for k, v in X.STRENGTH_MS.items()] + [("", 750)])
def test_break_forms(attrs, ms):
    d = _doc(f"One sentence that is long enough.<break {attrs}/>Another sentence, also long enough.")
    assert d.breaks == [None, ms, None]


@pytest.mark.parametrize("value,factor", [("50%", 0.5), ("150%", 1.5), ("+20%", 1.2), ("-20%", 0.8), ("2", 2.0),
                                          ("0.75", 0.75), ("x-slow", 0.5), ("slow", 0.75), ("medium", 1.0),
                                          ("fast", 1.25), ("x-fast", 1.75)])
def test_rate_forms(value, factor):
    assert _one(f"<prosody rate='{value}'>Some words here.</prosody>").speed == pytest.approx(factor)


@pytest.mark.parametrize("value,st", [("+2st", 2.0), ("-3st", -3.0), ("1.5st", 1.5), ("+10%", 12 * np.log2(1.1)),
                                      ("-10%", 12 * np.log2(0.9)), ("x-low", -6), ("low", -3), ("medium", 0),
                                      ("high", 3), ("x-high", 6)])
def test_pitch_forms(value, st):
    assert _one(f"<prosody pitch='{value}'>Some words here.</prosody>").pitch == pytest.approx(st)


@pytest.mark.parametrize("value,db", [("+6dB", 6.0), ("-6dB", -6.0), ("3.5dB", 3.5), ("silent", -96), ("x-soft", -12),
                                      ("soft", -6), ("medium", 0), ("loud", 6), ("x-loud", 12)])
def test_volume_forms(value, db):
    assert _one(f"<prosody volume='{value}'>Some words here.</prosody>").gain_db == pytest.approx(db)


def test_nested_prosody_composes():
    d = _doc("<prosody rate='1.5' pitch='-2st' volume='-3dB'>Outer words of the span. <prosody rate='50%' "
             "pitch='+1st' volume='-3dB'>Inner words of the span.</prosody></prosody>")
    assert [(s.speed, s.pitch, s.gain_db) for s in d.spans] == [(1.5, -2, -3), (0.75, -1, -6)]


def test_breaks_add_up_and_cap():
    d = _doc("<break time='100ms'/> <break strength='weak'/>\n <s>First sentence of the text.</s>"
             "<break time='1s'/>  <break time='2s'/><s>Second sentence of the text.</s><break/>")
    assert d.breaks == [600, 3000, 750]
    assert _doc("Text one.<break time='5s'/><break time='5s'/>Text two.").breaks == [None, 10000, None]
    with pytest.raises(ValueError, match="<break>.*10001 ms"):
        _doc("Text one.<break time='5s'/><break time='5001ms'/>Text two.")
    with pytest.raises(ValueError, match="<break>"):
        _doc("Text one.<break time='10001ms'/>Text two.")


def test_whitespace_sub_and_cuts():
    d = _doc("  Hello\n\n   big\tworld, <sub alias='World Health Organization'>WHO</sub>   says hi.  ")
    assert [s.text for s in d.spans] == ["Hello big world, World Health Organization says hi."]
    d = _doc("<p>One.</p><p><s>Two.</s><s>Three.</s></p>")
    assert [s.text for s in d.spans] == ["One.", "Two.", "Three."]   # forced cuts: no merge of short pieces
    assert d.breaks == [None] * 4


@pytest.mark.parametrize("tag,lang", list(X.LANGUAGES.items()) + [("en-US", "English"), ("zh-CN", "Chinese"),
                                                                   ("PT-br", "Portuguese")])
def test_language_map(tag, lang):
    assert _one(f"<s xml:lang='{tag}'>Some words here.</s>").language == lang


def test_language_precedence():
    # innermost xml:lang, then the voice spec's language, then the call's
    d = X.parse("<speak xml:lang='fr'><voice name='b'>Des mots ici.<s xml:lang='ja'>Words.</s></voice></speak>", V,
                "a", language="Spanish")
    assert [s.language for s in d.spans] == ["French", "Japanese"]
    d = X.parse("<speak><voice name='b'>Worte hier.</voice> Palabras aqui.</speak>", V, "a", language="Spanish")
    assert [(s.voice, s.language) for s in d.spans] == [("b", "German"), ("a", "Spanish")]


def test_voices_innermost_wins_and_default():
    d = _doc("Default voice. <voice name='b'>Voice b <voice name='d'>voice d</voice> back to b.</voice>")
    assert [(s.voice, s.text) for s in d.spans] == [("a", "Default voice."), ("b", "Voice b"), ("d", "voice d"),
                                                    ("b", "back to b.")]


@pytest.mark.parametrize("T", ["Hello there. How are you today? I am fine; thanks! And you?",
                               "no punctuation at all " * 40, "x" * 1000,
                               "Mr. Smith paid 3.50 dollars. e.g. this. Done"])
@pytest.mark.parametrize("max_chars", [7, 40, 400])
def test_plain_document_is_split_text(T, max_chars):
    d = X.parse(f"<speak>{T}</speak>", V, "a", max_segment_chars=max_chars)
    assert [s.text for s in d.spans] == split_text(T, max_chars)
    assert d.breaks == [None] * (len(d.spans) + 1)
    assert {(s.voice, s.speed, s.pitch, s.gain_db) for s in d.spans} == {("a", 1, 0, 0)}


# ---- parser: refusals -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("doc,names", [
    ("<speak><mark name='m'/>Hi.</speak>", "<mark>"),
    ("<speak><say-as interpret-as='date'>1/2</say-as></speak>", "<say-as>"),
    ("<speak><emphasis>Hi.</emphasis></speak>", "<emphasis>"),
    ("<speak><phoneme ph='x'>Hi.</phoneme></speak>", "<phoneme>"),
    ("<speak><audio src='a.wav'/>Hi.</speak>", "<audio>"),
    ("<speak><lang xml:lang='fr'>Hi.</lang></speak>", "<lang>"),
    ("<speak><amazon:effect name='whispered'>Hi.</amazon:effect></speak>", "<amazon:effect>"),
    ("<speak xmlns:amazon='x'>Hi.</speak>", "'xmlns:amazon'"),
    ("<speak><speak>Hi.</speak></speak>", "<speak>"),
    ("<p>Hi.</p>", "<p>"),
    ("<speak foo='1'>Hi.</speak>", "'foo'"),
    ("<speak><s lang='en'>Hi.</s></speak>", "'lang'"),
    ("<speak><break time='1s' foo='x'/>Hi.</speak>", "'foo'"),
    ("<speak><break time='-1s'/>Hi.</speak>", "<break> time"),
    ("<speak><break time='1 min'/>Hi.</speak>", "<break> time"),
    ("<speak><break strength='loud'/>Hi.</speak>", "<break> strength"),
    ("<speak><break>x</break>Hi.</speak>", "<break>"),
    ("<speak><prosody rate='0'>Hi.</prosody></speak>", "<prosody> rate"),
    ("<speak><prosody rate='-5'>Hi.</prosody></speak>", "<prosody> rate"),
    ("<speak><prosody rate='quick'>Hi.</prosody></speak>", "<prosody> rate"),
    ("<speak><prosody pitch='200Hz'>Hi.</prosody></speak>", "<prosody> pitch"),
    ("<speak><prosody pitch='+10Hz'>Hi.</prosody></speak>", "<prosody> pitch"),
    ("<speak><prosody pitch='10%'>Hi.</prosody></speak>", "<prosody> pitch"),
    ("<speak><prosody volume='+10%'>Hi.</prosody></speak>", "<prosody> volume"),
    ("<speak><prosody contour='(0%,+20Hz)'>Hi.</prosody></speak>", "'contour'"),
    ("<speak><prosody range='high'>Hi.</prosody></speak>", "'range'"),
    ("<speak><prosody duration='2s'>Hi.</prosody></speak>", "'duration'"),
    ("<speak><prosody rate='x-fast'><prosody rate='x-fast'><prosody rate='2'>Hi.</prosody></prosody></prosody></speak>",
     "<prosody>"),
    ("<speak><prosody pitch='+8st'><prosody pitch='+8st'>Hi.</prosody></prosody></speak>", "<prosody>"),
    ("<speak><prosody volume='silent'><prosody volume='x-soft'>Hi.</prosody></prosody></speak>", "<prosody>"),
    ("<speak><voice name='zzz'>Hi.</voice></speak>", "'zzz'"),
    ("<speak><voice name='a' gender='female'>Hi.</voice></speak>", "'gender'"),
    ("<speak><voice>Hi.</voice></speak>", "<voice>"),
    ("<speak><sub>WHO</sub></speak>", "<sub>"),
    ("<speak><sub alias='x'>W<s>H</s>O</sub></speak>", "<sub>"),
    ("<speak><s xml:lang='xx'>Hi.</s></speak>", "xml:lang"),
    ("<speak>Hi.", "malformed"),
    ("<speak>Hi &nbsp; there.</speak>", "malformed"),
    ("<speak>  <break/>  </speak>", "no text"),
    ("<speak><?pi data?>Hi.</speak>", "processing instruction"),
])
def test_refusals_name_the_element(doc, names):
    with pytest.raises(ValueError) as e:
        X.parse(doc, V, "a")
    assert names in str(e.value), str(e.value)
    if "malformed" not in names and "no text" not in names:
        assert re.search(r"line \d+, column \d+", str(e.value))


def test_unknown_voice_lists_the_known_ones_and_default_voice_is_needed():
    with pytest.raises(ValueError, match=r"\['a', 'b', 'd'\]"):
        X.parse("<speak><voice name='q'>Hi.</voice></speak>", V)
    with pytest.raises(ValueError, match="default voice"):
        X.parse("<speak>Hi.</speak>", V)
    with pytest.raises(ValueError, match="default voice"):
        X.parse("<speak>Hi.</speak>", V, "nope")
    assert X.parse("<speak><voice name='b'>Hi.</voice></speak>", V).spans[0].voice == "b"


@pytest.mark.parametrize("doc", [
    "<?xml version='1.0'?><!DOCTYPE speak [<!ENTITY x 'boom'>]><speak>&x;</speak>",
    "<!DOCTYPE speak SYSTEM 'http://example.invalid/x.dtd'><speak>Hi.</speak>",
    "<!DOCTYPE speak><speak>Hi.</speak>",
])
def test_doctype_and_entities_refused(doc):
    with pytest.raises(ValueError, match="DOCTYPE|entity"):
        X.parse(doc, V, "a")


# ---- voice specs ----------------------------------------------------------------------------------------------------
def test_voice_request_kinds(monkeypatch):
    import faster_qwen3_tts.serving as sv
    seen = []
    monkeypatch.setattr(sv, "voice_clone_request", lambda *a, **k: seen.append(("clone", a[1:], k)) or "c")
    monkeypatch.setattr(sv, "custom_voice_request", lambda *a, **k: seen.append(("custom", a[1:], k)) or "v")
    m = object()
    X.voice_request(m, {"ref_audio": "r.wav", "ref_text": "words", "xvec_only": True, "language": "English"}, "hi")
    X.voice_request(m, {"ref_audio": "r.wav"}, "hi", split=True)
    X.voice_request(m, {"speaker": "ryan", "instruct": "happy"}, "hi", "German")
    X.voice_request(m, {"design": "a calm voice", "max_new_tokens": 99}, "hi")
    assert seen == [("clone", ("hi", "English", "r.wav", "words"), {"xvec_only": True}),
                    ("clone", ("hi", "Auto", "r.wav", ""), {"split": True, "max_segment_chars": 400}),
                    ("custom", ("hi", "ryan", "German"), {"instruct": "happy"}),
                    ("custom", ("hi", None, "Auto"), {"instruct": "a calm voice"})]
    for bad in ({}, {"ref_audio": "r.wav", "speaker": "ryan"}, {"speaker": "ryan", "design": "x"}):
        with pytest.raises(ValueError, match="exactly one"):
            X.voice_request(m, bad, "hi")


# ---- join oracle and constants --------------------------------------------------------------------------------------
def test_constants_agree_with_the_header():
    h = open(os.path.join(ROOT, "include", "fq3_engine.h")).read()
    val = dict(re.findall(r"#define FQ3_JOIN_(\w+) (\d+)", h))
    assert int(val["BREAK_MAX_MS"]) == J.BREAK_MAX_MS == 10000
    assert "fq3_join_create_pauses" in h and "fq3_join_reset_pauses" in h
    from faster_qwen3_tts.engine import EXPORTS
    assert {"fq3_join_create_pauses", "fq3_join_reset_pauses"} <= set(EXPORTS)


@pytest.mark.parametrize("pause_ms", [0, 1, 37, 2000])
def test_uniform_plan_is_the_join(pause_ms):
    rng = np.random.default_rng(pause_ms)
    for n in (1, 2, 4):
        segs = [rng.standard_normal(int(rng.integers(0, 3000))).astype(np.float32) for _ in range(n)]
        assert np.array_equal(join_pauses(segs, [0] + [pause_ms] * (n - 1) + [0]), O.join(segs, pause_ms))


def test_leading_and_trailing_silence():
    rng = np.random.default_rng(3)
    segs = [rng.standard_normal(n).astype(np.float32) for n in (400, 50, 900)]
    plan = [200, 0, 10000, 500]
    y = join_pauses(segs, plan)
    assert len(y) == sum(map(len, segs)) + 24 * sum(plan)
    assert not y[:4800].any() and not y[-12000:].any()
    inner = O.join(segs, 0)
    assert np.array_equal(y[4800:4800 + 450], inner[:450])   # outer edges are not faded; inner ones are as in join
    assert np.array_equal(y[4800 + 450 + 240000:-12000], inner[450:])
    assert np.array_equal(y[4800:4800 + 400], segs[0][:400] * np.r_[np.ones(280, np.float32), O.fade()[::-1]])


def test_check_pauses():
    assert J.check_pauses([0, 10000, 5], 2) == [0, 10000, 5]
    for bad in ([0, 10001, 0], [0, -1, 0], [0, 1.5, 0], [0, True, 0], [0, 0]):
        with pytest.raises(ValueError):
            J.check_pauses(bad, 2)


# ---- a document through the batcher ---------------------------------------------------------------------------------
class _Req:
    def __init__(self, tag, total):
        self.tag, self.total, self.done, self.finished = tag, total, 0, False
        self.due, self.hold = 0.0, False


class _Sched:
    def __init__(self):
        self.active, self.submitted = [], []

    def capacity(self):
        return 16 - len(self.active)

    def has_capacity(self):
        return self.capacity() > 0

    def submit_many(self, reqs):
        out = []
        for r in reqs:
            rq = _Req(r["tag"], r["max_new_tokens"])
            self.submitted.append(r)
            self.active.append(rq)
            out.append(rq)
        return out

    def cancel(self, rq):
        self.active.remove(rq)

    def step(self, n):
        res = []
        for rq in list(self.active):
            k = min(n, rq.total - rq.done)
            codes = torch.arange(rq.done, rq.done + k)[:, None].repeat(1, 16) + 1000 * rq.tag
            rq.done += k
            rq.finished = rq.done >= rq.total
            if rq.finished:
                self.active.remove(rq)
            res.append((rq, codes))
        return res

    def __len__(self):
        return len(self.active)


class _Win:
    def __init__(self, gain=1.0):
        self.gain, self.finals = gain, []

    def push(self, codes, final=False):
        self.finals.append(final)
        return torch.repeat_interleave(codes[:, 0].float() * 1e-4 * self.gain, 4), 24000


class _Joiner:
    """a whole-array join once every segment ended, with the request's pause plan"""

    def __init__(self):
        self.plans = []

    def uniforms(self, seed, n):
        return ("uniforms", seed)

    def open(self, t, out_kw):
        self.plans.append(list(t.segments.pauses))
        return dict(n=len(t.segments), plan=t.segments.pauses, segs=[[] for _ in t.segments], ended=[False] * len(t.segments))

    def run(self, states, pushes):
        for st, k, pcm, ended in pushes:
            if pcm is not None:
                st["segs"][k].append(pcm.numpy())
            st["ended"][k] = st["ended"][k] or ended
        out = []
        for st in states:
            if all(st["ended"]) and not st.get("done"):
                st["done"] = True
                a = join_pauses([np.concatenate(s) if s else np.zeros(0, np.float32) for s in st["segs"]], st["plan"])
            else:
                a = np.zeros(0, np.float32)
            out.append((a, 24000, len(a)))
        return out

    def close(self, state):
        pass


def test_rows_get_their_voice_seed_and_prosody(monkeypatch):
    import faster_qwen3_tts.serving as sv
    made = []

    def fake_voice(model, spec, text, language=None, **kw):
        made.append((spec, text, language))
        return lambda: (torch.zeros(1, 3, 4), None, None, None, spec)   # ref_codes: the voice spec, seen by the window
    monkeypatch.setattr(X, "voice_request", fake_voice)
    windows = []

    def window(ref_codes, *a, **kw):
        windows.append((ref_codes, a, kw))
        return _Win(kw.get("gain_db", 0.0) and 10 ** (kw["gain_db"] / 20))
    doc = ("<speak><break time='200ms'/>Plain words of voice a.<break time='0s'/>"
           "<voice name='b'><prosody rate='1.5' pitch='-3st'>Faster and lower, voice b.</prosody></voice>"
           "<prosody volume='-6dB'>Softer words of voice a here.</prosody> Plain again, voice a.<break time='500ms'/>"
           "</speak>")
    segs = sv.ssml_request(object(), doc, V, "a")
    assert segs.texts == ["Plain words of voice a.", "Faster and lower, voice b.", "Softer words of voice a here.",
                          "Plain again, voice a."]
    assert [m[0] for m in made] == [V["a"], V["b"], V["a"], V["a"]]
    assert [m[2] for m in made] == ["Auto", "German", "Auto", "Auto"]
    assert segs.prosody == [(1, 0, 0), (1.5, -3, 0), (1, 0, -6), (1, 0, 0)]
    assert segs.breaks == [200, 0, None, None, 500]
    sched, joiner = _Sched(), _Joiner()
    b = ContinuousBatcher(sched, window, chunk_size=4, joiner=joiner, idle_sleep=0.0005)
    try:
        t = b.submit(segs, split=True, pause_ms=40, seed=17, max_new_tokens=6)
        chunks = list(t)
    finally:
        b.close()
    assert joiner.plans == [[200, 0, 40, 40, 500]]
    assert [r["uniforms"] for r in sched.submitted] == [("uniforms", segment_seed(17, k)) for k in range(4)]
    # identity rows: exactly the keywords of a split request; the others their prosody
    assert [w[0] for w in windows] == [V["a"], V["b"], V["a"], V["a"]]
    assert [w[2] for w in windows] == [{"segment": True},
                                       {"segment": True, "speed": 1.5, "pitch": -3.0, "gain_db": 0.0},
                                       {"segment": True, "speed": 1.0, "pitch": 0.0, "gain_db": -6.0},
                                       {"segment": True}]
    assert chunks[-1][2]["is_final"] and chunks[-1][2]["n_segments"] == 4
    assert len(np.concatenate([c[0] for c in chunks])) == 4 * 6 * 4 + 24 * (200 + 40 + 40 + 500)


def test_plain_split_request_is_unchanged():
    """a split request without a document: windows as before, the plan [0, P, ..., P, 0]"""
    windows = []

    def window(ref_codes, *a, **kw):
        windows.append(kw)
        return _Win()
    sched, joiner = _Sched(), _Joiner()
    b = ContinuousBatcher(sched, window, chunk_size=4, joiner=joiner, idle_sleep=0.0005)
    try:
        segs = Segments([lambda: (torch.zeros(1, 3, 4), None, None, None, None)] * 3, ["a", "b", "c"])
        list(b.submit(segs, split=True, pause_ms=25, max_new_tokens=3))
    finally:
        b.close()
    assert windows == [{"segment": True}] * 3 and joiner.plans == [[0, 25, 25, 0]]


def test_due_counts_row_rates_and_breaks():
    b = ContinuousBatcher(_Sched(), lambda *a, **k: _Win(), chunk_size=4, joiner=_Joiner(), sleep=lambda s: None,
                          clock=lambda: 0.0)
    b.close()
    mk = lambda: (torch.zeros(1, 3, 4), None, None, None, None)   # noqa: E731
    segs = Segments([mk] * 3, ["a" * 14, "b" * 28, "c" * 42], prosody=[(2.0, 0, 0), (0.5, 0, 0), (1, 0, 0)],
                    breaks=[300, 1500, None, 100])
    t = b.submit(segs, split=True, pause_ms=500, pace=1.0, speed=2.0)
    assert segs.pauses == [300, 1500, 500, 100]
    # segment 0: 14 chars at 14 / s, row rate 2 and request rate 2 -> 0.25 s; then 1.5 s of break at rate 2
    assert b._segment_due(t, 1, 0.0) == pytest.approx(0.25 + 0.75)
    # segment 1: 28 chars at row rate 0.5 and request rate 2 -> 2 s; then the 500 ms pause at rate 2
    assert b._segment_due(t, 2, 0.0) == pytest.approx(0.25 + 0.75 + 2.0 + 0.25)
    segs.frames[0], segs.ended[0] = 10, True   # 0.8 s of frames at rates 2 x 2
    t.first_chunk_at = 0.0
    assert b._segment_due(t, 2, 0.0) == pytest.approx(0.0 + 2.0 + 0.25)


def test_segments_refusals():
    mk = lambda: None   # noqa: E731
    with pytest.raises(ValueError):
        Segments([mk, mk], ["a", "b"], breaks=[None, None])
    with pytest.raises(ValueError):
        Segments([mk], ["a"], prosody=[(1, 0, 0), (1, 0, 0)])
    b = ContinuousBatcher(_Sched(), lambda *a, **k: _Win(), joiner=_Joiner())
    try:
        with pytest.raises(ValueError, match="pause"):
            b.submit(Segments([mk], ["a"], breaks=[10001, None]), split=True)
        with pytest.raises(ValueError):
            b.submit(Segments([mk], ["a"], prosody=[(4.0, -12, 0)]), split=True)
    finally:
        b.close()


def test_model_refuses_before_tokenizing():
    from faster_qwen3_tts.model import FasterQwen3TTS
    m = object.__new__(FasterQwen3TTS)
    for kw in (dict(speed=9.0), dict(pitch=13), dict(pause_ms=2001), dict(max_segment_chars=0), dict(sample_rate=1),
               dict(temprature=0.5)):
        with pytest.raises((ValueError, TypeError)):
            m.speak_ssml("<speak>Hi.</speak>", V, "a", **kw)
    with pytest.raises(ValueError, match="mark"):
        next(m.speak_ssml_streaming("<speak><mark name='x'/>Hi.</speak>", V, "a"))


# ---- server ---------------------------------------------------------------------------------------------------------
def _server():
    pytest.importorskip("fastapi")
    pytest.importorskip("httpx")
    import importlib.util
    spec = importlib.util.spec_from_file_location("openai_server", os.path.join(ROOT, "examples", "openai_server.py"))
    srv = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(srv)
    return srv


class _B:
    sched, max_concurrent = [], 0

    def __init__(self):
        self.calls = []

    def submit(self, prepare, **kw):
        from faster_qwen3_tts.serving import _DONE, Ticket
        self.calls.append((prepare, kw))
        t = Ticket(1, prepare, {})
        t.out.put(_DONE)
        return t


def test_server_input_format(monkeypatch):
    srv = _server()
    from fastapi.testclient import TestClient
    import faster_qwen3_tts.serving as sv
    monkeypatch.setattr(X, "voice_request", lambda m, spec, text, language=None, **kw: ("voice", spec, text, kw))
    voices = {"a": {"ref_audio": "a.wav"}, "b": {"speaker": "ryan", "max_new_tokens": 77}, "d": {"design": "calm"}}
    batcher = _B()
    c = TestClient(srv.build_app(object(), batcher, voices, "a"))
    doc = "<speak>Hello there.<break time='300ms'/><voice name='b'>Second voice.</voice></speak>"
    for fmt in ("wav", "pcm", "ulaw", "alaw", "flac"):
        r = c.post("/v1/audio/speech", json={"input": doc, "voice": "d", "input_format": "ssml", "pause_ms": 60,
                                             "response_format": fmt})
        assert r.status_code == 200, r.text
        segs, kw = batcher.calls[-1]
        assert isinstance(segs, sv.Segments) and kw["split"] is True and kw["pause_ms"] == 60
        assert [p[1] for p in segs] == [voices["d"], voices["b"]] and segs.breaks == [None, 300, None]
    # plain text through the voice resolver: custom and design entries, split as asked
    for name in ("a", "b", "d"):
        assert c.post("/v1/audio/speech", json={"input": "Hi there.", "voice": name}).status_code == 200
        prepare, kw = batcher.calls[-1]
        assert prepare == ("voice", voices[name], "Hi there.", {"split": False}) and kw["split"] is False
    assert batcher.calls[-2][1]["max_new_tokens"] == 77
    assert c.post("/v1/audio/speech", json={"input": "Hi.", "voice": "b", "split": True}).status_code == 200
    assert batcher.calls[-1][0][3] == {"split": True}
    n = len(batcher.calls)
    bad = [dict(input_format="xml"), dict(input_format="ssml", split=False),
           dict(input_format="ssml", input="<speak><mark name='x'/>Hi.</speak>"),
           dict(input_format="ssml", input="<speak><voice name='zzz'>Hi.</voice></speak>"),
           dict(input_format="ssml", input="<speak>Hi."),
           dict(input_format="ssml", input="<speak><break time='11s'/>Hi.</speak>")]
    for b in bad:
        r = c.post("/v1/audio/speech", json=dict({"input": doc, "voice": "a"}, **b))
        assert r.status_code == 400, (b, r.text)
    assert "mark" in c.post("/v1/audio/speech", json={"input": "<speak><mark name='x'/>Hi.</speak>", "voice": "a",
                                                      "input_format": "ssml"}).text
    assert len(batcher.calls) == n
